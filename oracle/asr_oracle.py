"""Torch restatement of the ASR-BLEU transcriber (asr_bleu/utils.py:220-288) for the tests: fairseq's Wav2VecCtc forward pass
(fairseq/models/wav2vec/wav2vec2.py ConvFeatureExtractionModel in "layer_norm" mode, feature LayerNorm, post_extract_proj,
TransformerEncoder with layer_norm_first, pos_conv with weight norm over dims 0 and 1, Wav2VecEncoder.proj) in any dtype, the beam-1 CTC
decoding rule and the letter post-processing.  Batch of one, no padding, as the reference calls it.  Pinned to fairseq's own modules and
torchaudio's own _get_tokens by tests/golden/asr_w2v.npz (oracle/gen_golden_asr.py, tests/test_asr_oracle_golden.py).
"""
from __future__ import annotations

import itertools
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

PRE = "w2v_encoder.w2v_model."
BLANK, UNK = 0, 3
SPECIALS = ["<s>", "<pad>", "</s>", "<unk>"]


def _p(sd, key, dtype, device):
    return sd[key].to(device=device, dtype=dtype)


def pos_conv_weight(sd: Dict[str, torch.Tensor], dtype=torch.float64, device="cpu") -> torch.Tensor:
    """torch.nn.utils.weight_norm(dim=2): w = g * v / ||v|| with the norm over dims 0 and 1"""
    if PRE + "encoder.pos_conv.0.weight" in sd:
        return _p(sd, PRE + "encoder.pos_conv.0.weight", dtype, device)
    v = _p(sd, PRE + "encoder.pos_conv.0.weight_v", dtype, device)
    g = _p(sd, PRE + "encoder.pos_conv.0.weight_g", dtype, device)
    return g * v / v.norm(dim=(0, 1), keepdim=True)


def n_layers(sd) -> int:
    return len({k.split(".")[4] for k in sd if k.startswith(PRE + "encoder.layers.")})


def n_conv(sd) -> int:
    return len({k.split(".")[4] for k in sd if k.startswith(PRE + "feature_extractor.conv_layers.")})


def num_frames(n: int, kernels: Sequence[int], strides: Sequence[int]) -> int:
    for k, s in zip(kernels, strides):
        n = (n - k) // s + 1 if n >= k else 0
    return n


@torch.no_grad()
def forward(sd: Dict[str, torch.Tensor], wav: torch.Tensor, strides: Sequence[int], normalize: bool = True, dtype=torch.float64,
            device="cpu") -> Dict[str, torch.Tensor]:
    """stages of one utterance: "extractor" [T][C], "proj" [T][D] (feature LN + post_extract_proj), "pos" [T][D], "layer{l}" [T][D],
    "final_ln" [T][D], "emissions" [T][V]"""
    p = lambda k: _p(sd, PRE + k, dtype, device)  # noqa: E731
    x = wav.to(device=device, dtype=dtype).reshape(1, -1)
    if normalize:
        x = F.layer_norm(x, x.shape)
    out = {}
    x = x.unsqueeze(1)  # B x 1 x L
    for i in range(n_conv(sd)):
        pre = f"feature_extractor.conv_layers.{i}."
        b = sd.get(PRE + pre + "0.bias")
        x = F.conv1d(x, p(pre + "0.weight"), None if b is None else b.to(device=device, dtype=dtype), stride=strides[i])
        x = F.layer_norm(x.transpose(1, 2), (x.shape[1],), p(pre + "2.1.weight"), p(pre + "2.1.bias"), 1e-5).transpose(1, 2)
        x = F.gelu(x)
    x = x.transpose(1, 2)[0]  # T x C
    out["extractor"] = x
    x = F.layer_norm(x, (x.shape[1],), p("layer_norm.weight"), p("layer_norm.bias"), 1e-5)
    x = F.linear(x, p("post_extract_proj.weight"), p("post_extract_proj.bias"))
    out["proj"] = x
    w = pos_conv_weight(sd, dtype, device)
    D, k = x.shape[1], w.shape[2]
    c = F.conv1d(x.t().unsqueeze(0), w, p("encoder.pos_conv.0.bias"), padding=k // 2, groups=D // w.shape[1])
    if k % 2 == 0:
        c = c[:, :, :-1]  # SamePad
    x = x + F.gelu(c[0].t())
    out["pos"] = x
    H = D // 64
    T = x.shape[0]
    for li in range(n_layers(sd)):
        pre = f"encoder.layers.{li}."
        r = x
        h = F.layer_norm(x, (D,), p(pre + "self_attn_layer_norm.weight"), p(pre + "self_attn_layer_norm.bias"), 1e-5)
        q = F.linear(h, p(pre + "self_attn.q_proj.weight"), p(pre + "self_attn.q_proj.bias")) * 64 ** -0.5
        kk = F.linear(h, p(pre + "self_attn.k_proj.weight"), p(pre + "self_attn.k_proj.bias"))
        v = F.linear(h, p(pre + "self_attn.v_proj.weight"), p(pre + "self_attn.v_proj.bias"))
        q, kk, v = (t.view(T, H, 64).transpose(0, 1) for t in (q, kk, v))
        a = torch.softmax(q @ kk.transpose(1, 2), dim=-1) @ v
        a = a.transpose(0, 1).reshape(T, D)
        x = r + F.linear(a, p(pre + "self_attn.out_proj.weight"), p(pre + "self_attn.out_proj.bias"))
        r = x
        h = F.layer_norm(x, (D,), p(pre + "final_layer_norm.weight"), p(pre + "final_layer_norm.bias"), 1e-5)
        h = F.gelu(F.linear(h, p(pre + "fc1.weight"), p(pre + "fc1.bias")))
        x = r + F.linear(h, p(pre + "fc2.weight"), p(pre + "fc2.bias"))
        out[f"layer{li}"] = x
    x = F.layer_norm(x, (D,), p("encoder.layer_norm.weight"), p("encoder.layer_norm.bias"), 1e-5)
    out["final_ln"] = x
    out["emissions"] = F.linear(x, sd["w2v_encoder.proj.weight"].to(device=device, dtype=dtype),
                                sd["w2v_encoder.proj.bias"].to(device=device, dtype=dtype))
    return out


def best_path(emissions: torch.Tensor) -> List[int]:
    """flashlight's lexicon-free beam-1 step without LM: per frame the highest emission, <unk> excluded (unk_score = -inf), the lowest
    index on ties"""
    e = emissions.clone()
    e[:, UNK] = float("-inf")
    return [int(i) for i in e.argmax(dim=1)]  # torch.argmax returns the first maximal index


def get_tokens(idxs: Sequence[int], blank: int = BLANK) -> List[int]:
    """torchaudio CTCDecoder._get_tokens: collapse repeats, then drop blanks"""
    return [g for g, _ in itertools.groupby(idxs) if g != blank]


def letters(tokens: Sequence[int], vocab: Sequence[str]) -> str:
    """post_process "collapse" (utils.py:79-82) + transcribe_audiofile's strip().lower()"""
    return "".join(vocab[t] for t in tokens).replace("|", " ").strip().lower()
