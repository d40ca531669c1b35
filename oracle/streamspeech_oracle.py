"""CPU oracle: a restatement of the reference's streaming S2ST hot path in plain PyTorch fp32.

TEST INFRASTRUCTURE ONLY.  Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s
CPU-baseline legs may import this file; the product path (`streamspeech_b200/`) never does
and fails loudly when its CUDA library is missing.

Every function cites the reference file:line it restates (paths relative to the
ictnlp/StreamSpeech tree).  The restatement is pinned two ways (see oracle/gen_golden.py):
  1. against the reference's *own module classes* imported from /root/reference through
     package stubs (ChunkConformerEncoderLayer, Conv1dSubsampler, RelPositionalEncoding,
     TransformerDecoderBase, CTCTransformerUnitDecoder, UniTransformerEncoderNoEmb,
     CodeGenerator/HiFi-GAN Generator, VariancePredictor) on seeded weights -> the outputs
     are committed as tests/golden/*.npz and re-checked by `pytest -m "not gpu"`;
  2. against the two known-answer tests the reference holds for this path
     (fairseq/tests/test_espnet_multihead_attention.py:99-147,
      fairseq/tests/test_positional_encoding.py:17-59).
The Kaldi fbank arithmetic lives in a third-party dependency (torchaudio.compliance.kaldi,
reference pins torch 2.0.1 / torchaudio 2.0.2; this image has 2.11.0): it is restated from
the published algorithm and checked against the installed torchaudio function.
Blocks with no reference test (everything except rel-pos MHA / RelPositionalEncoding) are
"parity unpinned" by the reference itself; pin (1) is the only anchor for them.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

NEG_INF = float("-inf")


# --------------------------------------------------------------------------------------
# F1/F2  fbank + global CMVN
# --------------------------------------------------------------------------------------
def num_fbank_frames(n_samples: int, sample_rate: int = 16000, window_ms: int = 25, shift_ms: int = 10) -> int:
    """agent/speech_to_speech.streamspeech.agent.py:70-73 (OnlineFeatureExtractor.__call__)."""
    return max(
        0,
        math.floor((n_samples - (window_ms - shift_ms) * sample_rate / 1000) / int(shift_ms * sample_rate / 1000)),
    )


def _mel_banks(num_bins=80, padded=512, sample_freq=16000.0, low_freq=20.0, high_freq=0.0) -> torch.Tensor:
    """torchaudio/compliance/kaldi.py get_mel_banks (vtln_warp == 1.0): [num_bins, padded/2]."""
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    fft_bin_width = sample_freq / padded
    mel = lambda f: 1127.0 * math.log(1.0 + f / 700.0)
    mel_lo, mel_hi = mel(low_freq), mel(high_freq)
    delta = (mel_hi - mel_lo) / (num_bins + 1)
    b = torch.arange(num_bins).unsqueeze(1)
    left = mel_lo + b * delta
    center = mel_lo + (b + 1.0) * delta
    right = mel_lo + (b + 2.0) * delta
    melf = (1127.0 * (1.0 + fft_bin_width * torch.arange(padded // 2) / 700.0).log()).unsqueeze(0)
    up = (melf - left) / (center - left)
    down = (right - melf) / (right - center)
    return torch.max(torch.zeros(1), torch.min(up, down))


def kaldi_fbank(waveform: torch.Tensor) -> torch.Tensor:
    """`ta_kaldi.fbank(waveform, num_mel_bins=80, sample_frequency=16000)` with all other
    arguments at their defaults (fairseq/fairseq/data/audio/audio_utils.py:241-247;
    arithmetic: torchaudio/compliance/kaldi.py fbank/_get_window, SURVEY.md Appendix B).
    waveform: fp32 [n], already multiplied by 2**15.  Returns fp32 [m, 80]."""
    n = waveform.numel()
    if n < 400:
        return torch.empty(0, 80)
    m = 1 + (n - 400) // 160
    frames = waveform.as_strided((m, 400), (160, 1))
    frames = frames - frames.mean(dim=1, keepdim=True)  # remove_dc_offset
    prev = torch.cat([frames[:, :1], frames[:, :-1]], dim=1)  # replicate pad on the left
    frames = frames - 0.97 * prev  # pre-emphasis
    window = torch.hann_window(400, periodic=False, dtype=torch.float32).pow(0.85)  # povey
    frames = frames * window
    frames = F.pad(frames, (0, 112))  # 400 -> 512
    spec = torch.fft.rfft(frames).abs().pow(2.0)  # [m, 257]
    banks = F.pad(_mel_banks(), (0, 1))  # [80, 257]
    mel = torch.mm(spec, banks.T)
    return torch.max(mel, torch.tensor(torch.finfo(torch.float32).eps)).log()


def online_features(samples: torch.Tensor, gcmvn: Optional[Dict[str, np.ndarray]]) -> torch.Tensor:
    """OnlineFeatureExtractor.__call__ + transform (agent:66-98) for 16 kHz mono input
    (convert_waveform is the identity there; resampling is out of scope, SURVEY.md §8c)."""
    F_ = num_fbank_frames(samples.numel())
    eff = int(F_ * 160 + 240)
    wav = samples[:eff].float() * (2 ** 15)  # data_utils.py:85
    feat = kaldi_fbank(wav).numpy()
    if feat.shape[0] == 0:
        return torch.zeros(0, 80)
    if gcmvn is not None:
        feat = np.divide(np.subtract(feat, gcmvn["mean"]), gcmvn["std"])  # agent:96-97
    return torch.from_numpy(np.ascontiguousarray(feat, dtype=np.float32))


# --------------------------------------------------------------------------------------
# small helpers
# --------------------------------------------------------------------------------------
def _ln(x, sd, prefix):
    return F.layer_norm(x, (x.shape[-1],), sd[prefix + ".weight"], sd[prefix + ".bias"], 1e-5)


def _lin(x, sd, prefix):
    return F.linear(x, sd[prefix + ".weight"], sd.get(prefix + ".bias"))


def chunk_causal_conv1d(x, weight, bias, stride: int, groups: int, chunk_size: Optional[int]):
    """ChunkCausalConv1d.forward (researches/chunk_unity/modules/chunk_causal_conv1d.py:39-78).
    x: [B, C, L]."""
    k = weight.shape[-1]
    pad = k // 2
    if chunk_size is not None and 0 < chunk_size < 999:
        kk = pad + chunk_size
        L = x.size(-1)
        out_len = (L + 2 * pad - k) // stride + 1
        xp = F.pad(x, (pad, 0))
        xp = F.pad(xp, (0, (chunk_size - (L % chunk_size)) % chunk_size))
        un = xp.unfold(-1, kk, kk - pad)
        un = F.pad(un, (0, pad))
        bsz, nch, chunks, seq = un.size()
        un = un.transpose(1, 2).contiguous().view(-1, nch, seq)
        res = F.conv1d(un, weight, bias, stride=stride, groups=groups)
        res = res.contiguous().view(bsz, chunks, weight.shape[0], -1).transpose(1, 2)
        return res.contiguous().view(bsz, weight.shape[0], -1)[:, :, :out_len]
    xp = F.pad(F.pad(x, (pad, 0)), (0, pad))
    return F.conv1d(xp, weight, bias, stride=stride, groups=groups)


def rel_positional_encoding(T: int, d_model: int) -> torch.Tensor:
    """RelPositionalEncoding.extend_pe/forward (fairseq/fairseq/modules/positional_encoding.py:82-129):
    returns [2T-1, d_model]; row k holds relative position (T-1-k)."""
    position = torch.arange(0, T, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float32) * -(math.log(10000.0) / d_model))
    pos = torch.zeros(T, d_model)
    neg = torch.zeros(T, d_model)
    pos[:, 0::2] = torch.sin(position * div)
    pos[:, 1::2] = torch.cos(position * div)
    neg[:, 0::2] = torch.sin(-1 * position * div)
    neg[:, 1::2] = torch.cos(-1 * position * div)
    return torch.cat([torch.flip(pos, [0]), neg[1:]], dim=0)


def rel_shift(x: torch.Tensor) -> torch.Tensor:
    """RelPositionMultiHeadedAttention.rel_shift (uni_unity/modules/espnet_multihead_attention.py:133-152)."""
    zero_pad = torch.zeros((*x.size()[:3], 1), dtype=x.dtype)
    xp = torch.cat([zero_pad, x], dim=-1)
    xp = xp.view(*x.size()[:2], x.size(3) + 1, x.size(2))
    return xp[:, :, 1:].view_as(x)[:, :, :, : x.size(-1) // 2 + 1]


def chunk_mask(T: int, chunk_size: int) -> torch.Tensor:
    """buffered_chunk_mask (chunk_unity/models/s2t_conformer.py:195-213): True = masked."""
    c = max(chunk_size, 1)
    idx = torch.arange(T).unsqueeze(1)
    idx = ((idx // c + 1) * c).clamp(1, T)
    return torch.arange(T).unsqueeze(0) >= idx


def sinusoidal_table(n: int, dim: int, padding_idx: int = 1) -> torch.Tensor:
    """SinusoidalPositionalEmbedding.get_embedding (fairseq/modules/sinusoidal_positional_embedding.py:43-63)."""
    half = dim // 2
    e = math.log(10000) / (half - 1)
    e = torch.exp(torch.arange(half, dtype=torch.float) * -e)
    e = torch.arange(n, dtype=torch.float).unsqueeze(1) * e.unsqueeze(0)
    e = torch.cat([torch.sin(e), torch.cos(e)], dim=1).view(n, -1)
    e[padding_idx, :] = 0
    return e


def make_positions(tokens: torch.Tensor, pad: int) -> torch.Tensor:
    """fairseq/utils.py:256-266."""
    mask = tokens.ne(pad).int()
    return (torch.cumsum(mask, dim=1).type_as(mask) * mask).long() + pad


def mha(sd, prefix, query, key, num_heads, attn_mask=None, key_padding_mask=None):
    """ctc_unity MultiheadAttention.forward without incremental state
    (researches/ctc_unity/modules/multihead_attention.py:439-784; fast path is commented
    out there, N11).  query [Tq,B,C], key [Tk,B,Ck]; attn_mask: bool [Tq,Tk] True=masked;
    key_padding_mask bool [B,Tk]."""
    hd = query.shape[2] // num_heads
    q = _lin(query, sd, prefix + ".q_proj") * (hd ** -0.5)
    k = _lin(key, sd, prefix + ".k_proj")
    v = _lin(key, sd, prefix + ".v_proj")
    return _lin(mha_core(q, k, v, num_heads, attn_mask, key_padding_mask), sd, prefix + ".out_proj")


def mha_core(q, k, v, num_heads, attn_mask=None, key_padding_mask=None):
    """The attention of `mha` between its projections: q [Tq,B,C] (already scaled), k / v [Tk,B,C] -> [Tq,B,C], in q's dtype."""
    Tq, B, C = q.shape
    Tk = k.shape[0]
    hd = C // num_heads
    q = q.contiguous().view(Tq, B * num_heads, hd).transpose(0, 1)
    k = k.contiguous().view(Tk, B * num_heads, hd).transpose(0, 1)
    v = v.contiguous().view(Tk, B * num_heads, hd).transpose(0, 1)
    w = torch.bmm(q, k.transpose(1, 2))
    if key_padding_mask is not None:
        w = w.view(B, num_heads, Tq, Tk).masked_fill(key_padding_mask[:, None, None, :], NEG_INF).view(B * num_heads, Tq, Tk)
    if attn_mask is not None:
        w = w.masked_fill(attn_mask.unsqueeze(0), NEG_INF)
    p = F.softmax(w, dim=-1, dtype=q.dtype)  # fp32 in the reference, whose activations are fp32
    return torch.bmm(p, v).transpose(0, 1).contiguous().view(Tq, B, C)


def rel_attention_core(q, k, v, pp, bias_u, bias_v, mask=None, key_padding_mask=None):
    """The attention of RelPositionMultiHeadedAttention.forward between its projections (espnet_multihead_attention.py:186-209):
    q [B,T,H,dk], k / v [B,H,T,dk], pp [1,H,2T-1,dk] projected position rows (row k: relative position T-1-k), bias_u / bias_v [H,dk],
    mask [T,T] / key_padding_mask [B,T] True = masked -> [B,T,H*dk], in q's dtype."""
    B, T, H, dk = q.shape
    qu = (q + bias_u).transpose(1, 2)
    qv = (q + bias_v).transpose(1, 2)
    ac = torch.matmul(qu, k.transpose(-2, -1))
    bd = rel_shift(torch.matmul(qv, pp.transpose(-2, -1)))
    scores = (ac + bd) / math.sqrt(dk)
    if mask is not None:
        scores = scores.masked_fill(mask[None, None], NEG_INF)
    if key_padding_mask is not None:
        scores = scores.masked_fill(key_padding_mask[:, None, None, :], NEG_INF)
    attn = torch.softmax(scores, dim=-1)
    return torch.matmul(attn, v).transpose(1, 2).contiguous().view(B, -1, H * dk)


def depthwise_bn_silu_core(y, w, bn_mean, bn_var, bn_weight, bn_bias, conv_chunk_size):
    """Depthwise conv + BatchNorm (eval) + SiLU of ConvolutionModule.forward (conformer_layer.py:106-111): y [B,C,T], w [C,1,k]
    -> [B,C,T], in y's dtype; conv_chunk_size None = the plain padded conv, else ChunkCausalConv1d."""
    if conv_chunk_size is None:
        y = F.conv1d(y, w, None, padding=(w.shape[-1] - 1) // 2, groups=w.shape[0])
    else:
        y = chunk_causal_conv1d(y, w, None, 1, w.shape[0], conv_chunk_size)
    return F.silu(F.batch_norm(y, bn_mean, bn_var, bn_weight, bn_bias, False, 0.0, 1e-5))


# --------------------------------------------------------------------------------------
# the model
# --------------------------------------------------------------------------------------
class StreamSpeechOracle:
    def __init__(self, cfg, model_sd: Dict[str, torch.Tensor], vocoder_sd: Optional[Dict[str, torch.Tensor]] = None,
                 gcmvn=None, chunk_size: Optional[int] = 8, conv_chunk_size: Optional[int] = None, dtype: torch.dtype = torch.float32):
        """dtype: the arithmetic of every block (float64 makes a high-precision reference of the fp32 model).  Weights are taken as
        fp32 and then converted, and the position tables are computed in fp32 and then converted, so a float64 oracle sees exactly
        the numbers the fp32 model (and the engine) see; inputs are converted on entry."""
        self.cfg = cfg
        self.dtype = dtype
        self.sd = {k: (v.float().to(dtype) if v.is_floating_point() else v) for k, v in model_sd.items()}
        self.vsd = None
        if vocoder_sd is not None:
            self.vsd = {k: v.to(dtype) for k, v in _remove_weight_norm({k: v.float() for k, v in vocoder_sd.items()}).items()}
        self.gcmvn = gcmvn
        self.set_chunk(chunk_size, conv_chunk_size)

    def set_chunk(self, chunk_size: Optional[int], conv_chunk_size: Optional[int] = None):
        """agent:395-413: encoder.chunk_size = segment_ms // 40; conv chunk = 16 if >= 16 else 8 (N8)."""
        self.chunk_size = chunk_size
        if conv_chunk_size is None and chunk_size is not None:
            conv_chunk_size = 16 if chunk_size >= 16 else 8
        self.conv_chunk_size = conv_chunk_size

    # ---- E1 Conv1dSubsampler (chunk_unity/modules/convolution.py:75-89)
    def subsample(self, feats: torch.Tensor, lengths: torch.Tensor):
        x = feats.to(self.dtype).transpose(1, 2).contiguous()  # B x C x T
        for i in range(2):
            w = self.sd[f"encoder.subsample.conv_layers.{i}.weight"]
            b = self.sd[f"encoder.subsample.conv_layers.{i}.bias"]
            if self.conv_chunk_size is None:  # plain nn.Conv1d(padding=k//2) when the model has no chunk
                x = F.conv1d(x, w, b, stride=2, padding=w.shape[-1] // 2)
            else:
                x = chunk_causal_conv1d(x, w, b, 2, 1, self.conv_chunk_size)
            x = F.glu(x, dim=1)
        out_len = lengths.clone()
        for _ in range(2):
            out_len = ((out_len.float() - 1) / 2 + 1).floor().long()
        return x.transpose(1, 2).transpose(0, 1).contiguous(), out_len  # T x B x C

    # ---- E3 FeedForwardModule (chunk_unity/modules/conformer_layer.py:152-164)
    def _ffn(self, x, p):
        y = _ln(x, self.sd, p + ".layer_norm")
        y = F.silu(_lin(y, self.sd, p + ".w_1"))  # N5: SiLU(inplace=<int>) is plain SiLU
        return _lin(y, self.sd, p + ".w_2")

    # ---- E4 RelPositionMultiHeadedAttention.forward (uni_unity/.../espnet_multihead_attention.py:154-209)
    def _rel_mha(self, x, pos_emb, p, mask, key_padding_mask):
        H = self.cfg.enc_heads
        T, B, C = x.shape
        dk = C // H
        xb = x.transpose(0, 1)
        q = _lin(xb, self.sd, p + ".linear_q").view(B, -1, H, dk)
        k = _lin(xb, self.sd, p + ".linear_k").view(B, -1, H, dk).transpose(1, 2)
        v = _lin(xb, self.sd, p + ".linear_v").view(B, -1, H, dk).transpose(1, 2)
        pe = pos_emb.transpose(0, 1)  # [1, 2T-1, C]
        pp = F.linear(pe, self.sd[p + ".linear_pos.weight"]).view(pe.size(0), -1, H, dk).transpose(1, 2)
        o = rel_attention_core(q, k, v, pp, self.sd[p + ".pos_bias_u"], self.sd[p + ".pos_bias_v"], mask, key_padding_mask)
        return _lin(o, self.sd, p + ".linear_out").transpose(0, 1)

    # ---- E5 ConvolutionModule.forward (conformer_layer.py:94-119)
    def _conv_module(self, x, p):
        y = _ln(x, self.sd, p + ".layer_norm").transpose(1, 2)  # B C T
        y = F.conv1d(y, self.sd[p + ".pointwise_conv1.weight"])
        y = F.glu(y, dim=1)
        y = depthwise_bn_silu_core(y, self.sd[p + ".depthwise_conv.weight"], self.sd[p + ".batch_norm.running_mean"],
                                   self.sd[p + ".batch_norm.running_var"], self.sd[p + ".batch_norm.weight"], self.sd[p + ".batch_norm.bias"],
                                   self.conv_chunk_size)
        y = F.conv1d(y, self.sd[p + ".pointwise_conv2.weight"])
        return y.transpose(1, 2)

    # ---- E6 ChunkConformerEncoderLayer.forward (conformer_layer.py:254-312)
    def conformer_layer(self, x, i, pos_emb, mask, key_padding_mask):
        p = f"encoder.conformer_layers.{i}"
        x = self._ffn(x, p + ".ffn1") * 0.5 + x
        res = x
        y = _ln(x, self.sd, p + ".self_attn_layer_norm")
        x = self._rel_mha(y, pos_emb, p + ".self_attn", mask, key_padding_mask) + res
        res = x
        x = res + self._conv_module(x.transpose(0, 1), p + ".conv_module").transpose(0, 1)
        res = x
        x = self._ffn(x, p + ".ffn2") * 0.5 + res
        return _ln(x, self.sd, p + ".final_layer_norm")

    # ---- E2 ChunkS2TConformerEncoder._forward (chunk_unity/models/s2t_conformer.py:111-163)
    def encoder(self, feats: torch.Tensor, lengths: torch.Tensor, return_layers: bool = False):
        """feats [B,F,80], lengths [B] -> dict like the fairseq encoder_out."""
        x, out_len = self.subsample(feats, lengths)
        T, B, C = x.shape
        pad_mask = torch.arange(T).unsqueeze(0) >= out_len.unsqueeze(1)  # lengths_to_padding_mask
        x = math.sqrt(C) * x
        pos = rel_positional_encoding(T, C).to(self.dtype).unsqueeze(1)  # [2T-1,1,C]
        x = _lin(x, self.sd, "encoder.linear")
        mask = chunk_mask(T, self.chunk_size) if self.chunk_size is not None else None
        layers = []
        for i in range(self.cfg.enc_layers):
            x = self.conformer_layer(x, i, pos, mask, pad_mask)
            if return_layers:
                layers.append(x)
        return {"encoder_out": [x], "encoder_padding_mask": [pad_mask] if pad_mask.any() else [],
                "encoder_states": layers, "out_lengths": out_len}

    # ---- C1 CTCDecoder.generate (agent/ctc_decoder.py:40-111)
    def ctc_logits(self, name: str, enc_out: torch.Tensor) -> torch.Tensor:
        return _lin(enc_out.to(self.dtype), self.sd, f"{name}_decoder.proj").transpose(0, 1)  # B x T x V

    def ctc_greedy(self, name: str, enc_out: torch.Tensor):
        lprobs = F.log_softmax(self.ctc_logits(name, enc_out), dim=-1)
        lprobs[:, :, self.cfg.pad] = NEG_INF
        lprobs[:, :, self.cfg.unk] = NEG_INF
        _, pred = torch.max(lprobs, dim=2)
        out = []
        for b in range(pred.size(0)):
            toks = pred[b].int().tolist()
            toks_out, index = ctc_collapse(toks, blank=0, pad=self.cfg.pad)
            out.append({"tokens": toks_out, "index": index, "org_tokens": toks})
        return out

    # ---- M2 TransformerDecoderBase.extract_features_scriptable (ctc_unity/modules/transformer_decoder.py:257-403)
    def _decoder_layer(self, x, enc, prefix, heads, self_mask, self_pad, enc_pad):
        """TransformerDecoderLayerBase.forward, normalize_before=True (transformer_layer.py:388-551)."""
        res = x
        y = _ln(x, self.sd, prefix + ".self_attn_layer_norm")
        x = res + mha(self.sd, prefix + ".self_attn", y, y, heads, self_mask, self_pad)
        res = x
        y = _ln(x, self.sd, prefix + ".encoder_attn_layer_norm")
        x = res + mha(self.sd, prefix + ".encoder_attn", y, enc, heads, None, enc_pad)
        res = x
        y = _ln(x, self.sd, prefix + ".final_layer_norm")
        y = _lin(F.relu(_lin(y, self.sd, prefix + ".fc1")), self.sd, prefix + ".fc2")
        return res + y

    def mt_features(self, prev_tokens: torch.Tensor, enc_out: torch.Tensor, enc_pad=None) -> torch.Tensor:
        """prev_tokens [B,L] -> features [B,L,512] (after the final layer_norm)."""
        c = self.cfg
        B, L = prev_tokens.shape
        pfx = "target_unigram_decoder"
        enc_out = enc_out.to(self.dtype)
        table = sinusoidal_table(max(1024, c.pad + 1 + L + 1), c.mt_dim, c.pad).to(self.dtype)
        pos = table.index_select(0, make_positions(prev_tokens, c.pad).view(-1)).view(B, L, -1)
        x = math.sqrt(c.mt_dim) * F.embedding(prev_tokens, self.sd[pfx + ".embed_tokens.weight"]) + pos
        x = x.transpose(0, 1)
        self_pad = prev_tokens.eq(c.pad) if prev_tokens.eq(c.pad).any() else None
        causal = torch.triu(torch.ones(L, L, dtype=torch.bool), 1)
        for i in range(c.mt_layers):
            x = self._decoder_layer(x, enc_out, f"{pfx}.layers.{i}", c.mt_heads, causal, self_pad, enc_pad)
        x = _ln(x, self.sd, pfx + ".layer_norm")
        return x.transpose(0, 1)

    def mt_logits(self, prev_tokens, enc_out, enc_pad=None):
        return F.linear(self.mt_features(prev_tokens, enc_out, enc_pad), self.sd["target_unigram_decoder.output_projection.weight"])

    # ---- M1 greedy specialisation (beam=1) of SequenceGenerator.generate_decoder
    #      (agent/sequence_generator.py:165-582, fairseq/sequence_generator.py:630-739, search.py:110-146)
    def mt_greedy(self, enc_out: torch.Tensor, prefix: Optional[List[int]], max_new_tokens: int,
                  max_len_b: int = 100, max_decoder_positions: int = 1024, min_len: int = 1) -> List[int]:
        """Returns the finalized hypothesis tokens INCLUDING the trailing eos (as `finalize_hypos` does)."""
        c = self.cfg
        prefix = list(prefix) if prefix is not None else []
        start = len(prefix)
        if max_new_tokens == -1:
            max_len = min(int(0 * enc_out.size(0) + max_len_b), max_decoder_positions - 1)
        else:
            max_len = start + max_new_tokens
        assert min_len <= max_len
        tokens = [c.eos] + prefix
        score = 0.0
        for step in range(start, max_len + 1):
            logits = self.mt_logits(torch.tensor([tokens], dtype=torch.long), enc_out)[:, -1, :]
            lprobs = F.log_softmax(logits, dim=-1)[0]
            lprobs[lprobs != lprobs] = NEG_INF
            lprobs[c.pad] = NEG_INF
            if step >= max_len:
                lprobs[: c.eos] = NEG_INF
                lprobs[c.eos + 1:] = NEG_INF
            elif step < min_len:
                lprobs[c.eos] = NEG_INF
            if step > 0:
                lprobs = lprobs + score  # BeamSearch.step adds the cumulative score
            best = int(torch.topk(lprobs, 2)[1][0])
            score = float(lprobs[best])
            if best == c.eos:
                return tokens[1:] + [c.eos]
            tokens.append(best)
        raise AssertionError("unreachable: eos is forced at step == max_len")

    # ---- M1 with incremental states (use_incremental_states=True: S2TT / ASR agents; SURVEY.md N12)
    def mt_incremental_state(self):
        """fresh `incremental_states[0]` of SequenceGenerator (agent/sequence_generator.py:180-195): per layer the self-attention
        prev_key / prev_value and the encoder-attention prev_key / prev_value."""
        L = self.cfg.mt_layers
        return {"self_k": [None] * L, "self_v": [None] * L, "cross_k": [None] * L, "cross_v": [None] * L}

    def _mt_step_incremental(self, state, token: int, step: int, enc_out: torch.Tensor) -> torch.Tensor:
        """One `decoder.forward(tokens[:, :step+1], encoder_out, incremental_state)` (transformer_decoder.py:257-403): only the
        LAST token is embedded (:305-308) at sinusoidal position pad + 1 + step; self-attention appends its k / v to the saved
        state (multihead_attention.py:599-640, no mask); encoder attention projects only encoder rows beyond the cached
        prev_key length and concatenates (transformer_layer.py:492-505, static_kv otherwise).  Returns logits [vocab]."""
        c = self.cfg
        pfx = "target_unigram_decoder"
        enc_out = enc_out.to(self.dtype)
        table = sinusoidal_table(max(1024, c.pad + 1 + step + 2), c.mt_dim, c.pad).to(self.dtype)
        p = c.pad if token == c.pad else c.pad + 1 + step
        x = math.sqrt(c.mt_dim) * self.sd[pfx + ".embed_tokens.weight"][token] + table[p]
        x = x.view(1, 1, -1)
        H, hd = c.mt_heads, c.mt_dim // c.mt_heads

        def attend(q, k, v, prefix):
            q = (q * hd ** -0.5).view(1, H, hd).transpose(0, 1)         # [H,1,hd]
            kk = k.view(-1, H, hd).transpose(0, 1)                       # [H,n,hd]
            vv = v.view(-1, H, hd).transpose(0, 1)
            w = F.softmax(torch.bmm(q, kk.transpose(1, 2)), dim=-1, dtype=torch.float32)
            a = torch.bmm(w, vv).transpose(0, 1).contiguous().view(1, 1, c.mt_dim)
            return _lin(a, self.sd, prefix + ".out_proj")

        for i in range(c.mt_layers):
            lp = f"{pfx}.layers.{i}"
            res = x
            y = _ln(x, self.sd, lp + ".self_attn_layer_norm")
            k = _lin(y, self.sd, lp + ".self_attn.k_proj").view(1, -1)
            v = _lin(y, self.sd, lp + ".self_attn.v_proj").view(1, -1)
            state["self_k"][i] = k if state["self_k"][i] is None else torch.cat([state["self_k"][i], k], 0)
            state["self_v"][i] = v if state["self_v"][i] is None else torch.cat([state["self_v"][i], v], 0)
            x = res + attend(_lin(y, self.sd, lp + ".self_attn.q_proj"), state["self_k"][i], state["self_v"][i], lp + ".self_attn")
            res = x
            y = _ln(x, self.sd, lp + ".encoder_attn_layer_norm")
            have = 0 if state["cross_k"][i] is None else state["cross_k"][i].size(0)
            if enc_out.size(0) > have:  # static_kv = False: only the new encoder rows are projected and appended
                e = enc_out[have:, 0]
                k = _lin(e, self.sd, lp + ".encoder_attn.k_proj")
                v = _lin(e, self.sd, lp + ".encoder_attn.v_proj")
                state["cross_k"][i] = k if have == 0 else torch.cat([state["cross_k"][i], k], 0)
                state["cross_v"][i] = v if have == 0 else torch.cat([state["cross_v"][i], v], 0)
            x = res + attend(_lin(y, self.sd, lp + ".encoder_attn.q_proj"), state["cross_k"][i], state["cross_v"][i], lp + ".encoder_attn")
            res = x
            y = _ln(x, self.sd, lp + ".final_layer_norm")
            x = res + _lin(F.relu(_lin(y, self.sd, lp + ".fc1")), self.sd, lp + ".fc2")
        x = _ln(x, self.sd, pfx + ".layer_norm")
        return F.linear(x.view(-1), self.sd[pfx + ".output_projection.weight"])

    def mt_greedy_incremental(self, state, enc_out: torch.Tensor, prefix: Optional[List[int]], max_new_tokens: int, max_len_full: int,
                              min_len: int = 1) -> List[int]:
        """generate_decoder (agent/sequence_generator.py:165-582) with use_incremental_states=True and beam 1: `state` persists
        across calls; step `start` feeds tokens[start] = the last prefix token AGAIN (it was fed by the previous call's final
        step), every step feeds exactly one token.  max_len_full = max_len when max_new_tokens == -1."""
        c = self.cfg
        prefix = list(prefix) if prefix is not None else []
        start = len(prefix)
        max_len = max_len_full if max_new_tokens == -1 else start + max_new_tokens
        assert min_len <= max_len
        tokens = [c.eos] + prefix
        for step in range(start, max_len + 1):
            logits = self._mt_step_incremental(state, tokens[step], step, enc_out)
            lprobs = F.log_softmax(logits, dim=-1)
            lprobs[lprobs != lprobs] = NEG_INF
            lprobs[c.pad] = NEG_INF
            if step >= max_len:
                lprobs[: c.eos] = NEG_INF
                lprobs[c.eos + 1:] = NEG_INF
            elif step < min_len:
                lprobs[c.eos] = NEG_INF
            best = int(torch.topk(lprobs, 2)[1][0])
            if best == c.eos:
                return tokens[1:] + [c.eos]
            tokens.append(best)
        raise AssertionError("unreachable: eos is forced at step == max_len")

    # ---- T1 UniTransformerEncoderNoEmb.forward (ctc_unity/modules/transformer_encoder.py:32-77)
    def t2u_encoder(self, x: torch.Tensor, pad_mask: Optional[torch.Tensor]) -> torch.Tensor:
        """x [S,B,512] -> [S,B,512]."""
        c = self.cfg
        x = x.to(self.dtype)
        S = x.size(0)
        causal = torch.triu(torch.ones(S, S, dtype=torch.bool), 1) if c.uni_encoder else None
        for i in range(c.t2u_layers):
            p = f"synthesizer_encoder.layers.{i}"
            res = x
            y = _ln(x, self.sd, p + ".self_attn_layer_norm")
            x = res + mha(self.sd, p + ".self_attn", y, y, c.unit_heads, causal, pad_mask)
            res = x
            y = _ln(x, self.sd, p + ".final_layer_norm")
            x = res + _lin(F.relu(_lin(y, self.sd, p + ".fc1")), self.sd, p + ".fc2")
        return _ln(x, self.sd, "synthesizer_encoder.layer_norm")

    # ---- U1 CTCTransformerUnitDecoder.extract_features_scriptable / forward
    #      (ctc_unity/modules/ctc_transformer_unit_decoder.py:53-260)
    def unit_decoder_logits(self, t2u_out: torch.Tensor, pad_mask: Optional[torch.Tensor]) -> torch.Tensor:
        """t2u_out [S,B,512] -> logits [B, 25*S, 1005]."""
        c = self.cfg
        t2u_out = t2u_out.to(self.dtype)
        S, B, E = t2u_out.shape
        R = c.ctc_upsample_rate
        x = t2u_out.unsqueeze(1).repeat(1, R, 1, 1).contiguous().view(S * R, B, E)
        # N1: positions are computed from x[:, :, 0] viewed as [bsz=T', seq=B]
        first = x[:, :, 0]
        table = sinusoidal_table(max(1200, c.pad + 1 + B + 1), E, c.pad).to(self.dtype)
        pos = table.index_select(0, make_positions(first, c.pad).view(-1)).view(S * R, B, -1)
        x = x + pos
        self_pad = None
        if pad_mask is not None and pad_mask.any():
            self_pad = pad_mask.unsqueeze(2).repeat(1, 1, R).contiguous().view(B, S * R)
        L = S * R
        causal = torch.triu(torch.ones(L, L, dtype=torch.bool), 1)
        enc_pad = pad_mask if (pad_mask is not None and pad_mask.any()) else None
        for i in range(c.unit_layers):
            x = self._decoder_layer(x, t2u_out, f"decoder.layers.{i}", c.unit_heads, causal, self_pad, enc_pad)
        x = _ln(x, self.sd, "decoder.layer_norm").transpose(0, 1)
        return F.linear(x, self.sd["decoder.output_projection.weight"])

    # ---- U2 CTCSequenceGenerator.generate (agent/ctc_generator.py:41-123); offline variant also masks eos (N3)
    def unit_ctc_greedy(self, logits: torch.Tensor, mask_eos: bool = False):
        c = self.cfg
        lprobs = F.log_softmax(logits.to(self.dtype), dim=-1)
        lprobs[:, :, c.pad] = NEG_INF
        lprobs[:, :, c.unk] = NEG_INF
        if mask_eos:
            lprobs[:, :, c.eos] = NEG_INF
        _, pred = torch.max(lprobs, dim=2)
        out = []
        for b in range(pred.size(0)):
            toks = pred[b].int().tolist()
            hyp, _ = ctc_collapse(toks, blank=c.unit_blank, pad=c.pad)
            out.append({"tokens": hyp, "org_tokens": toks})
        return out

    # ---- V1 CodeGenerator.forward + VariancePredictor (agent/tts/codehifigan.py:56-95, fastspeech2.py:117-151)
    def dur_predict(self, emb: torch.Tensor) -> torch.Tensor:
        """emb [1,U,128] -> log-dur [1,U]."""
        v = self.vsd
        pad = (v["dur_predictor.conv1.0.weight"].shape[-1] - 1) // 2
        x = F.relu(F.conv1d(emb.transpose(1, 2), v["dur_predictor.conv1.0.weight"], v["dur_predictor.conv1.0.bias"], padding=pad)).transpose(1, 2)
        x = _ln(x, v, "dur_predictor.ln1")
        x = F.relu(F.conv1d(x.transpose(1, 2), v["dur_predictor.conv2.0.weight"], v["dur_predictor.conv2.0.bias"], padding=1)).transpose(1, 2)
        x = _ln(x, v, "dur_predictor.ln2")
        return _lin(x, v, "dur_predictor.proj").squeeze(2)

    def vocoder(self, codes: List[int], dur_prediction: bool = True):
        """CodeHiFiGANVocoderWithDur.forward (agent/tts/vocoder.py:48-60): returns (wav [N*hop], dur [1,U])."""
        v = self.vsd
        code = torch.tensor([c for c in codes if c >= 0], dtype=torch.long).view(1, -1)
        x = F.embedding(code, v["dict.weight"]).transpose(1, 2)  # 1 x 128 x U
        dur = None
        if dur_prediction:
            log_dur = self.dur_predict(x.transpose(1, 2))
            dur = torch.clamp(torch.round(torch.exp(log_dur) - 1).long(), min=1)
            x = torch.repeat_interleave(x, dur.view(-1), dim=2)
        return self.hifigan(x).squeeze(), dur

    # ---- V2 Generator.forward / ResBlock.forward (fairseq/models/text_to_speech/hifigan.py:95-102,154-170)
    def hifigan(self, x: torch.Tensor) -> torch.Tensor:
        v, vc = self.vsd, self.cfg.vocoder
        x = F.conv1d(x, v["conv_pre.weight"], v["conv_pre.bias"], padding=3)
        nk = len(vc.resblock_kernel_sizes)
        for i, (u, k) in enumerate(zip(vc.upsample_rates, vc.upsample_kernel_sizes)):
            x = F.leaky_relu(x, 0.1)
            x = F.conv_transpose1d(x, v[f"ups.{i}.weight"], v[f"ups.{i}.bias"], stride=u, padding=(k - u) // 2)
            xs = None
            for j in range(nk):
                rb = i * nk + j
                rk, dils = vc.resblock_kernel_sizes[j], vc.resblock_dilation_sizes[j]
                y = x
                for m, d in enumerate(dils):
                    t = F.leaky_relu(y, 0.1)
                    t = F.conv1d(t, v[f"resblocks.{rb}.convs1.{m}.weight"], v[f"resblocks.{rb}.convs1.{m}.bias"], dilation=d, padding=(rk * d - d) // 2)
                    t = F.leaky_relu(t, 0.1)
                    t = F.conv1d(t, v[f"resblocks.{rb}.convs2.{m}.weight"], v[f"resblocks.{rb}.convs2.{m}.bias"], padding=(rk - 1) // 2)
                    y = t + y
                xs = y if xs is None else xs + y
            x = xs / nk
        x = F.leaky_relu(x)  # default slope 0.01 (hifigan.py:166)
        x = F.conv1d(x, v["conv_post.weight"], v["conv_post.bias"], padding=3)
        return torch.tanh(x)


def ctc_collapse(toks: List[int], blank: int, pad: int) -> Tuple[List[int], List[int]]:
    """_ctc_postprocess / _ctc_postprocess_index (agent/ctc_decoder.py:70-88)."""
    hyp, index = [], []
    for i, v in enumerate(toks):
        if i == 0 or v != toks[i - 1]:
            if v != blank and v != pad:
                hyp.append(v)
                index.append(i)
    return hyp, index


def _remove_weight_norm(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """`remove_weight_norm` at load (agent/tts/vocoder.py:45): w = g * v / ||v|| (norm over all dims but 0)."""
    out = dict(sd)
    for k in list(sd.keys()):
        if k.endswith(".weight_g"):
            base = k[: -len(".weight_g")]
            g, v = sd[k], sd[base + ".weight_v"]
            norm = v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))
            out[base + ".weight"] = v * (g / norm)
            del out[k], out[base + ".weight_v"]
    return out
