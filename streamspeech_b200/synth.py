"""Seeded synthetic checkpoints with the reference's exact state-dict keys and shapes.

There is no StreamSpeech `.pt`, no vocoder `g_00500000` and no network in the build or
GPU containers (SURVEY.md §8c), so parity and throughput runs use random-init weights of
the reference architecture.  Keys/shapes follow the reference modules
(`StreamSpeechModel.build_model`, researches/ctc_unity/models/streamspeech_model.py:182-258;
`CodeGenerator`, agent/tts/codehifigan.py:9-33) and are verified by loading the result
with `load_state_dict(strict=True)` into the real reference classes in oracle/gen_golden.py.

Plain xavier init makes the decoders degenerate (CTC never blank, MT never EOS, every unit
distinct), so a handful of *calibration* knobs bias the blank/EOS rows to give token rates
in the range of a trained model.  Both the CPU oracle and the CUDA engine load the same
tensors, so calibration cannot help or hurt parity.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch

from .config import ModelConfig, VocoderConfig


_CAL_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "synth_calibration.npz")


@dataclass
class Calibration:
    """Rows measured by oracle/calibrate_synth.py for ModelConfig() + seed 0 (committed npz)."""

    # The random NAR unit decoder emits ~1 unit per MT token (all 25 upsampled positions agree), a trained
    # one ~12 with durations 1-3; to keep the vocoder workload realistic (~50 frames per output second,
    # ~1 s of output per source second) the duration predictor is biased towards long units instead.
    dur_log_mean: float = 2.2  # mean of the predicted log(dur+1)
    dur_log_std: float = 0.35
    rows_file: str = _CAL_FILE


def _xavier(g, out_f, in_f, *rest, gain=1.0):
    fan_in = in_f
    fan_out = out_f
    for r in rest:
        fan_in *= r
        fan_out *= r
    a = gain * math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand((out_f, in_f, *rest), generator=g) * 2 - 1) * a


def _normal(g, shape, std):
    return torch.randn(shape, generator=g) * std


def _ln(g, sd, prefix, dim):
    sd[prefix + ".weight"] = 1.0 + 0.1 * torch.randn(dim, generator=g)
    sd[prefix + ".bias"] = 0.05 * torch.randn(dim, generator=g)


# The MT decoder ties its input and output embeddings; with unit-norm random rows the 22.6x-scaled
# input embedding dominates the residual stream and the arg-max simply copies the previous token
# forever (never EOS).  Tiny rows leave the sinusoidal position signal dominant instead, so greedy
# decoding yields a varied, position-driven token stream; EOS is a single positional feature
# (sin with period ~300 positions) whose gain `mt_eos_b` is calibrated so sentences end after ~30 tokens.
MT_EMBED_SCALE = 0.01
MT_EOS_DIM = 150
# ... and the decoder's final LayerNorm carries a gain so that the logits (features @ tiny rows) have a spread of
# ~0.15 instead of ~0.002: with log-probs near -8.7 an fp32 ulp is 1e-6, and logit gaps of 1e-5 would make the
# arg-max depend on summation order (a real model's logits span several units).
MT_FEATURE_GAIN = 64.0
# Read-out rows only look at the 12 highest-frequency sin/cos positional features, which decorrelate
# within 2-3 positions (most of the 256 frequencies are nearly constant over a sentence), and the
# cross-attention branches of the two decoders are initialised very small so that the arg-max of an
# already emitted token/unit does not flip when the encoder output grows by a chunk (the reference
# agent assumes unit-prefix stability, SURVEY.md N6; a trained model provides it, a random one must
# be built to).
READOUT_FREQS = 12
CROSS_ATTN_GAIN = {"target_unigram_decoder": 0.05, "decoder": 0.03}


def _positional_readout(g, vocab, dim, scale):
    half = dim // 2
    E = torch.zeros(vocab, dim)
    E[:, :READOUT_FREQS] = torch.randn((vocab, READOUT_FREQS), generator=g) * scale
    E[:, half:half + READOUT_FREQS] = torch.randn((vocab, READOUT_FREQS), generator=g) * scale
    return E


# Residual-branch output projections are initialised small (as trained nets behave): with unit
# gain a deep random pre-LN stack forgets its input within a few layers and every frame/token
# gets the same argmax, which would make the streaming policy degenerate.
BRANCH_GAIN = 0.3


def _linear(g, sd, prefix, out_f, in_f, bias=True, gain=1.0):
    sd[prefix + ".weight"] = _xavier(g, out_f, in_f, gain=gain)
    if bias:
        sd[prefix + ".bias"] = _normal(g, (out_f,), 0.02)


def make_model_state_dict(cfg: ModelConfig, seed: int = 0, calibration: Optional[Calibration] = Calibration()) -> Dict[str, torch.Tensor]:
    """`calibration=None` gives the raw seeded init (what oracle/calibrate_synth.py starts from)."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    D, F = cfg.enc_dim, cfg.enc_ffn
    # --- Conv1d subsampler (chunk_unity/modules/convolution.py:45-58)
    mid = cfg.conv_channels
    sd["encoder.subsample.conv_layers.0.weight"] = _xavier(g, mid, cfg.feat_dim, cfg.conv_kernel)
    sd["encoder.subsample.conv_layers.0.bias"] = _normal(g, (mid,), 0.02)
    sd["encoder.subsample.conv_layers.1.weight"] = _xavier(g, 2 * D, mid // 2, cfg.conv_kernel)
    sd["encoder.subsample.conv_layers.1.bias"] = _normal(g, (2 * D,), 0.02)
    _linear(g, sd, "encoder.linear", D, D)
    for i in range(cfg.enc_layers):
        p = f"encoder.conformer_layers.{i}"
        for ffn in ("ffn1", "ffn2"):
            _ln(g, sd, f"{p}.{ffn}.layer_norm", D)
            _linear(g, sd, f"{p}.{ffn}.w_1", F, D)
            _linear(g, sd, f"{p}.{ffn}.w_2", D, F, gain=BRANCH_GAIN)
        _ln(g, sd, f"{p}.self_attn_layer_norm", D)
        dk = D // cfg.enc_heads
        sd[f"{p}.self_attn.pos_bias_u"] = _xavier(g, cfg.enc_heads, dk)
        sd[f"{p}.self_attn.pos_bias_v"] = _xavier(g, cfg.enc_heads, dk)
        for n in ("linear_q", "linear_k", "linear_v", "linear_out"):
            _linear(g, sd, f"{p}.self_attn.{n}", D, D, gain=BRANCH_GAIN if n == "linear_out" else 1.0)
        _linear(g, sd, f"{p}.self_attn.linear_pos", D, D, bias=False)
        _ln(g, sd, f"{p}.conv_module.layer_norm", D)
        sd[f"{p}.conv_module.pointwise_conv1.weight"] = _xavier(g, 2 * D, D, 1)
        sd[f"{p}.conv_module.depthwise_conv.weight"] = _normal(g, (D, 1, cfg.dw_kernel), 1.0 / math.sqrt(cfg.dw_kernel))
        sd[f"{p}.conv_module.batch_norm.weight"] = 1.0 + 0.1 * torch.randn(D, generator=g)
        sd[f"{p}.conv_module.batch_norm.bias"] = 0.05 * torch.randn(D, generator=g)
        sd[f"{p}.conv_module.batch_norm.running_mean"] = 0.1 * torch.randn(D, generator=g)
        sd[f"{p}.conv_module.batch_norm.running_var"] = 0.5 + torch.rand(D, generator=g)
        sd[f"{p}.conv_module.batch_norm.num_batches_tracked"] = torch.tensor(1000)
        sd[f"{p}.conv_module.pointwise_conv2.weight"] = _xavier(g, D, D, 1, gain=BRANCH_GAIN)
        _ln(g, sd, f"{p}.final_layer_norm", D)

    # --- CTC heads: one Linear each (fairseq/models/speech_to_speech/modules/ctc_decoder.py:11-18)
    for name, V in (("source_unigram", cfg.src_vocab), ("ctc_target_unigram", cfg.tgt_vocab)):
        w = _xavier(g, V, D)
        b = _normal(g, (V,), 0.02)
        # index 0 (<s>) is the CTC blank (agent/ctc_decoder.py:72-76); its bias is calibrated below
        sd[f"{name}_decoder.proj.weight"] = w
        sd[f"{name}_decoder.proj.bias"] = b

    def dec_layer(prefix, dim, ffn, kdim, cross=True):
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            _linear(g, sd, f"{prefix}.self_attn.{n}", dim, dim, gain=BRANCH_GAIN if n == "out_proj" else 1.0)
        _ln(g, sd, f"{prefix}.self_attn_layer_norm", dim)
        if cross:
            _linear(g, sd, f"{prefix}.encoder_attn.k_proj", dim, kdim)
            _linear(g, sd, f"{prefix}.encoder_attn.v_proj", dim, kdim)
            _linear(g, sd, f"{prefix}.encoder_attn.q_proj", dim, dim)
            _linear(g, sd, f"{prefix}.encoder_attn.out_proj", dim, dim, gain=CROSS_ATTN_GAIN.get(prefix.split(".")[0], BRANCH_GAIN))
            _ln(g, sd, f"{prefix}.encoder_attn_layer_norm", dim)
        _linear(g, sd, f"{prefix}.fc1", ffn, dim)
        _linear(g, sd, f"{prefix}.fc2", dim, ffn, gain=BRANCH_GAIN)
        _ln(g, sd, f"{prefix}.final_layer_norm", dim)

    # --- first-pass MT decoder (target_unigram), tied in/out embedding
    M = cfg.mt_dim
    emb = _positional_readout(g, cfg.tgt_vocab, M, M ** -0.5 * MT_EMBED_SCALE)
    emb[cfg.pad].zero_()
    sd["target_unigram_decoder.embed_tokens.weight"] = emb
    sd["target_unigram_decoder.output_projection.weight"] = emb
    for i in range(cfg.mt_layers):
        dec_layer(f"target_unigram_decoder.layers.{i}", M, cfg.mt_ffn, D)
    _ln(g, sd, "target_unigram_decoder.layer_norm", M)
    sd["target_unigram_decoder.layer_norm.weight"] *= MT_FEATURE_GAIN
    sd["target_unigram_decoder.layer_norm.bias"] *= MT_FEATURE_GAIN

    # --- T2U encoder (UniTransformerEncoderNoEmb)
    for i in range(cfg.t2u_layers):
        dec_layer(f"synthesizer_encoder.layers.{i}", cfg.unit_dim, cfg.unit_ffn, cfg.unit_dim, cross=False)
    _ln(g, sd, "synthesizer_encoder.layer_norm", cfg.unit_dim)

    # --- NAR CTC unit decoder, tied in/out embedding (StackedEmbedding num_stacked=1)
    U = cfg.unit_dim
    uemb = _positional_readout(g, cfg.unit_vocab, U, U ** -0.5)
    uemb[cfg.pad].zero_()
    sd["decoder.embed_tokens.weight"] = uemb
    sd["decoder.output_projection.weight"] = uemb
    for i in range(cfg.unit_layers):
        dec_layer(f"decoder.layers.{i}", U, cfg.unit_ffn, U)
    _ln(g, sd, "decoder.layer_norm", U)
    if calibration is not None and os.path.exists(calibration.rows_file):
        rows = np.load(calibration.rows_file)
        if "unit_blank_row" in rows and rows["unit_blank_row"].shape[0] == U and M > MT_EOS_DIM:
            for name in ("source_unigram", "ctc_target_unigram"):
                sd[f"{name}_decoder.proj.bias"][cfg.bos] += float(rows[f"{name}_blank_bias_delta"])
            emb[cfg.eos].zero_()
            emb[cfg.eos, MT_EOS_DIM] = float(rows["mt_eos_b"])
            uemb[cfg.unit_blank] = torch.from_numpy(rows["unit_blank_row"])
    return {k: v.contiguous().float() if v.is_floating_point() else v for k, v in sd.items()}


# UnitY's synthetic unit decoder: its cross-attention branch at full branch gain, so that samples emit different units (the
# StreamSpeech decoder's is tiny for prefix stability, which an offline search does not need), and eos read from one slow positional
# feature (period ~1400 steps, rising over the first few hundred) plus the T2U states: with UNITY_EOS_GAIN some samples end within
# the first tens of units and others run to the forced eos at max_len.
UNITY_CROSS_GAIN = 1.0
UNITY_EOS_DIM = 150
UNITY_EOS_GAIN = 6.0
# ... and the MT decoder's eos output row (tied with its input row) scaled as oracle.mt_beam_oracle.early_eos_state_dict does, so that
# MT hypotheses end after 9-16 tokens at different lengths within a batch (the StreamSpeech rows run to max_len_b_mt) and the T2U
# encoder sees padded positions
UNITY_MT_EOS_SCALE = -0.15


def make_unity_state_dict(cfg: ModelConfig, seed: int = 0, eos_gain: float = UNITY_EOS_GAIN) -> Dict[str, torch.Tensor]:
    """A seeded UnitY (unity_conformer_modified) state dict at `cfg`'s dimensions (ModelConfig.unity_default(): the released
    checkpoints'): StreamSpeech's encoder, MT decoder and T2U encoder without the CTC heads, and the autoregressive unit decoder
    over cfg.unit_vocab symbols (4 specials + units, no blank) with its tied output projection."""
    assert cfg.unity
    sd = make_model_state_dict(cfg, seed=seed)
    for k in [k for k in sd if k.startswith(("source_unigram_decoder.", "ctc_target_unigram_decoder."))]:
        del sd[k]
    g = torch.Generator().manual_seed(seed + 7919)
    U = cfg.unit_dim
    for i in range(cfg.unit_layers):
        sd[f"decoder.layers.{i}.encoder_attn.out_proj.weight"] = _xavier(g, U, U, gain=UNITY_CROSS_GAIN)
    uemb = sd["decoder.embed_tokens.weight"].clone()
    uemb[cfg.eos] = 0.0
    uemb[cfg.eos, UNITY_EOS_DIM] = eos_gain
    uemb[cfg.eos, :READOUT_FREQS] = torch.randn(READOUT_FREQS, generator=g) * U ** -0.5
    sd["decoder.embed_tokens.weight"] = uemb
    sd["decoder.output_projection.weight"] = uemb
    memb = sd["target_unigram_decoder.embed_tokens.weight"].clone()
    memb[cfg.eos] *= UNITY_MT_EOS_SCALE
    sd["target_unigram_decoder.embed_tokens.weight"] = memb
    sd["target_unigram_decoder.output_projection.weight"] = memb
    return sd


# the stored model cfg of each UnitY-family recipe (researches/unitY, uni_unity and chunk_unity train_scripts): what
# ModelConfig.from_checkpoint reads back
UNITY_RECIPES = {
    "unity": {"arch": "unity_conformer_modified"},
    "uni_unity": {"arch": "uni_unity_conformer", "uni_encoder": True},
    "chunk_unity": {"arch": "chunk_unity_conformer", "uni_encoder": True, "chunk_size": 8},
}


def synthetic_unity_variant(user_dir: Optional[str]) -> str:
    """the UnitY-family model a `synthetic[:seed]` model path stands for: the one the --user-dir's research directory registers
    (researches/uni_unity, researches/chunk_unity), else UnitY"""
    name = os.path.basename(os.path.normpath(user_dir)) if user_dir else ""
    return name if name in ("uni_unity", "chunk_unity") else "unity"


def make_unity_checkpoint(variant: str = "unity", seed: int = 0) -> Dict[str, object]:
    """A seeded `torch.load(ckpt)` of a UnitY-family checkpoint: {"model": make_unity_state_dict (the same keys for every variant),
    "cfg": {"model": the recipe's stored settings}} at ModelConfig.unity_default(variant)'s dimensions"""
    cfg = ModelConfig.unity_default(variant)
    model_cfg = dict(UNITY_RECIPES[variant], max_target_positions=cfg.max_target_positions, pos_enc_type="rel_pos", attn_type="espnet",
                     conv_version="s2t_transformer")
    return {"model": make_unity_state_dict(cfg, seed=seed), "cfg": {"model": model_cfg}}


def make_vocoder_state_dict(vc: VocoderConfig, seed: int = 1, cal: Calibration = Calibration(), weight_norm: bool = False) -> Dict[str, torch.Tensor]:
    """`torch.load(ckpt)["generator"]` of the CodeHiFiGAN vocoder (agent/tts/vocoder.py:37-45).

    With weight_norm=True every conv carries `weight_g`/`weight_v` like the published
    checkpoint (before `remove_weight_norm`); otherwise plain `weight`.
    """
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def conv(prefix, w):
        # gain sqrt(3)-ish keeps activations O(1) through the leaky-relu stack
        if weight_norm:
            # torch.nn.utils.weight_norm(dim=0): w = g * v / ||v|| over all dims but 0
            norm = w.flatten(1).norm(dim=1).view(-1, *([1] * (w.dim() - 1)))
            sd[prefix + ".weight_g"] = norm.clone()
            sd[prefix + ".weight_v"] = w.clone()
        else:
            sd[prefix + ".weight"] = w
        sd[prefix + ".bias"] = _normal(g, (w.shape[0] if "ups" not in prefix else w.shape[1],), 0.02)

    E = vc.embedding_dim
    sd["dict.weight"] = _normal(g, (vc.num_embeddings, E), 1.0)
    H = vc.dur_hidden
    sd["dur_predictor.conv1.0.weight"] = _xavier(g, H, E, vc.dur_kernel, gain=1.4)
    sd["dur_predictor.conv1.0.bias"] = _normal(g, (H,), 0.1)
    _ln(g, sd, "dur_predictor.ln1", H)
    sd["dur_predictor.conv2.0.weight"] = _xavier(g, H, H, vc.dur_kernel, gain=1.4)
    sd["dur_predictor.conv2.0.bias"] = _normal(g, (H,), 0.1)
    _ln(g, sd, "dur_predictor.ln2", H)
    sd["dur_predictor.proj.weight"] = _normal(g, (1, H), cal.dur_log_std / math.sqrt(H))
    sd["dur_predictor.proj.bias"] = torch.tensor([cal.dur_log_mean])

    C0 = vc.upsample_initial_channel
    conv("conv_pre", _xavier(g, C0, vc.model_in_dim, 7, gain=1.0))
    ch = C0
    for i, (u, k) in enumerate(zip(vc.upsample_rates, vc.upsample_kernel_sizes)):
        cin, cout = C0 // (2 ** i), C0 // (2 ** (i + 1))
        # ConvTranspose1d weight is [Cin, Cout, k]; each output sees ~k/u taps
        a = math.sqrt(3.0 * u / (cin * k)) * 1.3
        w = (torch.rand((cin, cout, k), generator=g) * 2 - 1) * a
        if weight_norm:
            norm = w.flatten(1).norm(dim=1).view(-1, 1, 1)
            sd[f"ups.{i}.weight_g"] = norm.clone()
            sd[f"ups.{i}.weight_v"] = w.clone()
        else:
            sd[f"ups.{i}.weight"] = w
        sd[f"ups.{i}.bias"] = _normal(g, (cout,), 0.02)
        ch = cout
        for j, (rk, dil) in enumerate(zip(vc.resblock_kernel_sizes, vc.resblock_dilation_sizes)):
            rb = i * len(vc.resblock_kernel_sizes) + j
            for m in range(len(dil)):
                a2 = math.sqrt(3.0 / (ch * rk)) * 0.5
                conv(f"resblocks.{rb}.convs1.{m}", (torch.rand((ch, ch, rk), generator=g) * 2 - 1) * a2 * 1.6)
                conv(f"resblocks.{rb}.convs2.{m}", (torch.rand((ch, ch, rk), generator=g) * 2 - 1) * a2)
    conv("conv_post", (torch.rand((1, ch, 7), generator=g) * 2 - 1) * math.sqrt(3.0 / (ch * 7)) * 0.5)
    return {k: v.contiguous().float() for k, v in sd.items()}


def make_gcmvn(cfg: ModelConfig, seed: int = 2):
    """Stand-in for configs/<pair>/gcmvn.npz (fp32 mean/std of the log-mel features).
    The stats of `make_audio` signals were measured once by oracle/calibrate_synth.py and are
    stored with the calibration rows, so CMVN output is ~zero-mean/unit-variance as with real data."""
    if os.path.exists(_CAL_FILE):
        rows = np.load(_CAL_FILE)
        if "gcmvn_mean" in rows and rows["gcmvn_mean"].shape[0] == cfg.feat_dim:
            return {"mean": rows["gcmvn_mean"].astype(np.float32), "std": rows["gcmvn_std"].astype(np.float32)}
    g = torch.Generator().manual_seed(seed)
    mean = 14.0 + 6.0 * torch.linspace(0, 1, cfg.feat_dim) + 0.2 * torch.rand(cfg.feat_dim, generator=g)
    std = 1.3 + 0.3 * torch.rand(cfg.feat_dim, generator=g)
    return {"mean": mean.numpy(), "std": std.numpy()}


def make_audio(seconds: float, seed: int = 1234, sample_rate: int = 16000) -> torch.Tensor:
    """Seeded fp32 mono audio: band-limited noise bursts + sinusoids under an envelope, peak 0.3
    (SURVEY.md §8d synthetic inputs)."""
    g = torch.Generator().manual_seed(seed)
    n = int(round(seconds * sample_rate))
    t = torch.arange(n, dtype=torch.float64) / sample_rate
    x = torch.zeros(n, dtype=torch.float64)
    for _ in range(4):
        f = 100.0 + 3900.0 * float(torch.rand(1, generator=g))
        ph = 2 * math.pi * float(torch.rand(1, generator=g))
        x += torch.sin(2 * math.pi * f * t + ph) * (0.3 + 0.7 * float(torch.rand(1, generator=g)))
    noise = torch.randn(n, generator=g, dtype=torch.float64)
    # cheap band-limit: 5-tap moving average
    k = torch.ones(5, dtype=torch.float64) / 5
    noise = torch.nn.functional.conv1d(noise.view(1, 1, -1), k.view(1, 1, -1), padding=2).view(-1)
    env = 0.55 + 0.45 * torch.sin(2 * math.pi * 1.3 * t + 0.7) * torch.sin(2 * math.pi * 0.31 * t)
    x = (x + 2.0 * noise) * env
    x = x / x.abs().max() * 0.3
    return x.float()


# ---- the ASR-BLEU transcriber: wav2vec 2.0 Large (LV-60) + CTC, the `en` model of asr_bleu/asr_model_cfgs.json.  The published
# configuration (conv_feature_layers, 24 pre-LN layers of width 1024, 16 heads, FFN 4096, pos_conv k = 128 in 16 groups); the real
# checkpoint is not read here.
W2V_CONV_LAYERS = [(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2
W2V_LETTERS = ["|", "E", "T", "A", "O", "N", "I", "H", "S", "R", "D", "L", "U", "M", "W", "C", "F", "G", "Y", "P", "B", "V", "K", "'", "X",
               "J", "Q", "Z"]  # dict.ltr.txt's order


def make_w2v_ctc_state_dict(seed: int = 7, dim: int = 1024, ffn: int = 4096, layers: int = 24, conv_layers=None, pos_k: int = 128,
                            pos_groups: int = 16, vocab: int = 32) -> Dict[str, torch.Tensor]:
    """Seeded fp32 Wav2VecCtc state dict with fairseq's key names ("w2v_encoder.w2v_model.*", "w2v_encoder.proj.*"), pos_conv
    weight-normed (weight_g / weight_v).  Calibration: weights at std ~ 1/sqrt(fan_in) keep the pre-LN residual stream bounded over 24
    layers; the final LayerNorm's output then varies little from frame to frame, so the proj is scaled up (std 3 / sqrt(dim)) and the
    blank gets a small lead (+0.3): a frame's arg-max is blank about half the time (measured 4-62 % on make_audio inputs), not always."""
    g = torch.Generator().manual_seed(seed)
    conv_layers = conv_layers or W2V_CONV_LAYERS
    P = "w2v_encoder.w2v_model."
    sd: Dict[str, torch.Tensor] = {}
    cin = 1
    for i, (c, k, _) in enumerate(conv_layers):
        sd[f"{P}feature_extractor.conv_layers.{i}.0.weight"] = _normal(g, (c, cin, k), math.sqrt(2.0 / (cin * k)))
        sd[f"{P}feature_extractor.conv_layers.{i}.0.bias"] = _normal(g, (c,), 0.05)
        _ln(g, sd, f"{P}feature_extractor.conv_layers.{i}.2.1", c)
        cin = c
    _ln(g, sd, P + "layer_norm", cin)
    sd[P + "post_extract_proj.weight"] = _normal(g, (dim, cin), 1.0 / math.sqrt(cin))
    sd[P + "post_extract_proj.bias"] = _normal(g, (dim,), 0.02)
    cg = dim // pos_groups
    sd[P + "encoder.pos_conv.0.weight_v"] = _normal(g, (dim, cg, pos_k), math.sqrt(4.0 / (pos_k * dim)))
    sd[P + "encoder.pos_conv.0.weight_g"] = 0.5 + torch.rand((1, 1, pos_k), generator=g)
    sd[P + "encoder.pos_conv.0.bias"] = _normal(g, (dim,), 0.02)
    for li in range(layers):
        pre = f"{P}encoder.layers.{li}."
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[pre + f"self_attn.{nm}.weight"] = _normal(g, (dim, dim), 1.0 / math.sqrt(dim))
            sd[pre + f"self_attn.{nm}.bias"] = _normal(g, (dim,), 0.02)
        _ln(g, sd, pre + "self_attn_layer_norm", dim)
        sd[pre + "fc1.weight"] = _normal(g, (ffn, dim), 1.0 / math.sqrt(dim))
        sd[pre + "fc1.bias"] = _normal(g, (ffn,), 0.02)
        sd[pre + "fc2.weight"] = _normal(g, (dim, ffn), 0.5 / math.sqrt(ffn))
        sd[pre + "fc2.bias"] = _normal(g, (dim,), 0.02)
        _ln(g, sd, pre + "final_layer_norm", dim)
    _ln(g, sd, P + "encoder.layer_norm", dim)
    sd["w2v_encoder.proj.weight"] = _normal(g, (vocab, dim), 3.0 / math.sqrt(dim))
    bias = _normal(g, (vocab,), 0.1)
    bias[0] += 0.3
    sd["w2v_encoder.proj.bias"] = bias
    return sd


def w2v_letter_dict(vocab: int = 32) -> str:
    """dict.ltr.txt for a vocab of `vocab` entries (the 4 specials are added by the reader)"""
    return "".join(f"{c} {1000 - i}\n" for i, c in enumerate(W2V_LETTERS[:vocab - 4]))
