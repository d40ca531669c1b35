"""GPU: the front of the pipeline (fbank + CMVN -> Conv1dSubsampler -> 12 Conformer layers -> CTC heads) against a float64 reference
of the same operation, at the shapes, chunk geometries and step edges where its kernels switch.

Entry points and the routes they take:
- ss_fbank: the TMA-staged kernel (fbank_tma = 1 and a 16-byte aligned sample pointer) or the plain kernel (fbank_tma = 0, or any
  unaligned pointer); the pool's ms_fbank computes the new frames of every stream of a step;
- ss_encoder_stream_step (the streaming agents): the cluster kernel (persistent_encoder_cluster, 1 <= nA <= 16 active rows), the
  one-CTA-per-SM persistent kernel (FFN fused or not, nA <= 16) or the per-op layer loop (persistent_encoder = 0, or nA > 16: first
  steps of long segments, attention chunks > 16).  Rows are final in groups of G = lcm(attention chunk, conv chunk) rows; the
  provisional tail rows are recomputed on every call;
- ss_encoder_forward (full prefix: recompute agents, offline generator): linears on the bf16x6 wgmma GEMM from umma_min_rows = 128
  rows (umma_linear = 13) decided on the whole batch B * T; offline model (set_chunk(None, None)) and padded batches with lengths;
- ss_pool_step: one encoder pass over the M = sum nA rows of every stepping stream (skinny GEMMs at M <= 64, fp32 tiled at 65 .. 127,
  wgmma at M >= 128), subsampler groups keyed by (nA == 0, a0 == 0, nA, n1, nf, attention chunk, conv chunk);
- the CTC heads: ss_ctc_greedy, _rows (row0 > 0), _pair, _batch and the pool's packed output.

The reference is StreamSpeechOracle.subsample / encoder / conformer_layer / ctc_logits and kaldi_fbank / online_features
(oracle/streamspeech_oracle.py, pinned to the reference's fixtures and to torchaudio by test_oracle_golden.py) restated as float64
torch operations on the GPU, with an attention chunk, a conv chunk (None = offline) and per-sample lengths;
test_reference_matches_the_cpu_oracle checks it against the oracle's own float64 functions once.  Both sides get the same fp32
inputs: the engine's own fbank rows for the encoder cases, the engine's own encoder rows for the CTC cases, so each case measures one
stage.  Streaming steps are compared, all T rows with the provisional tail, with the float64 full-prefix encoder of feats[:F]: what the
reference recomputes on every policy() call.  A padded batch sample is compared with the float64 encoder of that sample alone, padded
to the batch's length (fairseq padding semantics: pad frames are zeros that the convolutions read; attention masks the pad keys).

An arg-max may differ from the float64 one only where the float64 top-2 margin of the masked log-probs is below MARGIN (near ties,
counted); tokens and indices must equal ctc_collapse of the engine's own arg-max.  The measured maxima, the case of each maximum and
the near-tie counts are printed as one JSON line per test (`pytest -s`), with the card's name and power limit, before the bars are
asserted.
"""
import ctypes
import json
import math
import subprocess

import pytest
import torch
import torch.nn.functional as F

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)
F64 = torch.float64
MARGIN = 1e-4
EPS32 = torch.finfo(torch.float32).eps
UMMA_MIN_ROWS = 128
# Max-abs bars against float64, about ten times the largest error measured on an H100 80GB HBM3 (700 W) over every case of this file
# (in the comments).  Log-mel bars by signal; encoder bars by route: "fp32" every linear on the fp32 kernels, "tc" some linear on the
# bf16x6 wgmma GEMM.
FBANK_TOL = {
    "speech": 3e-4,  # 2.8e-5 (raw log-mel, TMA kernel)
    "silence": 3e-5,  # 2.9e-6 (CMVN, n = 400): log of the eps clamp
    "near_silent": 4e-4,  # 3.6e-5 (raw)
    "full_scale": 4e-4,  # 3.3e-5 (raw)
    "dc_offset": 5e-4,  # 4.7e-5 (raw)
    # 3.4e-2 (raw), in mel bins some 12 decades of power below the tone's bin, where the fp32 FFT's rounding dominates: the
    # reference's own fp32 kaldi_fbank (torch) errs 5.4e-2 there
    "tone": 0.4,
    "pool": 7e-4,  # 6.6e-5 (ms_fbank, speech, 40 streams)
}
ENC_TOL = {
    "stream": 4e-5,  # 4.0e-6 (per-op and persistent steps, chunk 8/8, nA = 17); cluster 3.7e-6
    "fp32": 7e-5,  # 6.5e-6 (full prefix, chunk 4/8, T = 1024, umma_linear 0); pool 1.0e-5 (M = 78)
    "tc": 2e-4,  # 1.7e-5 (offline batch, T = 1024); pool 1.2e-5 (M >= 128)
}
CHUNKS = [(2, 8), (4, 8), (8, 8), (12, 8), (16, 16), (24, 16), (32, 16), (40, 16)]
STREAM_ROUTES = {  # (persistent_encoder, persistent_encoder_cluster, persistent_ffn_fused)
    "cluster": (1, 1, 1),
    "persistent_fused": (1, 0, 1),
    "persistent_unfused": (1, 0, 0),
    "per_op": (0, 0, 1),
}
MAX_PERSISTENT_ROWS = 16  # active rows the cluster and persistent kernels take (kernels_persist.cu PMR, kernels_persist_cl.cu NCL * CR)
ONE_LAUNCH_STEP = 8  # launches of a step that runs its layers as one kernel: subsampler, input linear, layer kernel
PER_OP_STEP = 100  # at least this many launches: 12 layers of about a dozen kernels each


def report(name, **kw):
    print(json.dumps({"test": name, **card(), **kw}))


def card():
    """the GPU's name and power limit, part of every measured number"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = out[0].split(", ")
        return {"gpu": name, "power_limit": power}
    except Exception:
        return {"gpu": torch.cuda.get_device_name() if torch.cuda.is_available() else None, "power_limit": None}


def maxdiff(a, b):
    """max-abs difference; a NaN counts as infinite"""
    d = float((a.double() - b.to(a.device).double()).abs().max()) if a.numel() else 0.0
    return float("inf") if d != d else d


class Worst:
    """the largest error per key and the case it came from"""

    def __init__(self):
        self.v = {}

    def add(self, key, err, case):
        if key not in self.v or err > self.v[key][0]:
            self.v[key] = (err, case)

    def get(self, key):
        return self.v.get(key, (0.0, None))[0]

    def as_dict(self):
        return {k: {"max_abs": v, "case": c} for k, (v, c) in sorted(self.v.items())}

    def check(self, bars):
        """every key within its bar"""
        for k, (v, c) in self.v.items():
            assert v < bars[k], (k, v, c, bars[k])


def out_frames(F_):
    return ((F_ - 1) // 2 + 1 - 1) // 2 + 1


def lcm(a, b):
    return a * b // math.gcd(a, b)


# --------------------------------------------------------------------------------------------------------------------------------
# float64 reference
# --------------------------------------------------------------------------------------------------------------------------------
class Ref64:
    """StreamSpeechOracle.encoder / ctc_logits and kaldi_fbank + CMVN in float64 on `device`: the weights are the fp32 checkpoint's and
    the constant tables (window, mel bank, relative positions) are computed in fp32 as the reference does, then converted"""

    def __init__(self, cfg, sd, gcmvn, device="cuda"):
        from oracle.streamspeech_oracle import _mel_banks

        self.cfg, self.dev = cfg, device
        self.w = {k: v.float().to(device, F64) for k, v in sd.items()
                  if k.startswith(("encoder.", "source_unigram_decoder.", "ctc_target_unigram_decoder.")) and v.is_floating_point()}
        self.window = torch.hann_window(400, periodic=False, dtype=torch.float32).pow(0.85).to(device, F64)
        self.banks = F.pad(_mel_banks(), (0, 1)).to(device, F64)  # [80, 257]
        self.cmvn = None if gcmvn is None else tuple(torch.as_tensor(gcmvn[k]).float().to(device, F64) for k in ("mean", "std"))
        self._pos = {}

    # ---- F1/F2
    def fbank(self, wav, cmvn=True):
        """kaldi_fbank(wav * 2**15) [+ (x - mean) / std]: wav fp32 [n] (unscaled) -> [1 + (n - 400) // 160, 80]"""
        n = wav.numel()
        if n < 400:
            return torch.zeros(0, 80, dtype=F64, device=self.dev)
        m = 1 + (n - 400) // 160
        x = wav.reshape(-1).to(self.dev, F64) * 32768.0
        frames = x.as_strided((m, 400), (160, 1))
        frames = frames - frames.mean(dim=1, keepdim=True)
        prev = torch.cat([frames[:, :1], frames[:, :-1]], dim=1)  # replicate pad
        frames = (frames - 0.97 * prev) * self.window
        spec = torch.fft.rfft(F.pad(frames, (0, 112))).abs().pow(2.0)
        out = torch.clamp_min(spec @ self.banks.T, EPS32).log()  # the fp32 eps of the reference's clamp
        if cmvn and self.cmvn is not None:
            out = (out - self.cmvn[0]) / self.cmvn[1]
        return out

    # ---- E1..E6
    def _lin(self, x, name):
        return F.linear(x, self.w[name + ".weight"], self.w.get(name + ".bias"))

    def _ln(self, x, name):
        return F.layer_norm(x, (x.shape[-1],), self.w[name + ".weight"], self.w[name + ".bias"], 1e-5)

    def pos(self, T):
        """rel_positional_encoding(T, C) (fp32, converted): row k holds relative position T - 1 - k"""
        from oracle.streamspeech_oracle import rel_positional_encoding

        if T not in self._pos:
            self._pos[T] = rel_positional_encoding(T, self.cfg.enc_dim).to(self.dev, F64)
        return self._pos[T]

    def _rel_mha(self, x, p, mask):
        """RelPositionMultiHeadedAttention: x [B, T, C], mask [B, T, T] True = masked.  Query i and key j score
        (q_i + u) k_j + (q_i + v) pos(i - j): the rel_shift of the reference as a gather"""
        B, T, C = x.shape
        H = self.cfg.enc_heads
        dk = C // H
        q = self._lin(x, p + ".linear_q").view(B, T, H, dk)
        k = self._lin(x, p + ".linear_k").view(B, T, H, dk).transpose(1, 2)
        v = self._lin(x, p + ".linear_v").view(B, T, H, dk).transpose(1, 2)
        pp = F.linear(self.pos(T), self.w[p + ".linear_pos.weight"]).view(2 * T - 1, H, dk).transpose(0, 1)  # [H, 2T-1, dk]
        ac = (q + self.w[p + ".pos_bias_u"]).transpose(1, 2) @ k.transpose(-2, -1)
        bd = (q + self.w[p + ".pos_bias_v"]).transpose(1, 2) @ pp.transpose(-2, -1)  # [B, H, T, 2T-1]
        ar = torch.arange(T, device=self.dev)
        idx = (T - 1 - ar[:, None] + ar[None, :]).expand(B, H, T, T)
        scores = (ac + torch.gather(bd, -1, idx)) / math.sqrt(dk)
        scores = scores.masked_fill(mask[:, None], float("-inf"))
        o = (torch.softmax(scores, dim=-1) @ v).transpose(1, 2).reshape(B, T, C)
        return self._lin(o, p + ".linear_out")

    def _conv_module(self, x, p, conv_chunk):
        from oracle.streamspeech_oracle import depthwise_bn_silu_core

        y = self._ln(x, p + ".layer_norm").transpose(1, 2)
        y = F.glu(F.conv1d(y, self.w[p + ".pointwise_conv1.weight"]), dim=1)
        y = depthwise_bn_silu_core(y, self.w[p + ".depthwise_conv.weight"], self.w[p + ".batch_norm.running_mean"],
                                   self.w[p + ".batch_norm.running_var"], self.w[p + ".batch_norm.weight"], self.w[p + ".batch_norm.bias"],
                                   conv_chunk)
        return F.conv1d(y, self.w[p + ".pointwise_conv2.weight"]).transpose(1, 2)

    def _ffn(self, x, p):
        return self._lin(F.silu(self._lin(self._ln(x, p + ".layer_norm"), p + ".w_1")), p + ".w_2")

    def encoder(self, feats, lengths=None, attn_chunk=8, conv_chunk=8):
        """feats [B, F, 80] (fp32, any device), lengths [B] frames (None: all F) -> [B, T, C] float64; attn_chunk None = full
        attention, conv_chunk None = plain padded convolutions (the offline model)"""
        from oracle.streamspeech_oracle import chunk_causal_conv1d

        if feats.dim() == 2:
            feats = feats.unsqueeze(0)
        B, F_, _ = feats.shape
        x = feats.to(self.dev, F64).transpose(1, 2)
        for i in range(2):
            w, b = self.w[f"encoder.subsample.conv_layers.{i}.weight"], self.w[f"encoder.subsample.conv_layers.{i}.bias"]
            if conv_chunk is None:
                x = F.conv1d(x, w, b, stride=2, padding=w.shape[-1] // 2)
            else:
                x = chunk_causal_conv1d(x, w, b, 2, 1, conv_chunk)
            x = F.glu(x, dim=1)
        x = x.transpose(1, 2)
        T, C = x.shape[1], x.shape[2]
        lens = torch.tensor([out_frames(int(l)) for l in (lengths if lengths is not None else [F_] * B)], device=self.dev)
        ar = torch.arange(T, device=self.dev)
        mask = (ar[None, :] >= lens[:, None])[:, None, :].expand(B, T, T)  # key padding
        if attn_chunk is not None:  # buffered_chunk_mask
            c = max(attn_chunk, 1)
            mask = mask | (ar[None, :] >= ((ar[:, None] // c + 1) * c).clamp(1, T))[None]
        x = self._lin(math.sqrt(C) * x, "encoder.linear")
        for i in range(self.cfg.enc_layers):
            p = f"encoder.conformer_layers.{i}"
            x = self._ffn(x, p + ".ffn1") * 0.5 + x
            x = self._rel_mha(self._ln(x, p + ".self_attn_layer_norm"), p + ".self_attn", mask) + x
            x = x + self._conv_module(x, p + ".conv_module", conv_chunk)
            x = self._ln(self._ffn(x, p + ".ffn2") * 0.5 + x, p + ".final_layer_norm")
        return x

    def ctc_lprobs(self, head, enc):
        """masked float64 log-probs of CTC head 0 (source_unigram) or 1 (ctc_target_unigram) over fp32 rows enc [T, C]: never pad, unk"""
        name = ("source_unigram", "ctc_target_unigram")[head]
        lp = F.log_softmax(self._lin(enc.to(self.dev, F64), f"{name}_decoder.proj"), dim=-1)
        lp[:, [self.cfg.pad, self.cfg.unk]] = float("-inf")
        return lp


def check_argmax(got, lp, what):
    """got [N] int, lp [N, V] float64 masked log-probs: got must be the arg-max wherever the top-2 margin is at least MARGIN; returns
    the number of near-tie positions where it is not"""
    top = lp.topk(2, dim=-1)
    bad = torch.as_tensor(got, device=lp.device).long() != top.indices[:, 0]
    hard = bad & (top.values[:, 0] - top.values[:, 1] >= MARGIN)
    assert not bool(hard.any()), (what, torch.nonzero(hard).flatten()[:10].tolist())
    return int(bad.sum())


def near_tie_rows(lp):
    top = lp.topk(2, dim=-1)
    return int((top.values[:, 0] - top.values[:, 1] < MARGIN).sum())


def collapse(argmax):
    from oracle.streamspeech_oracle import ctc_collapse

    return ctc_collapse([int(t) for t in argmax], blank=0, pad=ModelConfig().pad)


def wgmma_ran(e, fn):
    """(fn(), whether some wgmma GEMM ran in it): the umma2 kernels stamp a zeroed debug buffer when they start (option umma2_debug)"""
    e.set_option("umma2_debug", 1)
    stamps = (ctypes.c_uint64 * 16)()
    try:
        r = fn()
        torch.cuda.synchronize()
        e._check(e.lib.ss_debug_copy(e._h, b"umma2_ts", ctypes.cast(stamps, ctypes.c_void_p), ctypes.sizeof(stamps)))
    finally:
        e.set_option("umma2_debug", 0)
    return r, any(stamps)


def alias(ptr, shape):
    """a float32 tensor over device memory the engine owns"""
    n = 1
    for s in shape:
        n *= s

    class _A:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_A(), device="cuda").view(*shape)


def ctc_checkpoint(cfg, sd, top):
    """CTC heads whose pad and unk output rows are 1.02 and 1.03 times the row of token top[head] (weight and bias): wherever that
    token's logit is positive unk, then pad, outrank it, and only the pad / unk mask gives the row back"""
    sd = dict(sd)
    for head, name in enumerate(("source_unigram", "ctc_target_unigram")):
        for k in ("weight", "bias"):
            t = sd[f"{name}_decoder.proj.{k}"].clone()
            t[cfg.pad] = 1.02 * t[top[head]]
            t[cfg.unk] = 1.03 * t[top[head]]
            sd[f"{name}_decoder.proj.{k}"] = t
    return sd


class Setup:
    """one engine (CMVN on, the CTC checkpoint of ctc_checkpoint), one without CMVN (raw log-mel), the float64 reference, and the
    engine's fbank rows of a 41 s utterance (4094 frames: T = 1024 encoder rows, the engine's capacity)"""

    def __init__(self):
        from streamspeech_b200.engine import Engine

        c = self.cfg = ModelConfig()
        sd = synth.make_model_state_dict(c, 0)
        self.gc = synth.make_gcmvn(c)
        probe = Engine(c, sd, None, self.gc)
        try:
            probe.set_chunk(8)
            enc = probe.encoder(probe.fbank(synth.make_audio(3.0, seed=29).cuda().contiguous()).unsqueeze(0).contiguous())[0]
            top = []
            for head in (0, 1):
                am = probe.ctc_greedy(head, enc.contiguous())["argmax"]
                top.append(int(torch.bincount(am, minlength=c.src_vocab).argmax()))
        finally:
            probe.close()
        self.top = top
        self.sd = ctc_checkpoint(c, sd, top)
        self.e = Engine(c, self.sd, None, self.gc)
        self.e_raw = Engine(c, self.sd, None, None)
        for e in (self.e, self.e_raw):
            e.set_option("umma_min_rows", UMMA_MIN_ROWS)
            e.set_chunk(8)
        self.ref = Ref64(c, self.sd, self.gc)
        self.wav = synth.make_audio(41.0, seed=17)
        self.feats = self.e.fbank(self.wav.cuda().contiguous())[:4094].contiguous()
        assert out_frames(self.feats.shape[0]) == 1024
        self._enc = {}

    def enc64(self, F_, attn_chunk, conv_chunk):
        """float64 full-prefix encoder of feats[:F_] (cached)"""
        key = (F_, attn_chunk, conv_chunk)
        if key not in self._enc:
            self._enc[key] = self.ref.encoder(self.feats[:F_], None, attn_chunk, conv_chunk)[0]
        return self._enc[key]

    def close(self):
        self.e.close()
        self.e_raw.close()


@pytest.fixture(scope="module")
def enc():
    s = Setup()
    yield s
    s.close()


def test_reference_matches_the_cpu_oracle():
    """the float64 restatement against StreamSpeechOracle(dtype=float64).encoder on the CPU (chunk 8/8, 12/8, offline, a padded batch
    of two) and its CTC log-probs against ctc_logits; its fbank against the oracle's fp32 kaldi_fbank / online_features"""
    from oracle.streamspeech_oracle import StreamSpeechOracle, kaldi_fbank, online_features

    dev = "cuda" if torch.cuda.is_available() else "cpu"
    c = ModelConfig()
    sd = synth.make_model_state_dict(c, 0)
    gc = synth.make_gcmvn(c)
    ref = Ref64(c, sd, gc, dev)
    wav = synth.make_audio(1.3, seed=3)
    feats = online_features(wav, gc)
    res = {}
    for ac, cc in ((8, 8), (12, 8), (None, None)):
        o = StreamSpeechOracle(c, sd, None, gc, chunk_size=ac, conv_chunk_size=cc, dtype=F64)
        want = o.encoder(feats.unsqueeze(0), torch.tensor([feats.shape[0]]))["encoder_out"][0][:, 0]
        got = ref.encoder(feats, None, ac, cc)[0]
        res[f"chunk {ac}/{cc}"] = maxdiff(got.cpu(), want)
        if ac == 8:
            for head, name in enumerate(("source_unigram", "ctc_target_unigram")):
                lp = F.log_softmax(o.ctc_logits(name, want.float().double().unsqueeze(1))[0], dim=-1)
                lp[:, [c.pad, c.unk]] = float("-inf")
                got_lp = ref.ctc_lprobs(head, want.float()).cpu()
                assert torch.equal(torch.isinf(got_lp), torch.isinf(lp))
                res[f"ctc head {head}"] = maxdiff(got_lp.masked_fill(torch.isinf(lp), 0), lp.masked_fill(torch.isinf(lp), 0))
    lengths = [feats.shape[0], 70]
    batch = torch.zeros(2, feats.shape[0], c.feat_dim)
    batch[0], batch[1, :70] = feats, feats[:70]
    o = StreamSpeechOracle(c, sd, None, gc, chunk_size=8, dtype=F64)
    out = o.encoder(batch, torch.tensor(lengths))
    got = ref.encoder(batch, lengths, 8, 8)
    for b in range(2):
        n = int(out["out_lengths"][b])
        res[f"batch b={b}"] = maxdiff(got[b, :n].cpu(), out["encoder_out"][0][:n, b])
    fb32 = kaldi_fbank(wav * 2 ** 15)
    fb64 = ref.fbank(wav, cmvn=False).cpu()
    res["fbank vs fp32 kaldi_fbank"] = maxdiff(fb64, fb32)
    res["online_features vs fp32"] = maxdiff(ref.fbank(wav[:(feats.shape[0] * 160 + 240)]).cpu(), feats)
    report("encoder_fp64_reference_vs_cpu_oracle", **res)
    for k, v in res.items():
        assert v < (1e-3 if "fp32" in k else 1e-10), (k, v)


# --------------------------------------------------------------------------------------------------------------------------------
# fbank
# --------------------------------------------------------------------------------------------------------------------------------
def signals():
    """name -> fp32 [6000] unscaled 16 kHz signal"""
    n = 6000
    g = torch.Generator().manual_seed(41)
    t = torch.arange(n, dtype=F64) / 16000.0
    mel = lambda f: 1127.0 * math.log(1.0 + f / 700.0)
    lo, hi = mel(20.0), mel(8000.0)
    delta = (hi - lo) / 81
    f_edge = 700.0 * (math.exp((lo + 31 * delta) / 1127.0) - 1.0)  # bin 29's right edge = bin 30's center = bin 31's left edge
    return {
        "speech": synth.make_audio(n / 16000.0, seed=5)[:n],
        "silence": torch.zeros(n),
        "near_silent": (1e-6 * torch.randn(n, generator=g)).float(),
        "full_scale": torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).float(),
        "dc_offset": (0.9 + 0.05 * torch.randn(n, generator=g)).clamp(-1, 1).float(),
        "tone": (0.5 * torch.sin(2 * math.pi * f_edge * t)).float(),
    }


def fbank_cases():
    """(n_samples, frame0, n_frames): frame counts 0 / 1 / 2 at the 400 and 560 sample edges (last frame ending at the buffer end at
    400 and 560), whole signals and frame0 > 0 sub-ranges"""
    out = [(n, 0, None) for n in (399, 400, 401, 559, 560, 561, 6000)]
    out += [(6000, 1, 5), (6000, 17, None), (5840, 30, None)]  # 5840 = 35 * 160 + 240: frame 34 ends exactly at the end
    return out


@pytest.mark.gpu
def test_fbank_vs_fp64(enc):
    """ss_fbank on both kernels (fbank_tma 1 with an aligned pointer, fbank_tma 0, and fbank_tma 1 with an unaligned pointer, which takes
    the plain kernel), raw log-mel and with CMVN, against the float64 kaldi fbank of the same samples"""
    worst, n_cases = Worst(), 0
    for sig, wav in signals().items():
        for raw in (True, False):
            e = enc.e_raw if raw else enc.e
            for tma, aligned in ((1, True), (0, True), (1, False)):
                e.set_option("fbank_tma", tma)
                try:
                    for n, f0, nf in fbank_cases():
                        buf = torch.zeros(n + 4, device="cuda")
                        x = buf[:n] if aligned else buf[1:n + 1]
                        x.copy_(wav[:n].cuda())
                        assert (x.data_ptr() % 16 == 0) == aligned
                        got = e.fbank(x, f0, nf)
                        want = enc.ref.fbank(wav[:n], cmvn=not raw)
                        want = want[f0:f0 + got.shape[0]]
                        assert got.shape[0] == (want.shape[0] if nf is None else nf), (sig, n, f0, nf)
                        assert got.shape[0] == max(0, e.num_fbank_frames(n) - f0) or nf is not None
                        worst.add(sig, maxdiff(got, want), f"{'raw' if raw else 'cmvn'} tma={tma} aligned={aligned} n={n} frame0={f0}")
                        n_cases += 1
                finally:
                    e.set_option("fbank_tma", 1)
    enc.e.check_async_error()
    report("encoder_fbank_fp64", cases=n_cases, **worst.as_dict())
    worst.check(FBANK_TOL)


@pytest.mark.gpu
def test_pool_fbank_vs_fp64(enc):
    """the pool's ms_fbank: two slots fed pushes of 1, 159, 160, 161 and 5120 samples in turn (frame0 advancing across partial frames),
    their features after every step against the float64 fbank + CMVN of everything pushed so far"""
    e = enc.e
    sigs = signals()
    pushes = [1, 159, 160, 161, 5120, 160, 161, 159, 1, 5120]
    worst = Worst()
    e.pool_create(40, max_seconds=8)
    enc.pool_ready = True
    for slot, sig in ((0, "speech"), (1, "tone")):
        e.pool_reset(slot)
        wav = torch.cat([sigs[sig], synth.make_audio(1.0, seed=7)])
        n = 0
        for p in pushes:
            e.pool_push_audio(slot, wav[n:n + p].contiguous())
            n += p
            e.pool_step([slot], ctc_heads=0)
            info = e.pool_info(slot)
            assert info["n_audio"] == n and info["n_feat"] == e.num_fbank_frames(n)
            if info["n_feat"]:
                got = alias(info["feats_ptr"], (info["n_feat"], enc.cfg.feat_dim))
                worst.add("pool" if sig == "speech" else sig, maxdiff(got, enc.ref.fbank(wav[:n])), f"pool slot {slot} after {n} samples")
        e.pool_reset(slot)
    report("encoder_pool_fbank_fp64", **worst.as_dict())
    worst.check(FBANK_TOL)


# --------------------------------------------------------------------------------------------------------------------------------
# ss_encoder_stream_step
# --------------------------------------------------------------------------------------------------------------------------------
def stream_schedule(G):
    """fbank frame counts F of one stream's calls with lcm G: T = 1 twice (F < 4, repeated), ragged 17-frame steps, the first group
    final, then nA = 1, 16 and 17 from a final boundary, a repeated F, and 17-frame steps again"""
    Fs = [3, 3, 20, 37, 54]
    Tf = 0
    sched = []

    def step(F_):
        nonlocal Tf
        F_ = max(F_, sched[-1] if sched else F_)
        sched.append(F_)
        T = out_frames(F_)
        Tf = max(Tf, min(T, (F_ // (4 * G)) * G))

    for F_ in Fs:
        step(F_)
    step(4 * G * (sched[-1] // (4 * G) + 1))  # a group boundary: every row final
    for nA in (1, 16, 17):
        step(4 * (Tf + nA))
    step(sched[-1])
    for _ in range(2):
        step(sched[-1] + 17)
    return sched


def simulate(sched, G):
    """(nA, T, T_final) of every call, the engine's rule: a0 = min(T_final, T), T_final = max(T_final, min(T, F // (4 G) * G))"""
    Tf, out = 0, []
    for F_ in sched:
        T = out_frames(F_)
        nA = T - min(Tf, T)
        Tf = max(Tf, min(T, (F_ // (4 * G)) * G))
        out.append((nA, T, Tf))
    return out


def expected_route(route, nA):
    if nA == 0:
        return "none"
    if route == "per_op" or nA > MAX_PERSISTENT_ROWS:
        return "per_op"
    return "cluster" if route == "cluster" else "persistent"


def run_stream(enc, route, ac, cc, sched, compare):
    """one stream through `sched` on `route`; every call's route is proven from cluster_steps() and launch_count(), and the calls
    with compare(k) true are compared, all T rows, with the float64 full-prefix encoder.  Returns {(k, F): max-abs}"""
    e = enc.e
    G = lcm(ac, cc)
    pe, cl, ff = STREAM_ROUTES[route]
    e.set_chunk(ac, cc)
    e.set_option("persistent_encoder", pe)
    e.set_option("persistent_encoder_cluster", cl)
    e.set_option("persistent_ffn_fused", ff)
    buf = torch.full((1024, enc.cfg.enc_dim), float("nan"), device="cuda")
    errs, routes = {}, []
    try:
        e.encoder_stream_reset()
        for k, (F_, (nA, T, Tf)) in enumerate(zip(sched, simulate(sched, G))):
            n_cl, n_l = e.cluster_steps(), e.launch_count()
            T_got, Tf_got = e.encoder_stream_step(enc.feats[:F_], buf)
            d_cl, d_l = e.cluster_steps() - n_cl, e.launch_count() - n_l
            what = f"{route} chunk {ac}/{cc} call {k} F={F_} nA={nA}"
            assert (T_got, Tf_got) == (T, Tf), (what, T_got, Tf_got)
            want = expected_route(route, nA)
            got = "cluster" if d_cl == 1 else "per_op" if d_l >= PER_OP_STEP else "persistent" if 0 < d_l <= ONE_LAUNCH_STEP else f"? ({d_l})"
            if want == "none":
                got = want if d_l == 0 and d_cl == 0 else got
            assert got == want and d_cl == (want == "cluster"), (what, got, d_l, d_cl)
            routes.append(want)
            if compare(k) or k == len(sched) - 1:
                errs[(k, F_)] = maxdiff(buf[:T], enc.enc64(F_, ac, cc))
    finally:
        e.set_option("persistent_encoder", 1)
        e.set_option("persistent_encoder_cluster", 1)
        e.set_option("persistent_ffn_fused", 1)
        e.set_chunk(8)
        e.encoder_stream_reset()
    return errs, routes


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(STREAM_ROUTES))
def test_stream_step_vs_fp64(enc, route):
    """every chunk geometry of CHUNKS through stream_schedule on one route: every call's route proven, its T and T_final the engine's
    rule, all T rows (provisional tail included) within the bar of the float64 full-prefix encoder of feats[:F]"""
    worst, seen, counts = Worst(), set(), {}
    for ac, cc in CHUNKS:
        G = lcm(ac, cc)
        sched = stream_schedule(G)
        errs, routes = run_stream(enc, route, ac, cc, sched, lambda k: True)
        for (k, F_), d in errs.items():
            worst.add("stream", d, f"chunk {ac}/{cc} call {k} F={F_} nA={simulate(sched, G)[k][0]}")
        seen |= {nA for nA, _, _ in simulate(sched, G)}
        for r in routes:
            counts[r] = counts.get(r, 0) + 1
    enc.e.check_async_error()
    report(f"encoder_stream_step_fp64_{route}", routes=counts, nA_seen=sorted(seen), **worst.as_dict())
    assert {1, 16, 17} <= seen and max(seen) > 17, sorted(seen)
    if route != "per_op":
        assert counts.get("cluster" if route == "cluster" else "persistent", 0) > 0, counts
    worst.check(ENC_TOL)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["cluster", "per_op"])
def test_stream_to_capacity_vs_fp64(enc, route):
    """chunk 8/8 in 32-frame steps to F = 4094 (T = 1024, the engine's capacity): every 16th call and the last compared in full"""
    sched = list(range(30, 4094, 32)) + [4094]
    errs, routes = run_stream(enc, route, 8, 8, sched, lambda k: k % 16 == 0)
    worst = Worst()
    for (k, F_), d in errs.items():
        worst.add("stream", d, f"call {k} F={F_}")
    enc.e.check_async_error()
    report(f"encoder_stream_to_capacity_fp64_{route}", calls=len(sched), compared=len(errs), routes=sorted(set(routes)), **worst.as_dict())
    assert out_frames(sched[-1]) == 1024
    worst.check(ENC_TOL)


# --------------------------------------------------------------------------------------------------------------------------------
# ss_encoder_forward
# --------------------------------------------------------------------------------------------------------------------------------
FORWARD_F = [3, 508, 512, 4094]  # T = 1, 127, 128 (umma_min_rows), 1024


@pytest.mark.gpu
def test_encoder_forward_vs_fp64(enc):
    """ss_encoder_forward of one sample at every chunk geometry and offline, T = 1 / 127 / 128 / 1024, umma_linear 13 and 0: a wgmma
    GEMM runs exactly when umma_linear = 13 and T >= umma_min_rows"""
    e = enc.e
    worst = Worst()
    for ac, cc in CHUNKS + [(None, None)]:
        e.set_chunk(ac, cc)
        for F_ in FORWARD_F:
            T = out_frames(F_)
            for umma in (13, 0):
                e.set_option("umma_linear", umma)
                try:
                    out, ran = wgmma_ran(e, lambda: e.encoder(enc.feats[:F_].unsqueeze(0).contiguous()))
                finally:
                    e.set_option("umma_linear", 13)
                tc = umma == 13 and T >= UMMA_MIN_ROWS
                assert ran == tc, (ac, cc, F_, umma, ran)
                worst.add("tc" if tc else "fp32", maxdiff(out[0], enc.enc64(F_, ac, cc)), f"chunk {ac}/{cc} T={T} umma={umma}")
    e.set_chunk(8)
    report("encoder_forward_fp64", **worst.as_dict())
    worst.check(ENC_TOL)


# (F, lengths in frames): a sample of length 1; B * T >= 128 while every T < 128; T = 1024 with a ragged second sample
BATCHES = [(508, [508, 1, 300]), (60, [60, 33, 60, 9, 4, 57, 60, 41, 17, 60]), (4094, [4094, 2001])]


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [(8, 8), (12, 8), (None, None)], ids=["8-8", "12-8", "offline"])
def test_encoder_forward_batch_vs_fp64(enc, chunk):
    """ss_encoder_forward of padded batches with ragged lengths (pad frames zero): each sample's valid rows against the float64 encoder
    of that sample alone padded to the batch's length.  The linears are routed on the whole batch (B * T rows), not per sample as the
    decoder stages do: a full-length sample of a batch whose B * T reaches umma_min_rows while T does not takes the wgmma GEMM where its
    single-sample call does not; the difference between the two is recorded, both are held to the float64 bars."""
    e = enc.e
    ac, cc = chunk
    e.set_chunk(ac, cc)
    worst, vs_single = Worst(), {}
    try:
        for F_, lengths in BATCHES:
            B, T = len(lengths), out_frames(F_)
            x = torch.zeros(B, F_, enc.cfg.feat_dim, device="cuda")
            for b, l in enumerate(lengths):
                x[b, :l] = enc.feats[:l]
            out, ran = wgmma_ran(e, lambda: e.encoder(x, lengths))
            tc = B * T >= UMMA_MIN_ROWS
            assert ran == tc, (F_, lengths, ran)
            want = enc.ref.encoder(x, lengths, ac, cc)
            for b, l in enumerate(lengths):
                n = out_frames(l)
                worst.add("tc" if tc else "fp32", maxdiff(out[b, :n], want[b, :n]), f"F={F_} B={B} b={b} length={l}")
            b = lengths.index(F_)
            single = e.encoder(x[b:b + 1].contiguous())
            vs_single[f"F={F_} B={B}"] = {"batch_wgmma": ran, "single_wgmma": T >= UMMA_MIN_ROWS, "max_abs": maxdiff(out[b], single[0])}
    finally:
        e.set_chunk(8)
    report(f"encoder_forward_batch_fp64_{ac}_{cc}", batch_vs_single=vs_single, **worst.as_dict())
    worst.check(ENC_TOL)


# --------------------------------------------------------------------------------------------------------------------------------
# ss_pool_step
# --------------------------------------------------------------------------------------------------------------------------------
POOL_CHUNKS = [(8, 8), (12, 8), (4, 8), (16, 16), (24, 16), (2, 8), (8, 16)]  # (8, 8) and (8, 16) differ in the conv chunk only
POOL_PUSHES = [5120, 3000, 161, 6400, 2560, 159, 7000]


def gemm_class(M):
    return "skinny" if M <= 64 else "fp32" if M < UMMA_MIN_ROWS else "tc"


@pytest.mark.gpu
@pytest.mark.parametrize("n_streams, ctc_heads", [(1, 2), (6, 1), (12, 0), (40, 2)])
def test_pool_step_vs_fp64(enc, n_streams, ctc_heads):
    """n_streams slots of one 40-slot pool, each with its own chunk setting (several subsampler groups per step), starting at
    staggered steps (first steps next to later ones) with ragged pushes: after every step each stepping slot's rows against the float64
    encoder of its own features, its features against the float64 fbank, its CTC output against ctc_collapse of the float64 arg-max
    (sequences without near ties).  A wgmma GEMM runs exactly on steps with M = sum nA >= umma_min_rows."""
    e = enc.e
    if not getattr(enc, "pool_ready", False):
        e.pool_create(40, max_seconds=8)
        enc.pool_ready = True
    slots = list(range(n_streams))
    # slots s and s' with s // 7 == s' // 7 push the same sizes from the same step, each with its own chunk setting
    chunk = {s: POOL_CHUNKS[s % len(POOL_CHUNKS)] if n_streams > 1 else (8, 8) for s in slots}
    wavs = {s: synth.make_audio(2.0 + 0.1 * (s % 7), seed=100 + s) for s in slots}
    start = {s: (s // 7) % 3 for s in slots}
    pos = {s: 0 for s in slots}
    Tf = {s: 0 for s in slots}
    for s in slots:
        e.pool_reset(s)
        e.pool_set_chunk(s, *chunk[s])
    worst, classes, near, ctc_checked, groups_max = Worst(), {}, 0, 0, 0
    try:
        for step in range(12):
            active = [s for s in slots if step >= start[s]]
            for s in active:
                p = POOL_PUSHES[(s // 7 + step) % len(POOL_PUSHES)]
                if pos[s] < len(wavs[s]):
                    e.pool_push_audio(s, wavs[s][pos[s]:pos[s] + p].contiguous())
                    pos[s] = min(pos[s] + p, len(wavs[s]))
            nA = {}
            for s in active:
                F_ = e.num_fbank_frames(pos[s])
                T = out_frames(F_) if F_ > 0 else 0
                nA[s] = T - min(Tf[s], T)
            M = sum(nA.values())
            keys = {(nA[s] == 0, Tf[s] == 0, nA[s], chunk[s]) for s in active if nA[s] > 0}
            groups_max = max(groups_max, len(keys))
            res, ran = wgmma_ran(e, lambda: e.pool_step(active, ctc_heads=ctc_heads))
            if M > 0:
                assert ran == (M >= UMMA_MIN_ROWS), (step, M, ran)
                classes[gemm_class(M)] = classes.get(gemm_class(M), 0) + 1
            for s, r in zip(active, res):
                what = f"streams={n_streams} step={step} slot={s} chunk={chunk[s]} T={r['T']} nA={nA[s]} M={M}"
                Tf[s] = r["T_final"]
                info = e.pool_info(s)
                if info["n_feat"] == 0:
                    continue
                feats = alias(info["feats_ptr"], (info["n_feat"], enc.cfg.feat_dim)).clone()
                worst.add("fbank", maxdiff(feats, enc.ref.fbank(wavs[s][:pos[s]])), what)
                rows = e.pool_encoder_rows(s, r["T"]).clone()
                worst.add(gemm_class(M), maxdiff(rows, enc.ref.encoder(feats, None, *chunk[s])[0]), what)
                for head in range(ctc_heads):
                    lp = enc.ref.ctc_lprobs(head, rows)
                    if near_tie_rows(lp):
                        near += 1
                        continue
                    want = collapse(lp.argmax(-1).tolist())
                    assert tuple(map(list, r["ctc"][head])) == tuple(map(list, want)), (what, head)
                    ctc_checked += 1
    finally:
        for s in slots:
            e.pool_reset(s)
            e.pool_set_chunk(s, 0, 0)
    e.check_async_error()
    report(f"encoder_pool_step_fp64_{n_streams}", gemm_classes=classes, max_groups=groups_max, ctc_checked=ctc_checked,
           ctc_near_tie_sequences=near, **worst.as_dict())
    assert n_streams == 1 or groups_max > 2, groups_max
    worst.check({"fbank": FBANK_TOL["pool"], "skinny": ENC_TOL["fp32"], "fp32": ENC_TOL["fp32"], "tc": ENC_TOL["tc"]})


# --------------------------------------------------------------------------------------------------------------------------------
# CTC heads
# --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ctc_heads_vs_fp64(enc):
    """ss_ctc_greedy, _rows (row0 > 0), _pair (equal and different row0) and _batch over the engine's T = 1024 encoder rows: arg-max by
    the margin rule against float64 masked log-probs, tokens and indices exactly ctc_collapse of the engine's arg-max (of the float64
    arg-max for _batch, which returns no arg-max, in sequences without near ties).  The checkpoint's pad and unk rows outrank the most
    frequent token wherever its logit is positive, so the mask decides those rows."""
    e = enc.e
    c = enc.cfg
    rows = e.encoder(enc.feats.unsqueeze(0).contiguous())[0].contiguous()
    T = rows.shape[0]
    lps = [enc.ref.ctc_lprobs(h, rows) for h in (0, 1)]
    res = {"near_ties": {}}
    for h in (0, 1):
        name = ("source_unigram", "ctc_target_unigram")[h]
        raw = F.linear(rows.double(), enc.ref.w[f"{name}_decoder.proj.weight"], enc.ref.w[f"{name}_decoder.proj.bias"]).argmax(-1)
        res[f"head{h}_rows_won_by_pad_or_unk"] = n_masked = int(((raw == c.pad) | (raw == c.unk)).sum())
        assert n_masked > 0, h
    ams = []
    for h in (0, 1):
        r = e.ctc_greedy(h, rows)
        am = r["argmax"]
        res["near_ties"][f"ctc_greedy head{h}"] = check_argmax(am, lps[h], f"ctc_greedy head {h}")
        n = int(r["count"][0])
        assert (r["tokens"][:n].tolist(), r["index"][:n].tolist()) == collapse(am.tolist()), h
        ams.append(am)
        for row0 in (1, 517, T - 1, T):
            buf = torch.full((T,), -7, dtype=torch.int64, device="cuda")
            buf[:row0] = am[:row0]
            toks = e.ctc_greedy_rows(h, rows, row0, buf)
            assert torch.equal(buf[:row0], am[:row0]), (h, row0)
            res["near_ties"][f"rows head{h} row0={row0}"] = check_argmax(buf[row0:], lps[h][row0:], f"rows head {h} row0 {row0}")
            assert tuple(toks) == collapse(buf.tolist()), (h, row0)
    for r0 in ((0, 0), (300, 300), (300, 700)):
        bufs = [torch.full((T,), -7, dtype=torch.int64, device="cuda") for _ in (0, 1)]
        for h in (0, 1):
            bufs[h][:r0[h]] = ams[h][:r0[h]]
        pair = e.ctc_greedy_rows_pair(rows, r0, bufs)
        for h in (0, 1):
            res["near_ties"][f"pair head{h} row0={r0[h]}"] = check_argmax(bufs[h][r0[h]:], lps[h][r0[h]:], f"pair {r0} head {h}")
            assert tuple(pair[h]) == collapse(bufs[h].tolist()), (r0, h)
    lengths = [4094, 1, 2001]
    x = torch.zeros(3, 4094, c.feat_dim, device="cuda")
    for b, l in enumerate(lengths):
        x[b, :l] = enc.feats[:l]
    batch_rows = e.encoder(x, lengths).contiguous()
    out, _ = e.ctc_greedy_batch(batch_rows)
    checked = 0
    for b in range(3):
        for h in (0, 1):
            lp = enc.ref.ctc_lprobs(h, batch_rows[b])
            if near_tie_rows(lp):
                continue
            assert tuple(out[b][h]) == collapse(lp.argmax(-1).tolist()), (b, h)
            checked += 1
    report("encoder_ctc_fp64", batch_sequences_checked=checked, **res)
    assert checked >= 3


# --------------------------------------------------------------------------------------------------------------------------------
# capacity errors
# --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_capacity_errors_leave_state(enc):
    """an engine with max_enc_frames = 64: T = 65 in ss_encoder_forward, ss_encoder_stream_step and ss_pool_step fails with
    SS_ERR_CAPACITY, launches nothing and leaves the stream state as it was: the next valid call still matches float64"""
    from streamspeech_b200.engine import Engine, EngineError

    SS_ERR_CAPACITY = -5
    e = Engine(enc.cfg, enc.sd, None, enc.gc, max_enc_frames=64)
    res = {}
    try:
        e.set_chunk(8)

        def refused(fn, what):
            n = e.launch_count()
            with pytest.raises(EngineError) as err:
                fn()
            assert err.value.code == SS_ERR_CAPACITY, (what, err.value.code, err.value.detail)
            assert e.launch_count() == n, what

        assert out_frames(257) == 65 and out_frames(256) == 64
        refused(lambda: e.encoder(enc.feats[:257].unsqueeze(0).contiguous()), "forward")
        out = e.encoder(enc.feats[:256].unsqueeze(0).contiguous())[0]
        res["forward T=64"] = maxdiff(out, enc.enc64(256, 8, 8))
        buf = torch.zeros(128, enc.cfg.enc_dim, device="cuda")
        e.encoder_stream_reset()
        assert e.encoder_stream_step(enc.feats[:200], buf) == (50, 48)
        kept = buf.clone()
        refused(lambda: e.encoder_stream_step(enc.feats[:257], buf), "stream step")
        assert torch.equal(buf, kept)
        assert e.encoder_stream_step(enc.feats[:256], buf) == (64, 64)
        res["stream after refusal"] = maxdiff(buf[:64], enc.enc64(256, 8, 8))
        e.pool_create(2, max_seconds=4)
        long_wav, short_wav = synth.make_audio(2.7, seed=61), synth.make_audio(1.0, seed=62)
        e.pool_push_audio(0, long_wav)
        e.pool_push_audio(1, short_wav)
        refused(lambda: e.pool_step([1, 0], ctc_heads=1), "pool step")
        r = e.pool_step([1], ctc_heads=1)[0]
        info = e.pool_info(1)
        feats = alias(info["feats_ptr"], (info["n_feat"], enc.cfg.feat_dim)).clone()
        res["pool after refusal"] = maxdiff(e.pool_encoder_rows(1, r["T"]), enc.ref.encoder(feats, None, 8, 8)[0])
        e.check_async_error()
    finally:
        e.close()
    report("encoder_capacity_errors", **res)
    for k, v in res.items():
        assert v < ENC_TOL["fp32"], (k, v)


# --------------------------------------------------------------------------------------------------------------------------------
# one 38 s utterance through the agents' three encoder paths
# --------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def long38():
    """engine, float64 oracle, the utterance, its oracle features and the fp64 encoder output (computed once)"""
    from oracle.streamspeech_oracle import StreamSpeechOracle, online_features
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    gc = synth.make_gcmvn(cfg)
    e = Engine(cfg, sd, None, gc)
    e.set_chunk(8)
    o = StreamSpeechOracle(cfg, sd, None, gc, chunk_size=8, dtype=F64)
    wav = synth.make_audio(38.0, seed=11)
    feats = online_features(wav, gc)
    ref = o.encoder(feats.unsqueeze(0), torch.tensor([feats.size(0)]))["encoder_out"][0][:, 0]
    assert ref.shape[0] > 900
    yield cfg, e, o, wav, feats, ref
    e.close()


def ctc_lprobs(cfg, o, enc64):
    out = []
    for name in ("source_unigram", "ctc_target_unigram"):
        lp = F.log_softmax(o.ctc_logits(name, enc64.unsqueeze(1))[0], dim=-1)
        lp[:, cfg.pad] = float("-inf")
        lp[:, cfg.unk] = float("-inf")
        out.append(lp)
    return out


@pytest.mark.gpu
def test_encoders_vs_fp64_oracle(long38):
    """one 38 s utterance (T = 950, chunk 8) against StreamSpeechOracle(dtype=float64).encoder: the full-prefix encoder (wgmma
    linears), streaming in 32-frame steps with and without the cluster kernel, and a one-slot pool fed 320 ms pushes (its rows against
    the float64 encoder of the pool's own features); CTC arg-max of both heads by the margin rule"""
    cfg, e, o, wav, feats, ref = long38
    T = ref.shape[0]
    fd = feats.float().cuda().contiguous()
    got = {"per_op": e.encoder(fd.unsqueeze(0))[0]}
    for cluster in (1, 0):
        e.set_option("persistent_encoder_cluster", cluster)
        buf = torch.zeros(1024, cfg.enc_dim, device="cuda")
        e.encoder_stream_reset()
        n0 = e.cluster_steps()
        Ts = 0
        for F_ in list(range(30, fd.shape[0], 32)) + [fd.shape[0]]:
            Ts, _ = e.encoder_stream_step(fd[:F_].contiguous(), buf)
        assert Ts == T
        assert (e.cluster_steps() > n0) == bool(cluster)
        got[f"stream_cluster{cluster}"] = buf[:T].clone()
    e.set_option("persistent_encoder_cluster", 1)
    e.encoder_stream_reset()
    e.check_async_error()
    lps = ctc_lprobs(cfg, o, ref)
    res = {}
    for name, x in got.items():
        d = maxdiff(x.cpu(), ref)
        near = [check_argmax(e.ctc_greedy(head, x.contiguous())["argmax"].cpu(), lps[head], name) for head in (0, 1)]
        res[name] = {"maxdiff": d, "near_ties": near}
        assert d < ENC_TOL["tc" if name == "per_op" else "stream"], (name, d)
    e.pool_create(1, max_seconds=40)
    n = 5120
    for i in range(0, len(wav), n):
        e.pool_push_audio(0, wav[i:i + n].contiguous())
        r = e.pool_step([0], ctc_heads=0)[0]
    info = e.pool_info(0)
    Tp = r["T"]
    pool_feats = alias(info["feats_ptr"], (info["n_feat"], cfg.feat_dim)).cpu()
    assert abs(Tp - T) <= 1 and maxdiff(pool_feats, feats[:pool_feats.shape[0]]) < 2e-3
    ref_pool = o.encoder(pool_feats.unsqueeze(0), torch.tensor([pool_feats.size(0)]))["encoder_out"][0][:, 0]
    rows = e.pool_encoder_rows(0, Tp).clone()
    d = maxdiff(rows.cpu(), ref_pool)
    near = [check_argmax(e.ctc_greedy(head, rows)["argmax"].cpu(), lp, "pool") for head, lp in enumerate(ctc_lprobs(cfg, o, ref_pool))]
    res["pool"] = {"maxdiff": d, "near_ties": near}
    report("long38_encoders_fp64", T=T, **res)
    assert d < ENC_TOL["stream"], ("pool", d)
