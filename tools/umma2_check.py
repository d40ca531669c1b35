#!/usr/bin/env python
"""Parity and timing of the wgmma conv / linear kernel (kernels_umma2.cu) against an fp64 torch
reference and the fp32 CUDA-core kernel.  Parts: conv (single ops), time (single-op timing), e2e (vocoder + unit decoder
with the tensor-core routing switched on).  Run every part under `timeout` (a wrong mbarrier protocol would spin)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.nn.functional as F
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.engine import Engine

torch.set_grad_enabled(False)
part = sys.argv[1] if len(sys.argv) > 1 else "conv"
cfg = ModelConfig(); cfg.enc_layers = 2
e = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), None)
g = torch.Generator().manual_seed(0)
res, ok = {}, True


def ref_conv(x, w, b, k, dil, pad, slope):
    L, C = x.shape
    N = w.shape[0]
    xx = x.double()
    if slope != 1.0:
        xx = torch.where(xx > 0, xx, xx * slope)
    wt = w.double().view(N, k, C).permute(0, 2, 1).contiguous()
    xp = F.pad(xx.t().unsqueeze(0), (pad, (k - 1) * dil - pad))
    return (F.conv1d(xp, wt, b.double(), dilation=dil)[0].t()).float()


SHAPES = [  # L, C, N, k, dil, pad_left, slope
    (128, 32, 16, 1, 1, 0, 1.0), (100, 64, 128, 3, 1, 1, 0.1), (260, 256, 256, 11, 5, 25, 0.1), (1040, 128, 128, 7, 3, 9, 0.1),
    (4160, 64, 64, 3, 1, 1, 0.1), (8320, 32, 32, 11, 1, 5, 0.1), (16640, 16, 16, 7, 5, 15, 0.1), (300, 128, 512, 7, 1, 3, 1.0),
    (775, 512, 2048, 1, 1, 0, 1.0), (1250, 2048, 512, 1, 1, 0, 1.0), (200, 512, 1005, 1, 1, 0, 1.0), (261, 256, 128, 3, 1, 2, 0.1),
    (130, 48, 48, 5, 2, 4, 0.1),
]

if part == "conv":
    for (L, C, N, k, dil, pad, slope) in SHAPES:
        x = torch.randn(L, C, generator=g); w = torch.randn(N, k * C, generator=g) / (k * C) ** 0.5; b = torch.randn(N, generator=g)
        ref = ref_conv(x, w, b, k, dil, pad, slope)
        xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
        d32 = float((e.op_conv1d(xd, wd, bd, k, dil, pad, slope, 0).cpu() - ref).abs().max())
        row = {"fp32_simt": d32}
        for mode in (12, 13):
            e.set_option("umma2_cache_clear", 1)
            got = e.op_conv1d(xd, wd, bd, k, dil, pad, slope, mode).cpu()
            d = float((got - ref).abs().max())
            row[f"umma2_p{mode - 10}"] = d
            tol = 2e-4 if mode == 13 else 2e-3
            good = d < tol
            ok &= good
            print(f"L={L} C={C} N={N} k={k} dil={dil} pad={pad} mode={mode}: maxdiff {d:.3e} (fp32 SIMT {d32:.3e})", "OK" if good else "FAIL", flush=True)
        res[f"conv_L{L}_C{C}_N{N}_k{k}_d{dil}"] = row
elif part == "time":
    for (L, C, N, k, dil, pad, slope) in [(260, 256, 256, 11, 5, 25, 0.1), (260, 256, 256, 3, 1, 1, 0.1), (1040, 128, 128, 7, 3, 9, 0.1),
                                           (4160, 64, 64, 7, 1, 3, 0.1), (8320, 32, 32, 11, 1, 5, 0.1), (16640, 16, 16, 7, 5, 15, 0.1),
                                           (2500, 256, 256, 11, 1, 5, 0.1), (775, 512, 2048, 1, 1, 0, 1.0), (775, 2048, 512, 1, 1, 0, 1.0),
                                           (775, 512, 512, 1, 1, 0, 1.0), (1250, 512, 1536, 1, 1, 0, 1.0), (250, 256, 1024, 1, 1, 0, 1.0)]:
        x = torch.randn(L, C, device="cuda"); w = torch.randn(N, k * C, device="cuda") / (k * C) ** 0.5; b = torch.zeros(N, device="cuda")
        e.set_option("umma2_cache_clear", 1)
        row = {}
        for mode in (0, 2, 12, 13):
            fn = lambda: e.op_conv1d(x, w, b, k, dil, pad, slope, mode)
            for _ in range(3): fn()
            s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize(); s.record()
            for _ in range(20): fn()
            t.record(); torch.cuda.synchronize()
            us = s.elapsed_time(t) / 20 * 1e3
            row[f"mode{mode}_us"] = us
        row["gflop"] = 2.0 * L * C * k * N / 1e9
        res[f"time_L{L}_C{C}_N{N}_k{k}"] = row
        print(L, C, N, k, {kk: round(v, 2) for kk, v in row.items()}, flush=True)
elif part == "stamps":
    import ctypes
    e.set_option("umma2_debug", 1)
    names = ["start", "setup_done", "first_A_ready", "issuer_saw_A", "issuer_saw_B", "last_commit", "last_A_ready", "acc_full_seen", "epilogue_done", "tmem_ld_done", "transpose_written", "first_block_stored"]
    for (L, C, N, k, dil, pad, slope, mode) in [(160, 256, 1024, 1, 1, 0, 1.0, 13), (775, 512, 2048, 1, 1, 0, 1.0, 13), (775, 2048, 512, 1, 1, 0, 1.0, 13),
                                                (260, 256, 256, 11, 5, 25, 0.1, 12), (260, 256, 256, 3, 1, 1, 0.1, 12), (4160, 64, 64, 7, 1, 3, 0.1, 12)]:
        x = torch.randn(L, C, device="cuda"); w = torch.randn(N, k * C, device="cuda") / (k * C) ** 0.5; b = torch.zeros(N, device="cuda")
        e.set_option("umma2_cache_clear", 1)
        for _ in range(3): e.op_conv1d(x, w, b, k, dil, pad, slope, mode)
        torch.cuda.synchronize()
        buf = (ctypes.c_uint64 * 16)()
        e._check(e.lib.ss_debug_copy(e._h, b"umma2_ts", buf, ctypes.sizeof(buf)))
        t = [int(v) for v in buf[:12]]
        rel = {n: (t[i] - t[0]) for i, n in enumerate(names)}
        res[f"stamps_L{L}_C{C}_N{N}_k{k}"] = rel
        print(L, C, N, k, "ns from CTA start:", rel, flush=True)
    e.set_option("umma2_debug", 0)
else:
    gold = np.load(os.path.join(ROOT, "tests", "golden", "vocoder.npz"))
    codes = torch.from_numpy(gold["code"][0].astype(np.int64)).cuda()
    dur, cum = e.vocoder_durations(codes, True); total = int(cum[-1].item())
    base = e.vocoder_generate(total, 0, total, 0).cpu()
    for mode in (12, 13):
        e.set_option("umma_vocoder", mode)
        wav = e.vocoder_generate(total, 0, total, 0).cpu()
        d = float((wav - torch.from_numpy(gold["wav"])).abs().max())
        res[f"vocoder_umma2_mode{mode}"] = {"maxdiff_vs_reference_fixture": d, "maxdiff_vs_fp32_path": float((wav - base).abs().max())}
        print("vocoder mode", mode, res[f"vocoder_umma2_mode{mode}"], flush=True)
        ok &= d < 1e-3
        for fn_name, fn in (("full", lambda: e.vocoder_generate(total, 0, total, 0)), ("tail30", lambda: e.vocoder_generate(total, total - 30, 30, -1))):
            for _ in range(2): fn()
            s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize(); s.record()
            for _ in range(5): fn()
            t.record(); torch.cuda.synchronize()
            res[f"vocoder_umma2_mode{mode}"][f"ms_{fn_name}"] = s.elapsed_time(t) / 5
    e.set_option("umma_vocoder", 0)
    for fn_name, fn in (("full", lambda: e.vocoder_generate(total, 0, total, 0)), ("tail30", lambda: e.vocoder_generate(total, total - 30, 30, -1))):
        for _ in range(2): fn()
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); s.record()
        for _ in range(5): fn()
        t.record(); torch.cuda.synchronize()
        res.setdefault("vocoder_fp32", {})[f"ms_{fn_name}"] = s.elapsed_time(t) / 5
    print({k: v for k, v in res.items()}, flush=True)
    dec = np.load(os.path.join(ROOT, "tests", "golden", "decoders.npz"))
    feats = torch.from_numpy(dec["mt_feats"]).cuda()
    big = feats.repeat(6, 1).contiguous()  # 42 tokens -> 1050 unit positions
    ref = e.t2u_unit_decode(big, debug=True)
    for mode in (13, 0):
        e.set_option("umma_linear", mode)
        got = e.t2u_unit_decode(big, debug=True)
        for _ in range(2): e.t2u_unit_decode(big)
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); s.record()
        for _ in range(5): e.t2u_unit_decode(big)
        t.record(); torch.cuda.synchronize()
        d = float((got["logits"] - ref["logits"]).abs().max())
        same = got["argmax"].tolist() == ref["argmax"].tolist()
        res[f"unit_decoder_mode{mode}"] = {"logits_maxdiff_vs_fp32_path": d, "argmax_equal": same, "ms": s.elapsed_time(t) / 5}
        print("unit decoder mode", mode, res[f"unit_decoder_mode{mode}"], flush=True)
        ok &= same and d < 1e-3
    e.set_option("umma_linear", 0)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "gpurun_out", f"umma2_check_{part}.json"), "w"), indent=1)
print("UMMA2_CHECK", part, "PASS" if ok else "FAIL")
sys.exit(0 if ok else 1)
