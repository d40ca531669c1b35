"""Greedy MT search of the offline generator: one ss_mt_greedy call per sample vs one ss_mt_greedy_batch call per batch.

Workload: the offline model (uni_encoder = False, synthetic weights), B x 15 s utterances (synth.make_audio, seeds 7000 + b as
bench.py's offline leg), padded encoder output, max_len_b = 100.  For each B the two arms run alternately after a warm-up;
each call is timed with CUDA events and its kernel launches are counted.  The tokens of both arms must be identical.  For
B = 1 the batched call takes the single-token kernel (option mt_batch_min_rows = 2); the batched kernel is also timed there
with the option at 1, which is what that routing rests on.

A torch.profiler pass over one batched call per B gives the batched kernel's device time per decode step, and the MT weight
bytes one step reads (every GEMV weight of the 4 layers plus the tied output projection, read once per step: algorithmic
bytes, not measured DRAM traffic) over that time.

    python tools/offline_mt_bench.py [--batches 1 8 32] [--reps 5] [--out results/offline_mt_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.engine import Engine  # noqa: E402

MAX_LEN_B = 100


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def encode(eng, B, seconds=15.0):
    feats = [eng.fbank(synth.make_audio(seconds, seed=7000 + b).cuda()) for b in range(B)]
    F = max(f.shape[0] for f in feats)
    src = torch.zeros(B, F, eng.cfg.feat_dim, device="cuda")
    for b, f in enumerate(feats):
        src[b, : f.shape[0]] = f
    lens = [f.shape[0] for f in feats]
    return eng.encoder(src, lens), [eng.encoder_out_frames(n) for n in lens]


def timed(eng, fn):
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n0 = eng.launch_count()
    s.record()
    r = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), eng.launch_count() - n0, r


def mt_weight_bytes(cfg):
    d, f = cfg.mt_dim, cfg.mt_ffn
    per_layer = 3 * d * d + d * d + d * d + d * d + d * f + f * d  # QKV, Wo, Wcq, Wco, FC1, FC2
    return 4.0 * (cfg.mt_layers * per_layer + cfg.tgt_vocab * d)


def kernel_ms(fn, name):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total_us, n = 0.0, 0
    for ev in prof.events():
        if name in ev.name and ev.device_type.name == "CUDA":
            total_us += ev.device_time
            n += 1
    return total_us / 1e3, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    cfg = ModelConfig()
    cfg.uni_encoder = False
    eng = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    eng.set_chunk(None, None)
    result = {"gpu": gpu_info(), "max_len_b": MAX_LEN_B, "seconds": 15.0, "rows": []}
    wbytes = mt_weight_bytes(cfg)
    for B in args.batches:
        enc, lens = encode(eng, B)

        def loop():
            return [eng.mt_greedy(enc[b, : lens[b]].contiguous(), None, -1, max_len_b=MAX_LEN_B)[0] for b in range(B)]

        def batch():
            return eng.mt_greedy_batch(enc, lens, MAX_LEN_B)

        def batch_kernel():  # the batched kernel even for one row
            eng.set_option("mt_batch_min_rows", 1)
            try:
                return eng.mt_greedy_batch(enc, lens, MAX_LEN_B)
            finally:
                eng.set_option("mt_batch_min_rows", 2)

        arms = {"per_sample_loop": loop, "batch_call": batch}
        if B < 2:
            arms["batch_kernel_forced"] = batch_kernel
        times = {k: [] for k in arms}
        launches, toks = {}, {}
        for fn in arms.values():  # warm-up
            fn()
        for _ in range(args.reps):
            for k, fn in arms.items():
                ms, nl, r = timed(eng, fn)
                times[k].append(ms)
                launches[k] = nl
                toks[k] = r
        for k in arms:
            assert toks[k] == toks["per_sample_loop"], f"B={B}: {k} tokens differ from the per-sample search"
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        steps = min(MAX_LEN_B, max(len(h) for h in toks["batch_call"]) + 1)  # the forced-eos step needs no work
        kfn = batch if B >= 2 else batch_kernel
        k_ms, k_n = kernel_ms(kfn, "mt_decode_batch_kernel")
        row = {"B": B, "ms_median": med, "ms_all": times, "launches": launches, "speedup_batch_vs_loop": med["per_sample_loop"] / med["batch_call"],
               "tokens_identical": True, "hyp_lengths": [len(h) for h in toks["batch_call"]], "decode_steps": steps,
               "batch_call_path": "batched kernel" if B >= 2 else "single-token kernel (per sample)",
               "batched_kernel": {"launches": k_n, "ms_total": k_ms, "us_per_step": 1e3 * k_ms / steps,
                                  "mt_weight_bytes_per_step": wbytes,
                                  "algorithmic_GBps": wbytes / (k_ms / steps * 1e-3) / 1e9 if k_ms > 0 else None}}
        result["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"gpu": result["gpu"]}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
