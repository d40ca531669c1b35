#!/usr/bin/env python
"""16 kHz vs 48 kHz stream pool on one GPU: concurrent streaming-ASR utterances (default 32 x 10 s at 160 ms chunks, BASELINE
configs[3]) through a 16 kHz pool and through a 48 kHz pool fed the same synthetic signals upsampled to 48 kHz.  Each pool lives on its
own engine handle (one pool per handle); the timed runs alternate between the two.

Reports, as one JSON line on stdout:
  - ms per round of each pool (CUDA events around whole runs: every round is one push per stream + one ss_pool_step + the token read),
    best and median of --repeats runs, with the resample timing switched off;
  - the resample kernel (ms_resample_3to1, one launch per 48 kHz step) timed with CUDA events around its launch (engine option
    persistent_time) in one further run of the 48 kHz pool, and its share of that run's step time; then the kernel alone
    (torch.profiler, CUDA activities) in a run of its own;
  - its achieved bytes/s (12 B in + 4 B out per output sample) against the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s;
  - the card name, power limit and max SM clock, read in the same process.

  python tools/pool_rate_bench.py [--streams 32] [--seconds 10] [--chunk-ms 160] [--repeats 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torchaudio  # noqa: E402

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.engine import Engine  # noqa: E402
from streamspeech_b200.scheduler import StreamPool  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet (HBM3)


def card():
    """name, power limit and max SM clock of the device this process runs on"""
    p = torch.cuda.get_device_properties(0)
    info = {"name": p.name}
    try:
        bus = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
        out = subprocess.run(["nvidia-smi", f"--id={bus}", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60)
        limit, clock = (x.strip() for x in out.stdout.strip().split(","))
        info.update(power_limit=limit, max_sm_clock=clock)
    except Exception as e:  # the numbers below are still reported, marked as measured on an unidentified power limit
        info.update(power_limit=f"not read ({type(e).__name__})", max_sm_clock=None)
    return info


def make_pool(cfg, sd, gcmvn, rate, wavs, args):
    eng = Engine(cfg, sd, None, gcmvn)
    eng.set_chunk(args.chunk_ms // 40, min(args.chunk_ms // 40, 16))  # speech_to_text.asr agent :361-375
    pool = StreamPool(eng, n_slots=args.streams, max_seconds=int(args.seconds) + 1, ctc_heads=1, sample_rate=rate)
    slots = [pool.acquire() for _ in range(args.streams)]
    n = rate * args.chunk_ms // 1000

    def run():
        """one pass over all utterances; returns (ms, rounds, final tokens)"""
        for sl in slots:
            pool.reset(sl)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        rounds = 0
        for i in range(0, wavs[0].numel(), n):
            fin = i + n >= wavs[0].numel()
            for j, sl in enumerate(slots):
                pool.push(sl, wavs[j][i:i + n], finished=fin)
            pool.flush()
            rounds += 1
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e), rounds, sum(len(pool.results[sl]["ctc"][0][0]) for sl in slots)

    return eng, run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--chunk-ms", type=int, default=160)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pool_rate_bench needs a CUDA device: nothing is measured without one")
    torch.set_grad_enabled(False)
    cfg = ModelConfig()
    sd, gcmvn = synth.make_model_state_dict(cfg, 0), synth.make_gcmvn(cfg)
    wavs16 = [synth.make_audio(args.seconds, seed=5000 + j).contiguous() for j in range(args.streams)]
    # the same signals at 48 kHz (band-limited upsampling), so that both pools decode comparable audio
    wavs48 = [torchaudio.functional.resample(w, 16000, 48000).contiguous() for w in wavs16]
    eng16, run16 = make_pool(cfg, sd, gcmvn, 16000, wavs16, args)
    eng48, run48 = make_pool(cfg, sd, gcmvn, 48000, wavs48, args)
    run16()  # warm-up: workspaces, packed weight caches
    run48()
    t16, t48 = [], []
    for _ in range(args.repeats):  # alternate the pools: the host and GPU are shared
        ms, rounds, tok16 = run16()
        t16.append(ms / rounds)
        ms, rounds, tok48 = run48()
        t48.append(ms / rounds)
    # the resample kernel: CUDA events around each of its launches, in one more run of the 48 kHz pool
    eng48.set_option("persistent_time", 1)
    eng48.pool_resample_time()  # drop anything recorded before
    ms_run, rounds, _ = run48()
    r_ms, r_launches, r_bytes = eng48.pool_resample_time()
    eng48.set_option("persistent_time", 0)
    # The event window also holds the launch gap after ss_pool_step's entry synchronisation (the GPU is idle until the host has
    # enqueued the kernel), so it bounds the kernel time from above.  The kernel alone: torch.profiler over a run of its own.
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run48()
    ka = [k for k in prof.key_averages() if "ms_resample_3to1_kernel" in k.key]
    k_us, k_n = sum(k.device_time_total for k in ka), sum(k.count for k in ka)
    out = {
        "workload": f"streaming ASR, chunk {args.chunk_ms} ms, {args.streams} concurrent {args.seconds:g} s utterances, one GPU",
        "card": card(),
        "rounds": rounds,
        "ms_per_round_16k": {"best": min(t16), "median": statistics.median(t16), "runs": t16},
        "ms_per_round_48k": {"best": min(t48), "median": statistics.median(t48), "runs": t48},
        "tokens_final_16k": tok16,
        "tokens_final_48k": tok48,
        "resample": {
            "launches": r_launches,
            "ms_total": r_ms,
            "us_per_launch": 1e3 * r_ms / max(r_launches, 1),
            "share_of_step": r_ms / ms_run,
            "timed_run_ms_per_round": ms_run / rounds,
            "bytes": r_bytes,
            "achieved_bytes_per_s": r_bytes / (r_ms * 1e-3) if r_ms > 0 else None,
            "frac_of_3.35TB/s": r_bytes / (r_ms * 1e-3) / HBM_BYTES_PER_S if r_ms > 0 else None,
            "profiler_kernels": k_n,
            "profiler_us_per_kernel": k_us / max(k_n, 1),
            "profiler_bytes_per_s": r_bytes / (k_us * 1e-6) if k_us > 0 else None,
            "profiler_frac_of_3.35TB/s": r_bytes / (k_us * 1e-6) / HBM_BYTES_PER_S if k_us > 0 else None,
        },
    }
    print(json.dumps(out))
    eng16.close()
    eng48.close()


if __name__ == "__main__":
    main()
