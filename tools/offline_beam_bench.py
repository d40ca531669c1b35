"""MT beam search of the offline generator (ss_mt_beam_batch) against its greedy search (ss_mt_greedy_batch).

Workload: the offline model (uni_encoder = False, synthetic weights), B x 15 s utterances (synth.make_audio, seeds 7000 + b as
bench.py's offline leg), padded encoder output, max_len_b = 100; B in {1, 8, 32} and K in {1 (greedy), 2, 5, 10}.  The arms of
one B run alternately after a warm-up, each call timed with CUDA events (median of --reps), with its kernel launches counted.
Reported per arm: device time per search, decode steps (the longest finalized hypothesis, eos included), time per step, launches
and host synchronisations.  The synchronisations are counted from the burst structure of the calls, not traced: the beam search
makes one per burst of 16 steps and launch group (its done-flag read) and one for the final read-back; the greedy search one
per burst and group plus one for its initial token upload.  A first call that grows the buffers synchronises more.

To isolate what the beam phases cost (candidates, selection, self-attention reorder), K = 5 over B = 6 samples (30 rows, one
launch) is compared with greedy over B = 30 samples (30 rows, one launch), per decode step.

    python tools/offline_beam_bench.py [--batches 1 8 32] [--beams 1 2 5 10] [--reps 3] [--out results/offline_beam_bench.json]
"""
import argparse
import json
import math
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
BURST = 16
MAX_ROWS = 32


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        raise SystemExit("nvidia-smi unavailable: the card cannot be named")
    return q.stdout.strip().splitlines()[0]


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


def arm(eng, enc, lens, K):
    if K == 1:
        return lambda: eng.mt_greedy_batch(enc, lens, MAX_LEN_B)
    return lambda: eng.mt_beam_batch(enc, lens, K, MAX_LEN_B)


def steps_and_syncs(res, K, B):
    """decode steps of the search and the host synchronisations its calls make (see the module docstring)"""
    if K == 1:
        steps = min(MAX_LEN_B, max(len(h) for h in res) + 1)
        groups = [list(range(g, min(B, g + MAX_ROWS))) for g in range(0, B, MAX_ROWS)]
        syncs = sum(math.ceil(min(MAX_LEN_B, max(len(res[b]) for b in g) + 1) / BURST) + 1 for g in groups)
        return steps, syncs
    per = MAX_ROWS // K
    groups = [list(range(g, min(B, g + per))) for g in range(0, B, per)]
    last = [max(len(h["tokens"]) for b in g for h in res[b]) + 1 for g in groups]  # steps of each group (eos included)
    return max(last), sum(math.ceil(n / BURST) + 1 for n in last)


def run(eng, reps, cases):
    """cases: {name: (B, K)}; alternated after one warm-up each"""
    data = {n: encode(eng, B) for n, (B, _) in cases.items()}
    fns = {n: arm(eng, *data[n], K) for n, (_, K) in cases.items()}
    for f in fns.values():
        f()
    times = {n: [] for n in cases}
    out = {}
    for _ in range(reps):
        for n, f in fns.items():
            ms, nl, r = timed(eng, f)
            times[n].append(ms)
            out[n] = (nl, r)
    rows = []
    for n, (B, K) in cases.items():
        nl, r = out[n]
        med = sorted(times[n])[len(times[n]) // 2]
        steps, syncs = steps_and_syncs(r, K, B)
        rows.append({"case": n, "B": B, "K": K, "rows": B * K, "ms_median": med, "ms_all": times[n], "steps": steps,
                     "us_per_step": 1e3 * med / steps, "launches": nl, "host_syncs": syncs})
        print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--beams", type=int, nargs="+", default=[1, 2, 5, 10])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    info = gpu_info()
    cfg = ModelConfig()
    cfg.uni_encoder = False
    eng = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    eng.set_chunk(None, None)
    result = {"gpu": info, "max_len_b": MAX_LEN_B, "seconds": 15.0, "grid": [], "isolation": []}
    for B in args.batches:
        result["grid"] += run(eng, args.reps, {f"B{B}_K{K}": (B, K) for K in args.beams})
    result["isolation"] = run(eng, args.reps, {"beam_K5_B6": (6, 5), "greedy_B30": (30, 1)})
    print(json.dumps({"gpu": info}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
