"""Device time of one greedy step of the incremental MT search against the number of self-attention entries, across the 1024-entry
edge where the persistent MT kernels switch from the one-pass attention to the block loop (attend_head_long, kernels_persist_mt.cuh).

Arms: the single-token kernel (ss_mt_greedy_incremental) and the batched kernel (ss_pool_mt_greedy_incremental) with 8 and 32 rows, on
the synthetic 12-layer model with its eos row zeroed, so that a search always fills the length it is given.  A point is a burst of 16
steps in one launch whose self-attention spans 16 consecutive entry counts: [n - 15, n] for n <= 1024 and [n, n + 15] above, so no
burst straddles the edge.  Per repetition the state is rebuilt by an untimed search and the burst is timed with CUDA events around the
entry point (the launch, the token upload and the read-back of the burst); every point is warmed once and repeated until it has
run --steps steps.  Reported: microseconds per step (median and minimum over the repetitions) and the card's name, power limit and max
SM clock, read in the same run.  The point is the shape: growth roughly linear in the entries and no cliff between 1024 and 1025.

    python tools/mt_long_attention_bench.py [--entries 256 1000 1024 1025 1400 2000] [--rows 8 32] [--steps 208] [--out results/mt_long_attention.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.engine import Engine  # noqa: E402

BURST = 16


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return out, e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, nargs="+", default=[256, 1000, 1024, 1025, 1400, 2000])
    ap.add_argument("--rows", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--steps", type=int, default=208)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    for k in ("target_unigram_decoder.embed_tokens.weight", "target_unigram_decoder.output_projection.weight"):
        if k in sd:
            sd[k] = sd[k].clone()
            sd[k][cfg.eos] = 0.0  # the eos logit is 0, below the best of the others: no search ends before its max_len
    eng = Engine(cfg, sd, None, synth.make_gcmvn(cfg), max_mt_positions=max(a.entries) + BURST + 8)
    eng.set_chunk(8, 8)
    n_slots = max(a.rows)
    eng.pool_create(n_slots, max_seconds=3)
    slots = list(range(n_slots))
    for sl in slots:
        eng.pool_push_audio(sl, synth.make_audio(2.0, seed=700 + sl).contiguous())
    res = eng.pool_step(slots, ctc_heads=0)
    enc = eng.pool_encoder_rows(0, res[0]["T"]).clone()
    reps = -(-a.steps // BURST)
    result = {"gpu": gpu_info(), "steps_per_point": reps * BURST, "burst": BURST, "rows": []}
    for n in a.entries:
        lo = n - BURST + 1 if n <= 1024 else n
        fill = lo - 2  # a fresh search of `fill` tokens leaves fill + 1 entries; the next call's first step then attends over lo
        row = {"entries": [lo, lo + BURST - 1], "us_per_step": {}}
        for arm in ["single"] + [f"batched_{r}" for r in a.rows]:
            ms = []
            for rep in range(reps + 1):  # (the first repetition warms the point)
                if arm == "single":
                    eng.mt_incremental_reset()
                    hyp = eng.mt_greedy_incremental(enc, None, fill, fill)
                    out, t = timed(lambda: eng.mt_greedy_incremental(enc, hyp, BURST - 1, fill + BURST))
                    assert len(hyp) == fill and len(out) == fill + BURST - 1
                else:
                    sl = slots[:int(arm.split("_")[1])]
                    for s in sl:  # a slot's incremental state goes with its audio: start the utterance again
                        eng.pool_reset(s)
                        eng.pool_push_audio(s, synth.make_audio(2.0, seed=700 + s).contiguous())
                    eng.pool_step(sl, ctc_heads=0)
                    hyps = eng.pool_mt_greedy_incremental(sl, [None] * len(sl), [fill] * len(sl), [fill] * len(sl))
                    out, t = timed(lambda: eng.pool_mt_greedy_incremental(sl, hyps, [BURST - 1] * len(sl), [fill + BURST] * len(sl)))
                    assert all(len(h) == fill for h in hyps) and all(len(o) == fill + BURST - 1 for o in out)
                if rep:
                    ms.append(t)
            row["us_per_step"][arm] = {"median": statistics.median(ms) * 1e3 / BURST, "min": min(ms) * 1e3 / BURST}
        print(json.dumps(row), flush=True)
        result["rows"].append(row)
    print(json.dumps({"gpu": result["gpu"], "steps_per_point": result["steps_per_point"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
