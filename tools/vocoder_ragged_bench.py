"""The vocoder of n sequences in one ragged call (ss_vocoder_durations_ragged + ss_vocoder_generate_ragged) against the per-stream
loop of single calls (ss_vocoder_durations + host read of the cumsum + ss_vocoder_generate) on the same codes, synthetic vocoder.

Shapes:
  * streaming: n in {1, 8, 32} streams of 40 units (durations predicted), each emitting its last 28 frames with the receptive field
    of left context (the streaming agent's call);
  * offline: 32 utterances of 750 frames (one frame per code), whole-sequence passes.

The two arms alternate (--reps times each); each run is timed with CUDA events on the stream from the first call to the last
(one device synchronise per run) and its kernel launches are counted.  The outputs of the two arms are compared bit for bit first.
The card's name, power limit and max SM clock are read in the same run.

    python tools/vocoder_ragged_bench.py [--reps 20] [--out results/vocoder_ragged_bench.json]
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


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def per_stream(eng, codes, dp, window):
    out = []
    for c in codes:
        _, cum = eng.vocoder_durations(c, dp)
        total = int(cum[-1].item())  # the single agent's host read
        f0, nf, lc = window(total)
        out.append(eng.vocoder_generate(total, f0, nf, lc))
    return out


def ragged(eng, codes, dp, window):
    _, cums, _ = eng.vocoder_durations_ragged(codes, dp)
    args = [(cs[-1],) + window(cs[-1]) for cs in cums]
    return eng.vocoder_generate_ragged(*zip(*args))


def timed(eng, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = eng.launch_count()
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), eng.launch_count() - l0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    cfg = ModelConfig().tiny()  # the smallest model next to the vocoder (never run)
    eng = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), None)
    g = torch.Generator().manual_seed(0)
    V = cfg.vocoder.num_embeddings
    rf = eng.vocoder_receptive_field
    shapes = [(f"streaming_{n}x28_new_frames", [torch.randint(0, V, (40,), generator=g).cuda() for _ in range(n)], True,
               lambda t: (t - min(28, t), min(28, t), -1)) for n in (1, 8, 32)]
    shapes.append(("offline_32x750_frames", [torch.randint(0, V, (750,), generator=g).cuda() for _ in range(32)], False, lambda t: (0, t, 0)))
    result = {"gpu": gpu_info(), "receptive_field_frames": rf, "rows": []}
    for name, codes, dp, window in shapes:
        ref = [w.clone() for w in per_stream(eng, codes, dp, window)]
        got = ragged(eng, codes, dp, window)
        assert all(torch.equal(x, y) for x, y in zip(ref, got)), f"{name}: the ragged call differs from the per-stream loop"
        ms = {"per_stream": [], "ragged": []}
        launches = {}
        for _ in range(a.reps):
            for arm, fn in (("per_stream", per_stream), ("ragged", ragged)):
                t, n_launch = timed(eng, lambda: fn(eng, codes, dp, window))
                ms[arm].append(t)
                launches[arm] = n_launch
        med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
        row = {"shape": name, "streams": len(codes), "ms_median": med, "ms_min": {k: min(v) for k, v in ms.items()},
               "speedup_ragged_vs_per_stream": med["per_stream"] / med["ragged"], "launches_per_call": launches, "identical_outputs": True}
        print(json.dumps(row), flush=True)
        result["rows"].append(row)
    print(json.dumps({"gpu": result["gpu"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
