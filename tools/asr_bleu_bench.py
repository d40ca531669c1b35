"""Throughput of the ASR-BLEU transcriber (ss_asr_transcribe) on the seeded Large-shape wav2vec 2.0 CTC checkpoint.

Workload: N synthetic utterances of ragged length (synth.make_audio, uniform in [--min-s, --max-s]), the kind of wavs/ directory an
evaluation leaves.  Reported, with the card's name, power limit and max SM clock read in the same run:

  batched       audio-s/s of ASRTranscriber.transcribe over all N (batches of --batch-seconds of audio), device-synchronised wall clock
  per_file      audio-s/s of one call per utterance (what the reference does), same clock
  stages_ms     device time per stage over one batched pass (CUDA events: extractor, feature projection + positional conv, layers,
                final LayerNorm + proj + arg-max + collapse)
  launches      kernels per ss_asr_transcribe call in the batched pass
  identical     whether every utterance's letters agree between the two passes

    python tools/asr_bleu_bench.py --utterances 64 --json out.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.asr import ASRTranscriber  # noqa: E402
from streamspeech_b200.engine import load_library  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=64)
    ap.add_argument("--min-s", type=float, default=2.0)
    ap.add_argument("--max-s", type=float, default=12.0)
    ap.add_argument("--batch-seconds", type=float, default=160.0)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    g = np.random.default_rng(0)
    secs = g.uniform(a.min_s, a.max_s, a.utterances)
    waves = [synth.make_audio(float(s), seed=1000 + i).numpy() for i, s in enumerate(secs)]
    audio_s = float(sum(len(w) for w in waves)) / 16000
    tr = ASRTranscriber("synthetic", None, 0, max_batch_samples=int(a.batch_seconds * 16000), time_stages=True)
    lib = load_library()
    tr.transcribe(waves[:4])  # warm-up: module load, workspace, packed weights
    for w in waves[:2]:
        tr.transcribe([w])
    tr.engine.stage_ms()
    torch.cuda.synchronize()
    l0 = lib.ss_launch_count(None)
    t0 = time.perf_counter()
    batched = tr.transcribe(waves)
    torch.cuda.synchronize()
    t_b = time.perf_counter() - t0
    launches = lib.ss_launch_count(None) - l0
    calls = len(tr.batches([len(w) for w in waves]))
    stages = tr.engine.stage_ms()
    t0 = time.perf_counter()
    single = [tr.transcribe([w])[0] for w in waves]
    torch.cuda.synchronize()
    t_s = time.perf_counter() - t0
    tr.engine.stage_ms()
    res = {"card": card(), "utterances": a.utterances, "audio_s": round(audio_s, 1), "batch_calls": calls,
           "batched_audio_s_per_s": round(audio_s / t_b, 1), "batched_wall_s": round(t_b, 3),
           "per_file_audio_s_per_s": round(audio_s / t_s, 1), "per_file_wall_s": round(t_s, 3),
           "stages_ms": dict(zip(["extractor", "proj_pos_conv", "layers", "proj_argmax"], [round(x, 1) for x in stages])),
           "launches_per_call": round(launches / calls, 1), "identical": batched == single,
           "est_gflop_per_audio_s": 36.0}
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
