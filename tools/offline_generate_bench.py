"""Wall clock and device time of `python -m streamspeech_b200.generate` on a synthetic split, and the cost of the unit scores.

The workload is what pred.offline-s2st.sh runs at --max-tokens 10000: N synthetic utterances of 3-12 s (synth.make_audio, fbank on the
CPU) written as a stored-zip fbank split with gcmvn, then the whole front door in this process (reads, batches, generation, output
files).  Reported, with the card's name, power limit and max SM clock read in the same run:

  wall          seconds of main() and audio-s/s (source seconds over wall seconds), reads and writes included
  stages        device time per stage of generate() summed over the run (CUDA events around each engine call of the stage)
  unit_scores   the T2U + unit-decoder call of every batch without scores (ss_t2u_unit_decode_batch) and with them
                (ss_t2u_unit_decode_batch_scored), alternated, median of --reps runs of the whole split, device time

    python tools/offline_generate_bench.py --utterances 256 --reps 5 --json out.json
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import zipfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from streamspeech_b200 import generate as G  # noqa: E402
from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.engine import Engine  # noqa: E402

STAGES = {"encoder": "encoder", "ctc_greedy_batch": "ctc", "mt_greedy_batch": "mt_search", "mt_beam_batch": "mt_search",
          "mt_features_batch": "mt_features", "t2u_unit_decode_batch_scored": "t2u_units"}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"torch_name": torch.cuda.get_device_name(0), "name_power_limit_max_sm_clock": q}


def write_split(root: str, n: int, seed: int):
    from oracle.streamspeech_oracle import online_features

    cfg = ModelConfig()
    rng = np.random.default_rng(seed)
    gcmvn = synth.make_gcmvn(cfg)
    np.savez(os.path.join(root, "gcmvn.npz"), mean=gcmvn["mean"], std=gcmvn["std"])
    with open(os.path.join(root, "config_gcmvn.yaml"), "w") as f:
        f.write(f"global_cmvn:\n  stats_npz_path: {os.path.join(root, 'gcmvn.npz')}\ntransforms:\n  '*':\n  - global_cmvn\n")
    zpath = os.path.join(root, "fbank80.zip")
    frames, seconds = [], 0.0
    with zipfile.ZipFile(zpath, "w", compression=zipfile.ZIP_STORED) as z:
        for i in range(n):
            sec = float(rng.uniform(3.0, 12.0))
            wav = synth.make_audio(sec, seed=1000 + i)
            x = online_features(wav, None).numpy()  # Kaldi fbank without CMVN: the split's config applies it
            seconds += len(wav) / 16000
            frames.append(x.shape[0])
            with z.open(f"u{i}.npy", "w") as e:
                np.save(e, x)
    with zipfile.ZipFile(zpath) as z, open(os.path.join(root, "test.tsv"), "w") as f:
        f.write("id\tsrc_audio\tsrc_n_frames\ttgt_audio\ttgt_n_frames\n")
        for info in z.infolist():
            i = int(info.filename[1:-4])
            off = info.header_offset + 30 + len(info.filename.encode()) + len(info.extra)
            f.write(f"u{i}\t{zpath}:{off}:{info.file_size}\t{frames[i]}\t\t100\n")
    return seconds


def timed_engine_calls(times):
    """wrap the Engine methods of each stage with CUDA events; times[stage] collects milliseconds"""
    originals = {}
    for name, stage in STAGES.items():
        fn = getattr(Engine, name)
        originals[name] = fn

        def wrapper(self, *a, _fn=fn, _stage=stage, **k):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = _fn(self, *a, **k)
            e.record()
            e.synchronize()
            times[_stage] = times.get(_stage, 0.0) + s.elapsed_time(e)
            return out

        setattr(Engine, name, wrapper)
    return originals


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=256)
    ap.add_argument("--max-tokens", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    out = {"card": card()}
    with tempfile.TemporaryDirectory() as root:
        seconds = write_split(root, a.utterances, a.seed)
        argv = [root, "--config-yaml", "config_gcmvn.yaml", "--task", "speech_to_speech_ctc", "--target-is-code", "--path", "synthetic",
                "--gen-subset", "test", "--beam-mt", "1", "--beam", "1", "--max-len-a", "1", "--max-tokens", str(a.max_tokens),
                "--required-batch-size-multiple", "1", "--results-path", os.path.join(root, "res")]
        with open(os.devnull, "w") as null:
            G.main(argv, stdout=null)  # warm-up: module loads, workspace growth
            t0 = time.perf_counter()
            split = G.main(argv, stdout=null)
            wall = time.perf_counter() - t0
            times = {}
            originals = timed_engine_calls(times)
            try:
                G.main(argv, stdout=null)
            finally:
                for name, fn in originals.items():
                    setattr(Engine, name, fn)
        out["workload"] = {"utterances": a.utterances, "source_seconds": round(seconds, 2), "batches": len(split.batches),
                           "max_tokens": a.max_tokens}
        out["wall"] = {"seconds": round(wall, 3), "audio_s_per_s": round(seconds / wall, 1)}
        out["stages_ms"] = {k: round(v, 2) for k, v in times.items()}

        # ---- the unit stage with and without scores, on every batch's MT features
        from streamspeech_b200.offline import OfflineS2STGenerator

        cfg = ModelConfig()
        cfg.uni_encoder = False
        eng = Engine(cfg, synth.make_model_state_dict(cfg, 0), None, None)
        gen = OfflineS2STGenerator(eng)
        inputs = []
        for batch in split.batches:
            res = G.run_batch(gen, split, batch)
            hyps = [r["mt_tokens"] for r in res]
            S = max(len(h) for h in hyps) + 1
            inputs.append((torch.stack([r["mt_feats"] for r in res]).contiguous(), [S - (len(h) + 1) for h in hyps]))
        arms = {"plain": lambda f, p: eng.t2u_unit_decode_batch(f, p, mask_eos=True),
                "scored": lambda f, p: eng.t2u_unit_decode_batch_scored(f, p, mask_eos=True)}
        ms = {k: [] for k in arms}
        for rep in range(a.reps + 1):
            for k, fn in arms.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                s.record()
                for f, p in inputs:
                    fn(f, p)
                e.record()
                e.synchronize()
                if rep:
                    ms[k].append(s.elapsed_time(e))
        for f, p in inputs[:4]:
            u0, a0, _ = eng.t2u_unit_decode_batch(f, p, mask_eos=True)
            u1, a1, _, _ = eng.t2u_unit_decode_batch_scored(f, p, mask_eos=True)
            assert u0 == u1 and a0 == a1
        eng.close()
        out["unit_scores_ms"] = {k: {"median": round(statistics.median(v), 3), "runs": [round(x, 3) for x in v]} for k, v in ms.items()}
        med = {k: statistics.median(v) for k, v in ms.items()}
        out["unit_scores_ms"]["scored_over_plain"] = round(med["scored"] / med["plain"], 4)
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
