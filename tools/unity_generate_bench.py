"""UnitY offline generation on the synthetic UnitY checkpoint (released dimensions): device time per stage (encoder, MT search, MT
features, T2U encoder, unit search), unit-search time per step at 8 and 32 rows, launches and host synchronisations per batch, and
whole-split audio-s/s through `python -m streamspeech_b200.generate --task speech_to_speech_modified`.  Prints one JSON line; the
card's name and power limit are read in the same run.

    python tools/unity_generate_bench.py [--samples 32] [--seconds 6] [--beam-mt 10]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=6.0)
    ap.add_argument("--beam-mt", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--variant", choices=("unity", "uni_unity"), default="unity",
                    help="the synthetic checkpoint: UnitY, or Uni-UnitY (future-masked encoder, causal T2U encoder)")
    a = ap.parse_args()
    from streamspeech_b200 import generate as G
    from streamspeech_b200 import synth
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.engine import Engine
    from streamspeech_b200.offline import UnitYGenerator

    torch.set_grad_enabled(False)
    cfg = ModelConfig.unity_default(a.variant)
    eng = Engine(cfg, synth.make_unity_state_dict(cfg, 0), None, None, device=0)
    gen = UnitYGenerator(eng, beam_size_mt=a.beam_mt, max_len_a=1.0, max_len_b=200)
    rng = np.random.default_rng(0)
    F = int(a.seconds * 100)
    x = torch.from_numpy(rng.standard_normal((a.samples, F, 80)).astype(np.float32)).cuda()
    lens = [F - int(v) for v in rng.integers(0, F // 4, a.samples)]
    lens[0] = F
    res = {"card": card(), "variant": a.variant, "samples": a.samples, "fbank_frames": F, "beam_mt": a.beam_mt}
    gen.generate(x, lens)  # warm-up of every shape
    stages = {k: [] for k in ("encoder", "mt_search", "mt_features", "t2u_encoder", "unit_search")}
    for _ in range(a.reps):
        enc, t = timed(lambda: eng.encoder(x, lens))
        stages["encoder"].append(t)
        out_len = [eng.encoder_out_frames(n) for n in lens]
        nb, t = timed(lambda: eng.mt_beam_batch(enc, out_len, a.beam_mt, 200, 1.0))
        stages["mt_search"].append(t)
        hyps = [n[0]["tokens"] for n in nb]
        S = max(len(h) for h in hyps) + 1
        toks = [[cfg.eos] + h + [cfg.pad] * (S - 1 - len(h)) for h in hyps]
        feats, t = timed(lambda: eng.mt_features_batch(enc, out_len, toks))
        stages["mt_features"].append(t)
        t2u_len = [len(h) + 1 for h in hyps]
        t2u, t = timed(lambda: eng.t2u_encode_batch(feats, t2u_len))
        stages["t2u_encoder"].append(t)
        l0 = eng.launch_count()
        units, t = timed(lambda: eng.unit_search_batch(t2u, t2u_len, gen.unit_max_len(F)))
        stages["unit_search"].append(t)
        res["unit_search_launches"] = eng.launch_count() - l0
        res["unit_steps"] = max(len(u["tokens"]) for u in units)
    res["stage_ms"] = {k: round(float(np.median(v)), 3) for k, v in stages.items()}
    l0 = eng.launch_count()
    gen.generate(x, lens)
    res["launches_per_batch"] = eng.launch_count() - l0
    # bursts of 16 steps the unit search's burst loop ran, each ending in one host read of the done flags (not a traced count)
    res["unit_search_bursts_per_batch"] = -(-res["unit_steps"] // 16)
    # per-step cost of the unit search: every row runs to the forced eos at max_len = steps (eos's output row zeroed, as
    # tests/test_unity_gpu.py's long_search_state_dict), checked below, so the time covers that many steps over a growing cache
    sd = synth.make_unity_state_dict(cfg, 1)
    e = sd["decoder.embed_tokens.weight"].clone()
    e[cfg.eos] = 0.0
    sd["decoder.embed_tokens.weight"] = sd["decoder.output_projection.weight"] = e
    flat = Engine(cfg, sd, None, None, device=0)
    per_step = {}
    g = torch.Generator(device="cuda").manual_seed(3)
    for rows in (8, 32):
        st = torch.randn(rows, 40, 512, device="cuda", generator=g)
        flat.unit_search_batch(st, [40] * rows, 64)
        for steps in (256, 1024):
            out, t = timed(lambda: flat.unit_search_batch(st, [40] * rows, steps))
            assert all(len(u["tokens"]) == steps + 1 for u in out), [len(u["tokens"]) for u in out]
            per_step[f"{rows}_rows_{steps}_steps_us"] = round(1000 * t / (steps + 1), 1)
    res["unit_search_per_step"] = per_step
    flat.close()
    eng.close()
    # whole split through the front door
    with tempfile.TemporaryDirectory() as d:
        data = os.path.join(d, "data")
        os.makedirs(data)
        with open(os.path.join(data, "test.tsv"), "w") as f:
            f.write("id\tsrc_audio\tsrc_n_frames\ttgt_audio\ttgt_n_frames\n")
            for i, n in enumerate(lens):
                p = os.path.join(data, f"u{i}.npy")
                np.save(p, rng.standard_normal((n, 80)).astype(np.float32))
                f.write(f"u{i}\t{p}\t{n}\t\t0\n")
        argv = [data, "--user-dir", f"researches/{a.variant}", "--task", "speech_to_speech_modified", "--target-is-code", "--target-code-size", "1000", "--path", "synthetic",
                "--gen-subset", "test", "--beam-mt", str(a.beam_mt), "--beam", "1", "--max-len-a", "1", "--max-tokens", "10000",
                "--required-batch-size-multiple", "1", "--results-path", os.path.join(d, "out")]
        with open(os.devnull, "w") as null:
            G.main(argv, stdout=null)  # warm-up
            t0 = time.perf_counter()
            G.main(argv, stdout=null)
            wall = time.perf_counter() - t0
        res["split_audio_s_per_s"] = round(sum(lens) / 100.0 / wall, 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
