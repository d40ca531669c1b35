"""Throughput of the front doors with and without `--devices`: one process against several worker processes on one GPU (0,0 and
0,0,0,0), and against one worker per GPU (0,1,...) when more than one device is visible.

Each arm is the whole command a user runs (`python -m streamspeech_b200.{evaluate,generate,asr_bleu} ...`) in a fresh process, and
its wall clock covers everything the command does: interpreter start, imports, checkpoint build, every engine build (one per
worker), the run, the output files.  Rate = source audio seconds over that wall clock.  The arms of a workload alternate within each
repetition, so a slow period of the shared host falls on all of them.  Every worker pays the start-up and its own engine build once,
so on a short list that fixed cost decides the rate.  The defaults are sized so that the run outweighs it, and the fixed cost is also
measured on its own: each arm's S2ST command on the list's first utterance alone (`startup`).  For the S2ST workloads each arm then
also reports the rate past it, (audio seconds - first utterance) / (wall - that arm's startup wall).  Workloads:

  evaluate   pool_eval_bench.py's synthetic list (--utterances WAVs of 3-8 s, 16-bit PCM, seeds 5000 + i) at 320 ms on the calibrated
             synthetic checkpoint: S2ST and S2TT at --streams 1 and 32, and the wait-k S2ST agent (synthetic UnitY) at --streams 1 on
             the list's first --waitk-utterances
  generate   offline_generate_bench.py's split (--gen-utterances fbank utterances of 3-12 s, stored zip, gcmvn) at --max-tokens 10000
  asr_bleu   asr_bleu_bench.py's files (--asr-utterances WAVs of 2-12 s, seeds 1000 + i) on the synthetic transcriber

Each arm's outputs are compared with the single-process arm's in every repetition: instances.log (text `elapsed` aside), generate's
stdout and results file, asr_bleu's transcripts and score line must be equal, and the waveforms' largest difference is reported in PCM
steps (0 at one stream; pooled runs are held to one step by the tests).  The card's name, power limit and max SM clock are read in the same run.

    python tools/devices_bench.py [--utterances 160] [--waitk-utterances 40] [--gen-utterances 64] [--asr-utterances 160] [--reps 1]
                                  [--json out.json]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from offline_generate_bench import write_split  # noqa: E402
from pool_eval_bench import gpu_info, write_sources  # noqa: E402

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.evaluate import read_wav  # noqa: E402
from streamspeech_b200.generate_waveform_from_code import write_wav  # noqa: E402

AGENTS = os.path.join(ROOT, "streamspeech_b200", "agents")
EVALUATE = {"s2st": "speech_to_speech.streamspeech.agent.py", "s2tt": "speech_to_text.s2tt.streamspeech.agent.py",
            "waitk_s2st": "waitk/speech_to_speech.wait-k-stride-n.agent.py"}


def arms(n_devices):
    out = [None, "0,0", "0,0,0,0"]
    if n_devices > 1:
        out.append(",".join(str(d) for d in range(n_devices)))
    return out


def timed(cmd):
    t0 = time.perf_counter()
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        raise SystemExit(f"{' '.join(cmd)} failed:\n{p.stderr[-3000:]}")
    return wall, p.stdout


def evaluate_cmd(d, kind, streams, out, devices):
    cmd = [sys.executable, "-m", "streamspeech_b200.evaluate", "--agent", os.path.join(AGENTS, EVALUATE[kind]), "--source",
           os.path.join(d, "src.txt"), "--target", os.path.join(d, "tgt.txt"), "--output", out, "--source-segment-size", "320",
           "--streams", str(streams), "--model-path", "synthetic", "--data-bin", ".", "--vocoder", "synthetic", "--vocoder-cfg", "none",
           "--dur-prediction", "--sample-rate", "16000"]
    return cmd + (["--devices", devices] if devices else [])


def evaluate_outputs(out, speech):
    """{"log": instances.log without text `elapsed`, "wavs": the waveforms' samples}"""
    rows, wavs = [], {}
    with open(os.path.join(out, "instances.log")) as f:
        for line in f:
            r = json.loads(line)
            if speech:
                r["prediction"] = os.path.basename(r["prediction"])
                p = os.path.join(out, "wavs", r["prediction"])
                wavs[r["prediction"]] = read_wav(p)[0] if os.path.exists(p) else None
            else:
                r.pop("elapsed")
            rows.append(r)
    return {"log": rows, "wavs": wavs}


def max_pcm_steps(a, b):
    """the largest sample difference between two {name: samples} maps, in PCM steps; inf where the files or lengths differ"""
    if a.keys() != b.keys():
        return float("inf")
    worst = 0.0
    for k in a:
        if (a[k] is None) != (b[k] is None) or (a[k] is not None and a[k].shape != b[k].shape):
            return float("inf")
        if a[k] is not None and len(a[k]):
            worst = max(worst, float(np.abs(a[k] - b[k]).max()) * 32768)
    return worst


def run_workload(base, name, make_cmd, outputs, audio_s, devices_arms, reps):
    """outputs(out dir, stdout) -> {part: value}; each arm reports per part whether it equalled the single-process arm's in every
    repetition (waveforms: the largest difference in PCM steps)"""
    res = {"audio_s": round(audio_s, 1), "arms": {}}
    ref = None
    for rep in range(reps):
        for devices in devices_arms:
            key = devices or "none"
            out = tempfile.mkdtemp(prefix=f"{name}_{key.replace(',', '')}_", dir=base)
            wall, stdout = timed(make_cmd(out, devices))
            got = outputs(out, stdout)
            if devices is None and ref is None:
                ref = got
            arm = res["arms"].setdefault(key, {"wall_s": [], "audio_s_per_s": [], "equal_to_single": {}})
            arm["wall_s"].append(round(wall, 2))
            arm["audio_s_per_s"].append(round(audio_s / wall, 1))
            for part in got:
                if part == "wavs":
                    arm["wav_max_pcm_steps"] = max(arm.get("wav_max_pcm_steps", 0.0), max_pcm_steps(got[part], ref[part]))
                else:
                    arm["equal_to_single"][part] = arm["equal_to_single"].get(part, True) and bool(got[part] == ref[part])
    print(json.dumps({name: res}), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=160)
    ap.add_argument("--waitk-utterances", type=int, default=40)
    ap.add_argument("--gen-utterances", type=int, default=64)
    ap.add_argument("--asr-utterances", type=int, default=160)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    n_dev = torch.cuda.device_count()
    result = {"card": gpu_info(), "visible_devices": n_dev, "workloads": {}}
    print(json.dumps({"card": result["card"], "visible_devices": n_dev}), flush=True)
    devices_arms = arms(n_dev)
    with tempfile.TemporaryDirectory() as d:
        write_sources(d, a.utterances, 3.0, 8.0)
        with open(os.path.join(d, "src.txt")) as f:
            seconds = [read_wav(p.strip(), header_only=True)[1].frames / 16000 for p in f if p.strip()]
        startup = run_workload(d, "startup", lambda out, dev: evaluate_cmd(d, "s2st", 1, out, dev) + ["--end-index", "1"],
                               lambda out, stdout: {}, seconds[0], devices_arms, a.reps)
        result["workloads"]["startup"] = startup
        for kind, streams in (("s2st", 1), ("s2st", 32), ("s2tt", 1), ("s2tt", 32), ("waitk_s2st", 1)):
            speech = kind != "s2tt"
            n = a.waitk_utterances if kind == "waitk_s2st" else a.utterances
            name = f"evaluate_{kind}_{streams}"
            res = result["workloads"][name] = run_workload(
                d, name, lambda out, dev, k=kind, s=streams, n=n: evaluate_cmd(d, k, s, out, dev) + ["--end-index", str(n)],
                lambda out, stdout, sp=speech: evaluate_outputs(out, sp), sum(seconds[:n]), devices_arms, a.reps)
            if kind == "s2st":
                for key, arm in res["arms"].items():
                    fixed = min(startup["arms"][key]["wall_s"])
                    arm["past_startup_audio_s_per_s"] = [round((sum(seconds[:n]) - seconds[0]) / (w - fixed), 1) if w > fixed else None
                                                         for w in arm["wall_s"]]
                print(json.dumps({name: res}), flush=True)

        data = os.path.join(d, "split")
        os.makedirs(data)
        gen_s = write_split(data, a.gen_utterances, 0)

        def generate_cmd(out, devices):
            cmd = [sys.executable, "-m", "streamspeech_b200.generate", data, "--config-yaml", "config_gcmvn.yaml", "--task",
                   "speech_to_speech_ctc", "--target-is-code", "--target-code-size", "1000", "--path", "synthetic", "--gen-subset", "test",
                   "--beam", "1", "--max-len-a", "1", "--max-tokens", "10000", "--required-batch-size-multiple", "1", "--results-path", out]
            return cmd + (["--devices", devices] if devices else [])

        result["workloads"]["generate"] = run_workload(
            d, "generate", generate_cmd, lambda out, stdout: {"stdout": stdout, "results_file": open(os.path.join(out, "generate-test.txt")).read()}, gen_s,
            devices_arms, a.reps)

        wavs = os.path.join(d, "asr")
        os.makedirs(wavs)
        secs = np.random.default_rng(0).uniform(2.0, 12.0, a.asr_utterances)
        for i, s in enumerate(secs):
            write_wav(os.path.join(wavs, f"{i}_pred.wav"), synth.make_audio(float(s), seed=1000 + i).numpy())
        with open(os.path.join(d, "asr_ref.txt"), "w") as f:
            f.write("".join(f"reference {i}\n" for i in range(a.asr_utterances)))

        def asr_cmd(out, devices):
            cmd = [sys.executable, "-m", "streamspeech_b200.asr_bleu", "--lang", "en", "--audio_dirpath", wavs, "--reference_path",
                   os.path.join(d, "asr_ref.txt"), "--reference_format", "txt", "--asr-model", "synthetic", "--transcripts_path",
                   os.path.join(out, "t.txt")]
            return cmd + (["--devices", devices] if devices else [])

        result["workloads"]["asr_bleu"] = run_workload(
            d, "asr_bleu", asr_cmd, lambda out, stdout: {"score_line": stdout, "transcripts": open(os.path.join(out, "t.txt")).read()}, float(secs.sum()),
            devices_arms, a.reps)
    result["card_after"] = gpu_info()
    print(json.dumps(result))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
