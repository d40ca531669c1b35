"""Wall time of the evaluator's scoring stage: the reference's S2ST recipe metrics (ASR_BLEU and the twelve latency metrics) on
pool_eval_bench.py's source list (64 synthetic utterances of 3 to 8 s, 16-bit PCM WAV).

One `python -m streamspeech_b200.evaluate` run per repetition at --streams 32 with `--quality-metrics ASR_BLEU --latency-metrics
...` and `--asr-model synthetic` (the seeded wav2vec 2.0 Large-shape CTC model).  The scoring stage starts after the agents' engine is
closed and covers building the transcriber, reading and transcribing every wav in one batched pass, the latency metrics, and writing
scores.tsv, metrics.tsv, asr_transcripts.txt and wavs/{k}_pred.txt; the run's JSON line reports it as `scoring_seconds`.  The first
repetition also loads the ASR kernels' module; every repetition is printed and kept in the JSON, none is dropped, and
`scoring_seconds_best` is the least of them.  The card's name, power limit and max SM clock are read in the same run.

    python tools/scoring_bench.py [--utterances 64] [--streams 32] [--reps 3] [--out results/scoring_bench.json]
"""
import argparse
import contextlib
import io
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pool_eval_bench import AGENT_FILES, gpu_info, write_sources  # noqa: E402
from streamspeech_b200 import evaluate as ev  # noqa: E402

LATENCY = ["AL", "AP", "DAL", "StartOffset", "EndOffset", "LAAL", "ATD", "NumChunks", "DiscontinuitySum", "DiscontinuityAve",
           "DiscontinuityNum", "RTF"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=64)
    ap.add_argument("--streams", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    runs = []
    with tempfile.TemporaryDirectory() as d:
        write_sources(d, a.utterances, 3.0, 8.0)
        for r in range(a.reps):
            argv = ["--agent", os.path.join(ROOT, "streamspeech_b200", "agents", AGENT_FILES["s2st"]), "--source",
                    os.path.join(d, "src.txt"), "--target", os.path.join(d, "tgt.txt"), "--output", os.path.join(d, f"out{r}"),
                    "--source-segment-size", "320", "--streams", str(a.streams), "--model-path", "synthetic", "--data-bin", ".",
                    "--vocoder", "synthetic", "--vocoder-cfg", "none", "--dur-prediction", "--sample-rate", "16000",
                    "--quality-metrics", "ASR_BLEU", "--latency-metrics", *LATENCY, "--asr-model", "synthetic"]
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                ev.main(argv)
            printed = buf.getvalue().splitlines()
            line = json.loads(printed[-1])
            runs.append({"run_wall_seconds": line["wall_seconds"], "scoring_seconds": line["scoring_seconds"],
                         "table": printed[:-1]})
            print(json.dumps(runs[-1]))
    res = {"gpu": gpu_info(), "utterances": a.utterances, "streams": a.streams, "runs": runs,
           "scoring_seconds_best": min(r["scoring_seconds"] for r in runs)}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
