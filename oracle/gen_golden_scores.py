"""Pin the evaluator's scoring to SimulEval's own scorers and evaluator (build container only).

Run:  python -m oracle.gen_golden_scores        (needs the reference tree; CPU only, a few seconds)

Loads the reference's SimulEval/simuleval/evaluator/instance.py, scorers/latency_scorer.py, scorers/quality_scorer.py and
evaluator.py unchanged by stub import.  Stubbed: the `simuleval` package __init__ files, `simuleval.data.dataloader` (a scripted
source list), `textgrid`, and `soundfile` (write() writes 16-bit PCM through streamspeech_b200.generate_waveform_from_code).
`sacrebleu.metrics.bleu.BLEU` is backed by streamspeech_b200.sacrebleu_compat, which tests/test_asr_bleu.py pins by known answers;
its corpus_score raises as sacrebleu 2.x's argument check does ("Each element of `hyps` should be a string"), so a live speech
run's BLEU reaches SimulEval's `except` branch.  pandas, yaml and tqdm are the installed packages.  For ASR_BLEU, `fairseq` is a
stand-in package in a temporary directory whose examples/speech_to_speech/asr_bleu/compute_asr_bleu.py is fairseq's own script
(copied from the reference at run time) and whose utils.ASRGenerator returns scripted transcripts per file; SimulEval runs it with
bash as it does.

Each case drives scripted instances (seeded audio, scripted predictions per call, a scripted clock) through SimulEval's live
instance classes, writes instances.log with its write_log, and calls dump_results and dump_metrics; then it builds a
`--score-only` evaluator on the same directory (LogInstances).  SimulEval's ATD and ASR_BLEU read `instances[0]`, which raises
KeyError when the run starts past index 0; those two are scored there with instances[0] read as the first instance, which is
what the evaluator does (DESIGN.md §14).

Recorded per case and mode: the scores, every instance's metrics, the bytes of scores.tsv, metrics.tsv and the printed table, the
instances.log lines (the output directory as {OUT}), asr_transcripts.txt and wavs/{k}_pred.txt.

Writes tests/golden/simuleval_scores.json.
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import shutil
import sys
import tempfile
import types
from argparse import Namespace

import numpy as np

from oracle.ref_loader import REF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "simuleval_scores.json")
ALL_LATENCY = ["AL", "AP", "DAL", "StartOffset", "EndOffset", "LAAL", "ATD", "NumChunks", "DiscontinuitySum", "DiscontinuityAve",
               "DiscontinuityNum", "RTF"]  # the order of simuleval.simul-s2st.sh
TEXT_LATENCY = ["AL", "AP", "DAL", "StartOffset", "EndOffset", "LAAL", "ATD", "NumChunks", "RTF"]  # simul-s2tt / streaming-asr
LOG_LATENCY = [m for m in ALL_LATENCY if not m.startswith("Discontinuity")]


def seeded(n: int, seed: int) -> list:
    return np.random.RandomState(seed).uniform(-0.5, 0.5, n).astype(np.float32).tolist()


# An instance: source rate / length / seed, reference, and the scripted predictions by call number.  Speech predictions are
# (samples, seed) at 16 kHz; calls go on until the source is read, as SimulEval's loop does.
def _speech(n, seed, ref, writes):
    return dict(rate=16000, n=n, seed=seed, ref=ref, writes=writes)


S2ST_INSTANCES = [
    _speech(16000 * 2 + 300, 11, "Hello world, this is a test.", {0: (3000, 1), 3: (12000, 2), 4: (800, 3), 6: (9000, 4)}),
    _speech(16000 + 5000, 12, "Good morning everyone", {1: (20000, 5), 2: (1600, 6), 3: (4000, 7)}),
    _speech(16000 * 3, 13, "The cat sat on the mat", {2: (500, 8), 8: (6000, 9), 9: (7000, 10)}),
]
S2ST_WITH_EMPTY = S2ST_INSTANCES[:2] + [_speech(16000 + 77, 14, "Nothing came out", {})] + S2ST_INSTANCES[2:]
TEXT_INSTANCES = [
    dict(rate=16000, n=16000 * 2 + 1234, seed=21, ref="the quick brown fox jumps", writes={0: "▁the ▁quick", 3: "▁brown", 6: "▁fox ▁jumps"}),
    dict(rate=16000, n=16000 + 800, seed=22, ref="hello  there", writes={}),
    dict(rate=16000, n=16000 * 3 + 7, seed=23, ref="a man walks  into a bar", writes={1: "▁a ▁man", 2: "▁walks", 9: "▁into ▁a ▁bar"}),
    dict(rate=16000, n=16000 + 2, seed=24, ref="late words", writes={3: "▁late ▁words ▁here"}),
]
ASR_INSTANCES = [
    dict(rate=16000, n=16000 * 2 + 5, seed=31, ref="bonjour tout le monde", writes={1: "▁bon jour", 4: "▁tout ▁le", 6: "▁monde"}),
    dict(rate=16000, n=16000 + 321, seed=32, ref="il fait beau", writes={0: "▁il", 3: "▁fait ▁beau"}),
    dict(rate=16000, n=9000, seed=33, ref="oui", writes={}),
]
# transcripts the stand-in ASR model returns, per wav file name (lower-cased letters, as the en model writes them)
TRANSCRIPTS = {"0_pred.wav": "hello world this is a test", "1_pred.wav": "good morning every one", "2_pred.wav": "the cat sat on a mat",
               "3_pred.wav": "the cat sat on the mat", "4_pred.wav": "four"}

CASES = [
    dict(name="s2st_all_wavs", kind="speech", seg=320, unit="word", instances=S2ST_INSTANCES, quality=["ASR_BLEU", "BLEU"],
         latency=ALL_LATENCY, log_quality=["ASR_BLEU"], log_latency=LOG_LATENCY),
    dict(name="s2st_empty_prediction", kind="speech", seg=320, unit="word", instances=S2ST_WITH_EMPTY, quality=["ASR_BLEU", "BLEU"],
         latency=ALL_LATENCY, log_quality=["ASR_BLEU"], log_latency=LOG_LATENCY),
    dict(name="s2st_start_index", kind="speech", seg=640, unit="word", instances=S2ST_WITH_EMPTY, start=2, quality=["ASR_BLEU"],
         latency=ALL_LATENCY, log_quality=["ASR_BLEU"], log_latency=LOG_LATENCY),
    dict(name="s2st_bleu_defaults", kind="speech", seg=640, unit="char", instances=S2ST_INSTANCES, quality=["BLEU"],
         latency=["LAAL", "AL", "AP", "DAL", "ATD"], log_quality=["BLEU"], log_latency=["LAAL", "AL", "AP", "DAL", "ATD"],
         log_paths="/data/run/wavs"),
    dict(name="s2tt_word", kind="text", seg=320, unit="word", instances=TEXT_INSTANCES, quality=["BLEU"], latency=TEXT_LATENCY,
         log_quality=["BLEU"], log_latency=TEXT_LATENCY),
    dict(name="s2tt_char", kind="text", seg=320, unit="char", instances=TEXT_INSTANCES, quality=["BLEU"], latency=TEXT_LATENCY,
         log_quality=["BLEU"], log_latency=TEXT_LATENCY),
    dict(name="s2tt_word_no_ref_len", kind="text", seg=160, unit="word", instances=TEXT_INSTANCES, quality=["BLEU"],
         latency=TEXT_LATENCY, no_use_ref_len=True, log_quality=["BLEU"], log_latency=TEXT_LATENCY),
    dict(name="asr_word", kind="text", seg=320, unit="word", instances=ASR_INSTANCES, quality=["BLEU"], latency=TEXT_LATENCY,
         log_quality=["BLEU"], log_latency=TEXT_LATENCY),
    dict(name="asr_char", kind="text", seg=640, unit="char", instances=ASR_INSTANCES, quality=["BLEU"], latency=TEXT_LATENCY,
         log_quality=["BLEU"], log_latency=TEXT_LATENCY),
]

# instances.log lines written by hand: delays past the source end (AL's and LAAL's early return), a line without intervals or
# delays, and a line without a reference
LOG_ONLY = dict(name="log_delays_past_source_end", quality=["BLEU"], latency=LOG_LATENCY, lines=[
    {"index": 0, "prediction": "a b c", "delays": [1500.0, 1500.0, 2100.0], "elapsed": [], "prediction_length": 3,
     "reference": "a b c d", "source": ["x"], "source_length": 1200.0, "metric": {}},
    {"index": 1, "prediction": "e f", "delays": [300.0, 900.0], "elapsed": [], "prediction_length": 2, "reference": "e f g",
     "source": ["x"], "source_length": 1000.0, "metric": {}, "intervals": [[300.0, 400.0], [900.0, 700.0]]},
    {"index": 2, "prediction": "", "delays": [], "reference": "h", "source_length": 800.0},
    {"index": 3, "prediction": "i j", "delays": [200.0, 800.0], "source_length": 900.0},
])


class ScriptedClock:
    def __init__(self):
        self.t = 1000.0

    def __call__(self) -> float:
        t = self.t
        self.t += 0.125
        return t


class StubInfo:
    def __init__(self, rate: int, n: int):
        self.samplerate = rate
        self.text = f"src/utt.wav\nsamplerate: {rate} Hz\nchannels: 1\nframes: {n}"

    def __str__(self):
        return self.text


class StubDataloader:
    def __init__(self, instances):
        self.instances = instances

    def __len__(self):
        return len(self.instances)

    def __getitem__(self, index):
        t = self.instances[index]
        return {"source": seeded(t["n"], t["seed"]), "target": t["ref"]}

    def get_source_audio_info(self, index):
        return StubInfo(self.instances[index]["rate"], self.instances[index]["n"])

    def get_source_audio_path(self, index):
        return f"src/{index}.wav"


def _bleu_module():
    """sacrebleu's surface that quality_scorer.py and compute_asr_bleu.py use, on sacrebleu_compat"""
    from streamspeech_b200.sacrebleu_compat import corpus_bleu

    class BLEU:
        TOKENIZER_DEFAULT, TOKENIZERS = "13a", ["13a"]

        def __init__(self, tokenize="13a"):
            assert tokenize == "13a", tokenize

        def corpus_score(self, hyps, refs):
            # sacrebleu 2.x Metric._check_corpus_score_args
            if not isinstance(hyps[0], str):
                raise TypeError("BLEU: Each element of `hyps` should be a string.")
            if not isinstance(refs[0][0], str):
                raise TypeError("BLEU: `refs` should be a sequence of sequence of strings.")
            return corpus_bleu(hyps, refs)

    sb = types.ModuleType("sacrebleu")
    metrics = types.ModuleType("sacrebleu.metrics")
    bleu = types.ModuleType("sacrebleu.metrics.bleu")
    bleu.BLEU = BLEU
    metrics.bleu, metrics.METRICS = bleu, {"BLEU": BLEU}
    sb.metrics, sb.corpus_bleu = metrics, corpus_bleu
    return {"sacrebleu": sb, "sacrebleu.metrics": metrics, "sacrebleu.metrics.bleu": bleu}


STUB_SACREBLEU = '''import sys
sys.path.insert(0, {root!r})
from streamspeech_b200.sacrebleu_compat import corpus_bleu
'''

STUB_UTILS = '''import json, os


def retrieve_asr_config(lang_key, asr_version, json_path):
    with open(json_path) as f:
        return json.load(f)[lang_key][asr_version]


class ASRGenerator:
    """scripted transcripts per wav file name (SCRIPTED_TRANSCRIPTS)"""

    def __init__(self, cfg):
        with open(os.environ["SCRIPTED_TRANSCRIPTS"]) as f:
            self.transcripts = json.load(f)

    def transcribe_audiofile(self, audio_path, lower=True):
        return self.transcripts[os.path.basename(audio_path)]
'''


def make_fairseq_standin(tmp: str) -> None:
    """tmp/fairseq (the package SimulEval imports), tmp/examples/speech_to_speech/asr_bleu/ (fairseq's script, the stand-in utils.py),
    tmp/stubs/sacrebleu, tmp/bin/python (runs this interpreter); the environment the script's subprocess inherits"""
    os.makedirs(os.path.join(tmp, "fairseq"))
    open(os.path.join(tmp, "fairseq", "__init__.py"), "w").close()
    asr_dir = os.path.join(tmp, "examples", "speech_to_speech", "asr_bleu")
    os.makedirs(asr_dir)
    src = os.path.join(REF, "fairseq", "examples", "speech_to_speech", "asr_bleu")
    for name in ("compute_asr_bleu.py", "asr_model_cfgs.json"):
        shutil.copy(os.path.join(src, name), asr_dir)
    with open(os.path.join(asr_dir, "utils.py"), "w") as f:
        f.write(STUB_UTILS)
    os.makedirs(os.path.join(tmp, "stubs", "sacrebleu"))
    with open(os.path.join(tmp, "stubs", "sacrebleu", "__init__.py"), "w") as f:
        f.write(STUB_SACREBLEU.format(root=ROOT))
    os.makedirs(os.path.join(tmp, "bin"))
    with open(os.path.join(tmp, "bin", "python"), "w") as f:  # this interpreter, with its site-packages
        f.write(f'#!/bin/sh\nexec "{sys.executable}" "$@"\n')
    os.chmod(os.path.join(tmp, "bin", "python"), 0o755)
    with open(os.path.join(tmp, "transcripts.json"), "w") as f:
        json.dump(TRANSCRIPTS, f)
    os.environ["PATH"] = os.path.join(tmp, "bin") + os.pathsep + os.environ["PATH"]
    os.environ["PYTHONPATH"] = os.path.join(tmp, "stubs")
    os.environ["SCRIPTED_TRANSCRIPTS"] = os.path.join(tmp, "transcripts.json")
    sys.path.insert(0, tmp)


def load_simuleval(dataloaders: list):
    """the reference's evaluator.py, scorers and instance.py behind stub packages; build_dataloader returns dataloaders[-1]"""
    from streamspeech_b200.generate_waveform_from_code import write_wav

    root = os.path.join(REF, "SimulEval", "simuleval")

    def package(name, path):
        m = types.ModuleType(name)
        m.__path__ = [path]
        sys.modules[name] = m
        return m

    package("simuleval", root)
    package("simuleval.data", os.path.join(root, "data"))
    package("simuleval.evaluator", os.path.join(root, "evaluator"))
    dl = types.ModuleType("simuleval.data.dataloader")
    dl.SpeechToTextDataloader = dl.TextToTextDataloader = dl.GenericDataloader = object
    dl.build_dataloader = lambda args: dataloaders[-1]
    sys.modules["simuleval.data.dataloader"] = dl
    sf = types.ModuleType("soundfile")
    sf.write = lambda path, samples, rate: write_wav(str(path), np.asarray(samples, dtype=np.float32), rate)
    sys.modules["soundfile"] = sf
    sys.modules["textgrid"] = types.ModuleType("textgrid")
    sys.modules.update(_bleu_module())
    import simuleval.data.segments as segments
    import simuleval.evaluator.evaluator as evaluator
    import simuleval.evaluator.instance as instance
    import simuleval.evaluator.scorers.latency_scorer as latency_scorer

    return evaluator, instance, latency_scorer, segments


class FirstIsZero(dict):
    """instances[0] read as the first instance: what ATD and ASR_BLEU see here when the run starts past index 0"""

    def __getitem__(self, key):
        if key == 0 and 0 not in self:
            return next(iter(self.values()))
        return super().__getitem__(key)


def _args(case, out, score_only, quality, latency):
    return Namespace(score_only=score_only, output=out, quality_metrics=quality, latency_metrics=latency,
                     no_use_ref_len=case.get("no_use_ref_len", False), computation_aware=False, sacrebleu_tokenizer="13a",
                     target_speech_lang="en", source_type=None if score_only else "speech",
                     target_type=None if score_only else case.get("kind"), start_index=case.get("start", 0), end_index=-1,
                     no_progress_bar=True, continue_unfinished=False, eval_latency_unit=case.get("unit", "word"),
                     source_segment_size=case.get("seg", 320))


def _dump(ev, out):
    """dump_results + dump_metrics -> what they wrote and printed"""
    if ev.args.start_index > 0:
        ev.instances = FirstIsZero(ev.instances)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        ev.dump_results()
        ev.dump_metrics()

    def read(name):
        p = os.path.join(out, name)
        return open(p).read() if os.path.exists(p) else None

    wav_dir = os.path.join(out, "wavs")
    pred_txt = {f: open(os.path.join(wav_dir, f)).read() for f in sorted(os.listdir(wav_dir)) if f.endswith("_pred.txt")} \
        if os.path.isdir(wav_dir) else {}
    # the scores as written: an int64 column holds digits only
    head, row = read("scores.tsv").splitlines()
    scores = {k: int(v) if v.lstrip("-").isdigit() else float(v) for k, v in zip(head.split("\t"), row.split("\t"))}
    return {"printed": buf.getvalue(), "scores_tsv": read("scores.tsv"), "metrics_tsv": read("metrics.tsv"),
            "metrics": [ins.metrics for ins in ev.instances.values()], "scores": scores,
            "asr_transcripts": read("asr_transcripts.txt"), "pred_txt": pred_txt}


def run_case(case, evaluator, instance_mod, seg_mod, dataloaders, tmp):
    out = os.path.join(tmp, case["name"])
    os.makedirs(out)
    dataloaders.append(StubDataloader(case["instances"]))
    instance_mod.time = types.SimpleNamespace(time=ScriptedClock())
    ev = evaluator.SentenceLevelEvaluator.from_args(_args(case, out, False, case["quality"], case["latency"]))
    for ins in ev.instance_iterator:
        writes = case["instances"][ins.index]["writes"]
        k = 0
        while not ev.is_finished(ins):
            ins.send_source(ev.source_segment_size)
            w = writes.get(k)
            if w is None:
                pred = seg_mod.EmptySegment()
            elif case["kind"] == "speech":
                pred = seg_mod.SpeechSegment(content=seeded(*w), sample_rate=16000, finished=False)
            else:
                pred = seg_mod.TextSegment(content=w, finished=False)
            ins.receive_prediction(pred)
            k += 1
        ev.write_log(ins)
    live = _dump(ev, out)
    log_lines = open(os.path.join(out, "instances.log")).read().splitlines()
    for f in os.listdir(out):  # the score-only pass starts from what the run wrote
        if f in ("scores.tsv", "metrics.tsv", "asr_transcripts.txt", "asr_cmd.bash"):
            os.remove(os.path.join(out, f))
    if os.path.isdir(os.path.join(out, "wavs")):
        for f in os.listdir(os.path.join(out, "wavs")):
            if f.endswith("_pred.txt"):
                os.remove(os.path.join(out, "wavs", f))
    if case.get("log_paths"):  # BLEU of the path strings, at a path that does not depend on where this ran
        with open(os.path.join(out, "instances.log"), "w") as f:
            for line in log_lines:
                f.write(line.replace(os.path.join(out, "wavs"), case["log_paths"]) + "\n")
    log = _dump(evaluator.SentenceLevelEvaluator.from_args(_args(case, out, True, case["log_quality"], case["log_latency"])), out)
    return {"live": live, "log": log, "instances_log": [ln.replace(out, "{OUT}") for ln in log_lines]}


def run_log_only(case, evaluator, tmp):
    out = os.path.join(tmp, case["name"])
    os.makedirs(out)
    with open(os.path.join(out, "config.yaml"), "w") as f:
        f.write("source_type: speech\ntarget_type: text\n")
    with open(os.path.join(out, "instances.log"), "w") as f:
        for line in case["lines"]:
            f.write(json.dumps(line) + "\n")
    return {"log": _dump(evaluator.SentenceLevelEvaluator.from_args(
        _args(dict(unit="word"), out, True, case["quality"], case["latency"])), out)}


def main():
    dataloaders: list = []
    with tempfile.TemporaryDirectory() as tmp:
        make_fairseq_standin(tmp)
        evaluator, instance_mod, _, seg_mod = load_simuleval(dataloaders)
        out = []
        for case in CASES:
            rec = run_case(case, evaluator, instance_mod, seg_mod, dataloaders, tmp)
            out.append({**{k: v for k, v in case.items() if k != "instances"}, "instances": [
                {**t, "writes": {str(k): v for k, v in t["writes"].items()}} for t in case["instances"]], **rec})
            print(case["name"], rec["live"]["scores"], rec["log"]["scores"])
        rec = run_log_only(LOG_ONLY, evaluator, tmp)
        out.append({**LOG_ONLY, **rec})
        print(LOG_ONLY["name"], rec["log"]["scores"])
    with open(GOLD, "w") as f:
        json.dump({"clock": {"start": 1000.0, "step": 0.125}, "transcripts": TRANSCRIPTS, "cases": out}, f, indent=1,
                  ensure_ascii=False)
        f.write("\n")
    print("wrote", GOLD)


if __name__ == "__main__":
    main()
