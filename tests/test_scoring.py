"""streamspeech_b200.simuleval_scoring and the scoring stage of streamspeech_b200.evaluate (CPU).

The scorers against SimulEval's own evaluator and scorers (tests/golden/simuleval_scores.json, oracle/gen_golden_scores.py): every
case's scripted instances are replayed through the evaluator's instance classes, scored live and then from the instances.log they
wrote (`--score-only`), and every score, per-instance metric, file and printed table must equal the fixture's, byte for byte.
ASR_BLEU runs the evaluator's transcription path with a scripted transcriber in place of the GPU one.  Then the refusals, and the
front door with fake agents: an unscored run is unchanged, a scored run writes the files, `--score-only` rescores it, and a pooled
run whose instances finish out of index order is scored in index order, as one stream scores it."""
import contextlib
import io
import json
import os
import shutil
from pathlib import Path

import numpy as np
import pytest

from streamspeech_b200 import evaluate as ev
from streamspeech_b200 import simuleval_scoring as sc
from streamspeech_b200.simuleval_compat import EmptySegment, SpeechSegment, TextSegment

AGENT_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "streamspeech_b200", "agents")
S2ST, ASR = "speech_to_speech.streamspeech.agent.py", "speech_to_text.asr.streamspeech.agent.py"


def _golden():
    with open(os.path.join(os.path.dirname(__file__), "golden", "simuleval_scores.json")) as f:
        return json.load(f)


G = _golden()


def _seeded(n, seed):
    return np.random.RandomState(seed).uniform(-0.5, 0.5, n).astype(np.float32).tolist()


class ScriptedTranscriber:
    """the transcriber surface transcribe_simuleval uses, answering from the fixture's transcripts per file name"""

    def __init__(self, transcripts):
        self.transcripts, self.calls = transcripts, []

    def load_audio(self, path):
        assert os.path.exists(path)
        return os.path.basename(path)

    def num_frames(self, n):
        return n

    def transcribe(self, waves):
        self.calls.append(list(waves))
        return [self.transcripts[w] for w in waves]


class Info:
    def __init__(self, rate, n):
        self.samplerate = rate
        self.text = f"src/utt.wav\nsamplerate: {rate} Hz\nchannels: 1\nframes: {n}"

    def __str__(self):
        return self.text


def _replay(case, out: Path):
    """the case's instances through evaluate's instance classes, as the oracle drove SimulEval's -> (live instances, log lines)"""
    t_now = [G["clock"]["start"]]

    def clock():
        t = t_now[0]
        t_now[0] += G["clock"]["step"]
        return t

    (out / "wavs").mkdir(parents=True, exist_ok=True)
    kept, lines = {}, []
    for i in range(case.get("start", 0), len(case["instances"])):
        t = case["instances"][i]
        common = dict(info=Info(t["rate"], t["n"]), source_path=f"src/{i}.wav", reference=t["ref"], latency_unit=case["unit"],
                      clock=clock)
        if case["kind"] == "speech":
            inst = ev.SpeechToSpeechInstance(i, _seeded(t["n"], t["seed"]), wav_path=(out / "wavs" / f"{i}_pred.wav").absolute(), **common)
        else:
            inst = ev.SpeechToTextInstance(i, _seeded(t["n"], t["seed"]), **common)
        k = 0
        while not inst.source_finished_reading:
            inst.send_source(case["seg"])
            w = t["writes"].get(str(k))
            if w is None:
                pred = EmptySegment()
            elif case["kind"] == "speech":
                pred = SpeechSegment(content=_seeded(*w), sample_rate=16000, finished=False)
            else:
                pred = TextSegment(content=w, finished=False)
            inst.receive_prediction(pred)
            k += 1
        summary = inst.summarize()
        if case["kind"] == "text":  # SimulEval logs soundfile.info's text; the oracle's stub info has its own
            summary["source"] = str(common["info"]).split("\n")
        lines.append(json.dumps(summary))
        kept[i] = sc.live_instance(summary, case["unit"], getattr(inst, "silences", None))
    with open(out / "instances.log", "w") as f:
        f.write("".join(ln + "\n" for ln in lines))
    return kept, lines


def _score(instances, out, quality, latency, use_ref_len=True):
    tr = ScriptedTranscriber(G["transcripts"])
    scores = sc.score(instances, quality, latency, use_ref_len=use_ref_len, make_transcriber=lambda: tr)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        sc.dump(out, instances, scores)

    def read(name):
        p = out / name
        return p.read_text() if p.exists() else None

    pred_txt = {f: (out / "wavs" / f).read_text() for f in sorted(os.listdir(out / "wavs")) if f.endswith("_pred.txt")} \
        if (out / "wavs").is_dir() else {}
    return {"printed": buf.getvalue(), "scores_tsv": read("scores.tsv"), "metrics_tsv": read("metrics.tsv"),
            "metrics": [ins.metrics for ins in instances.values()], "scores": scores, "asr_transcripts": read("asr_transcripts.txt"),
            "pred_txt": pred_txt}


def _check(got, want):
    assert got["scores"] == want["scores"]
    assert [type(v) is int for v in got["scores"].values()] == [type(v) is int for v in want["scores"].values()]
    assert json.loads(json.dumps(got["metrics"])) == want["metrics"]
    for key in ("printed", "scores_tsv", "metrics_tsv", "asr_transcripts", "pred_txt"):
        assert got[key] == want[key], key


LIVE_CASES = [c["name"] for c in G["cases"] if "live" in c]


@pytest.mark.parametrize("name", LIVE_CASES)
def test_live_and_score_only_equal_simulevals(name, tmp_path):
    case = next(c for c in G["cases"] if c["name"] == name)
    out = tmp_path / "run"
    kept, lines = _replay(case, out)
    assert [ln.replace(str(out), "{OUT}") for ln in lines] == case["instances_log"]
    _check(_score(kept, out, case["quality"], case["latency"], not case.get("no_use_ref_len", False)), case["live"])

    for f in ("scores.tsv", "metrics.tsv", "asr_transcripts.txt"):
        (out / f).unlink(missing_ok=True)
    for f in (out / "wavs").glob("*_pred.txt"):
        f.unlink()
    if case.get("log_paths"):
        (out / "instances.log").write_text("".join(ln.replace(str(out / "wavs"), case["log_paths"]) + "\n" for ln in lines))
    _check(_score(sc.read_log(out), out, case["log_quality"], case["log_latency"], not case.get("no_use_ref_len", False)), case["log"])


def test_hand_written_log_equals_simulevals(tmp_path):
    case = next(c for c in G["cases"] if c["name"] == "log_delays_past_source_end")
    (tmp_path / "instances.log").write_text("".join(json.dumps(x) + "\n" for x in case["lines"]))
    _check(_score(sc.read_log(tmp_path), tmp_path, case["quality"], case["latency"]), case["log"])


def test_fixture_covers_the_cases_the_scorers_branch_on():
    cases = {c["name"]: c for c in G["cases"]}
    live = cases["s2st_all_wavs"]["live"]
    assert live["scores"]["ASR_BLEU"] > 0 and live["scores"]["BLEU"] == 0  # BLEU of a live speech run: sacrebleu refuses a Path
    assert live["asr_transcripts"] and len(live["pred_txt"]) == 3
    assert live["scores"]["DiscontinuitySum"] > 0  # silences occur
    assert cases["s2st_empty_prediction"]["live"]["scores"]["ASR_BLEU"] == 0.0  # a missing wav fails the script
    assert cases["s2st_empty_prediction"]["live"]["asr_transcripts"] is None
    assert cases["s2st_start_index"]["log"]["scores"]["ASR_BLEU"] == 0.0  # wav 0 absent
    assert cases["s2st_bleu_defaults"]["log"]["scores"]["BLEU"] > 0  # --score-only scores the path strings
    assert any(c["live"]["scores"]["ATD"] != c["log"]["scores"]["ATD"] for c in cases.values() if c.get("kind") == "speech")
    assert cases["s2tt_char"]["live"]["scores"]["AL"] != cases["s2tt_char"]["log"]["scores"]["AL"]  # LogInstance counts words
    assert {c["unit"] for c in cases.values() if c.get("kind") == "text"} == {"word", "char"}
    assert any(c.get("no_use_ref_len") for c in cases.values())
    assert any("" in c["live"]["metrics_tsv"].split("\n")[1].split("\t") or "\t\t" in c["live"]["metrics_tsv"]
               for c in cases.values() if "live" in c)  # a skipped instance: empty fields
    log = cases["log_delays_past_source_end"]["lines"][0]
    assert log["delays"][0] > log["source_length"]


# --------------------------------------------------------------------------------------------------------------- formatting edges

def test_table_and_tsv_formatting_edges():
    scores = {"A": 3, "B": 2.5, "C": 0.0, "LongerName": -12.25, "E": 1234567.891}
    assert sc.results_table(scores) == " A   B   C  LongerName           E\n 3 2.5 0.0      -12.25 1234567.891"  # pandas 3.0.2
    assert sc.scores_tsv(scores) == "A\tB\tC\tLongerName\tE\n3\t2.5\t0.0\t-12.25\t1234567.891\n"
    assert sc.results_table({"X": 123456789.123}) == "           X\n1.234568e+08"
    ins = [sc.ScoredInstance("text", i, [1.0], "r", 1.0, "p", 1) for i in range(2)]
    ins[0].metrics = {"AL": 1.23456, "N": 3}
    assert sc.metrics_tsv({0: ins[0], 1: ins[1]}) == "AL\tN\n1.235\t3.0\n\t\n"
    assert sc.metrics_tsv({1: ins[1]}) == "\n\n"
    ins[1].metrics = {"AL": 0.0005}
    assert sc.metrics_tsv({1: ins[1]}) == "AL\n0.0\n"


# ------------------------------------------------------------------------------------------------------------------------ refusals

@pytest.mark.parametrize("kw,match", [
    (dict(quality=["METEOR"]), "--quality-metrics METEOR: no quality metric called METEOR"),
    (dict(latency=["XL"]), "--latency-metrics XL: no latency metric called XL"),
    (dict(latency=["AL_SpeechAlign_BOW"]), "AL_SpeechAlign_BOW is not offered.*Montreal Forced Aligner"),
    (dict(quality=["WHISPER_ASR_BLEU"]), "WHISPER_ASR_BLEU is not offered"),
    (dict(target_speech_lang="de"), "--target-speech-lang de"),
    (dict(tokenizer="intl"), "--sacrebleu-tokenizer intl: only the 13a tokenizer"),
    (dict(quality=["ASR_BLEU"], speech_output=True), "ASR_BLEU needs --asr-model"),
    (dict(quality=["ASR_BLEU"], speech_output=False, asr_model="synthetic"), "ASR_BLEU needs speech output"),
    (dict(latency=["DiscontinuityAve"], score_only=True), "DiscontinuityAve cannot be scored with --score-only"),
    (dict(latency=["DiscontinuityNum"], speech_output=False), "DiscontinuityNum needs speech output"),
    (dict(latency=["AL"], n_instances=0), "--latency-metrics AL: there are no instances"),
])
def test_refusals_name_the_metric_or_flag(kw, match):
    kw = {"quality": ["BLEU"], "latency": ["AL"], **kw}
    with pytest.raises(SystemExit, match=match):
        sc.check_request(kw.pop("quality"), kw.pop("latency"), **kw)


def test_a_latency_metric_without_any_delays_is_refused_by_name():
    ins = {0: sc.ScoredInstance("text", 0, [], "r", 1000.0, "", 1)}
    with pytest.raises(SystemExit, match="--latency-metrics LAAL: no instance has delays"):
        sc.score(ins, [], ["LAAL"])
    with pytest.raises(SystemExit, match="--latency-metrics ATD: no instance has delays"):
        sc.score(ins, [], ["ATD"])


def test_asr_bleu_failure_names_the_missing_file(tmp_path, caplog):
    case = next(c for c in G["cases"] if c["name"] == "s2st_all_wavs")
    out = tmp_path / "run"
    kept, _ = _replay(case, out)
    (out / "wavs" / "2_pred.wav").unlink()  # the last one: the count no longer matches instances.log
    with caplog.at_level("ERROR", logger="streamspeech_b200.scoring"):
        s = sc.score(kept, ["ASR_BLEU"], [], make_transcriber=lambda: pytest.fail("the transcriber must not be built"))
    assert s == {"ASR_BLEU": 0.0}
    assert "ASR on target speech failed" in caplog.text and "missing: 2_pred.wav" in caplog.text
    assert not (out / "asr_transcripts.txt").exists()


# ----------------------------------------------------------------------------------------------------------------- the front door

class FakeAgent:
    """a text agent: one word per second segment, the last one finished"""

    class engine:  # noqa: N801
        closed = 0

        @classmethod
        def close(cls):
            cls.closed += 1

    def __init__(self):
        self.reset()

    def reset(self):
        self.calls, self.finished = 0, False

    def push(self, seg):
        self.calls += 1
        self.finished = seg.finished

    def pop(self):
        if self.finished:
            return TextSegment(content=f"▁w{self.calls} ▁end", finished=True)
        return TextSegment(content=f"▁w{self.calls}") if self.calls % 2 == 0 else EmptySegment()


class FakeSpeechAgent(FakeAgent):
    """a speech agent: 100 ms of output every second segment, 200 ms more at the end of the source"""

    def pop(self):
        if self.finished:
            return SpeechSegment(content=[0.25] * 3200, sample_rate=16000, finished=True)
        if self.calls % 2 == 0:
            return SpeechSegment(content=[0.25] * 1600, sample_rate=16000, finished=False)
        return EmptySegment()


def _front_door(tmp_path, monkeypatch, *extra, streams=1, speech=False):
    """the front door over four sources on `streams` fake agents; with 2 or more, instance 1 (0.96 s) finishes before instance 0 (2 s)"""
    from streamspeech_b200.generate_waveform_from_code import write_wav

    paths = []
    for i, n in enumerate([16000 * 2 + 1, 5120 * 3, 16000 + 2, 9999]):
        p = tmp_path / f"u{i}.wav"
        write_wav(str(p), np.random.RandomState(i).uniform(-0.3, 0.3, n).astype(np.float32), 16000)
        paths.append(str(p))
    (tmp_path / "src.txt").write_text("\n".join(paths) + "\n")
    (tmp_path / "tgt.txt").write_text("w2 w4 end\nthe w2 end\nw2 end here\nw2 w4 w6 end\n")
    cls = FakeSpeechAgent if speech else FakeAgent
    monkeypatch.setattr(ev, "build_agents", lambda args, max_seconds: ([cls() for _ in range(args.streams)], None,
                                                                       "speech" if speech else "text"))
    argv = ["--agent", os.path.join(AGENT_DIR, S2ST if speech else ASR), "--source", str(tmp_path / "src.txt"), "--target",
            str(tmp_path / "tgt.txt"), "--output", str(tmp_path / "out"), "--source-segment-size", "320", "--model-path", "synthetic",
            "--data-bin", ".", "--sample-rate", "16000", "--streams", str(streams), *extra]
    if speech:
        argv += ["--vocoder", "synthetic", "--vocoder-cfg", "none"]
    return argv


def _finish_order(monkeypatch):
    """the indices in the order their instances finish (the run keeps each one as it finishes)"""
    order = []
    live = sc.live_instance

    def record(summary, *a, **k):
        order.append(summary["index"])
        return live(summary, *a, **k)

    monkeypatch.setattr(sc, "live_instance", record)
    return order


def test_a_pooled_run_is_scored_in_index_order(tmp_path, monkeypatch, capsys):
    order = _finish_order(monkeypatch)
    run = ev.main(_front_door(tmp_path, monkeypatch, "--latency-metrics", "AL", "ATD", "NumChunks", "RTF", streams=2))
    assert order != sorted(order)  # the streams finish out of index order
    assert list(run.kept) == [0, 1, 2, 3]
    live_metrics = (tmp_path / "out" / "metrics.tsv").read_text()
    scores = ev.main(["--score-only", "--output", str(tmp_path / "out"), "--latency-metrics", "AL", "ATD", "NumChunks", "RTF"])
    assert scores == run.scores
    assert (tmp_path / "out" / "metrics.tsv").read_text() == live_metrics
    single = tmp_path / "single"
    single.mkdir()
    run1 = ev.main(_front_door(single, monkeypatch, "--latency-metrics", "AL", "ATD", "NumChunks", "RTF", streams=1))
    assert run1.scores == run.scores
    assert (single / "out" / "metrics.tsv").read_text() == live_metrics  # row i is instance i's


def test_a_pooled_speech_run_pairs_each_transcript_with_its_reference(tmp_path, monkeypatch, capsys):
    refs = ["w2 w4 end", "the w2 end", "w2 end here", "w2 w4 w6 end"]
    transcripts = {f"{i}_pred.wav": r for i, r in enumerate(refs)}  # transcript i is reference i: ASR_BLEU 100 when paired right
    monkeypatch.setattr(ev, "_transcriber_factory", lambda args: (lambda: ScriptedTranscriber(transcripts)))
    order = _finish_order(monkeypatch)
    run = ev.main(_front_door(tmp_path, monkeypatch, "--quality-metrics", "ASR_BLEU", "--latency-metrics", "AL", "DiscontinuityNum",
                              "--asr-model", "synthetic", streams=3, speech=True))
    assert order != sorted(order) and list(run.kept) == [0, 1, 2, 3]
    assert run.scores["ASR_BLEU"] == 100.0
    assert (tmp_path / "out" / "asr_transcripts.txt").read_text() == "".join(r + "\n" for r in refs)
    single = tmp_path / "single"
    single.mkdir()
    run1 = ev.main(_front_door(single, monkeypatch, "--quality-metrics", "ASR_BLEU", "--latency-metrics", "AL", "DiscontinuityNum",
                               "--asr-model", "synthetic", streams=1, speech=True))
    assert run1.scores == run.scores
    assert (single / "out" / "metrics.tsv").read_text() == (tmp_path / "out" / "metrics.tsv").read_text()


def test_a_transcriber_error_is_raised_not_scored_as_zero(tmp_path):
    case = next(c for c in G["cases"] if c["name"] == "s2st_all_wavs")
    out = tmp_path / "run"
    kept, _ = _replay(case, out)

    class Broken(ScriptedTranscriber):
        def transcribe(self, waves):
            raise ValueError("device error")

    with pytest.raises(ValueError, match="device error"):
        sc.score(kept, ["ASR_BLEU"], [], make_transcriber=lambda: Broken({}))


def test_a_run_without_metric_flags_is_not_scored(tmp_path, monkeypatch, capsys):
    ev.main(_front_door(tmp_path, monkeypatch))
    lines = capsys.readouterr().out.splitlines()
    assert len(lines) == 1 and set(json.loads(lines[0])) == {"instances", "streams", "source_seconds", "wall_seconds",
                                                              "audio_s_per_s", "output"}
    assert sorted(os.listdir(tmp_path / "out")) == ["config.yaml", "instances.log"]


def test_a_scored_run_and_score_only_agree(tmp_path, monkeypatch, capsys):
    run = ev.main(_front_door(tmp_path, monkeypatch, "--latency-metrics", "AL", "ATD", "NumChunks", "RTF"))
    out = capsys.readouterr().out.splitlines()
    assert json.loads(out[-1])["scoring_seconds"] >= 0 and "scoring_seconds" in json.loads(out[-1])
    assert out[:2] == sc.results_table(run.scores).split("\n")
    assert list(run.scores) == ["BLEU", "AL", "ATD", "NumChunks", "RTF"]  # BLEU: SimulEval's default quality metric
    assert run.scores["BLEU"] > 0
    assert (tmp_path / "out" / "scores.tsv").read_text() == sc.scores_tsv(run.scores)
    live_metrics = (tmp_path / "out" / "metrics.tsv").read_text()
    assert len(live_metrics.splitlines()) == 5
    scores = ev.main(["--score-only", "--output", str(tmp_path / "out"), "--latency-metrics", "AL", "ATD", "NumChunks", "RTF"])
    assert scores == run.scores  # word latency unit: LogInstance's reference length is the live one
    assert (tmp_path / "out" / "metrics.tsv").read_text() == live_metrics


def test_score_only_keeps_the_log_instance_quirks(tmp_path, monkeypatch, capsys):
    run = ev.main(_front_door(tmp_path, monkeypatch, "--latency-metrics", "AL", "--eval-latency-unit", "char"))
    scores = ev.main(["--score-only", "--output", str(tmp_path / "out"), "--latency-metrics", "AL", "--eval-latency-unit", "char"])
    assert scores["BLEU"] == run.scores["BLEU"] and scores["AL"] != run.scores["AL"]  # the log counts reference words
    words = sc.read_log(tmp_path / "out")
    assert all(ins.reference_length == len(ins.reference.split(" ")) for ins in words.values())


def test_front_door_refusals_come_before_the_run(tmp_path, monkeypatch):
    argv = _front_door(tmp_path, monkeypatch)
    monkeypatch.setattr(ev, "build_agents", lambda *a, **k: pytest.fail("refused after the model was loaded"))
    with pytest.raises(SystemExit, match="ASR_BLEU needs speech output"):
        ev.main(argv + ["--quality-metrics", "ASR_BLEU", "--asr-model", "synthetic"])
    with pytest.raises(SystemExit, match="--latency-metrics DiscontinuitySum needs speech output"):
        ev.main(argv + ["--latency-metrics", "DiscontinuitySum"])
    with pytest.raises(SystemExit, match="no latency metric called Foo"):
        ev.main(argv + ["--latency-metrics", "Foo"])
    with pytest.raises(SystemExit, match="there are no instances"):
        ev.main(argv + ["--latency-metrics", "AL", "--start-index", "3", "--end-index", "3"])
    s2st = [a if not a.endswith(ASR) else os.path.join(AGENT_DIR, S2ST) for a in argv] + ["--vocoder", "synthetic", "--vocoder-cfg", "x"]
    with pytest.raises(SystemExit, match="ASR_BLEU needs --asr-model"):
        ev.main(s2st + ["--quality-metrics", "ASR_BLEU"])
    with pytest.raises(SystemExit, match="--asr-setting bogus=1"):
        ev.main(s2st + ["--quality-metrics", "ASR_BLEU", "--asr-model", "synthetic", "--asr-setting", "bogus=1"])
    with pytest.raises(SystemExit, match="cannot be scored with --score-only"):
        ev.main(["--score-only", "--output", str(tmp_path), "--latency-metrics", "DiscontinuityNum"])
    with pytest.raises(SystemExit):
        ev.main(["--score-only", "--output", str(tmp_path), "--computation-aware"])


S2ST_RECIPE_METRICS = ["--quality-metrics", "ASR_BLEU", "--target-speech-lang", "en", "--latency-metrics", "AL", "AP", "DAL",
                       "StartOffset", "EndOffset", "LAAL", "ATD", "NumChunks", "DiscontinuitySum", "DiscontinuityAve",
                       "DiscontinuityNum", "RTF"]  # researches/ctc_unity/test_scripts/simuleval.simul-s2st.sh


def test_reference_s2st_metric_flags_parse_and_need_an_asr_model():
    base = ["--agent", os.path.join(AGENT_DIR, S2ST), "--source", "s", "--target", "t", "--output", "o", "--model-path", "M",
            "--data-bin", ".", "--vocoder", "V", "--vocoder-cfg", "C"]
    args = ev.parse_args(base + S2ST_RECIPE_METRICS)
    metrics = sc.metric_lists(args.quality_metrics, args.latency_metrics)
    assert metrics == (["ASR_BLEU"], S2ST_RECIPE_METRICS[5:])
    with pytest.raises(SystemExit, match="ASR_BLEU needs --asr-model"):
        ev._check_scoring(args, metrics, True, False, None)
    args = ev.parse_args(base + S2ST_RECIPE_METRICS + ["--asr-model", "w2v.pt", "--asr-dict", "dict.ltr.txt"])
    ev._check_scoring(args, metrics, True, False, 4)
    assert sc.metric_lists(None, None) is None
    assert sc.metric_lists(["BLEU"], None) == (["BLEU"], ["LAAL", "AL", "AP", "DAL", "ATD"])
