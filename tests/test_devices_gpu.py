"""The front doors with `--devices` on the GPU, against the same run without it, on the synthetic checkpoints as the front-door tests
build them.  evaluate with two workers on one GPU (--devices 0,0): every agent kind, --streams 1 and 2, the wait-k agents at 1, on
test_evaluate.py's ragged six-utterance list; instances.log equal but for text `elapsed` (wall clock), waveforms bit-identical at one
stream and within one PCM step pooled (the pooled tests' bar), scores.tsv and metrics.tsv equal.  generate --devices 0,0,0 on a
split of at least 6 batches, StreamSpeech and UnitY: stdout and generate-{subset}.txt byte-identical.  asr_bleu --devices 0,0 and
evaluate --score-only --devices 0,0 with ASR_BLEU: transcripts and score line identical.  No child process is left after any run.
A variant over two distinct GPUs (--devices 0,1) runs where two are visible."""
import io
import json
import multiprocessing
import os

import numpy as np
import pytest
import torch

from streamspeech_b200 import asr_bleu
from streamspeech_b200 import evaluate as ev
from streamspeech_b200 import generate as G
from streamspeech_b200 import synth
from test_evaluate import ASR, S2ST, S2TT, UTTERANCES, write_float_wav, write_pcm_wav

pytestmark = pytest.mark.gpu
AGENTS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "streamspeech_b200", "agents")
WAITK_S2ST, WAITK_S2TT = "waitk/speech_to_speech.wait-k-stride-n.agent.py", "waitk/speech_to_text.wait-k-stride-n.agent.py"
SPEECH_LATENCY = ["AL", "AP", "DAL", "StartOffset", "EndOffset", "LAAL", "ATD", "NumChunks", "DiscontinuitySum", "DiscontinuityAve",
                  "DiscontinuityNum", "RTF"]
TEXT_LATENCY = ["AL", "AP", "DAL", "StartOffset", "EndOffset", "LAAL", "ATD", "NumChunks", "RTF"]


@pytest.fixture(autouse=True)
def no_child_left():
    yield
    assert multiprocessing.active_children() == []


def _sources(tmp_path, rate, float_wav):
    src = tmp_path / f"src{rate}.txt"
    paths = []
    for i, sec in enumerate(UTTERANCES):  # test_evaluate.py's list
        n = int(sec * rate)
        x = synth.make_audio(n / rate + 0.001, seed=700 + i, sample_rate=rate)[:n].numpy()
        p = tmp_path / f"utt{rate}_{i}.wav"
        (write_float_wav if float_wav else write_pcm_wav)(p, x, rate)
        paths.append(str(p))
    src.write_text("\n".join(paths) + "\n")
    (tmp_path / "tgt.txt").write_text("".join(f"reference {i}\n" for i in range(len(UTTERANCES))))
    return src


def _evaluate(tmp_path, src, agent, seg_ms, rate, streams, name, *extra):
    out = tmp_path / name
    ev.main(["--agent", os.path.join(AGENTS, agent), "--source", str(src), "--target", str(tmp_path / "tgt.txt"), "--output", str(out),
             "--source-segment-size", str(seg_ms), "--streams", str(streams), "--model-path", "synthetic", "--data-bin", ".",
             "--vocoder", "synthetic", "--vocoder-cfg", "none", "--dur-prediction", "--sample-rate", str(rate), *extra])
    return out


def _log(out, speech):
    lines = []
    for x in (out / "instances.log").read_text().splitlines():
        d = json.loads(x)
        if speech:
            assert d["prediction"] == (out / "wavs" / f"{d['index']}_pred.wav").absolute().as_posix()
            d["prediction"] = os.path.basename(d["prediction"])
        else:
            d.pop("elapsed")
        lines.append(d)
    return lines


def _compare_evaluations(ref, got, speech, streams):
    a, b = _log(ref, speech), _log(got, speech)
    assert [d["index"] for d in a] == list(range(len(UTTERANCES))) and sum(d["prediction_length"] for d in a) > 0
    assert a == b
    worst = 0.0
    if speech:
        assert sorted(os.listdir(ref / "wavs")) == sorted(os.listdir(got / "wavs"))
        for d in a:
            if not d["delays"]:
                continue
            if streams == 1:
                assert (ref / "wavs" / d["prediction"]).read_bytes() == (got / "wavs" / d["prediction"]).read_bytes(), d["index"]
            else:
                x, _ = ev.read_wav(str(ref / "wavs" / d["prediction"]))
                y, _ = ev.read_wav(str(got / "wavs" / d["prediction"]))
                assert x.shape == y.shape
                worst = max(worst, float(np.abs(x - y).max()) * 32768)
    assert worst <= 1.0, worst
    for name in ("scores.tsv", "metrics.tsv"):
        assert (got / name).read_bytes() == (ref / name).read_bytes(), name
    return worst


CASES = [(S2ST, 320, 16000, 1), (S2ST, 320, 16000, 2), (S2ST, 640, 48000, 1), (S2ST, 640, 48000, 2), (S2TT, 320, 16000, 1),
         (S2TT, 320, 16000, 2), (ASR, 160, 16000, 1), (ASR, 160, 16000, 2), (WAITK_S2ST, 320, 16000, 1), (WAITK_S2TT, 320, 16000, 1)]


@pytest.mark.parametrize("agent,seg_ms,rate,streams", CASES,
                         ids=["s2st320_16k_1", "s2st320_16k_2", "s2st640_48k_1", "s2st640_48k_2", "s2tt320_1", "s2tt320_2", "asr160_1",
                              "asr160_2", "waitk_s2st_1", "waitk_s2tt_1"])
def test_evaluate_on_two_workers_equals_one_process(tmp_path, agent, seg_ms, rate, streams):
    speech = "speech_to_speech" in agent
    src = _sources(tmp_path, rate, float_wav=rate == 48000)
    metrics = ["--latency-metrics", *(SPEECH_LATENCY if speech else TEXT_LATENCY)] + ([] if speech else ["--quality-metrics", "BLEU"])
    ref = _evaluate(tmp_path, src, agent, seg_ms, rate, streams, "single", *metrics)
    got = _evaluate(tmp_path, src, agent, seg_ms, rate, streams, "devices", *metrics, "--devices", "0,0")
    worst = _compare_evaluations(ref, got, speech, streams)
    print(json.dumps({"test": "evaluate_devices", "agent": agent, "streams": streams, "worst_pcm_steps": worst}))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
@pytest.mark.parametrize("agent,seg_ms,rate,streams", [(S2ST, 320, 16000, 1), (S2TT, 320, 16000, 2)], ids=["s2st_1", "s2tt_2"])
def test_evaluate_on_two_gpus_equals_one_process(tmp_path, agent, seg_ms, rate, streams):
    speech = agent == S2ST
    src = _sources(tmp_path, rate, float_wav=False)
    metrics = ["--latency-metrics", *(SPEECH_LATENCY if speech else TEXT_LATENCY)]
    ref = _evaluate(tmp_path, src, agent, seg_ms, rate, streams, "single", *metrics)
    got = _evaluate(tmp_path, src, agent, seg_ms, rate, streams, "devices", *metrics, "--devices", "0,1")
    _compare_evaluations(ref, got, speech, streams)


# ------------------------------------------------------------------------------------------------------------------------- generate

def write_split(root, n=24, seed=3):
    """n utterances of random fbank rows, 60-400 frames: with --max-tokens 800 they make 8 batches of 2 to 5"""
    g = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "test.tsv"), "w") as f:
        f.write("id\tsrc_audio\tsrc_n_frames\ttgt_audio\ttgt_n_frames\n")
        for i, F in enumerate(int(x) for x in g.integers(60, 400, n)):
            p = os.path.join(root, f"utt{i}.npy")
            np.save(p, g.standard_normal((F, 80)).astype(np.float32))
            f.write(f"utt{i}\t{p}\t{F}\t\t0\n")
    return root


def _generate(argv, out, *extra):
    buf = io.StringIO()
    split = G.main(argv + ["--results-path", out, *extra], stdout=buf)
    with open(os.path.join(out, "generate-test.txt"), "rb") as f:
        return buf.getvalue(), f.read(), split


@pytest.mark.parametrize("task", ["speech_to_speech_ctc", "speech_to_speech_modified"], ids=["streamspeech", "unity"])
def test_generate_on_three_workers_is_byte_identical(tmp_path, task):
    data = write_split(str(tmp_path / "data"))
    argv = [data, "--task", task, "--target-is-code", "--target-code-size", "1000", "--path", "synthetic", "--gen-subset", "test",
            "--beam", "1", "--max-len-a", "1", "--max-len-b", "20", "--max-len-b-mt", "60", "--max-tokens", "800",
            "--required-batch-size-multiple", "1"]
    out1, file1, split = _generate(argv, str(tmp_path / "one"))
    assert len(split.batches) >= 6 and max(len(b) for b in split.batches) > 1
    out3, file3, _ = _generate(argv, str(tmp_path / "three"), "--devices", "0,0,0")
    assert out1 and out3 == out1
    assert file3 == file1
    assert sum(line.startswith("H-") for line in file1.decode().splitlines()) == len(split.rows)


# ------------------------------------------------------------------------------------------------------------------------ ASR-BLEU

def test_asr_bleu_on_two_workers_is_identical(tmp_path, capsys):
    d = tmp_path / "wavs"
    d.mkdir()
    refs = []
    for i in range(9):
        x = synth.make_audio(1.0 + 0.4 * i, seed=900 + i).numpy() if i != 4 else np.full(300, 0.1, dtype=np.float32)  # 4: too short
        write_pcm_wav(d / f"{i}_pred.wav", x, 16000)
        refs.append(f"reference number {i}")
    (tmp_path / "ref.txt").write_text("\n".join(refs) + "\n")
    argv = ["--lang", "en", "--audio_dirpath", str(d), "--reference_path", str(tmp_path / "ref.txt"), "--reference_format", "txt",
            "--asr-model", "synthetic"]
    runs = {}
    for name, extra in (("one", []), ("two", ["--devices", "0,0"])):
        transcripts, bleu = asr_bleu.main(argv + ["--results_dirpath", str(tmp_path / name), *extra])
        runs[name] = (transcripts, str(bleu), (d / "pred.txt").read_bytes(), (tmp_path / name / "txt_en_bleu.txt").read_bytes(),
                      capsys.readouterr().out)
    assert runs["two"] == runs["one"]
    assert runs["one"][0][4] == "" and any(runs["one"][0])


def test_score_only_on_two_workers_is_identical(tmp_path):
    src = _sources(tmp_path, 16000, float_wav=False)
    out = _evaluate(tmp_path, src, S2ST, 320, 16000, 2, "run")
    flags = ["--score-only", "--output", str(out), "--quality-metrics", "ASR_BLEU", "--latency-metrics", "AL", "LAAL", "RTF",
             "--asr-model", "synthetic"]
    files = ("scores.tsv", "metrics.tsv", "asr_transcripts.txt")
    scores1 = ev.main(flags)
    one = {n: (out / n).read_bytes() for n in files}
    one_txt = sorted((p.name, p.read_bytes()) for p in (out / "wavs").glob("*_pred.txt"))
    for n in files:
        (out / n).unlink()
    scores2 = ev.main(flags + ["--devices", "0,0"])
    assert scores2 == scores1
    assert {n: (out / n).read_bytes() for n in files} == one
    assert sorted((p.name, p.read_bytes()) for p in (out / "wavs").glob("*_pred.txt")) == one_txt
    assert any(line.strip() for line in one["asr_transcripts.txt"].decode().splitlines())


def test_evaluate_scores_asr_bleu_on_its_workers(tmp_path):
    src = _sources(tmp_path, 16000, float_wav=False)
    flags = ["--quality-metrics", "ASR_BLEU", "--latency-metrics", *SPEECH_LATENCY, "--asr-model", "synthetic"]
    ref = _evaluate(tmp_path, src, S2ST, 320, 16000, 1, "single", *flags)
    got = _evaluate(tmp_path, src, S2ST, 320, 16000, 1, "devices", *flags, "--devices", "0,0")
    _compare_evaluations(ref, got, True, 1)
    assert (got / "asr_transcripts.txt").read_bytes() == (ref / "asr_transcripts.txt").read_bytes()


def test_a_refused_file_stops_every_asr_worker(tmp_path):
    from streamspeech_b200.workers import WorkerFailed

    d = tmp_path / "wavs"
    d.mkdir()
    for i in range(8):
        write_pcm_wav(d / f"{i}_pred.wav", synth.make_audio(1.0 + 0.2 * i, seed=950 + i).numpy(), 22050 if i == 5 else 16000)
    (tmp_path / "ref.txt").write_text("".join(f"reference {i}\n" for i in range(8)))
    argv = ["--lang", "en", "--audio_dirpath", str(d), "--reference_path", str(tmp_path / "ref.txt"), "--reference_format", "txt",
            "--asr-model", "synthetic"]
    with pytest.raises(asr_bleu.AudioRefused, match="5_pred.wav: 22050 Hz"):
        asr_bleu.main(argv)
    with pytest.raises(WorkerFailed, match=r"worker on device 0 failed: \S*AudioRefused: .*5_pred\.wav: 22050 Hz"):
        asr_bleu.main(argv + ["--devices", "0,0"])
