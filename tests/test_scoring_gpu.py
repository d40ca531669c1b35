"""The scoring stage of streamspeech_b200.evaluate on the GPU: the reference's S2ST recipe flags (simuleval.simul-s2st.sh, without
--computation-aware) on the synthetic checkpoint with the synthetic ASR model, and the S2TT and ASR recipes' flags.

ASR_BLEU's transcripts must equal the oracle pipeline's (read_wav of the 16-bit files, the float64 wav2vec 2.0 forward pass, best
path), with the engine's letter taken only at fp64 near-ties; the score must be BLEU of those transcripts against the raw references;
the latency columns must equal the CPU scorers applied to the run's own instances.log; --streams 1 and 2 (whose instances finish out
of index order) must write the same scores.tsv, metrics.tsv and asr_transcripts.txt; and --score-only after a wav is deleted must report ASR_BLEU 0.0 and name the file."""
import json
import os

import pytest
import torch

from oracle import asr_oracle as ao
from streamspeech_b200 import evaluate as ev
from streamspeech_b200 import simuleval_scoring as sc
from streamspeech_b200 import synth
from streamspeech_b200.asr import SPECIALS, ASRTranscriber
from streamspeech_b200.generate_waveform_from_code import write_wav
from streamspeech_b200.sacrebleu_compat import corpus_bleu

pytestmark = pytest.mark.gpu

AGENTS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "streamspeech_b200", "agents")
S2ST, S2TT, ASR = ("speech_to_speech.streamspeech.agent.py", "speech_to_text.s2tt.streamspeech.agent.py",
                   "speech_to_text.asr.streamspeech.agent.py")
# (seconds, audio seed): the longest first, so with --streams 2 instance 1 finishes before instance 0 and the run completes out of
# index order (1, 0, 2, 3, 4)
SOURCES = [(4.2, 904), (1.6, 902), (3.4, 901), (2.1, 900), (2.8, 903)]
SECONDS = [sec for sec, _ in SOURCES]
REFS = ["So on, and so on.", "The end", "o no", "Son of a son!", "no one knows"]  # not lower-cased or normalised
S2ST_LATENCY = ["AL", "AP", "DAL", "StartOffset", "EndOffset", "LAAL", "ATD", "NumChunks", "DiscontinuitySum", "DiscontinuityAve",
                "DiscontinuityNum", "RTF"]
TEXT_LATENCY = ["AL", "AP", "DAL", "StartOffset", "EndOffset", "LAAL", "ATD", "NumChunks", "RTF"]
STRIDES = [s for (_, _, s) in synth.W2V_CONV_LAYERS]
KERNELS = [k for (_, k, _) in synth.W2V_CONV_LAYERS]
TIE_MARGIN = 1e-2  # as tests/test_asr_bleu_e2e.py


def _sources(tmp_path):
    paths = []
    for i, (sec, seed) in enumerate(SOURCES):
        p = tmp_path / f"utt{i}.wav"
        write_wav(str(p), synth.make_audio(sec, seed=seed).numpy(), 16000)
        paths.append(str(p))
    (tmp_path / "src.txt").write_text("\n".join(paths) + "\n")
    (tmp_path / "tgt.txt").write_text("\n".join(REFS) + "\n")


def _run(tmp_path, agent, streams, *extra):
    out = tmp_path / f"{agent.split('.')[0]}_{agent.split('.')[1]}_{streams}"
    argv = ["--agent", os.path.join(AGENTS, agent), "--source", str(tmp_path / "src.txt"), "--target", str(tmp_path / "tgt.txt"),
            "--output", str(out), "--source-segment-size", "320", "--streams", str(streams), "--model-path", "synthetic",
            "--data-bin", ".", "--vocoder", "synthetic", "--vocoder-cfg", "none", "--dur-prediction", "--sample-rate", "16000", *extra]
    return ev.main(argv), out


def oracle_transcripts(files, sd64, vocab, engine):
    """the oracle pipeline's transcript per file; the engine's per-frame arg-max may differ from fp64's only at near-ties"""
    out, ties = [], 0
    for fp in files:
        x, _ = ev.read_wav(fp)
        assert ao.num_frames(len(x), KERNELS, STRIDES) > 0
        e = ao.forward(sd64, torch.from_numpy(x), STRIDES, normalize=True, dtype=torch.float64, device="cuda")["emissions"]
        m = e.clone()
        m[:, ao.UNK] = float("-inf")
        top2 = m.topk(2, dim=1).values
        margin = (top2[:, 0] - top2[:, 1]).cpu()
        bp = ao.best_path(e)
        _, am = engine.transcribe_tokens([x])[0]
        diff = [t for t in range(len(bp)) if am[t] != bp[t]]
        assert all(float(margin[t]) < TIE_MARGIN for t in diff), [(t, float(margin[t])) for t in diff]
        ties += len(diff)
        out.append(ao.letters(ao.get_tokens(am if diff else bp), vocab))
    return out, ties


def _cpu_latency(out, unit, latency):
    """the CPU scorers on the run's own instances.log: live instances from its summaries, speech silences from the intervals"""
    instances = {}
    for line in (out / "instances.log").read_text().splitlines():
        d = json.loads(line)
        silences = []
        for (s0, d0), (s1, _) in zip(d.get("intervals", []), d.get("intervals", [])[1:]):
            if s1 > s0 + d0:
                silences.append(s1 - (s0 + d0))
        instances[d["index"]] = sc.live_instance(d, unit, silences)
    return sc.score(instances, [], latency), instances


def _finish_order(monkeypatch):
    """the indices in the order their instances finish (the run keeps each one as it finishes)"""
    order = []
    live = sc.live_instance

    def record(summary, *a, **k):
        order.append(summary["index"])
        return live(summary, *a, **k)

    monkeypatch.setattr(sc, "live_instance", record)
    return order


def test_s2st_recipe_scores_asr_bleu_and_latency(tmp_path, caplog, monkeypatch):
    _sources(tmp_path)
    flags = ["--quality-metrics", "ASR_BLEU", "--target-speech-lang", "en", "--latency-metrics", *S2ST_LATENCY, "--asr-model", "synthetic"]
    runs, orders = {}, {}
    order = _finish_order(monkeypatch)
    for n in (1, 2):
        order.clear()
        runs[n] = _run(tmp_path, S2ST, n, *flags)
        orders[n] = list(order)
    assert orders[1] == list(range(len(SOURCES))) and orders[2] != sorted(orders[2])  # the pooled run finishes out of order
    assert list(runs[2][0].kept) == list(range(len(SOURCES)))  # ... and is scored in index order
    run, out = runs[1]
    assert list(run.scores) == ["ASR_BLEU"] + S2ST_LATENCY
    wavs = out / "wavs"
    files = [str(wavs / f"{i}_pred.wav") for i in range(len(SECONDS))]
    assert all(os.path.exists(f) for f in files), "every utterance must produce speech for this test"
    sd64 = {k: v.to("cuda", torch.float64) for k, v in synth.make_w2v_ctc_state_dict().items()}
    vocab = SPECIALS + [ln.split()[0] for ln in synth.w2v_letter_dict().splitlines()]
    want, ties = oracle_transcripts(files, sd64, vocab, ASRTranscriber("synthetic", None, 0))
    assert any(want)
    assert (out / "asr_transcripts.txt").read_text() == "".join(w + "\n" for w in want)
    for k, w in enumerate(want):
        assert (wavs / f"{k}_pred.txt").read_text() == w.lower() + "\n"
    assert run.scores["ASR_BLEU"] == round(corpus_bleu(want, [REFS]).score, 3)
    latency, _ = _cpu_latency(out, "word", S2ST_LATENCY)
    assert {k: v for k, v in run.scores.items() if k != "ASR_BLEU"} == latency
    assert run.scores["DiscontinuityNum"] >= 0 and run.scores["NumChunks"] > 1
    assert (runs[2][1] / "scores.tsv").read_bytes() == (out / "scores.tsv").read_bytes()
    assert (runs[2][1] / "metrics.tsv").read_bytes() == (out / "metrics.tsv").read_bytes()  # rows in index order
    assert (runs[2][1] / "asr_transcripts.txt").read_bytes() == (out / "asr_transcripts.txt").read_bytes()
    print(json.dumps({"test": "s2st_recipe_scores", "scores": run.scores, "near_tie_frames": ties, "finish_order_2": orders[2]}))

    (wavs / "1_pred.wav").unlink()
    with caplog.at_level("ERROR", logger="streamspeech_b200.scoring"):
        scores = ev.main(["--score-only", "--output", str(out), "--quality-metrics", "ASR_BLEU", "--latency-metrics", "AL", "RTF",
                          "--asr-model", "synthetic"])
    assert scores["ASR_BLEU"] == 0.0
    assert "ASR on target speech failed" in caplog.text and "1_pred.wav" in caplog.text


@pytest.mark.parametrize("agent", [S2TT, ASR])
def test_text_recipes_score_bleu_and_latency(tmp_path, agent):
    _sources(tmp_path)
    run, out = _run(tmp_path, agent, 2, "--quality-metrics", "BLEU", "--latency-metrics", *TEXT_LATENCY)
    latency, instances = _cpu_latency(out, "word", TEXT_LATENCY)
    preds = [ins.prediction for ins in instances.values()]
    assert any(preds)
    assert run.scores == {"BLEU": round(corpus_bleu(preds, [REFS]).score, 3), **latency}
    assert (out / "scores.tsv").read_text() == sc.scores_tsv(run.scores)
    print(json.dumps({"test": "text_recipe_scores", "agent": agent, "scores": run.scores}))
