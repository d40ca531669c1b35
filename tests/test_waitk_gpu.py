"""The wait-k-stride-n agents on the H100 against tests/golden/waitk_policy.npz (the reference's own policy() on the synthetic UnitY
checkpoint): every action, token, text, unit and duration exact and the waveform within 1e-3, a unit or token decision that differs
accepted only where the float64 oracle shows it is a near tie; and `python -m streamspeech_b200.evaluate` with each wait-k agent,
whose instances.log must be the fixture's actions played through the same SimulEval bookkeeping."""
import argparse
import json
import os
import struct

import numpy as np
import pytest
import torch

from oracle.waitk_oracle import OracleWaitkS2STAgent, OracleWaitkS2TTAgent
from streamspeech_b200 import evaluate as ev
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.dictionary import Dictionary
from streamspeech_b200.simuleval_compat import EmptySegment, SpeechSegment, TextSegment

pytestmark = pytest.mark.gpu
AGENT_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "streamspeech_b200", "agents", "waitk")
FILES = {"s2st": "speech_to_speech.wait-k-stride-n.agent.py", "s2tt": "speech_to_text.wait-k-stride-n.agent.py"}
TAGS = ["s2st_default", "s2st_k5n2", "s2tt_default", "s2tt_k5n2"]
MARGIN = 1e-4  # float64 decisions closer than this may go either way in fp32


@pytest.fixture(scope="module")
def fixture(gold):
    return gold["waitk_policy"]


def _setting(g, tag):
    k1, k2, n, n2, ups, seg, chunk, seed = g[f"{tag}_setting"].tolist()
    return dict(k1=k1, k2=k2, n=n, n2=n2, ups=ups, seg=seg, chunk=chunk, seed=seed, kind=str(g[f"{tag}_kind"]),
                seconds=float(g[f"{tag}_seconds"]))


def _flags(s):
    return ["--model-path", "synthetic", "--data-bin", ".", "--vocoder", "synthetic", "--vocoder-cfg", "none", "--dur-prediction",
            "--lagging-k1", str(s["k1"]), "--lagging-k2", str(s["k2"]), "--stride-n", str(s["n"]), "--stride-n2", str(s["n2"]),
            "--unit-per-subword", str(s["ups"]), "--segment-size", str(s["seg"])]


def _agent(s):
    from streamspeech_b200.waitk import WaitkS2STAgent, WaitkS2TTAgent, add_waitk_args

    p = argparse.ArgumentParser()
    add_waitk_args(p)
    args = p.parse_args(_flags(s))
    return WaitkS2STAgent(args) if s["kind"] == "s2st" else WaitkS2TTAgent(args)


def _float64_margins(s, wav, upto):
    """the float64 oracle's smallest unit-search margin and MT trace per call, calls 0 .. upto"""
    cfg = ModelConfig.unity_default()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    kw = dict(lagging_k1=s["k1"], lagging_k2=s["k2"], stride_n=s["n"], stride_n2=s["n2"], unit_per_subword=s["ups"], segment_size=s["seg"],
              dtype=torch.float64)
    o = (OracleWaitkS2STAgent(cfg, sd, synth.make_gcmvn(cfg), synth.make_vocoder_state_dict(cfg.vocoder, 1), **kw) if s["kind"] == "s2st"
         else OracleWaitkS2TTAgent(cfg, sd, synth.make_gcmvn(cfg), **kw))
    step, out = 16 * s["chunk"], []
    for ci, i in enumerate(range(0, len(wav), step)):
        o.push(wav[i:i + step].tolist(), finished=i + step >= len(wav))
        out.append(o.policy().trace)
        if ci == upto:
            break
    return out


@pytest.mark.parametrize("tag", TAGS)
def test_engine_agent_reproduces_the_reference_policy(fixture, tag):
    g, s = fixture, _setting(fixture, tag)
    agent = _agent(s)
    wav = synth.make_audio(s["seconds"], seed=s["seed"])
    step = 16 * s["chunk"]
    kinds, flags, texts = g[f"{tag}_kinds"], g[f"{tag}_flags"], g[f"{tag}_texts"]
    worst, n_write = 0.0, 0
    try:
        for ci, i in enumerate(range(0, len(wav), step)):
            fin = i + step >= len(wav)
            agent.push(SpeechSegment(content=wav[i:i + step].tolist(), sample_rate=16000, finished=fin))
            action = agent.policy()
            tr = agent.trace
            # decisions first: a differing MT token or unit is accepted only at a float64 near tie, and the run ends there
            for k in ("mt_tokens", "units"):
                key = f"{tag}_call{ci}_{k}"
                if key in g and k in tr and list(tr[k]) != g[key].tolist():
                    o = _float64_margins(s, wav, ci)[ci]
                    assert k == "units" and o.get("unit_margin", np.inf) < MARGIN, (tag, ci, k, "differs away from a tie")
                    pytest.skip(f"{tag}: call {ci} is a float64 near tie ({o['unit_margin']:.2e}); the trajectories part there")
            for k in ("new_subword_tokens", "new_unit_tokens", "mt_tokens", "units", "dur"):
                key = f"{tag}_call{ci}_{k}"
                assert (key in g) == (k in tr), (key, sorted(tr))
                if key in g:
                    assert np.array(tr[k]).reshape(-1).tolist() == g[key].reshape(-1).tolist(), key
            assert action.is_read() == (kinds[ci] == 0), (tag, ci)
            if action.is_read():
                continue
            n_write += 1
            if s["kind"] == "s2st":
                seg = action.content
                assert [action.finished, seg.finished] == flags[ci].tolist(), (tag, ci)
                ref = g[f"{tag}_call{ci}_wav"]
                assert len(seg.content) == len(ref), (tag, ci)
                if len(ref):
                    worst = max(worst, float(np.abs(np.asarray(seg.content, dtype=np.float32) - ref).max()))
            else:
                assert action.content == str(texts[ci]) and action.finished == bool(flags[ci][0]), (tag, ci)
        assert ci + 1 == len(kinds) and n_write == int(kinds.sum())
        assert worst < 1e-3, (tag, worst)
    finally:
        agent.engine.close()


def test_step_resident_matches_policy(fixture):
    """the S2ST agent's device-resident entry (the source already in HBM) takes the same actions"""
    tag = "s2st_default"
    g, s = fixture, _setting(fixture, tag)
    agent = _agent(s)
    try:
        wav = synth.make_audio(s["seconds"], seed=s["seed"])
        dev = wav.to(agent.torch_device)
        step = 16 * s["chunk"]
        for ci, i in enumerate(range(0, len(wav), step)):
            n = min(i + step, len(wav))
            is_write, out = agent.step_resident(dev, n, n == len(wav))
            assert is_write == bool(g[f"{tag}_kinds"][ci]), ci
            if is_write:
                ref = g[f"{tag}_call{ci}_wav"]
                got = out.cpu().numpy() if out is not None else np.zeros(0, np.float32)
                assert len(got) == len(ref) and (len(ref) == 0 or np.abs(got - ref).max() < 1e-3), ci
    finally:
        agent.engine.close()


def write_float_wav(path, x, rate):
    data = np.asarray(x, dtype="<f4").tobytes()
    fmt = struct.pack("<HHIIHH", 3, 1, rate, rate * 4, 4, 32)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt) + 8 + len(data)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(data)) + data)


def _expected_log(g, tag, s, src_path, out_dir, index):
    """the fixture's actions played through evaluate's SimulEval instance bookkeeping"""
    samples, info = ev.read_wav(src_path)
    common = dict(info=info, source_path=src_path, reference=f"reference {index}", latency_unit="word")
    if s["kind"] == "s2st":
        inst = ev.SpeechToSpeechInstance(index, samples.tolist(), wav_path=(out_dir / f"{index}_expected.wav").absolute(), **common)
    else:
        inst = ev.SpeechToTextInstance(index, samples.tolist(), **common)
    kinds, flags, texts = g[f"{tag}_kinds"], g[f"{tag}_flags"], g[f"{tag}_texts"]
    for ci in range(len(kinds)):
        inst.send_source(s["chunk"])
        if kinds[ci] == 0:
            inst.receive_prediction(EmptySegment())
        elif s["kind"] == "s2st":
            inst.receive_prediction(SpeechSegment(content=g[f"{tag}_call{ci}_wav"].tolist(), sample_rate=16000, finished=bool(flags[ci][1])))
        else:
            inst.receive_prediction(TextSegment(index=0, content=str(texts[ci]), finished=bool(flags[ci][0])))
    assert inst.source_finished_reading
    return inst.summarize()


@pytest.mark.parametrize("tag", ["s2st_default", "s2tt_k5n2"])
def test_evaluate_front_door_writes_the_fixtures_instances(fixture, tag, tmp_path):
    """two copies of the fixture's utterance in one list: the second also checks the agent's state between instances"""
    g, s = fixture, _setting(fixture, tag)
    wav = synth.make_audio(s["seconds"], seed=s["seed"]).numpy()
    src = tmp_path / "utt.wav"
    write_float_wav(src, wav, 16000)
    (tmp_path / "src.txt").write_text(f"{src}\n{src}\n")
    (tmp_path / "tgt.txt").write_text("reference 0\nreference 1\n")
    out = tmp_path / "out"
    ev.main(["--agent", os.path.join(AGENT_DIR, FILES[s["kind"]]), "--source", str(tmp_path / "src.txt"), "--target", str(tmp_path / "tgt.txt"),
             "--output", str(out), "--source-segment-size", str(s["chunk"]), "--sample-rate", "16000", *_flags(s)])
    assert (out / "config.yaml").exists()
    lines = [json.loads(x) for x in (out / "instances.log").read_text().splitlines()]
    assert [d["index"] for d in lines] == [0, 1]
    for d in lines:
        want = _expected_log(g, tag, s, str(src), tmp_path, d["index"])
        if s["kind"] == "s2st":
            got_wav, _ = ev.read_wav(d["prediction"])
            want_wav, _ = ev.read_wav(want["prediction"])
            assert len(got_wav) == len(want_wav) and np.abs(np.asarray(got_wav) - np.asarray(want_wav)).max() <= 2 / 32768
            assert os.path.dirname(d["prediction"]) == (out / "wavs").absolute().as_posix()
            for k in ("prediction", "elapsed"):
                d.pop(k), want.pop(k)
        else:
            assert len(d.pop("elapsed")) == len(want.pop("elapsed"))
        assert d == want, d["index"]
