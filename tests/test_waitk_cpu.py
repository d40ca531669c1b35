"""The wait-k-stride-n agents on UnitY without a GPU: the float32 oracle (oracle/waitk_oracle.py) replays every action of
tests/golden/waitk_policy.npz (the reference's own policy(), oracle/gen_golden_waitk.py), the gate arithmetic against the reference's
expressions, the flags and their defaults, and the refusals of the front door and of a StreamSpeech checkpoint."""
import argparse
import os

import numpy as np
import pytest
import torch

from oracle.waitk_oracle import OracleWaitkS2STAgent, OracleWaitkS2TTAgent
from streamspeech_b200 import evaluate as ev
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.dictionary import Dictionary
from streamspeech_b200.waitk import load_unity_checkpoint, waitk_counts

AGENT_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "streamspeech_b200", "agents", "waitk")
S2ST, S2TT = "speech_to_speech.wait-k-stride-n.agent.py", "speech_to_text.wait-k-stride-n.agent.py"


@pytest.fixture(scope="module")
def fixture(gold):
    return gold["waitk_policy"]


def fixture_settings(g):
    return [str(t) for t in g["tags"]]


def test_fixture_covers_the_issue_settings(fixture):
    tags = fixture_settings(fixture)
    assert set(tags) == {"s2st_default", "s2st_k5n2", "s2tt_default", "s2tt_k5n2"}
    for t in tags:
        k1, k2, n, n2, ups, seg, chunk, _ = fixture[f"{t}_setting"].tolist()
        kinds = fixture[f"{t}_kinds"]
        assert kinds.sum() >= 2 and (kinds == 0).any(), t
        samples = int(round(float(fixture[f"{t}_seconds"]) * 16000))
        if t.endswith("default"):
            assert (k1, k2, n, n2, ups, seg, chunk) == (3, 1, 1, 1, 15, 320, 320)
            assert samples % (16 * seg) != 0  # the source ends in the middle of a segment
        else:
            assert (k1, n, n2, seg, chunk) == (5, 2, 2, 640, 320)


def _oracle(cfg, sd, gcmvn, vsd, g, tag, dtype=torch.float32):
    k1, k2, n, n2, ups, seg, _, _ = g[f"{tag}_setting"].tolist()
    kw = dict(lagging_k1=k1, lagging_k2=k2, stride_n=n, stride_n2=n2, unit_per_subword=ups, segment_size=seg, sample_rate=16000, dtype=dtype)
    if str(g[f"{tag}_kind"]) == "s2st":
        return OracleWaitkS2STAgent(cfg, sd, gcmvn, vsd, **kw)
    d = Dictionary.synthetic(cfg.tgt_vocab)
    return OracleWaitkS2TTAgent(cfg, sd, gcmvn, symbols=lambda t: d[t], **kw)


@pytest.mark.parametrize("tag", ["s2st_default", "s2st_k5n2", "s2tt_default", "s2tt_k5n2"])
def test_oracle_replays_the_reference_policy(fixture, tag):
    g = fixture
    cfg = ModelConfig.unity_default()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    vsd = synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=True)
    agent = _oracle(cfg, sd, synth.make_gcmvn(cfg), vsd, g, tag)
    _, _, _, _, _, _, chunk, seed = g[f"{tag}_setting"].tolist()
    wav = synth.make_audio(float(g[f"{tag}_seconds"]), seed=seed)
    step = 16 * chunk
    kinds, flags, texts = g[f"{tag}_kinds"], g[f"{tag}_flags"], g[f"{tag}_texts"]
    s2st = str(g[f"{tag}_kind"]) == "s2st"
    for ci, i in enumerate(range(0, len(wav), step)):
        agent.push(wav[i:i + step].tolist(), finished=i + step >= len(wav))
        a = agent.policy()
        assert (a.kind == "write") == bool(kinds[ci]), (tag, ci)
        for k in ("new_subword_tokens", "new_unit_tokens", "mt_tokens", "units", "dur"):
            key = f"{tag}_call{ci}_{k}"
            assert (key in g) == (k in a.trace), (key, a.trace.keys())
            if key in g:
                assert np.array(a.trace[k]).reshape(-1).tolist() == g[key].reshape(-1).tolist(), key
        if a.kind == "read":
            continue
        if s2st:
            assert [a.finished, a.seg_finished] == flags[ci].tolist(), (tag, ci)
            ref = g[f"{tag}_call{ci}_wav"]
            assert len(a.wav) == len(ref)
            if len(ref):
                assert np.abs(np.array(a.wav) - ref).max() < 1e-5, (tag, ci)
        else:
            assert a.wav == str(texts[ci]) and a.finished == bool(flags[ci][0]), (tag, ci)
    assert ci + 1 == len(kinds)


def _reference_gate(n_samples, segment_size, k1, n, k2, n2, ups, rate=16000):
    """agent:359-384 as written (floats from `//` with a float divisor)"""
    src_seg_num = n_samples // (segment_size * rate / 1000)
    subword_tokens = ((src_seg_num - k1) // n) * n
    unit_tokens = ((subword_tokens - k2) // n2) * n2 * ups
    return src_seg_num, subword_tokens, unit_tokens


@pytest.mark.parametrize("k1,n,k2,n2,ups,seg", [(3, 1, 1, 1, 15, 320), (5, 2, 1, 2, 15, 640), (0, 3, 0, 1, 10, 160), (7, 4, 3, 3, 25, 480),
                                                (1, 1, 2, 1, 1, 40), (4, 2, 0, 5, 15, 1000)])
def test_gate_arithmetic_matches_the_reference(k1, n, k2, n2, ups, seg):
    for n_samples in list(range(0, 16 * seg * 12, 16 * seg // 4 + 7)) + [16 * seg * m + d for m in range(1, 12) for d in (-1, 0, 1)]:
        ref = _reference_gate(n_samples, seg, k1, n, k2, n2, ups)
        got = waitk_counts(n_samples, seg, 16000, k1, n, k2, n2, ups)
        assert got == tuple(int(x) for x in ref), (n_samples, got, ref)
    # 48 kHz sources count segments of 48 kHz samples
    assert waitk_counts(3 * 16 * seg * 5, seg, 48000, k1, n, k2, n2, ups) == waitk_counts(16 * seg * 5, seg, 16000, k1, n, k2, n2, ups)


def _parse(agent, *extra):
    return ev.parse_args(["--agent", os.path.join(AGENT_DIR, agent), "--source", "s.txt", "--target", "t.txt", "--output", "o",
                          "--model-path", "synthetic", "--data-bin", ".", *extra])


def test_flags_and_defaults_are_the_references():
    a = _parse(S2ST, "--vocoder", "v", "--vocoder-cfg", "c", "--dur-prediction")
    assert (a.lagging_k1, a.lagging_k2, a.stride_n, a.stride_n2, a.unit_per_subword, a.segment_size) == (3, 1, 1, 1, 15, 320)
    assert (a.sample_rate, a.max_len, a.force_finish, a.dur_prediction, a.streams) == (16000, 200, False, True, 1)
    a = _parse(S2ST, "--vocoder", "v", "--vocoder-cfg", "c", "--lagging-k1", "5", "--lagging-k2", "2", "--stride-n", "2", "--stride-n2", "3",
               "--unit-per-subword", "10", "--segment-size", "640", "--source-segment-size", "320")
    assert (a.lagging_k1, a.lagging_k2, a.stride_n, a.stride_n2, a.unit_per_subword, a.segment_size) == (5, 2, 2, 3, 10, 640)
    assert a.source_segment_size == 320 and not a.dur_prediction
    with pytest.raises(SystemExit):  # the S2ST agent needs its vocoder
        _parse(S2ST)
    a = _parse(S2TT)  # the S2TT agent accepts --vocoder / --vocoder-cfg and does not need them
    assert a.vocoder is None and a.lagging_k1 == 3
    a = _parse(S2TT, "--vocoder", "v", "--vocoder-cfg", "c")
    assert a.vocoder == "v"


@pytest.mark.parametrize("agent", [S2ST, S2TT])
def test_more_than_one_stream_is_refused(agent, capsys):
    with pytest.raises(SystemExit):
        _parse(agent, "--vocoder", "v", "--vocoder-cfg", "c", "--streams", "2")
    err = capsys.readouterr().err
    assert "wait-k" in err and "one stream" in err
    assert _parse(agent, "--vocoder", "v", "--vocoder-cfg", "c", "--streams", "1").streams == 1


def test_a_streamspeech_checkpoint_is_refused(tmp_path):
    cfg = ModelConfig()
    path = tmp_path / "streamspeech.pt"
    torch.save({"model": synth.make_model_state_dict(cfg, seed=0)}, path)
    args = argparse.Namespace(model_path=str(path), data_bin=str(tmp_path), config_yaml=None, multitask_config_yaml=None)
    with pytest.raises(ValueError, match="StreamSpeech"):
        load_unity_checkpoint(args)


def test_the_synthetic_checkpoint_is_unity():
    cfg, sd, gcmvn, dicts = load_unity_checkpoint(argparse.Namespace(model_path="synthetic:3"))
    assert cfg.unity and cfg.max_target_positions == 1200 and gcmvn is not None
    assert torch.equal(sd["decoder.embed_tokens.weight"], synth.make_unity_state_dict(cfg, seed=3)["decoder.embed_tokens.weight"])
    assert len(dicts["tgt"]) == cfg.unit_vocab and dicts["tgt"][4] == "0"


def test_agent_files_load_the_way_simuleval_loads_them():
    """`simuleval --agent FILE` imports the file as a top-level module named "agents" and requires exactly one @entrypoint class"""
    import importlib.util

    from streamspeech_b200 import simuleval_compat as sc

    expected = {S2ST: ("WaitkS2STAgent", "speech"), S2TT: ("WaitkS2TTAgent", "text")}
    assert sorted(f for f in os.listdir(AGENT_DIR) if f.endswith(".py")) == sorted(expected)
    for fname, (cls_name, target) in expected.items():
        before = len(sc.EVALUATION_SYSTEM_LIST)
        spec = importlib.util.spec_from_file_location("agents", os.path.join(AGENT_DIR, fname))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        new = sc.EVALUATION_SYSTEM_LIST[before:]
        assert len(new) == 1 and new[0].__name__ == cls_name, (fname, new)
        assert new[0].source_type == "speech" and new[0].target_type == target
        p = argparse.ArgumentParser()
        new[0].add_args(p)
        a = p.parse_args(["--model-path", "m", "--data-bin", "d", "--vocoder", "v", "--vocoder-cfg", "c"])
        assert (a.lagging_k1, a.lagging_k2, a.segment_size, a.sample_rate) == (3, 1, 320, 16000)
