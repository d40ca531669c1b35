"""UnitY against tests/golden/unity_generate.npz (oracle/gen_golden_unity.py: the reference's own encoder, MT decoder, T2U
encoder and unit decoder classes under MultiDecoderSequenceGenerator and fairseq's unity SequenceGenerator).  CPU: the oracle
against the fixture, and the stored max_target_positions.  GPU: the `--task speech_to_speech_modified` front door on the fixture's
split, for every setting the fixture holds."""
import importlib.util
import io
import math
import os

import numpy as np
import pytest
import torch

from oracle.unity_oracle import UnitYOracle, unity_generate
from streamspeech_b200 import generate as G
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.dictionary import Dictionary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "unity_generate.npz")


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLD))


def _write_split(g, root):
    """the split writer of tests/test_generate.py (raw fbank files, a stored zip, gcmvn stats, config yaml)"""
    spec = importlib.util.spec_from_file_location("_test_generate_split", os.path.join(ROOT, "tests", "test_generate.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.write_split(g, root)


def _batches(g, k):
    mt, _, _ = (int(v) for v in g["settings"][k])
    return G.make_batches(g["n_frames"].tolist(), [0] * len(g["n_frames"]), mt, None, 1, (6000, 1024), False)


def _features(g, i):
    raw = g[f"raw_{i}"].astype(np.float32) / np.float32(int(g["raw_scale"]))
    return G.apply_cmvn(raw, (g["gcmvn_mean"], g["gcmvn_std"])).astype(np.float32)


def test_fixture_pins_the_padded_batch_limit(g):
    """every sample ends at the forced eos of its BATCH's padded length: a short sample's limit follows its batch"""
    for k, (_, _, mlb) in enumerate(g["settings"].tolist()):
        for batch in _batches(g, k):
            F = max(int(g["n_frames"][i]) for i in batch)
            for i in batch:
                assert len(g[f"s{k}_units_{i}"]) == F + mlb + 1, (k, i)
    assert int(g["n_forced_eos"]) == sum(len(b) for k in range(len(g["settings"])) for b in _batches(g, k))


@pytest.mark.parametrize("k,bi", [(2, 2), (4, 3)])
def test_oracle_against_fixture(g, k, bi):
    """the float32 oracle reproduces the reference's D- prints, units, scores and positional scores on two of the fixture's batches
    (a lone sample, and four samples with ragged MT hypotheses under --beam-mt 4)"""
    cfg = ModelConfig.unity_default()
    o = UnitYOracle(cfg, synth.make_unity_state_dict(cfg, seed=0), torch.float32)
    _, beam_mt, mlb = (int(v) for v in g["settings"][k])
    batch = _batches(g, k)[bi]
    fl = [torch.from_numpy(_features(g, i)) for i in batch]
    x = torch.zeros(len(fl), max(f.shape[0] for f in fl), 80)
    for b, f in enumerate(fl):
        x[b, :f.shape[0]] = f
    mine = unity_generate(o, x, [f.shape[0] for f in fl], beam_mt, 1.0, mlb, int(g["max_len_b_mt"]))
    tdict = Dictionary.synthetic(cfg.tgt_vocab)
    stdout = g[f"s{k}_stdout"].tolist()
    for i, h, u in zip(batch, mine["mt_hyps"], mine["units"]):
        assert "D-{}\t{}".format(i, G.ctc_text(tdict, h)) in stdout
        assert u["tokens"] == g[f"s{k}_units_{i}"].tolist(), (k, i)
        assert abs(u["score"] - float(g[f"s{k}_score_{i}"])) < 1e-5
        bar = 1e-5 + 2.4e-7 * abs(u["score"]) * len(u["tokens"])
        assert np.abs(np.array(u["positional_scores"]) - g[f"s{k}_positional_{i}"]).max() < bar
    if len(batch) > 1:
        assert len({len(h) for h in mine["mt_hyps"]}) > 1  # ragged MT lengths: padded T2U positions are masked keys


def test_from_checkpoint_reads_max_target_positions():
    cfg = ModelConfig.unity_default()
    cfg.enc_layers = cfg.mt_layers = 1
    sd = synth.make_unity_state_dict(cfg, seed=0)
    assert ModelConfig.from_state_dict(sd).max_target_positions == 1024
    assert ModelConfig.from_checkpoint({"model": sd, "cfg": {"model": {"max_target_positions": 1200}}}).max_target_positions == 1200
    assert ModelConfig.from_checkpoint({"model": sd, "args": type("A", (), {"max_target_positions": 1100})()}).max_target_positions == 1100
    assert ModelConfig.from_checkpoint({"model": sd}).max_target_positions == 1024


@pytest.mark.gpu
def test_front_door_against_fixture(g, tmp_path):
    """every setting of the fixture through `python -m streamspeech_b200.generate`: stdout and the texts / units of the results
    file identical, H- / P- scores within test_front_door_end_to_end's tolerances (P- scaled by the cumulative score: positional
    scores are differences of fp32 cumulative sums)"""
    data = _write_split(g, str(tmp_path / "data"))
    for k, (mt, beam_mt, mlb) in enumerate(g["settings"].tolist()):
        out = str(tmp_path / f"out{k}")
        buf = io.StringIO()
        G.main([data, "--config-yaml", "config_gcmvn.yaml", "--task", "speech_to_speech_modified", "--target-is-code",
                "--target-code-size", "1000", "--path", "synthetic", "--gen-subset", "test", "--beam-mt", str(beam_mt), "--beam", "1",
                "--max-len-a", "1", "--max-len-b", str(mlb), "--max-len-b-mt", str(int(g["max_len_b_mt"])), "--max-tokens", str(mt),
                "--required-batch-size-multiple", "1", "--results-path", out], stdout=buf)
        assert buf.getvalue().splitlines() == g[f"s{k}_stdout"].tolist(), k
        got = open(os.path.join(out, "generate-test.txt")).read().splitlines()
        want = g[f"s{k}_file_lines"].tolist()
        assert len(got) == len(want) + 1 and got[-1].startswith("Generate test with beam=1: BLEU4 = ")
        for a, b in zip(got, want):
            fa, fb = a.split("\t"), b.split("\t")
            assert fa[0] == fb[0], (k, a[:60], b[:60])
            if fa[0][0] in "HD":
                assert fa[2] == fb[2], (k, fa[0])  # the units
                n = len(fb[2].split()) + 1
                assert abs(float(fa[1]) - float(fb[1])) * math.log(2) < 1e-5 * n, (k, fa[0], fa[1], fb[1])
            elif fa[0][0] == "P":
                pa, pb = np.array(fa[1].split(), dtype=np.float64), np.array(fb[1].split(), dtype=np.float64)
                assert pa.shape == pb.shape
                bar = 2e-4 + 2.4e-7 * abs(pb.sum()) * math.log(2)
                assert np.abs(pa - pb).max() < bar, (k, fa[0], float(np.abs(pa - pb).max()))
            else:
                assert a == b
