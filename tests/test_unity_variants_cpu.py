"""Uni-UnitY and Chunk-UnitY on the CPU: recognition of the UnitY family from a checkpoint's stored cfg, the refusals, and the float32
oracle (oracle/unity_variant_oracle.py) against tests/golden/unity_variants.npz, which oracle/gen_golden_unity_variants.py writes
from the reference's own uni_unity / chunk_unity modules, fairseq's MultiDecoderSequenceGenerator and the wait-k agents' policy()."""
import math
import os

import numpy as np
import pytest
import torch

from oracle.unity_variant_oracle import VariantUnitYOracle, VariantWaitkS2STAgent, VariantWaitkS2TTAgent
from oracle.unity_oracle import unity_generate
from streamspeech_b200 import generate as G
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig, unity_variant_of
from streamspeech_b200.dictionary import Dictionary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def g():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "unity_variants.npz")))


@pytest.fixture(scope="module")
def split():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "unity_generate.npz")))


@pytest.fixture(scope="module")
def sd():
    return synth.make_unity_state_dict(ModelConfig.unity_default(), seed=0)


# stored model cfg -> (unity_variant, uni_encoder, chunk_size, Engine.set_chunk geometry)
TABLE = [
    ({}, ("unity", False, 0, (None, None))),
    ({"arch": "unity_conformer_modified"}, ("unity", False, 0, (None, None))),
    ({"arch": "unity_conformer_modified", "uni_encoder": True, "chunk_size": 8}, ("unity", False, 0, (None, None))),
    ({"arch": "unity_conformer", "pos_enc_type": "rel_pos", "attn_type": "espnet"}, ("unity", False, 0, (None, None))),
    ({"arch": "uni_unity_conformer", "uni_encoder": True}, ("uni_unity", True, 0, (1, 0))),
    ({"arch": "uni_unity_conformer_waitk", "uni_encoder": True}, ("uni_unity", True, 0, (1, 0))),
    ({"arch": "uni_unity_conformer"}, ("uni_unity", False, 0, (None, None))),
    ({"arch": "chunk_unity_conformer", "uni_encoder": True, "chunk_size": 8}, ("chunk_unity", True, 8, (8, 8))),
    ({"arch": "chunk_unity_conformer", "chunk_size": 16}, ("chunk_unity", False, 16, (16, 16))),
]


@pytest.mark.parametrize("stored,want", TABLE)
def test_recognition_from_the_stored_cfg(sd, stored, want):
    for state in ({"model": sd, "cfg": {"model": stored}}, {"model": sd, "args": type("A", (), dict(stored))()}):
        c = ModelConfig.from_checkpoint(state)
        assert c.unity and (c.unity_variant, c.uni_encoder, c.chunk_size, c.encoder_chunk()) == want, stored


def test_released_unity_takes_the_old_path(sd):
    """a UnitY checkpoint (no arch, or unity_conformer_modified) gives the config the engine had before the variants existed"""
    old = ModelConfig.from_state_dict(sd)
    old.max_target_positions = 1200
    for stored in ({"max_target_positions": 1200}, {"arch": "unity_conformer_modified", "max_target_positions": 1200}):
        assert ModelConfig.from_checkpoint({"model": sd, "cfg": {"model": stored}}) == old
    assert ModelConfig.unity_default() == ModelConfig.from_checkpoint(synth.make_unity_checkpoint("unity"))


@pytest.mark.parametrize("stored,setting", [
    ({"arch": "unity_transformer_modified"}, "arch"),
    ({"arch": "s2ut_conformer"}, "arch"),
    ({"arch": "uni_unity_conformer", "pos_enc_type": "abs"}, "pos_enc_type"),
    ({"arch": "unity_conformer_modified", "pos_enc_type": "rope"}, "pos_enc_type"),
    ({"arch": "uni_unity_conformer", "attn_type": None, "conv_version": "convtransformer"}, "conv_version"),
    ({"arch": "chunk_unity_conformer", "attn_type": "abs"}, "attn_type"),
    ({"arch": "chunk_unity_conformer"}, "chunk_size"),
    ({"arch": "chunk_unity_conformer", "chunk_size": 7}, "chunk_size"),
    ({"arch": "chunk_unity_conformer", "chunk_size": 999999}, "chunk_size"),
])
def test_unsupported_settings_are_refused_by_name(stored, setting):
    with pytest.raises(ValueError, match=setting):
        unity_variant_of(stored.get)


def test_synthetic_variants_share_the_keys():
    keys = {v: {k: tuple(t.shape) for k, t in synth.make_unity_checkpoint(v)["model"].items()} for v in ("unity", "uni_unity", "chunk_unity")}
    assert keys["unity"] == keys["uni_unity"] == keys["chunk_unity"]
    assert synth.synthetic_unity_variant("researches/uni_unity") == "uni_unity"
    assert synth.synthetic_unity_variant("/x/researches/chunk_unity/") == "chunk_unity"
    assert synth.synthetic_unity_variant("researches/translatotron") == synth.synthetic_unity_variant(None) == "unity"


def test_generate_refuses_chunk_unity_offline():
    args = G.parse_args(["D", "--task", "speech_to_speech_modified", "--path", "synthetic", "--user-dir", "researches/chunk_unity",
                         "--target-is-code", "--target-code-size", "1000", "--beam", "1", "--max-tokens", "1000"])
    with pytest.raises(ValueError, match="chunk-size 8"):
        G.load_offline_checkpoint(args, 1024)


def _features(split, i):
    raw = split[f"raw_{i}"].astype(np.float32) / np.float32(int(split["raw_scale"]))
    return G.apply_cmvn(raw, (split["gcmvn_mean"], split["gcmvn_std"])).astype(np.float32)


def test_fixture_split_is_unity_generate_split(g, split):
    """the generate settings ran on unity_generate.npz's split: same frame counts, quantisation and per-sample checksums"""
    assert g["gen_n_frames"].tolist() == split["n_frames"].tolist() and int(g["gen_raw_scale"]) == int(split["raw_scale"])
    for i, (s1, s2) in enumerate(g["gen_raw_sums"].tolist()):
        x = split[f"raw_{i}"].astype(np.int64)
        assert [int(x.sum()), int((x ** 2).sum())] == [s1, s2], i


def stored_wav_or_count(g, key):
    """(the stored waveform or None, its sample count): one WRITE of the fixture keeps its samples, every other its count"""
    if key + "_wav" in g:
        return g[key + "_wav"], len(g[key + "_wav"])
    return None, int(g[key + "_wav_n"])


@pytest.mark.parametrize("k", [0, 1, 2])
def test_uni_unity_oracle_reproduces_the_generate_fixture(g, split, k):
    """prints, units, scores and positional scores of every batch of a setting"""
    cfg = ModelConfig.from_checkpoint(synth.make_unity_checkpoint("uni_unity"))
    o = VariantUnitYOracle(cfg, synth.make_unity_state_dict(cfg, seed=0), torch.float32)
    mt, beam_mt, mlb = (int(v) for v in g["gen_settings"][k])
    n_frames = g["gen_n_frames"].tolist()
    batches = G.make_batches(n_frames, [0] * len(n_frames), mt, None, 1, (6000, 1024), False)
    tdict = Dictionary.synthetic(cfg.tgt_vocab)
    stdout = []
    for batch in batches[:3]:
        fl = [torch.from_numpy(_features(split, i)) for i in batch]
        x = torch.zeros(len(fl), max(f.shape[0] for f in fl), 80)
        for b, f in enumerate(fl):
            x[b, :f.shape[0]] = f
        mine = unity_generate(o, x, [f.shape[0] for f in fl], beam_mt, 1.0, mlb, int(g["gen_max_len_b_mt"]))
        for i, h, u in zip(batch, mine["mt_hyps"], mine["units"]):
            stdout.append(G.mt_print_line(cfg, i, G.ctc_text(tdict, h)))
            assert u["tokens"] == g[f"gen{k}_units_{i}"].tolist(), (k, i)
            assert abs(u["score"] - float(g[f"gen{k}_score_{i}"])) < 1e-5
            bar = 1e-5 + 2.4e-7 * abs(u["score"]) * len(u["tokens"])
            assert np.abs(np.array(u["positional_scores"]) - g[f"gen{k}_positional_{i}"]).max() < bar
    assert stdout == g[f"gen{k}_stdout"].tolist()[:len(stdout)]
    assert all(line.endswith(")") and " (None-" in line for line in stdout)


@pytest.mark.parametrize("variant", ["uni_unity", "chunk_unity"])
@pytest.mark.parametrize("tag", ["s2st_default", "s2st_k5n2", "s2tt_k5n2"])
def test_waitk_oracle_reproduces_the_fixture(g, variant, tag):
    """every action of the float32 oracle against the reference's policy() on the model: kinds, flags, texts, tokens, units,
    durations and sample counts exact, and the stored waveform within 1e-5"""
    p = f"{variant}_{tag}"
    k1, k2, n, n2, ups, seg, chunk_ms, seed = g[f"{p}_setting"].tolist()
    kind = str(g[f"{p}_kind"])
    cfg = ModelConfig.from_checkpoint(synth.make_unity_checkpoint(variant))
    sd = synth.make_unity_state_dict(cfg, seed=0)
    tdict = Dictionary.synthetic(cfg.tgt_vocab)
    kw = dict(lagging_k1=k1, lagging_k2=k2, stride_n=n, stride_n2=n2, unit_per_subword=ups, segment_size=seg, symbols=lambda t: tdict[t])
    o = (VariantWaitkS2STAgent(cfg, sd, synth.make_gcmvn(cfg), synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=True), **kw)
         if kind == "s2st" else VariantWaitkS2TTAgent(cfg, sd, synth.make_gcmvn(cfg), **kw))
    wav = synth.make_audio(float(g[f"{p}_seconds"]), seed=seed)
    step = math.ceil(chunk_ms / 1000 * 16000)
    kinds = []
    for ci, i in enumerate(range(0, len(wav), step)):
        o.push(wav[i:i + step].tolist(), finished=i + step >= len(wav))
        a = o.policy()
        kinds.append(int(a.kind == "write"))
        for key in ("new_subword_tokens", "new_unit_tokens", "mt_tokens", "units", "dur"):
            assert (f"{p}_call{ci}_{key}" in g) == (key in a.trace), (p, ci, key)
            if key in a.trace:
                assert np.array(a.trace[key]).reshape(-1).tolist() == g[f"{p}_call{ci}_{key}"].reshape(-1).tolist(), (p, ci, key)
        if a.kind == "write":
            if kind == "s2st":
                ref, n = stored_wav_or_count(g, f"{p}_call{ci}")
                assert len(a.wav) == n, (p, ci)
                if ref is not None:
                    assert n and np.abs(np.array(a.wav) - ref).max() < 1e-5, (p, ci)
                assert [a.finished, a.seg_finished] == g[f"{p}_flags"][ci].tolist()
            else:
                assert a.wav == str(g[f"{p}_texts"][ci]) and a.finished == bool(g[f"{p}_flags"][ci][0])
    assert kinds == g[f"{p}_kinds"].tolist()
