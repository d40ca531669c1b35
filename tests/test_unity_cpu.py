"""UnitY offline generation, CPU side: state-dict recognition of both model kinds, the front door's argument rules and refusals, the
unit search's max_len rule on padded batches, and the float32 oracle of the unit search against its float64 restatement."""
import argparse
import math

import pytest
import torch

from oracle.unity_oracle import UnitYOracle, unity_max_len
from streamspeech_b200 import generate as G
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.dictionary import Dictionary


def _small_unity_cfg():
    c = ModelConfig.unity_default()
    c.enc_layers, c.mt_layers, c.t2u_layers = 1, 1, 1
    return c


def test_state_dict_recognition_both_kinds():
    ss = synth.make_model_state_dict(ModelConfig().tiny(), seed=0)
    c = ModelConfig.from_state_dict(ss)
    assert not c.unity and c.unit_vocab == 1005 and c.src_vocab == 6000
    u = synth.make_unity_state_dict(_small_unity_cfg(), seed=0)
    assert not any(k.startswith(("source_unigram_decoder.", "ctc_target_unigram_decoder.")) for k in u)
    c = ModelConfig.from_state_dict(u)
    assert c.unity and not c.uni_encoder and c.unit_vocab == 4 + 1000 and c.unit_layers == 2 and (c.unit_dim, c.unit_ffn) == (512, 2048)
    one_head = dict(ss)
    del one_head["source_unigram_decoder.proj.weight"]
    with pytest.raises(KeyError, match="both CTC heads"):
        ModelConfig.from_state_dict(one_head)


def test_unit_dictionary_has_no_blank():
    d = Dictionary.units(1000, blank=False)
    assert len(d) == 1004 and d.blank_index is None and d[4] == "0" and d[1003] == "999"
    assert len(Dictionary.units(1000)) == 1005


PRED_SH = ["DATA", "--user-dir", "researches/translatotron", "--config-yaml", "config_gcmvn.yaml", "--multitask-config-yaml",
           "config_unity.yaml", "--task", "speech_to_speech_modified", "--target-is-code", "--target-code-size", "1000", "--vocoder",
           "code_hifigan", "--path", "CKPT", "--gen-subset", "test", "--beam-mt", "10", "--beam", "1", "--max-len-a", "1",
           "--max-tokens", "10000", "--required-batch-size-multiple", "1", "--results-path", "OUT"]


def test_pred_sh_flags_are_accepted():
    a = G.parse_args(PRED_SH)
    assert (a.task, a.beam_mt, a.beam, a.max_len_a, a.max_len_b) == ("speech_to_speech_modified", 10, 1, 1.0, 200)
    a = G.parse_args(PRED_SH + ["--max-len-b", "50"])
    assert a.max_len_b == 50


@pytest.mark.parametrize("extra,msg", [(["--beam", "5"], "beam 1 only"), (["--nbest", "2"], "nbest"), (["--task", "speech_to_text"], "only"),
                                       (["--max-len-a", "nan"], "finite")])
def test_argument_refusals(extra, msg, capsys):
    with pytest.raises(SystemExit):
        G.parse_args(PRED_SH + extra)
    assert msg in capsys.readouterr().err


def test_task_must_match_checkpoint(tmp_path):
    """a UnitY checkpoint under --task speech_to_speech_ctc and a StreamSpeech one under speech_to_speech_modified are refused"""
    ss = synth.make_model_state_dict(ModelConfig().tiny(), seed=0)
    un = synth.make_unity_state_dict(_small_unity_cfg(), seed=0)
    for sd, task, kind in ((un, "speech_to_speech_ctc", "UnitY"), (ss, "speech_to_speech_modified", "StreamSpeech")):
        path = str(tmp_path / f"{kind}.pt")
        torch.save({"model": sd, "cfg": {"model": {"max_target_positions": 1200}}}, path)
        args = argparse.Namespace(path=path, task=task, data=str(tmp_path), multitask_config_yaml="x.yaml")
        with pytest.raises(ValueError, match=f"does not match the checkpoint .*{kind} model"):
            G.load_offline_checkpoint(args, 1024)


def test_max_len_uses_the_padded_batch_length():
    """generate_decoder's max_len takes src_tokens.size(1): a short sample in a batch with a long one gets the long one's limit"""
    assert unity_max_len(1.0, 200, 300, 1200) == 500
    assert unity_max_len(1.0, 200, 1500, 1200) == 1199
    assert unity_max_len(0.5, 10, 101, 1200) == 60  # int(60.5)
    from streamspeech_b200.offline import UnitYGenerator

    gen = UnitYGenerator.__new__(UnitYGenerator)
    gen.cfg, gen.max_len_a, gen.max_len_b = ModelConfig.unity_default(), 1.0, 200
    assert [gen.unit_max_len(f) for f in (10, 300, 999, 2000)] == [210, 500, 1199, 1199]


def test_oracle_fp32_follows_fp64():
    """the float32 unit search takes the float64 one's decisions wherever their margin is clear, and ends rows both ways"""
    cfg = _small_unity_cfg()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    g = torch.Generator().manual_seed(5)
    feats = torch.randn(6, 10, 512, generator=g)
    lens = [10, 10, 7, 3, 10, 5]
    r32 = UnitYOracle(cfg, sd, torch.float32).generate_units(feats, lens, 120)
    r64 = UnitYOracle(cfg, sd, torch.float64).generate_units(feats, lens, 120)
    assert any(len(r["tokens"]) < 121 for r in r64) and any(len(r["tokens"]) == 121 for r in r64)
    for a, b in zip(r32, r64):
        assert a["tokens"][-1] == b["tokens"][-1] == cfg.eos
        n = next((i for i, m in enumerate(b["margins"]) if m < 1e-4), len(b["margins"]))
        assert a["tokens"][:n] == b["tokens"][:n]
        if n == len(b["margins"]):
            assert abs(a["score"] - b["score"]) < 1e-4
            assert max(abs(x - y) for x, y in zip(a["positional_scores"], b["positional_scores"])) < 1e-4
            assert math.isclose(sum(b["positional_scores"]) / len(b["tokens"]), b["score"], rel_tol=1e-9, abs_tol=1e-9)
