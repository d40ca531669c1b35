"""Offline batched generator (SURVEY.md §8 row O1): oracle vs the fixture dumped from the reference's own modules on a padded
batch (CPU), and the engine's per-sample reproduction of the batch (GPU)."""
import numpy as np
import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)


def offline_cfg():
    cfg = ModelConfig()
    cfg.uni_encoder = False  # offline model (N10)
    return cfg


def test_offline_oracle_matches_reference_fixture(gold):
    """oracle/offline_oracle.py on the padded batch == the chain of reference modules (oracle/gen_golden_offline.py):
    encoder 0-tolerance class, CTC prints / MT hypotheses / units token-exact including the batch quirks N1-N3."""
    from oracle.offline_oracle import offline_generate
    from oracle.streamspeech_oracle import StreamSpeechOracle

    g = gold["offline_batch"]
    cfg = offline_cfg()
    o = StreamSpeechOracle(cfg, synth.make_model_state_dict(cfg, 0), None, synth.make_gcmvn(cfg), chunk_size=None, conv_chunk_size=None)
    r = offline_generate(o, torch.from_numpy(g["feats"]), torch.from_numpy(g["lengths"]), max_len_b_mt=int(g["max_len_b_mt"]))
    assert float((r["enc_out"] - torch.from_numpy(g["enc_out"])).abs().max()) < 2e-5
    assert r["prev_output_tokens_mt"].tolist() == g["prev_output_tokens_mt"].tolist()
    assert float((r["mt_feats"] - torch.from_numpy(g["mt_feats"])).abs().max()) < 5e-5
    B = g["feats"].shape[0]
    lens = [len(r["mt_hyps"][b]) for b in range(B)]
    assert len(set(lens)) > 1  # the fixture exercises padded MT rows (N2)
    for b in range(B):
        assert r["asr"][b]["tokens"] == g[f"asr_tokens_{b}"].tolist()
        assert r["st"][b]["tokens"] == g[f"st_tokens_{b}"].tolist()
        assert r["mt_hyps"][b] == g[f"mt_hyp_{b}"].tolist()
        assert r["units"][b]["org_tokens"] == g[f"unit_argmax_{b}"].tolist()
        assert r["units"][b]["tokens"] == g[f"units_{b}"].tolist()


def test_unit_positions_depend_on_batch_index(gold):
    """N1: the same T2U states decode differently at batch index 0 and 1 (position b + 2 at every step), which is why the
    engine needs ss_unit_position_row; guards against 'fixing' the quirk in the oracle."""
    from oracle.streamspeech_oracle import StreamSpeechOracle

    cfg = offline_cfg()
    o = StreamSpeechOracle(cfg, synth.make_model_state_dict(cfg, 0), None, synth.make_gcmvn(cfg), chunk_size=None, conv_chunk_size=None)
    t2u = torch.from_numpy(gold["decoders"]["t2u_out"]).unsqueeze(1)  # [S, 1, 512]
    both = o.unit_decoder_logits(t2u.repeat(1, 2, 1), None)
    single = o.unit_decoder_logits(t2u, None)
    assert float((both[0] - single[0]).abs().max()) < 1e-5
    assert float((both[1] - single[0]).abs().max()) > 1e-3


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_offline_generator_engine_vs_fixture(gold):
    from streamspeech_b200.engine import Engine
    from streamspeech_b200.offline import OfflineS2STGenerator

    g = gold["offline_batch"]
    cfg = offline_cfg()
    e = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    try:
        gen = OfflineS2STGenerator(e, max_len_b_mt=int(g["max_len_b_mt"]))
        feats = torch.from_numpy(g["feats"]).cuda()
        B = feats.shape[0]
        forced = [[int(t) for t in g[f"mt_hyp_{b}"][:-1]] if g[f"mt_hyp_{b}"][-1] == cfg.eos else g[f"mt_hyp_{b}"].tolist() for b in range(B)]
        for run, fm in (("forced", forced), ("search", None)):
            res = gen.generate(feats, g["lengths"].tolist(), forced_mt=fm)
            for b in range(B):
                assert res[b]["asr_tokens"] == g[f"asr_tokens_{b}"].tolist(), (run, b)
                assert res[b]["st_tokens"] == g[f"st_tokens_{b}"].tolist(), (run, b)
                assert res[b]["mt_tokens"] == forced[b], (run, b)
                d = float((res[b]["mt_feats"].cpu() - torch.from_numpy(g["mt_feats"][b])).abs().max())
                assert d < 2e-4, (run, b, d)
                assert res[b]["unit_argmax"] == g[f"unit_argmax_{b}"].tolist(), (run, b)
                assert res[b]["units"] == g[f"units_{b}"].tolist(), (run, b)
        wav = gen.synthesize(gen.units_to_codes(res[0]["units"]))
        assert wav.numel() > 0 and bool(torch.isfinite(wav).all())
    finally:
        e.close()
