"""MT beam search of the offline generator (ss_mt_beam_batch / Engine.mt_beam_batch / OfflineS2STGenerator(beam_size_mt=K)):
the oracle against the reference's own n-best (tests/golden/mt_beam.npz, CPU), the engine against the same fixture on the
stored encoder rows, samples independent of their batch and launch group, the forced-eos edges, argument errors before any
launch, the generator's wiring and a streaming agent on the same engine left undisturbed."""
import ctypes
import math

import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)

gpu = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")


def offline_cfg():
    cfg = ModelConfig()
    cfg.uni_encoder = False  # offline model
    return cfg


def fixture_cases(g, early=False):
    """(K, len_penalty, key prefix, max_len_b) of the fixture's plain cases, or of its early-eos cases"""
    pfx = "early_" if early else ""
    mlb = int(g["early_max_len_b_mt"] if early else g["max_len_b_mt"])
    for K in g["beams"].tolist():
        for lp in g["len_penalties"].tolist():
            yield K, lp, f"{pfx}k{K}_lp{lp}", mlb


def model_sd(g, early):
    """the synthetic offline checkpoint, or its early-eos variant the fixture's early_ cases were made on"""
    from oracle.mt_beam_oracle import early_eos_state_dict

    cfg = offline_cfg()
    sd = synth.make_model_state_dict(cfg, 0)
    return early_eos_state_dict(sd, cfg.eos, float(g["eos_row_scale"])) if early else sd


@pytest.mark.parametrize("early", [False, True])
def test_oracle_reproduces_reference_nbest(gold, early):
    """the float32 restatement gives the reference's n-best (tokens, order, scores, positional scores) on the stored encoder
    rows; early: the checkpoint on which samples finalize hypotheses at two steps before max_len"""
    from oracle.mt_beam_oracle import mt_beam
    from oracle.streamspeech_oracle import StreamSpeechOracle

    g = gold["mt_beam"]
    cfg = offline_cfg()
    o = StreamSpeechOracle(cfg, model_sd(g, early), None, synth.make_gcmvn(cfg), chunk_size=None, conv_chunk_size=None)
    B = len(g["enc_lengths"])
    lengths = set()
    for K, lp, tag, mlb in fixture_cases(g, early):
        for b in range(B):
            enc = torch.from_numpy(g[f"enc_{b}"]).unsqueeze(1)
            hyps = mt_beam(o, enc, K, mlb, lp)["hyps"]
            for i, h in enumerate(hyps):
                assert h["tokens"] == g[f"{tag}_tokens_{b}_{i}"].tolist(), (tag, b, i)
                assert abs(h["score"] - float(g[f"{tag}_score_{b}_{i}"])) < 1e-5, (tag, b, i)
                pos = g[f"{tag}_pos_{b}_{i}"].tolist()
                assert len(pos) == len(h["positional_scores"]) and max(abs(x - y) for x, y in zip(pos, h["positional_scores"])) < 1e-5
            lengths.add(tuple(len(h["tokens"]) for h in hyps))
    if early:  # a sample finalizes at step 1, searches on and finalizes again before max_len
        assert any(min(n) < max(n) < int(g["early_max_len_b_mt"]) + 1 for n in lengths), lengths


def test_generator_argument_checks():
    from streamspeech_b200.offline import OfflineS2STGenerator

    class Stub:  # the checks run before the engine is touched
        cfg = offline_cfg()

    for bad in (0, 33, 2.5):
        with pytest.raises(ValueError):
            OfflineS2STGenerator(Stub(), beam_size_mt=bad)
    with pytest.raises(ValueError):
        OfflineS2STGenerator(Stub(), beam_size_mt=2, len_penalty=math.nan)
    with pytest.raises(NotImplementedError):
        OfflineS2STGenerator(Stub(), beam_size_mt=2, beam_size=2)
    with pytest.raises(NotImplementedError):
        OfflineS2STGenerator(Stub(), beam_size_mt=2, max_len_a_mt=1.0)


def make_engine(sd):
    from streamspeech_b200.engine import Engine

    cfg = offline_cfg()
    e = Engine(cfg, sd, synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    e.set_chunk(None, None)
    return e


@pytest.fixture(scope="module")
def eng():
    e = make_engine(synth.make_model_state_dict(offline_cfg(), 0))
    yield e
    e.close()


def oracle64(sd=None):
    from oracle.streamspeech_oracle import StreamSpeechOracle

    cfg = offline_cfg()
    sd = synth.make_model_state_dict(cfg, 0) if sd is None else sd
    return StreamSpeechOracle(cfg, sd, None, synth.make_gcmvn(cfg), chunk_size=None, conv_chunk_size=None, dtype=torch.float64)


def assert_matches_oracle(res, want, what):
    """engine hypotheses (tokens without eos) against the oracle's: same tokens in the same order, scores within 1e-4"""
    assert len(res) == len(want), what
    for i, (h, w) in enumerate(zip(res, want)):
        assert h["tokens"] + [offline_cfg().eos] == w["tokens"], (what, i)
        assert abs(h["score"] - w["score"]) < 1e-4, (what, i)
        assert max(abs(x - y) for x, y in zip(h["positional_scores"], w["positional_scores"])) < 1e-4, (what, i)


def encode(e, seconds, seed0):
    feats = [e.fbank(synth.make_audio(s, seed=seed0 + b).cuda()) for b, s in enumerate(seconds)]
    F = max(f.shape[0] for f in feats)
    src = torch.zeros(len(feats), F, e.cfg.feat_dim, device="cuda")
    for b, f in enumerate(feats):
        src[b, : f.shape[0]] = f
    lens = [f.shape[0] for f in feats]
    return e.encoder(src, lens), [e.encoder_out_frames(n) for n in lens], src, lens


@pytest.mark.parametrize("early", [False, True])
@pytest.mark.gpu
@gpu
def test_fixture_parity(eng, gold, early):
    """the reference's K hypotheses per sample, same tokens in the same order; scores and positional scores within 1e-4 (the
    engine's log-softmax and sums are fp32 on the GPU, the reference's fp32 on the CPU).  early: an engine on the fixture's
    early-eos checkpoint, where samples finalize hypotheses at step 1 and again at step 8 < max_len"""
    g = gold["mt_beam"]
    T_b = g["enc_lengths"].tolist()
    B, T = len(T_b), max(T_b)
    enc = torch.zeros(B, T, eng.cfg.enc_dim)
    for b in range(B):
        enc[b, : T_b[b]] = torch.from_numpy(g[f"enc_{b}"])
    enc = enc.cuda().contiguous()
    e = make_engine(model_sd(g, True)) if early else eng
    try:
        for K, lp, tag, mlb in fixture_cases(g, early):
            check_fixture_case(e, g, enc, T_b, K, lp, tag, mlb)
    finally:
        if early:
            e.close()


def check_fixture_case(eng, g, enc, T_b, K, lp, tag, mlb):
    res = eng.mt_beam_batch(enc, T_b, K, mlb, lp)
    for b in range(len(T_b)):
        assert len(res[b]) == K
        for i, h in enumerate(res[b]):
            want = g[f"{tag}_tokens_{b}_{i}"].tolist()
            assert want[-1] == eng.cfg.eos
            assert h["tokens"] == want[:-1], (tag, b, i)
            assert abs(h["score"] - float(g[f"{tag}_score_{b}_{i}"])) < 1e-4, (tag, b, i)
            assert max(abs(x - y) for x, y in zip(h["positional_scores"], g[f"{tag}_pos_{b}_{i}"].tolist())) < 1e-4, (tag, b, i)


@pytest.mark.gpu
@gpu
def test_samples_independent_of_batch_and_group(eng):
    """B = 7 at K = 5: launch groups of 6 and 1 samples; one sample with a single encoder row, one filling the stride"""
    enc, lens, _, _ = encode(eng, [1.2, 0.8, 1.6, 0.6, 1.0, 1.4, 0.9], 900)
    T = enc.shape[1]
    lens[1] = 1
    lens[2] = T
    res = eng.mt_beam_batch(enc, lens, 5, 20)
    for b in range(7):
        one = eng.mt_beam_batch(enc[b:b + 1].contiguous(), lens[b:b + 1], 5, 20)[0]
        assert one == res[b], b  # tokens, scores and positional scores bit for bit


@pytest.mark.gpu
@gpu
def test_widths_and_long_encoder_against_float64_oracle(eng, gold):
    """K = 32 (one sample per launch, 32 rows on one cross K / V block; two launch groups), K = 2 with B = 1, and a 1024-row
    encoder output, each against the float64 restatement (float32 and float64 select the same hypotheses in all three; the
    float64 oracle's smallest score gap among the 2K + 1 best candidates of a step is in the failure message)"""
    from oracle.mt_beam_oracle import mt_beam

    g = gold["mt_beam"]
    o = oracle64()
    rows = [torch.from_numpy(g[f"enc_{b}"]) for b in (0, 2)]
    T = max(r.shape[0] for r in rows)
    enc = torch.zeros(2, T, eng.cfg.enc_dim)
    for b, r in enumerate(rows):
        enc[b, : r.shape[0]] = r
    wide = eng.mt_beam_batch(enc.cuda().contiguous(), [r.shape[0] for r in rows], 32, 6)
    for b, r in enumerate(rows):
        want = mt_beam(o, r.unsqueeze(1), 32, 6)
        assert_matches_oracle(wide[b], want["hyps"], f"K=32 sample {b}, float64 margin {want['margin']:.2e}")
    r1 = torch.from_numpy(g["enc_1"])
    two = eng.mt_beam_batch(r1.unsqueeze(0).cuda().contiguous(), [r1.shape[0]], 2, 12)[0]
    want = mt_beam(o, r1.unsqueeze(1), 2, 12)
    assert_matches_oracle(two, want["hyps"], f"K=2 B=1, float64 margin {want['margin']:.2e}")
    long = torch.randn(1024, eng.cfg.enc_dim, generator=torch.Generator().manual_seed(11))
    res = eng.mt_beam_batch(long.unsqueeze(0).cuda().contiguous(), [1024], 3, 8)[0]
    want = mt_beam(o, long.unsqueeze(1), 3, 8)
    assert_matches_oracle(res, want["hyps"], f"1024 rows, float64 margin {want['margin']:.2e}")


@pytest.mark.gpu
@gpu
def test_forced_eos_edges(eng):
    enc, lens, _, _ = encode(eng, [1.0, 0.7], 950)
    for mlb in (1, 2):
        for hyps in eng.mt_beam_batch(enc, lens, 4, mlb):
            assert all(len(h["tokens"]) == mlb for h in hyps)  # every beam ends at the forced eos
            assert all(len(h["positional_scores"]) == mlb + 1 for h in hyps)
            for h in hyps:
                assert abs(h["score"] - sum(h["positional_scores"]) / (mlb + 1)) < 1e-4


@pytest.mark.gpu
@gpu
def test_argument_errors_before_any_launch(eng):
    enc, lens, _, _ = encode(eng, [1.0, 0.8], 960)
    T = enc.shape[1]
    lib = eng.lib
    K, cap = 3, 64
    tl = (ctypes.c_int32 * 2)(*lens)
    out = (ctypes.c_int64 * (2 * K * cap))()
    n = (ctypes.c_int32 * (2 * K))()
    sc = (ctypes.c_float * (2 * K))()
    pos = (ctypes.c_float * (2 * K * (cap + 1)))()
    torch.cuda.synchronize()
    l0 = eng.launch_count()

    def call(B=2, lengths=tl, beam=K, mlb=20, lp=1.0, max_out=cap, ptr_out=out):
        return lib.ss_mt_beam_batch(eng._h, eng._stream(), enc.data_ptr(), B, T, lengths, beam, mlb, lp, ptr_out, max_out, n, sc, pos)

    assert call(beam=1) == -1  # SS_ERR_INVALID: beam 1 is ss_mt_greedy_batch
    assert call(beam=33) == -1
    assert call(lp=math.inf) == -1 and call(lp=math.nan) == -1
    assert call(lengths=(ctypes.c_int32 * 2)(0, lens[1])) == -1
    assert call(lengths=(ctypes.c_int32 * 2)(T + 1, lens[1])) == -1
    assert call(B=0) == -1
    assert call(ptr_out=None) == -1
    assert call(mlb=60, max_out=8) == -5  # SS_ERR_CAPACITY
    assert eng.launch_count() == l0
    eng.set_option("persistent_mt", 0)
    try:
        assert call() == -3  # SS_ERR_CUDA: no other beam implementation
        assert b"persistent" in lib.ss_last_error(eng._h)
    finally:
        eng.set_option("persistent_mt", 1)
    assert eng.launch_count() == l0
    assert call() == 0


@pytest.mark.gpu
@gpu
def test_offline_generator_uses_best_hypothesis(eng):
    from streamspeech_b200.offline import OfflineS2STGenerator

    enc, out_len, src, lengths = encode(eng, [1.4, 0.9, 1.1], 970)
    gen = OfflineS2STGenerator(eng, beam_size_mt=4, len_penalty=0.8, max_len_b_mt=25)
    res = gen.generate(src, lengths)
    best = [n[0]["tokens"] for n in eng.mt_beam_batch(enc, out_len, 4, 25, 0.8)]
    ref = gen.generate(src, lengths, forced_mt=best)
    for b in range(len(lengths)):
        assert res[b]["mt_tokens"] == best[b]
        assert res[b]["units"] == ref[b]["units"] and res[b]["unit_argmax"] == ref[b]["unit_argmax"], b


@pytest.mark.gpu
@gpu
def test_streaming_agent_state_untouched():
    import argparse

    from streamspeech_b200.agent import StreamSpeechS2STAgent
    from streamspeech_b200.simuleval_compat import SpeechSegment

    args = argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, global_stats=None,
                              tgt_splitter_type="SentencePiece", tgt_splitter_path=None, user_dir="", agent_dir="", max_len=200,
                              force_finish=False, shift_size=10, window_size=25, sample_rate=16000, feature_dim=80, vocoder="synthetic",
                              vocoder_cfg=None, dur_prediction=True, lagging_k1=0, lagging_k2=0, segment_size=320, stride_n=1,
                              stride_n2=1, unit_per_subword=15, extra_output_dir=None, output_asr_translation=False,
                              source_segment_size=320, vocoder_context="receptive-field", device_index=0, device="gpu")
    g = torch.Generator().manual_seed(5)
    enc = torch.randn(3, 40, ModelConfig().enc_dim, generator=g).cuda()

    def run(interrupt):
        agent = StreamSpeechS2STAgent(args)
        e = agent.engine
        wav = synth.make_audio(4.0, seed=1234)
        n = 16 * 320
        starts = list(range(0, len(wav), n))
        out = []
        try:
            for ci, i in enumerate(starts):
                if interrupt and ci == len(starts) // 2:
                    e.mt_beam_batch(enc, [40, 17, 33], 5, 30)
                seg = agent.pushpop(SpeechSegment(content=wav[i:i + n].tolist(), sample_rate=16000, finished=i + n >= len(wav)))
                out.append((agent.trace.get("mt_tokens"), agent.trace.get("units"), list(seg.content)))
        finally:
            e.close()
        return out

    base = run(False)
    assert any(len(w) for _, _, w in base)
    assert run(True) == base
