"""Batched decoder stages of the offline generator (ss_ctc_greedy_batch, ss_mt_features_batch, ss_t2u_unit_decode_batch): every
sample must equal the per-sample calls (ctc_greedy_rows, mt_features + set_unit_batch_index(b) + t2u_unit_decode) and the CPU
oracle at batch indices the reference fixture does not reach, across workspace groups, without disturbing a streaming agent
that shares the engine."""
import argparse
import ctypes

import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)

SS_ERR_INVALID = -1
UNIT_BATCH_ROWS = 32768  # SS_UNIT_BATCH_ROWS


def offline_cfg():
    cfg = ModelConfig()
    cfg.uni_encoder = False  # offline model
    return cfg


@pytest.fixture(scope="module")
def eng():
    from streamspeech_b200.engine import Engine

    cfg = offline_cfg()
    e = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    e.set_chunk(None, None)
    yield e
    e.close()


def encode(e, seconds, seed0):
    """padded offline encoder output [B, T, C], each sample's rows, and the fbank batch"""
    feats = [e.fbank(synth.make_audio(s, seed=seed0 + b).cuda()) for b, s in enumerate(seconds)]
    F = max(f.shape[0] for f in feats)
    src = torch.zeros(len(feats), F, e.cfg.feat_dim, device="cuda")
    for b, f in enumerate(feats):
        src[b, : f.shape[0]] = f
    lens = [f.shape[0] for f in feats]
    return e.encoder(src, lens), [e.encoder_out_frames(n) for n in lens], src, lens


def forced(cfg, B, n, seed):
    """B hypotheses of n ordinary tokens (no specials)"""
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(4, cfg.tgt_vocab, (n,), generator=g).tolist() for _ in range(B)]


def prev_tokens(cfg, hyps):
    S = max(len(h) for h in hyps) + 1
    pads = [S - 1 - len(h) for h in hyps]
    return [[cfg.eos] + h + [cfg.pad] * p for h, p in zip(hyps, pads)], pads


def per_sample(e, enc, lens, hyps):
    """the per-sample calls the batched ones replace"""
    prev, pads = prev_tokens(e.cfg, hyps)
    out = {"ctc": [], "feats": [], "units": [], "argmax": []}
    try:
        for b in range(enc.shape[0]):
            eb = enc[b].contiguous()
            am = torch.zeros(eb.shape[0], dtype=torch.int64, device="cuda")
            out["ctc"].append((e.ctc_greedy_rows(0, eb, 0, am), e.ctc_greedy_rows(1, eb, 0, am)))
            f = e.mt_features(enc[b, : lens[b]].contiguous(), prev[b])
            e.set_unit_batch_index(b)
            r = e.t2u_unit_decode(f.contiguous(), n_pad_tail=pads[b], mask_eos=True)
            out["feats"].append(f)
            out["units"].append(e.units_to_host(r))
            out["argmax"].append(r["argmax"].tolist())
    finally:
        e.set_unit_batch_index(0)
    return out


def batched(e, enc, lens, hyps):
    prev, pads = prev_tokens(e.cfg, hyps)
    ctc, _ = e.ctc_greedy_batch(enc)
    feats = e.mt_features_batch(enc, lens, prev)
    units, argmax, _ = e.t2u_unit_decode_batch(feats, pads, mask_eos=True)
    return {"ctc": ctc, "feats": [feats[b] for b in range(enc.shape[0])], "units": units, "argmax": argmax}


def assert_same(ref, got, tol=2e-4):
    worst = 0.0
    for b in range(len(ref["units"])):
        assert got["ctc"][b] == ref["ctc"][b], b
        assert got["argmax"][b] == ref["argmax"][b], b
        assert got["units"][b] == ref["units"][b], b
        worst = max(worst, float((got["feats"][b] - ref["feats"][b]).abs().max()))
    assert worst < tol, worst
    print(f"mt_feats max-abs difference batched vs per-sample: {worst:.3e}")
    return worst


@pytest.mark.parametrize("case", ["search", "equal_length"])
@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_ragged_batch_equals_per_sample(eng, case):
    """B = 5 with T_b = 1, T_b = T_stride and (search case) an empty hypothesis: S_b = 1, every other position a pad"""
    enc, lens, _, _ = encode(eng, [3.0, 1.2, 2.4, 0.8, 1.9], 300)
    lens[1] = 1
    lens[0] = enc.shape[1]
    if case == "search":
        hyps = eng.mt_greedy_batch(enc, lens, 40)
        hyps[3] = []
    else:  # forced MT, every hypothesis of the same length: no pad tail
        hyps = forced(eng.cfg, 5, 23, 11)
    assert_same(per_sample(eng, enc, lens, hyps), batched(eng, enc, lens, hyps))


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_single_sample_equals_per_sample(eng):
    enc, lens, _, _ = encode(eng, [2.2], 77)
    hyps = eng.mt_greedy_batch(enc, lens, 40)
    assert_same(per_sample(eng, enc, lens, hyps), batched(eng, enc, lens, hyps))


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_groups_keep_the_global_batch_index(eng):
    """B = 16 with searched hypotheses of about 110 tokens -> about 2800 unit rows per sample -> groups of about 11 samples: the
    samples of the second group must still get the positional rows of their batch indices (N1)"""
    B = 16
    enc, lens, _, _ = encode(eng, [1.0 + 0.05 * b for b in range(B)], 4100)
    hyps = eng.mt_greedy_batch(enc, lens, 200)
    S = max(len(h) for h in hyps) + 1
    assert UNIT_BATCH_ROWS // (S * eng.cfg.ctc_upsample_rate) < B, S
    assert_same(per_sample(eng, enc, lens, hyps), batched(eng, enc, lens, hyps))


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_units_match_oracle_beyond_fixture_batch(eng):
    """B = 6 (the fixture has 3): the engine's batched stages vs oracle/streamspeech_oracle.py on the same padded batch, with the
    MT hypotheses of the GPU search forced into both.  Units token-exact, including N1 positions b + 2 for b = 3 .. 5."""
    from oracle.streamspeech_oracle import StreamSpeechOracle
    from streamspeech_b200.offline import OfflineS2STGenerator

    cfg = eng.cfg
    B = 6
    enc, lens, src, flen = encode(eng, [1.1, 0.7, 1.6, 0.9, 1.3, 1.0], 6100)
    hyps = eng.mt_greedy_batch(enc, lens, 25)
    res = OfflineS2STGenerator(eng, max_len_b_mt=25).generate(src, flen, forced_mt=hyps)
    o = StreamSpeechOracle(cfg, synth.make_model_state_dict(cfg, 0), None, synth.make_gcmvn(cfg), chunk_size=None, conv_chunk_size=None)
    prev, _ = prev_tokens(cfg, hyps)
    prev = torch.tensor(prev, dtype=torch.long)
    eo = enc.cpu().transpose(0, 1).contiguous()  # [T, B, C]
    enc_pad = torch.arange(eo.shape[0])[None, :] >= torch.tensor(lens)[:, None]
    x = o.mt_features(prev, eo, enc_pad if enc_pad.any() else None)
    mt_pad = prev.eq(cfg.pad) if prev.eq(cfg.pad).any() else None
    t2u = o.t2u_encoder(x.transpose(0, 1), mt_pad)
    logits = o.unit_decoder_logits(t2u, mt_pad)
    want = o.unit_ctc_greedy(logits, mask_eos=True)
    worst = max(float((res[b]["mt_feats"].cpu() - x[b]).abs().max()) for b in range(B))
    print(f"mt_feats max-abs difference vs oracle: {worst:.3e}")
    for b in range(B):
        got = res[b]["unit_argmax"]
        if got != want[b]["org_tokens"]:
            i = next(i for i, (p, q) in enumerate(zip(got, want[b]["org_tokens"])) if p != q)
            lp = torch.log_softmax(logits[b, i].float(), -1)
            lp[[cfg.pad, cfg.unk, cfg.eos]] = float("-inf")
            top = torch.topk(lp, 2)
            raise AssertionError(f"sample {b} position {i}: engine {got[i]}, oracle {want[b]['org_tokens'][i]}, oracle log-prob margin "
                                 f"{float(top.values[0] - top.values[1]):.3e} (engine's token at {float(lp[got[i]]):.4f})")
        assert res[b]["units"] == want[b]["tokens"], b


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_launches_do_not_grow_with_batch(eng):
    """B = 4 and B = 16 in one group: no stage launches more kernels at B = 16.  (A GEMM adds a split-K reduce launch when its
    tile grid is too small to fill the GPU, which happens at fewer rows, so B = 4 may launch a few more.)"""
    enc16, lens16, _, _ = encode(eng, [1.5] * 16, 9100)
    hyps16 = forced(eng.cfg, 16, 39, 3)
    counts = []
    for B in (4, 16):
        enc, lens, hyps = enc16[:B].contiguous(), lens16[:B], hyps16[:B]
        prev, pads = prev_tokens(eng.cfg, hyps)
        assert B * len(prev[0]) * eng.cfg.ctc_upsample_rate <= UNIT_BATCH_ROWS
        c = []
        n0 = eng.launch_count()
        eng.ctc_greedy_batch(enc)
        c.append(eng.launch_count() - n0)
        n0 = eng.launch_count()
        feats = eng.mt_features_batch(enc, lens, prev)
        c.append(eng.launch_count() - n0)
        n0 = eng.launch_count()
        eng.t2u_unit_decode_batch(feats, pads, mask_eos=True)
        c.append(eng.launch_count() - n0)
        counts.append(c)
    print("launches (ctc, mt features, t2u + unit decoder) at B = 4 / 16:", counts)
    assert all(n16 <= n4 for n4, n16 in zip(*counts)), counts


def _agent_args():
    return argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, global_stats=None,
                              tgt_splitter_type="SentencePiece", tgt_splitter_path=None, user_dir="", agent_dir="", max_len=200,
                              force_finish=False, shift_size=10, window_size=25, sample_rate=16000, feature_dim=80, vocoder="synthetic",
                              vocoder_cfg=None, dur_prediction=True, lagging_k1=0, lagging_k2=0, segment_size=320, stride_n=1,
                              stride_n2=1, unit_per_subword=15, extra_output_dir=None, output_asr_translation=False,
                              source_segment_size=320, vocoder_context="receptive-field", device_index=0, device="gpu")


def _run_agent(interrupt=None):
    from streamspeech_b200.agent import StreamSpeechS2STAgent
    from streamspeech_b200.simuleval_compat import SpeechSegment

    agent = StreamSpeechS2STAgent(_agent_args())
    e = agent.engine
    wav = synth.make_audio(4.0, seed=1234)
    n = 16 * 320
    starts = list(range(0, len(wav), n))
    out = []
    try:
        for ci, i in enumerate(starts):
            if interrupt is not None and ci == len(starts) // 2:
                enc, lens = interrupt
                hyps = e.mt_greedy_batch(enc, lens, 30)
                batched(e, enc, lens, hyps)
            fin = i + n >= len(wav)
            seg = agent.pushpop(SpeechSegment(content=wav[i:i + n].tolist(), sample_rate=16000, finished=fin))
            out.append((agent.trace.get("asr_tokens"), agent.trace.get("mt_tokens"), agent.trace.get("units"), list(seg.content)))
    finally:
        e.close()
    return out


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_streaming_agent_state_untouched():
    """the offline batch's decoder stages between two policy() calls of a streaming S2ST agent on the same engine leave its
    outputs unchanged (positional row, MT cross K / V cache, stable-rows state)"""
    g = torch.Generator().manual_seed(8)
    enc = torch.randn(3, 40, ModelConfig().enc_dim, generator=g).cuda()
    base = _run_agent()
    assert any(len(w) for _, _, _, w in base)
    assert _run_agent((enc, [40, 17, 33])) == base


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_invalid_arguments(eng):
    cfg = eng.cfg
    lib, h, st = eng.lib, eng._h, eng._stream()
    enc, lens, _, _ = encode(eng, [1.0, 1.4], 55)
    B, T = enc.shape[0], enc.shape[1]
    out = torch.empty(B * 2 * (2 * T + 2), dtype=torch.int64, device="cuda")
    assert lib.ss_ctc_greedy_batch(h, st, enc.data_ptr(), 0, T, out.data_ptr()) == SS_ERR_INVALID
    assert lib.ss_ctc_greedy_batch(h, st, enc.data_ptr(), B, 0, out.data_ptr()) == SS_ERR_INVALID
    assert lib.ss_ctc_greedy_batch(h, st, None, B, T, out.data_ptr()) == SS_ERR_INVALID
    assert lib.ss_ctc_greedy_batch(h, st, enc.data_ptr(), B, T, None) == SS_ERR_INVALID

    S = 5
    feats = torch.empty(B, S, cfg.mt_dim, device="cuda")

    def mtf(Bv=B, T_stride=T, tl=lens, toks=None, Sv=S, enc_p=enc.data_ptr(), out_p=feats.data_ptr()):
        toks = toks if toks is not None else [[cfg.eos, 10, 11, 12, 13]] * B
        tl_c = (ctypes.c_int32 * B)(*tl) if tl is not None else None
        tk_c = (ctypes.c_int64 * (B * S))(*[t for r in toks for t in r]) if toks != "null" else None
        return lib.ss_mt_features_batch(h, st, enc_p, Bv, T_stride, tl_c, tk_c, Sv, out_p)

    assert mtf() == 0
    for kw in (dict(Bv=0), dict(Sv=0), dict(Sv=eng.max_mt_positions + 1), dict(T_stride=0), dict(tl=[0, lens[1]]), dict(tl=[T + 1, lens[1]]),
               dict(tl=None), dict(toks="null"), dict(enc_p=None), dict(out_p=None),
               dict(toks=[[cfg.eos, 10, cfg.pad, 12, 13]] * B), dict(toks=[[cfg.eos, 10, 11, 12, cfg.tgt_vocab]] * B)):
        assert mtf(**kw) == SS_ERR_INVALID, kw

    L = S * cfg.ctc_upsample_rate
    rows = torch.zeros(B, cfg.unit_dim, device="cuda")
    am = torch.empty(B, L, dtype=torch.int64, device="cuda")
    packed = torch.empty(B, L + 1, dtype=torch.int64, device="cuda")

    def t2u(Bv=B, Sv=S, pads=(0, 2), f=feats.data_ptr(), r=rows.data_ptr(), a=am.data_ptr(), p=packed.data_ptr()):
        pc = (ctypes.c_int32 * B)(*pads) if pads is not None else None
        return lib.ss_t2u_unit_decode_batch(h, st, f, Bv, Sv, pc, r, 1, a, p)

    assert t2u() == 0
    for kw in (dict(Bv=0), dict(Sv=0), dict(Sv=eng.max_mt_positions + 1), dict(pads=(-1, 0)), dict(pads=(0, S)), dict(pads=None), dict(f=None),
               dict(r=None), dict(a=None), dict(p=None)):
        assert t2u(**kw) == SS_ERR_INVALID, kw
    # the handle stays usable
    hyps = [[10, 11, 12, 13], [10, 11]]
    assert_same(per_sample(eng, enc, lens, hyps), batched(eng, enc, lens, hyps))
