"""Batched greedy MT search of the offline generator (ss_mt_greedy_batch / Engine.mt_greedy_batch): every row must equal the
single-sample search of that sample, on the batched kernel, on the per-sample fallback, across several launch groups, and
without disturbing a streaming agent that shares the engine."""
import argparse
import ctypes

import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)

BMAX = 32  # MT_BATCH_MAX_ROWS


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
    """padded offline encoder output [B, T, C] and each sample's rows"""
    feats = [e.fbank(synth.make_audio(s, seed=seed0 + b).cuda()) for b, s in enumerate(seconds)]
    F = max(f.shape[0] for f in feats)
    src = torch.zeros(len(feats), F, e.cfg.feat_dim, device="cuda")
    for b, f in enumerate(feats):
        src[b, : f.shape[0]] = f
    lens = [f.shape[0] for f in feats]
    return e.encoder(src, lens), [e.encoder_out_frames(n) for n in lens]


def per_sample(e, enc, lens, max_len_b):
    return [e.mt_greedy(enc[b, : lens[b]].contiguous(), None, -1, max_len_b=max_len_b)[0] for b in range(enc.shape[0])]


@pytest.mark.parametrize("max_len_b", [60, 100])
@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_batch_equals_per_sample_search(eng, max_len_b):
    enc, lens = encode(eng, [3.0, 1.2, 2.4, 0.8, 1.9], 300)
    T = enc.shape[1]
    lens[1] = 1  # one encoder row
    lens[0] = T  # the whole padded stride
    ref = per_sample(eng, enc, lens, max_len_b)
    assert eng.mt_greedy_batch(enc, lens, max_len_b) == ref
    # a single row on the batched kernel too (by default one sample takes the single-token kernel)
    eng.set_option("mt_batch_min_rows", 1)
    try:
        assert eng.mt_greedy_batch(enc[2:3].contiguous(), lens[2:3], max_len_b) == ref[2:3]
        assert eng.mt_greedy_batch(enc, lens, max_len_b) == ref
    finally:
        eng.set_option("mt_batch_min_rows", 2)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_batch_vs_reference_fixture(eng, gold):
    """tests/golden/offline_batch.npz: hypotheses of the reference generator (lengths 53, 61, 61 with eos: one row ends by eos,
    two by the forced eos at max_len_b_mt = 60)"""
    g = gold["offline_batch"]
    feats = torch.from_numpy(g["feats"]).cuda()
    lengths = g["lengths"].tolist()
    enc = eng.encoder(feats.contiguous(), lengths)
    lens = [eng.encoder_out_frames(n) for n in lengths]
    B = feats.shape[0]
    want = []
    for b in range(B):
        h = g[f"mt_hyp_{b}"].tolist()
        assert h[-1] == eng.cfg.eos
        want.append(h[:-1])
    assert sorted(len(h) for h in want) == [52, 60, 60]
    assert eng.mt_greedy_batch(enc, lens, int(g["max_len_b_mt"])) == want


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_more_rows_than_one_launch(eng):
    enc5, lens5 = encode(eng, [2.0, 1.5, 2.6, 1.1, 0.7], 500)
    B = 2 * BMAX + 3
    idx = [b % 5 for b in range(B)]
    enc = enc5[idx].contiguous()
    lens = [max(1, lens5[i] - (b // 5) % 7) for b, i in enumerate(idx)]  # ragged within each group
    ref = per_sample(eng, enc, lens, 40)
    assert eng.mt_greedy_batch(enc, lens, 40) == ref


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_decode_launches_do_not_grow_with_batch(eng):
    """B = 32 vs B = 1 on the batch's longest hypothesis: the difference is exactly the cross K / V projections of the 31
    other samples (one linear per MT layer each, with that sample's row count)"""
    enc, lens = encode(eng, [15.0] * BMAX, 7000)
    hyps = eng.mt_greedy_batch(enc, lens, 100)
    longest = max(range(BMAX), key=lambda b: len(hyps[b]))
    n0 = eng.launch_count()
    eng.mt_greedy_batch(enc, lens, 100)
    n32 = eng.launch_count() - n0
    n0 = eng.launch_count()
    one = eng.mt_greedy_batch(enc[longest:longest + 1].contiguous(), lens[longest:longest + 1], 100)
    n1 = eng.launch_count() - n0
    assert one[0] == hyps[longest]
    w = torch.randn(2 * eng.cfg.mt_dim, eng.cfg.enc_dim, device="cuda")
    bias = torch.zeros(2 * eng.cfg.mt_dim, device="cuda")
    proj = 0
    for b in range(BMAX):
        if b != longest:
            n0 = eng.launch_count()
            eng.op_linear(enc[b, : lens[b]].contiguous(), w, bias)
            proj += (eng.launch_count() - n0) * eng.cfg.mt_layers
    assert n32 - n1 == proj, (n32, n1, proj)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_fallback_without_persistent_kernel(eng):
    enc, lens = encode(eng, [2.2, 1.4, 3.1], 900)
    on = eng.mt_greedy_batch(enc, lens, 60)
    eng.set_option("persistent_mt", 0)
    try:
        off = eng.mt_greedy_batch(enc, lens, 60)
    finally:
        eng.set_option("persistent_mt", 1)
    assert off == on


def _agent_args():
    return argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, global_stats=None,
                              tgt_splitter_type="SentencePiece", tgt_splitter_path=None, user_dir="", agent_dir="", max_len=200,
                              force_finish=False, shift_size=10, window_size=25, sample_rate=16000, feature_dim=80, vocoder="synthetic",
                              vocoder_cfg=None, dur_prediction=True, lagging_k1=0, lagging_k2=0, segment_size=320, stride_n=1,
                              stride_n2=1, unit_per_subword=15, extra_output_dir=None, output_asr_translation=False,
                              source_segment_size=320, vocoder_context="receptive-field", device_index=0, device="gpu")


def _run_agent(interrupt_with=None, persistent_mt=1):
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
            if interrupt_with is not None and ci == len(starts) // 2:
                enc, lens = interrupt_with
                e.set_option("persistent_mt", persistent_mt)
                e.mt_greedy_batch(enc, lens, 60)
                e.set_option("persistent_mt", 1)
            fin = i + n >= len(wav)
            seg = agent.pushpop(SpeechSegment(content=wav[i:i + n].tolist(), sample_rate=16000, finished=fin))
            out.append((agent.trace.get("mt_tokens"), agent.trace.get("units"), list(seg.content)))
    finally:
        e.close()
    return out


@pytest.mark.parametrize("persistent_mt", [1, 0])
@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_streaming_agent_state_untouched(persistent_mt):
    g = torch.Generator().manual_seed(5)
    enc = torch.randn(3, 40, ModelConfig().enc_dim, generator=g).cuda()
    base = _run_agent()
    assert any(len(w) for _, _, w in base)
    assert _run_agent((enc, [40, 17, 33]), persistent_mt) == base


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_errors_leave_the_handle_usable(eng):
    from streamspeech_b200.engine import EngineError

    enc, lens = encode(eng, [1.5, 2.0], 40)
    T = enc.shape[1]
    with pytest.raises(EngineError):
        eng.mt_greedy_batch(enc[:0].contiguous(), [], 60)
    with pytest.raises(EngineError):
        eng.mt_greedy_batch(enc, [0, lens[1]], 60)
    with pytest.raises(EngineError):
        eng.mt_greedy_batch(enc, [T + 1, lens[1]], 60)
    lib = eng.lib
    tl = (ctypes.c_int32 * 2)(*lens)
    out = (ctypes.c_int64 * 2 * 8)()
    n = (ctypes.c_int32 * 2)()
    rc = lib.ss_mt_greedy_batch(eng._h, eng._stream(), enc.data_ptr(), 2, T, tl, 60, out, 8, n)
    assert rc == -5  # SS_ERR_CAPACITY: a 60-token hypothesis does not fit 8 slots
    assert b"capacity" in lib.ss_last_error(eng._h)
    assert eng.mt_greedy_batch(enc, lens, 60) == per_sample(eng, enc, lens, 60)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_offline_generator_batched_search_at_bench_size(eng):
    from streamspeech_b200.offline import OfflineS2STGenerator

    B = 8
    feats = [eng.fbank(synth.make_audio(15.0, seed=7000 + b).cuda()) for b in range(B)]
    F = max(f.shape[0] for f in feats)
    src = torch.zeros(B, F, eng.cfg.feat_dim, device="cuda")
    for b, f in enumerate(feats):
        src[b, : f.shape[0]] = f
    lengths = [f.shape[0] for f in feats]
    gen = OfflineS2STGenerator(eng, max_len_b_mt=100)
    res = gen.generate(src, lengths)
    enc = eng.encoder(src, lengths)
    forced = per_sample(eng, enc, [eng.encoder_out_frames(n) for n in lengths], 100)
    ref = gen.generate(src, lengths, forced_mt=forced)
    for b in range(B):
        assert res[b]["mt_tokens"] == forced[b], b
        assert res[b]["units"] == ref[b]["units"], b
        assert res[b]["unit_argmax"] == ref[b]["unit_argmax"], b
