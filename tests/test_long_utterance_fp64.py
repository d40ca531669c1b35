"""GPU: the fused encoder and MT search paths against the float64 oracle on one 38 s utterance (T = 950 encoder rows, chunk 8,
the 12-layer synthetic model).  The T2U + unit-decoder call has its float64 tests in test_t2u_fp64.py.

The other long-utterance tests compare GPU paths with each other; here each one is compared with the float64 oracle
(StreamSpeechOracle(dtype=float64), pinned to the reference fixtures by test_oracle_golden.py).  Both sides get the same inputs:
the oracle's fbank features (the pool's own features for the pool) and fp32-rounded fp64 encoder rows for the MT search.  An arg-max
may differ from the fp64 one only where the fp64 top-2 log-prob margin is below MARGIN; such positions are counted and printed with
the measured maxima as JSON lines (`pytest -s`).
"""
import json

import pytest
import torch
import torch.nn.functional as F

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

pytestmark = pytest.mark.gpu

torch.set_grad_enabled(False)
# max-abs bars; measured on an H100 80GB HBM3 (700 W): encoder 1.1e-5 (per-op) and 2.9e-6 .. 3.4e-6 (streaming steps, pool), MT features
# 8.0e-5
ENC_TOL = 1e-4
MT_FEAT_TOL = 2e-4
MARGIN = 1e-4
CHUNK = 8


def report(name, **kw):
    print(json.dumps({"test": name, **kw}))


def maxdiff(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def cuda(x):
    return x.float().cuda().contiguous()


def alias(ptr, shape):
    """a float32 tensor over device memory the engine owns"""
    n = 1
    for s in shape:
        n *= s

    class _A:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_A(), device="cuda").view(*shape)


def check_argmax(got, lprobs):
    """got [N] int, lprobs [N, V] float64 log-probs with masked entries at -inf: got must be the arg-max wherever the top-2 margin is
    at least MARGIN; returns the number of near-tie positions where it is not"""
    top = lprobs.topk(2, dim=-1)
    want, margin = top.indices[:, 0], top.values[:, 0] - top.values[:, 1]
    bad = torch.as_tensor(got).cpu().long() != want
    assert not bool((bad & (margin >= MARGIN)).any()), torch.nonzero(bad & (margin >= MARGIN)).flatten()[:10].tolist()
    return int(bad.sum())


@pytest.fixture(scope="module")
def long38():
    """engine, float64 oracle, the utterance, its oracle features and the fp64 encoder output (computed once)"""
    from oracle.streamspeech_oracle import StreamSpeechOracle, online_features
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    gc = synth.make_gcmvn(cfg)
    e = Engine(cfg, sd, None, gc)
    e.set_chunk(CHUNK)
    o = StreamSpeechOracle(cfg, sd, None, gc, chunk_size=CHUNK, dtype=torch.float64)
    wav = synth.make_audio(38.0, seed=11)
    feats = online_features(wav, gc)
    ref = o.encoder(feats.unsqueeze(0), torch.tensor([feats.size(0)]))["encoder_out"][0][:, 0]
    assert ref.shape[0] > 900
    yield cfg, e, o, wav, feats, ref
    e.close()


def ctc_lprobs(cfg, o, enc64):
    out = []
    for name in ("source_unigram", "ctc_target_unigram"):
        lp = F.log_softmax(o.ctc_logits(name, enc64.unsqueeze(1))[0], dim=-1)
        lp[:, cfg.pad] = float("-inf")
        lp[:, cfg.unk] = float("-inf")
        out.append(lp)
    return out


def test_encoders_vs_fp64_oracle(long38):
    cfg, e, o, wav, feats, ref = long38
    T = ref.shape[0]
    got = {"per_op": e.encoder(cuda(feats).unsqueeze(0))[0]}
    fd = cuda(feats)
    for cluster in (1, 0):
        e.set_option("persistent_encoder_cluster", cluster)
        buf = torch.zeros(1024, cfg.enc_dim, device="cuda")
        e.encoder_stream_reset()
        n0 = e.cluster_steps()
        Ts = 0
        for F_ in list(range(30, fd.shape[0], 32)) + [fd.shape[0]]:
            Ts, _ = e.encoder_stream_step(fd[:F_].contiguous(), buf)
        assert Ts == T
        assert (e.cluster_steps() > n0) == bool(cluster)
        got[f"stream_cluster{cluster}"] = buf[:T].clone()
    e.set_option("persistent_encoder_cluster", 1)
    e.encoder_stream_reset()
    e.check_async_error()
    lps = ctc_lprobs(cfg, o, ref)
    res = {}
    for name, enc in got.items():
        d = maxdiff(enc, ref)
        near = [check_argmax(e.ctc_greedy(head, enc.contiguous())["argmax"], lps[head]) for head in (0, 1)]
        res[name] = {"maxdiff": d, "near_ties": near}
        assert d < ENC_TOL, (name, d)
    # a one-slot pool fed the audio in 320 ms pushes; its rows are compared with the fp64 encoder of the pool's own features
    e.pool_create(1, max_seconds=40)
    n = 5120
    for i in range(0, len(wav), n):
        e.pool_push_audio(0, wav[i:i + n].contiguous())
        r = e.pool_step([0], ctc_heads=0)[0]
    info = e.pool_info(0)
    Tp = r["T"]
    pool_feats = alias(info["feats_ptr"], (info["n_feat"], cfg.feat_dim)).cpu()
    assert abs(Tp - T) <= 1 and maxdiff(pool_feats, feats[:pool_feats.shape[0]]) < 2e-3
    ref_pool = o.encoder(pool_feats.unsqueeze(0), torch.tensor([pool_feats.size(0)]))["encoder_out"][0][:, 0]
    rows = e.pool_encoder_rows(0, Tp).clone()
    d = maxdiff(rows, ref_pool)
    near = [check_argmax(e.ctc_greedy(head, rows)["argmax"], lp) for head, lp in enumerate(ctc_lprobs(cfg, o, ref_pool))]
    res["pool"] = {"maxdiff": d, "near_ties": near}
    report("long38_encoders_fp64", T=T, **res)
    assert d < ENC_TOL, ("pool", d)


def mt_check(cfg, o, enc64, tokens, max_len):
    """teacher-forced fp64 pass over [eos] + tokens: token s (eos after the last one) must be the masked arg-max at step s; returns
    (near ties, fp64 features)"""
    seq = torch.tensor([[cfg.eos] + list(tokens)], dtype=torch.long)
    feats = o.mt_features(seq, enc64.unsqueeze(1))[0]
    lp = F.log_softmax(F.linear(feats, o.sd["target_unigram_decoder.output_projection.weight"]), dim=-1)
    lp[:, cfg.pad] = float("-inf")
    lp[0, cfg.eos] = float("-inf")  # min_len = 1: no eos at step 0
    n = len(tokens)
    if n == max_len:  # eos forced at max_len
        keep = lp[n, cfg.eos].clone()
        lp[n] = float("-inf")
        lp[n, cfg.eos] = keep
    return check_argmax(torch.tensor(list(tokens) + [cfg.eos]), lp), feats


def test_mt_search_vs_fp64_oracle(long38):
    cfg, e, o, wav, feats, ref = long38
    enc32 = ref.float()  # both sides get these rows
    enc64 = enc32.double()
    max_len = 200
    toks, f = e.mt_greedy(cuda(enc32), None, -1, max_len_b=max_len)
    assert 1 <= len(toks) <= max_len
    near, f64 = mt_check(cfg, o, enc64, toks, max_len)
    dfeat = maxdiff(f, f64)
    T1 = 700  # second sample of the batch: a shorter source
    batch = torch.zeros(2, enc32.shape[0], cfg.enc_dim)
    batch[0] = enc32
    batch[1, :T1] = enc32[:T1]
    hyps = e.mt_greedy_batch(cuda(batch), [enc32.shape[0], T1], max_len)
    near_b = [mt_check(cfg, o, enc64[:Tb], h, max_len)[0] for h, Tb in zip(hyps, (enc32.shape[0], T1))]
    report("long38_mt_fp64", tokens=len(toks), batch_tokens=[len(h) for h in hyps], feat_maxdiff=dfeat, near_ties=near, batch_near_ties=near_b)
    assert dfeat < MT_FEAT_TOL, dfeat
