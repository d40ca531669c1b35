"""GPU: the MT search paths against the float64 oracle on one 38 s utterance (T = 950 encoder rows, chunk 8, the 12-layer synthetic
model).  The encoder paths have their float64 tests in test_encoder_fp64.py, the T2U + unit-decoder call in test_t2u_fp64.py.

The other long-utterance tests compare GPU paths with each other; here each one is compared with the float64 oracle
(StreamSpeechOracle(dtype=float64), pinned to the reference fixtures by test_oracle_golden.py).  Both sides get the same inputs:
fp32-rounded fp64 encoder rows of the oracle's fbank features.  An arg-max
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
# max-abs bar; measured on an H100 80GB HBM3 (700 W): MT features 8.0e-5
MT_FEAT_TOL = 2e-4
MARGIN = 1e-4
CHUNK = 8


def report(name, **kw):
    print(json.dumps({"test": name, **kw}))


def maxdiff(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def cuda(x):
    return x.float().cuda().contiguous()


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
