"""S2TT utterances whose finishing MT call is allowed more than 1024 positions (longer than about 8 s), and incremental MT searches
that really fill more than 1024 self-attention entries.

The incremental search reserves max_len + kv_off + 2 cache entries before it starts, wherever eos will fall, so a 10 s utterance
(max_len = 1198) needs an engine built with max_mt_positions above the default 1024, and the persistent MT kernels need a
self-attention that is not limited to the 1024 scores a CTA keeps in shared memory (attend_head_long in kernels_persist_mt.cuh).

Two checkpoints.  The calibrated synthetic one ends its sentences (eos is a positional feature, synth.py): the reference's own
policy() on the 10 s bench utterance stops at 91 tokens (tests/golden/agent_policy_s2tt_long.npz, written by
oracle/gen_golden_s2tt_long.py), and the agents must reproduce that fixture call by call.  To fill the cache, the same checkpoint with
its eos row zeroed never ends a sentence (the eos logit is exactly 0, below the best of 6000 others); on it the searches are driven
through the entry points to 1023, 1024, 1025 and 2049 entries; the single-token kernel is compared with the float64 oracle by the rule
of test_long_utterance_fp64.py (a token may differ from the teacher-forced fp64 arg-max only where the fp64 top-2 margin is below
1e-4), the batched kernel with the single-token kernel token for token.
"""
import argparse
import ctypes
import json

import pytest
import torch
import torch.nn.functional as F

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)
gpu = pytest.mark.gpu
TRACE_KEYS = ("asr_tokens", "st_tokens", "mt_tokens")
SS_ERR_INVALID = -1
SS_ERR_CAPACITY = -5
MARGIN = 1e-4
LONG_POSITIONS = 2048


def report(name, **kw):
    """the measured values of a test as one JSON line on stdout (shown with `pytest -s`)"""
    print(json.dumps({"test": name, **kw}))


def s2tt_args(seg_ms=320, max_mt_positions=None):
    a = argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, global_stats=None,
                           tgt_splitter_type="SentencePiece", tgt_splitter_path=None, user_dir="", agent_dir="", max_len=200,
                           force_finish=False, shift_size=10, window_size=25, sample_rate=16000, feature_dim=80, vocoder="synthetic",
                           vocoder_cfg=None, dur_prediction=True, lagging_k1=0, lagging_k2=0, segment_size=seg_ms, stride_n=1, stride_n2=1,
                           unit_per_subword=15, extra_output_dir=None, output_asr_translation=False, source_segment_size=seg_ms,
                           vocoder_context="receptive-field", device_index=0, device="gpu")
    if max_mt_positions is not None:
        a.max_mt_positions = max_mt_positions
    return a


def record(seg, agent):
    """one call's observable output: (is write, text, finished, trace)"""
    return (not seg.is_empty, seg.content if not seg.is_empty else None, bool(seg.finished), dict((k, agent.trace.get(k)) for k in TRACE_KEYS))


def run_single(agent, wav, seg_ms):
    """a whole utterance through the single agent at this latency; returns its calls"""
    from streamspeech_b200.simuleval_compat import SpeechSegment

    c = seg_ms // 40
    agent.engine.set_chunk(c, min(c, 16))
    agent.reset()
    n = 16 * seg_ms
    return [record(agent.pushpop(SpeechSegment(content=wav[i:i + n].tolist(), sample_rate=16000, finished=i + n >= len(wav))), agent)
            for i in range(0, len(wav), n)]


def run_pooled(agents, wavs, seg_ms=320):
    """rounds of seg_ms: every agent pushes the next segment of its current utterance (agent j plays wavs[j] one after the other);
    returns each agent's calls"""
    from streamspeech_b200.scheduler import pushpop_many
    from streamspeech_b200.simuleval_compat import SpeechSegment

    queues = [list(w) for w in wavs]
    pos = [0] * len(agents)
    got = [[] for _ in agents]
    n = 16 * seg_ms
    while any(queues):
        due, segs = [], []
        for j, q in enumerate(queues):
            if not q:
                continue
            if pos[j] == 0 and agents[j].states.source_finished:  # the previous utterance ended without the reset quirk
                agents[j].reset()
            fin = pos[j] + n >= len(q[0])
            segs.append(SpeechSegment(content=q[0][pos[j]:pos[j] + n].tolist(), sample_rate=16000, finished=fin))
            due.append(j)
            pos[j] += n
            if fin:
                q.pop(0)
                pos[j] = 0
        for j, seg in zip(due, pushpop_many([agents[j] for j in due], segs)):
            got[j].append(record(seg, agents[j]))
    return got


def oracle_calls(wav, seg_ms):
    """the same utterance through OracleS2TTAgent (fp32, CPU): (is write, text, finished, trace) per call"""
    from oracle.agent_oracle import OracleS2TTAgent
    from oracle.streamspeech_oracle import StreamSpeechOracle
    from streamspeech_b200.dictionary import Dictionary

    cfg = ModelConfig()
    d = Dictionary.synthetic(cfg.tgt_vocab)
    o = OracleS2TTAgent(StreamSpeechOracle(cfg, synth.make_model_state_dict(cfg, 0), None, synth.make_gcmvn(cfg)), seg_ms, symbols=lambda t: d[t])
    n = 16 * seg_ms
    calls = []
    for i in range(0, len(wav), n):
        o.push(wav[i:i + n].tolist(), finished=i + n >= len(wav))
        a = o.policy()
        calls.append((a.kind == "write", a.wav if a.kind == "write" else None, bool(a.finished), dict((k, a.trace.get(k)) for k in TRACE_KEYS)))
    return calls


def compare(got, ref, tag):
    assert len(got) == len(ref), (tag, len(got), len(ref))
    for ci, (g, r) in enumerate(zip(got, ref)):
        assert g == r, (tag, ci, g, r)


def compare_with_fixture(calls, g):
    """every action, text delta, CTC and MT token of the reference's policy() fixture"""
    kinds, texts = g["kinds"].tolist(), g["texts"].tolist()
    assert len(calls) == len(kinds)
    for ci, (is_write, text, finished, tr) in enumerate(calls):
        assert is_write == bool(kinds[ci]), ci
        for k in ("asr_tokens", "st_tokens"):
            assert (tr[k] or []) == g[f"call{ci}_{k}"].tolist(), (ci, k)
        if kinds[ci]:
            assert text == texts[ci], (ci, text, texts[ci])
            assert tr["mt_tokens"] == g[f"call{ci}_mt_tokens"].tolist(), ci
            assert finished == bool(g[f"call{ci}_finished"]), ci
    assert len(calls[-1][3]["mt_tokens"]) == int(g["final_len"])


def bench_utterance(g):
    return synth.make_audio(float(g["seconds"]), seed=int(g["seed"]))


def test_oracle_agent_reproduces_the_long_reference_fixture(gold):
    g = gold["agent_policy_s2tt_long"]
    assert int(g["final_max_len"]) > 1024 and int(g["self_attention_entries"]) == int(g["final_len"]) + int(g["mt_calls"])
    compare_with_fixture(oracle_calls(bench_utterance(g), int(g["segment_ms"])), g)


# ---------------------------------------------------------------------------------------------------------------- agents (GPU)
@pytest.fixture(scope="module")
def long_agent():
    """a single S2TT agent on an engine with 2048 MT positions and, on that engine, an 8-slot pool for 13 s streams"""
    from streamspeech_b200.agent import StreamSpeechS2TTAgent
    from streamspeech_b200.scheduler import StreamPool

    agent = StreamSpeechS2TTAgent(s2tt_args(320, LONG_POSITIONS))
    pool = StreamPool(agent.engine, n_slots=8, max_seconds=13, ctc_heads=2)
    yield agent, pool
    agent.engine.close()


@pytest.fixture(scope="module")
def default_agent():
    """the same agent as every other test builds it: 1024 MT positions"""
    from streamspeech_b200.agent import StreamSpeechS2TTAgent

    agent = StreamSpeechS2TTAgent(s2tt_args(320))
    yield agent
    agent.engine.close()


@gpu
def test_agent_reproduces_the_reference_fixture_on_the_10s_utterance(long_agent, gold):
    agent, _ = long_agent
    g = gold["agent_policy_s2tt_long"]
    calls = run_single(agent, bench_utterance(g), int(g["segment_ms"]))
    compare_with_fixture(calls, g)
    report("s2tt_long_reference_fixture", calls=len(calls), writes=sum(c[0] for c in calls), final_tokens=len(calls[-1][3]["mt_tokens"]))


@gpu
@pytest.mark.parametrize("seconds,seed,seg_ms", [(10.0, 1234, 160), (12.0, 77, 320)])
def test_agent_equals_oracle_agent(long_agent, seconds, seed, seg_ms):
    """more calls (a larger kv_off) at 160 ms, and a 12 s utterance"""
    agent, _ = long_agent
    wav = synth.make_audio(seconds, seed=seed)
    compare(run_single(agent, wav, seg_ms), oracle_calls(wav, seg_ms), (seconds, seg_ms))


@gpu
def test_pooled_agents_equal_the_single_agent_on_long_utterances(long_agent):
    """4 s, 10 s and 12 s streams share every flush of one pool; the 4 s agents play a second utterance on their slot"""
    from streamspeech_b200.scheduler import PooledS2TTAgent

    agent, pool = long_agent
    plan = [[(10.0, 1234)], [(12.0, 801)], [(4.0, 802), (4.0, 803)], [(10.0, 804)], [(4.0, 805), (3.0, 806)], [(12.0, 807)]]
    wavs = [[synth.make_audio(sec, seed=sd) for sec, sd in p] for p in plan]
    refs = [sum((run_single(agent, w, 320) for w in ws), []) for ws in wavs]
    agents = [PooledS2TTAgent(pool, agent.dict["target_unigram"], s2tt_args(320)) for _ in plan]
    steps0 = pool.steps
    got = run_pooled(agents, wavs)
    assert max(pool.rows_per_step[steps0:]) == len(plan)
    for j, (g, r) in enumerate(zip(got, refs)):
        compare(g, r, j)
    report("pool_s2tt_long_vs_single", calls=sum(len(c) for c in got), writes=sum(c[0] for calls in got for c in calls))
    for a in agents:
        pool.release(a.slot)


@gpu
def test_results_below_1024_positions_do_not_depend_on_the_capacity(long_agent, default_agent):
    """an engine with 2048 positions and one with 1024: identical calls on a 6.4 s S2TT utterance, bit-identical MT feature rows from
    ss_mt_greedy and ss_mt_features (the S2ST agents' calls)"""
    agent, _ = long_agent
    wav = synth.make_audio(6.4, seed=1234)
    compare(run_single(agent, wav, 320), run_single(default_agent, wav, 320), "6.4 s")
    enc = torch.randn(120, agent.cfg.enc_dim, generator=torch.Generator().manual_seed(5)).cuda()
    outs = []
    for a in (agent, default_agent):
        toks, feats = a.engine.mt_greedy(enc, None, 40, max_len_b=100)
        toks2, feats2 = a.engine.mt_greedy(enc, toks[:7], 12, max_len_b=100)
        outs.append((toks, feats.clone(), toks2, feats2.clone(), a.engine.mt_features(enc, [a.cfg.eos] + toks).clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y
    assert len(outs[0][0]) >= 5


@gpu
def test_capacity_error_names_max_mt_positions(default_agent):
    """the default engine on the 10 s utterance: the agents say what the call needed and which setting to raise"""
    from streamspeech_b200.engine import EngineError
    from streamspeech_b200.scheduler import PooledS2TTAgent, StreamPool

    wav = synth.make_audio(10.0, seed=1234)
    with pytest.raises(EngineError, match=r"max_mt_positions = 1024.*needs 12\d\d self-attention entries.*args\.max_mt_positions") as ei:
        run_single(default_agent, wav, 320)
    assert ei.value.__cause__.code == SS_ERR_CAPACITY
    default_agent.reset()
    pool = StreamPool(default_agent.engine, n_slots=2, max_seconds=11, ctc_heads=2)
    pooled = [PooledS2TTAgent(pool, default_agent.dict["target_unigram"], s2tt_args(320)) for _ in range(2)]
    with pytest.raises(EngineError, match=r"max_mt_positions = 1024.*needs 12\d\d self-attention entries"):
        run_pooled(pooled, [[wav], [wav[:64000]]])


# ------------------------------------------------------------------- searches that fill more than 1024 entries (GPU, no-eos checkpoint)
NOEOS_POSITIONS = 2304
N_SLOTS = 12
BOUNDARY_ENTRIES = (1023, 1024, 1025, 2 * 1024 + 1)
WARMUP_CALLS = ((None, 2), (2, 3))  # (prefix length, max_new_tokens) of the calls before the finishing one: kv_off = 2 there


@pytest.fixture(scope="module")
def noeos():
    """an engine with room for 2049 entries and the float64 oracle, both on the checkpoint whose eos row is zero; a 12-slot pool on the
    engine"""
    from oracle.streamspeech_oracle import StreamSpeechOracle
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    for k in ("target_unigram_decoder.embed_tokens.weight", "target_unigram_decoder.output_projection.weight"):
        if k in sd:
            sd[k] = sd[k].clone()
            sd[k][cfg.eos] = 0.0
    gc = synth.make_gcmvn(cfg)
    e = Engine(cfg, sd, None, gc, max_mt_positions=NOEOS_POSITIONS)
    e.set_chunk(8, 8)
    o = StreamSpeechOracle(cfg, sd, None, gc, dtype=torch.float64)
    e.pool_create(N_SLOTS, max_seconds=3)
    yield cfg, e, o
    e.close()


def finishing_max_len(entries):
    """max_len of the finishing call that leaves `entries` cache entries: entries = final length + calls of the utterance"""
    return entries - (len(WARMUP_CALLS) + 1)


def single_search(e, enc, entries):
    """the utterance's calls on the handle's incremental state; returns the calls [(prefix, max_new, max_len, tokens)]"""
    e.mt_incremental_reset()
    calls, hyp = [], None
    for _, max_new in WARMUP_CALLS + ((None, -1),):
        ml = finishing_max_len(entries)
        toks = e.mt_greedy_incremental(enc, hyp, max_new, ml)
        calls.append((hyp, max_new, ml, toks))
        hyp = toks
    e.mt_incremental_reset()
    return calls


def fp64_lprobs(cfg, o, enc, toks):
    """[eos] + toks teacher-forced through the float64 decoder: the masked log-probs [len(toks) + 1, vocab] of every position"""
    seq = torch.tensor([[cfg.eos] + list(toks)], dtype=torch.long)
    feats = o.mt_features(seq, enc.double().cpu().unsqueeze(1))[0]
    lp = F.log_softmax(F.linear(feats, o.sd["target_unigram_decoder.output_projection.weight"]), dim=-1)
    lp[:, cfg.pad] = float("-inf")
    lp[0, cfg.eos] = float("-inf")  # min_len = 1: no eos at step 0
    return lp


def near_ties(toks, lp):
    """toks[s] must be the arg-max of lp[s] wherever the fp64 top-2 margin is at least MARGIN; returns the positions where it is not"""
    top = lp[:len(toks)].topk(2, dim=-1)
    bad = torch.tensor(toks) != top.indices[:, 0]
    margin = top.values[:, 0] - top.values[:, 1]
    assert not bool((bad & (margin >= MARGIN)).any()), torch.nonzero(bad & (margin >= MARGIN)).flatten()[:10].tolist()
    return int(bad.sum())


@gpu
def test_searches_to_the_block_edges_vs_fp64_oracle(noeos):
    """The single-token kernel to 1023, 1024, 1025 and 2049 entries against the float64 oracle, and the batched kernel against the
    single-token kernel with all four lengths and eight short rows in one launch.
    fp64: one call on a fresh state (kv_off = 0, entries = max_len + 1) is the plain causal decoder, which the float64 oracle
    teacher-forces in one pass; the four searches feed the same positions as far as they go, so the pass over the longest serves all.
    With earlier calls in the state (kv_off = 2, one duplicate entry per call) the pooled search must equal the handle's token for token."""
    cfg, e, o = noeos
    slots = list(range(N_SLOTS))
    # slots 0..3 hold the same utterance and run the four lengths, slots 4..11 stay short: rows below and above 1024 entries in one
    # launch of the batched kernel.  The handle's searches run on copies of the slots' own encoder rows.
    for sl in slots:
        k = 0 if sl < 4 else sl
        e.pool_reset(sl)
        e.pool_push_audio(sl, synth.make_audio(1.6 + 0.08 * k, seed=900 + k).contiguous())
    res = e.pool_step(slots, ctc_heads=0)
    rows = [e.pool_encoder_rows(sl, r["T"]).clone() for sl, r in zip(slots, res)]
    fresh = {}
    for sl, E in enumerate(BOUNDARY_ENTRIES):
        e.mt_incremental_reset()
        fresh[E] = e.mt_greedy_incremental(rows[3], None, -1, E - 1)
        assert len(fresh[E]) == E - 1  # (this checkpoint never emits eos: the search fills its max_len)
        assert fresh[E][:BOUNDARY_ENTRIES[0] - 1] == fresh[BOUNDARY_ENTRIES[0]]
    lp = fp64_lprobs(cfg, o, rows[3], fresh[BOUNDARY_ENTRIES[-1]])
    near = {E: near_ties(toks, lp) for E, toks in fresh.items()}
    singles = {E: single_search(e, rows[sl], E) for sl, E in enumerate(BOUNDARY_ENTRIES)}
    for E, calls in singles.items():
        assert len(calls[-1][3]) + len(calls) == E
    hyp = [None] * len(slots)
    pooled = [[] for _ in slots]
    for _, max_new in WARMUP_CALLS + ((None, -1),):
        mls = [finishing_max_len(BOUNDARY_ENTRIES[sl]) if sl < 4 else 40 + 3 * sl for sl in slots]
        out = e.pool_mt_greedy_incremental(slots, hyp, [max_new] * len(slots), mls)
        for sl, toks in zip(slots, out):
            pooled[sl].append((hyp[sl], max_new, mls[sl], toks))
            hyp[sl] = toks
    for sl, E in enumerate(BOUNDARY_ENTRIES):
        assert [c[3] for c in pooled[sl]] == [c[3] for c in singles[E]], E
    for sl in slots[4:]:  # the short rows of the same launches, against the handle's search on the same encoder rows
        e.mt_incremental_reset()
        for prefix, max_new, ml, toks in pooled[sl]:
            assert e.mt_greedy_incremental(rows[sl], prefix, max_new, ml) == toks, sl
    e.mt_incremental_reset()
    report("mt_long_attention_fp64", entries=list(BOUNDARY_ENTRIES), near_ties=near)


@gpu
def test_capacity_is_checked_before_any_launch(noeos):
    """max_len + kv_off + 2 > max_mt_positions: SS_ERR_CAPACITY with nothing launched, on the handle and in the pool, and the state as it was;
    the same for a token outside the vocabulary (SS_ERR_INVALID) in ss_mt_greedy_incremental, ss_mt_greedy and ss_mt_features"""
    cfg, e, o = noeos
    lib, h, st = e.lib, e._h, e._stream()
    I32, I64 = ctypes.c_int32, ctypes.c_int64
    cap = NOEOS_POSITIONS
    e.mt_incremental_reset()
    e.pool_reset(1)
    e.pool_push_audio(1, synth.make_audio(1.68, seed=901).contiguous())
    enc = e.pool_encoder_rows(1, e.pool_step([1], ctc_heads=0)[0]["T"]).clone()
    h1 = e.mt_greedy_incremental(enc, None, 3, 100)
    p1 = e.pool_mt_greedy_incremental([1], [None], [3], [100])[0]
    assert h1 == p1 and len(h1) == 3
    out, n_out, n_one = (I64 * cap)(), (I32 * 1)(), I32(0)
    pf = (I64 * 3)(*h1)
    torch.cuda.synchronize()
    l0 = e.launch_count()
    max_len = cap - 2  # kv_off = 1: the largest max_len that fits is cap - 3
    assert lib.ss_mt_greedy_incremental(h, st, enc.data_ptr(), enc.shape[0], pf, 3, -1, max_len, out, cap, ctypes.byref(n_one)) == SS_ERR_CAPACITY
    assert b"needs %d self-attention entries" % (cap + 1) in lib.ss_last_error(h)
    assert lib.ss_pool_mt_greedy_incremental(h, st, 1, (I32 * 1)(1), pf, (I32 * 1)(3), (I32 * 1)(-1), (I32 * 1)(max_len), out, cap,
                                             n_out) == SS_ERR_CAPACITY
    assert b"max_mt_positions = %d" % cap in lib.ss_last_error(h)
    # a caller token outside [0, tgt_vocab) would index the embedding table out of bounds: SS_ERR_INVALID, also before any launch
    feats = torch.empty(2, cfg.mt_dim, device="cuda")
    for bad in (cfg.tgt_vocab, -1):
        pb = (I64 * 3)(h1[0], h1[1], bad)
        assert lib.ss_mt_greedy_incremental(h, st, enc.data_ptr(), enc.shape[0], pb, 3, 3, 100, out, cap, ctypes.byref(n_one)) == SS_ERR_INVALID
        assert b"outside the vocabulary" in lib.ss_last_error(h)
        assert lib.ss_mt_greedy(h, st, enc.data_ptr(), enc.shape[0], pb, 3, 3, 100, out, cap, ctypes.byref(n_one), None) == SS_ERR_INVALID
        assert b"outside the vocabulary" in lib.ss_last_error(h)
        assert lib.ss_mt_features(h, st, enc.data_ptr(), enc.shape[0], (I64 * 2)(cfg.eos, bad), 2, feats.data_ptr(), None) == SS_ERR_INVALID
        assert b"outside the vocabulary" in lib.ss_last_error(h)
    assert e.launch_count() == l0
    # both states are intact: the largest search that fits continues them and the two agree
    a = e.mt_greedy_incremental(enc, h1, -1, cap - 3)
    b = e.pool_mt_greedy_incremental([1], [h1], [-1], [cap - 3])[0]
    assert a == b and len(a) == cap - 3 and a[:3] == h1
    e.mt_incremental_reset()


@gpu
def test_ss_create_refuses_max_mt_positions_out_of_range():
    from streamspeech_b200.engine import Engine, EngineError

    cfg = ModelConfig()
    for bad in (2, 1 << 20):
        with pytest.raises(EngineError, match="max_mt_positions = %d is outside" % bad):
            Engine(cfg, {}, None, None, max_mt_positions=bad)
