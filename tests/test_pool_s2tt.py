"""Simultaneous S2TT streams in one stream pool (PooledS2TTAgent): one pool step and one incremental MT search
(ss_pool_mt_greedy_incremental) per flush, each stream on its slot's own incremental decoder state (SURVEY.md N12).  Every pooled
stream must give what the single StreamSpeechS2TTAgent gives on that stream alone -- actions, text deltas, flags and the CTC / MT
token traces identical -- and the new entry point must equal ss_mt_greedy_incremental call by call, both quirks included."""
import argparse
import ctypes
import json

import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)
gpu = pytest.mark.gpu
TRACE_KEYS = ("asr_tokens", "st_tokens", "mt_tokens")
SS_ERR_INVALID, SS_ERR_STATE, SS_ERR_CAPACITY = -1, -4, -5


def report(name, **kw):
    """the measured maxima of a test as one JSON line on stdout (shown with `pytest -s`)"""
    print(json.dumps({"test": name, **kw}))


def s2tt_args(seg_ms=320, lagging_k1=0, vocoder="synthetic"):
    return argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, global_stats=None,
                              tgt_splitter_type="SentencePiece", tgt_splitter_path=None, user_dir="", agent_dir="", max_len=200,
                              force_finish=False, shift_size=10, window_size=25, sample_rate=16000, feature_dim=80, vocoder=vocoder,
                              vocoder_cfg=None, dur_prediction=True, lagging_k1=lagging_k1, lagging_k2=0, segment_size=seg_ms, stride_n=1,
                              stride_n2=1, unit_per_subword=15, extra_output_dir=None, output_asr_translation=False, source_segment_size=seg_ms,
                              vocoder_context="receptive-field", device_index=0, device="gpu")


def configure_single(agent, seg_ms, lagging_k1):
    """the single agent as if built with source_segment_size = seg_ms and this lagging_k1 (:359-366)"""
    c = seg_ms // 40
    agent.engine.set_chunk(c, min(c, 16))
    agent.lagging_k1 = lagging_k1
    agent.reset()


def record(seg, agent):
    """one call's observable output: (is write, text, finished, trace)"""
    return (not seg.is_empty, seg.content if not seg.is_empty else None, bool(seg.finished), dict((k, agent.trace.get(k)) for k in TRACE_KEYS))


def run_single(agent, wav, seg_ms):
    from streamspeech_b200.simuleval_compat import SpeechSegment

    n = 16 * seg_ms
    return [record(agent.pushpop(SpeechSegment(content=wav[i:i + n].tolist(), sample_rate=16000, finished=i + n >= len(wav))), agent)
            for i in range(0, len(wav), n)]


def run_pooled(agents, wavs, specs, between_rounds=None, record_s2st=None):
    """rounds of 320 ms; agent j pushes its own segment on the rounds it is due (a 640 ms agent every second round), starting `delay`
    rounds late, and a second utterance on the same agent once the first is done.  Returns each agent's calls."""
    from streamspeech_b200.scheduler import pushpop_many
    from streamspeech_b200.simuleval_compat import SpeechSegment

    queues = [list(w) for w in wavs]
    pos = [0] * len(agents)
    got = [[] for _ in agents]
    rnd = 0
    while any(queues):
        due, segs = [], []
        for j, s in enumerate(specs):
            every = s["seg"] // 320
            if not queues[j] or rnd < s["delay"] or (rnd - s["delay"]) % every:
                continue
            w = queues[j][0]
            if pos[j] == 0 and agents[j].states.source_finished:  # the previous utterance ended without the reset quirk
                agents[j].reset()
            n = 16 * s["seg"]
            fin = pos[j] + n >= len(w)
            segs.append(SpeechSegment(content=w[pos[j]:pos[j] + n].tolist(), sample_rate=16000, finished=fin))
            due.append(j)
            pos[j] += n
            if fin:
                queues[j].pop(0)
                pos[j] = 0
        if due:
            for j, seg in zip(due, pushpop_many([agents[j] for j in due], segs)):
                got[j].append((record_s2st if specs[j].get("kind") == "s2st" else record)(seg, agents[j]))
        if between_rounds is not None:
            between_rounds(rnd)
        rnd += 1
    return got


def compare(got, ref, tag):
    assert len(got) == len(ref), (tag, len(got), len(ref))
    for ci, (g, r) in enumerate(zip(got, ref)):
        assert g == r, (tag, ci, g, r)


@pytest.fixture(scope="module")
def single():
    """one single-stream S2TT agent and, on its engine, a 40-slot pool with both CTC heads"""
    from streamspeech_b200.agent import StreamSpeechS2TTAgent
    from streamspeech_b200.scheduler import StreamPool

    agent = StreamSpeechS2TTAgent(s2tt_args(320))
    pool = StreamPool(agent.engine, n_slots=40, max_seconds=9, ctc_heads=2)
    yield agent, pool
    agent.engine.close()


# ragged lengths (one shorter than its 320 ms chunk), late joiners, 320 / 640 ms mixed, lagging_k1 0 / 2, and one agent that plays a
# second utterance after the first one's reset quirk
SPECS = [dict(sec=[4.0, 2.2], seed=[101, 102], seg=320, k1=0, delay=0), dict(sec=[2.6], seed=[103], seg=320, k1=2, delay=0),
         dict(sec=[0.25], seed=[104], seg=320, k1=0, delay=1), dict(sec=[5.12], seed=[105], seg=640, k1=0, delay=0),
         dict(sec=[3.84], seed=[106], seg=640, k1=2, delay=3), dict(sec=[3.3], seed=[107], seg=320, k1=0, delay=4),
         dict(sec=[4.4], seed=[108], seg=320, k1=2, delay=0)]


def single_refs(agent, specs, wavs):
    refs = []
    for s, ws in zip(specs, wavs):
        calls = []
        for w in ws:
            configure_single(agent, s["seg"], s["k1"])
            calls += run_single(agent, w, s["seg"])
        refs.append(calls)
    return refs


@gpu
def test_pooled_s2tt_agents_equal_single_agent(single):
    from streamspeech_b200.scheduler import PooledS2TTAgent

    agent, pool = single
    wavs = [[synth.make_audio(sec, seed=sd) for sec, sd in zip(s["sec"], s["seed"])] for s in SPECS]
    refs = single_refs(agent, SPECS, wavs)
    agents = [PooledS2TTAgent(pool, agent.dict["target_unigram"], s2tt_args(s["seg"], s["k1"])) for s in SPECS]
    steps0 = pool.steps
    got = run_pooled(agents, wavs, SPECS)
    assert max(pool.rows_per_step[steps0:]) >= 4  # the streams really shared flushes
    for j, (g, r) in enumerate(zip(got, refs)):
        compare(g, r, j)
    writes = sum(c[0] for calls in got for c in calls)
    report("pool_s2tt_vs_single", writes=writes, calls=sum(len(c) for c in got))
    assert writes >= 10, writes
    for a in agents:
        pool.release(a.slot)


@gpu
def test_single_s2tt_agent_interleaved_with_pooled_flushes(single):
    """the single agent's incremental MT state on the handle survives pooled S2TT flushes in between its calls"""
    from streamspeech_b200.scheduler import PooledS2TTAgent
    from streamspeech_b200.simuleval_compat import SpeechSegment

    agent, pool = single
    w = synth.make_audio(4.2, seed=201)
    configure_single(agent, 320, 0)
    ref = run_single(agent, w, 320)
    configure_single(agent, 320, 0)
    specs = [dict(seg=320, delay=0), dict(seg=640, delay=0), dict(seg=320, delay=0)]
    others = [PooledS2TTAgent(pool, agent.dict["target_unigram"], s2tt_args(s["seg"])) for s in specs]
    pw = [[synth.make_audio(4.5, seed=202 + j)] for j in range(len(specs))]
    got, n = [], 5120

    def single_call(rnd):
        i = rnd * n
        if i < len(w):
            seg = agent.pushpop(SpeechSegment(content=w[i:i + n].tolist(), sample_rate=16000, finished=i + n >= len(w)))
            got.append(record(seg, agent))

    run_pooled(others, pw, specs, between_rounds=single_call)
    compare(got, ref, "single")
    for a in others:
        pool.release(a.slot)


@gpu
def test_pooled_s2tt_agent_reproduces_reference_policy_fixture(single, gold):
    """the s2tt320 utterance of the reference's own policy() fixture shares one pool with three other streams and reproduces every
    text delta and hypothesis of the fixture"""
    from streamspeech_b200.scheduler import PooledS2TTAgent

    agent, pool = single
    g = gold["agent_policy"]
    tag = "s2tt320"
    specs = [dict(seg=int(g[f"{tag}_segment_ms"]), delay=0), dict(seg=320, delay=1), dict(seg=640, delay=0), dict(seg=320, delay=0)]
    wavs = [[synth.make_audio(float(g[f"{tag}_seconds"]), seed=int(g[f"{tag}_seed"]))], [synth.make_audio(3.0, seed=301)],
            [synth.make_audio(2.56, seed=302)], [synth.make_audio(3.5, seed=303)]]
    agents = [PooledS2TTAgent(pool, agent.dict["target_unigram"], s2tt_args(s["seg"])) for s in specs]
    got = run_pooled(agents, wavs, specs)
    kinds, texts = g[f"{tag}_kinds"].tolist(), g[f"{tag}_texts"].tolist()
    assert len(got[0]) == len(kinds)
    writes = 0
    for ci, (is_write, text, _, tr) in enumerate(got[0]):
        assert is_write == bool(kinds[ci]), ci
        if kinds[ci]:
            assert text == texts[ci], (ci, text, texts[ci])
            assert tr["mt_tokens"] == g[f"{tag}_call{ci}_mt_tokens"].tolist(), ci
            writes += 1
    report("pool_s2tt_reference_fixture", writes=writes)
    assert writes >= 2
    for a in agents:
        pool.release(a.slot)


def _step(pool, slots, wavs, k, n):
    """push piece k (n samples) of every slot's utterance and run one pool step; returns each slot's encoder rows (a copy)"""
    for sl, w in zip(slots, wavs):
        pool.push(sl, w[k * n:(k + 1) * n])
    pool.flush()
    return [pool.engine.pool_encoder_rows(sl, pool.results[sl]["T"]).clone() for sl in slots]


@gpu
def test_pool_mt_greedy_incremental_equals_single_stream_calls(single):
    """34 streams, four calls each with a pool step before every call: 33 in one call (32 on the batched kernel, 1 on the single-token
    path, in reversed order every second call) and 1 alone.  Each stream's call sequence is replayed on the handle after mt_incremental_reset with copies of the slot's
    encoder rows at each call; every call's tokens must be identical, and both quirks of the incremental state must occur."""
    agent, pool = single
    eng = pool.engine
    slots = [pool.acquire() for _ in range(34)]
    group, alone = slots[:33], slots[33:]
    wavs = [synth.make_audio(3.2, seed=400 + j) for j in range(len(slots))]
    g = torch.Generator().manual_seed(7)
    hyp = [None] * len(slots)     # each stream's hypothesis so far: the next call's prefix
    calls = [[] for _ in slots]   # per stream: (encoder rows, prefix, max_new_tokens, max_len, tokens)
    self_len = [0] * len(slots)   # entries of each slot's self-attention cache (the engine's rule)
    cross_rows = [0] * len(slots)
    kv_offs, stale = [], 0
    for k in range(4):
        encs = _step(pool, slots, wavs, k, 8000)
        mnt = [int(torch.randint(1, 4, (1,), generator=g)) if k < 3 else -1 for _ in slots]
        mls = [(len(hyp[j] or []) + 3 + j % 5) for j in range(len(slots))]
        # the group's order alternates, so a stream moves between rows and between the batched and the single-token path
        for sel in (list(range(33)) if k % 2 == 0 else list(range(33))[::-1], [33]):
            out = eng.pool_mt_greedy_incremental([slots[j] for j in sel], [hyp[j] for j in sel], [mnt[j] for j in sel], [mls[j] for j in sel])
            for j, toks in zip(sel, out):
                start = len(hyp[j] or [])
                kv_off = self_len[j] - start
                kv_offs.append(kv_off)
                self_len[j] = len(toks) + kv_off + 1
                if calls[j]:  # an encoder row whose cross K / V were projected by an earlier call changed since
                    rows = calls[j][-1][0]
                    stale += int(not torch.equal(rows[:cross_rows[j]], encs[j][:cross_rows[j]]))
                cross_rows[j] = max(cross_rows[j], encs[j].shape[0])
                calls[j].append((encs[j], hyp[j], mnt[j], mls[j], toks))
                hyp[j] = toks
    checked = 0
    for j in range(len(slots)):
        eng.mt_incremental_reset()
        for ci, (enc, prefix, mn, ml, toks) in enumerate(calls[j]):
            ref = eng.mt_greedy_incremental(enc, prefix, mn, ml)
            assert toks == ref, (j, ci, toks, ref)
            checked += 1
    eng.mt_incremental_reset()
    report("pool_mt_greedy_incremental_vs_single", checked=checked, max_kv_off=max(kv_offs), stale_rows_streams=stale)
    assert max(kv_offs) > 0 and stale > 0, (max(kv_offs), stale)
    for sl in slots:
        pool.release(sl)


@gpu
def test_s2st_and_s2tt_agents_share_one_pool(single):
    """pooled S2ST and S2TT agents in one pool: each equals its own single agent (S2ST: actions, flags, MT tokens, units, durations
    identical and waveforms within 1e-3, as in test_pool_s2st.py)"""
    import numpy as np

    from streamspeech_b200.agent import StreamSpeechS2STAgent
    from streamspeech_b200.scheduler import PooledS2STAgent, PooledS2TTAgent, StreamPool

    agent, _ = single
    s2st = StreamSpeechS2STAgent(s2tt_args(320))
    pool = StreamPool(s2st.engine, n_slots=6, max_seconds=6, ctc_heads=2)
    specs = [dict(sec=[3.0], seed=[501], seg=320, k1=0, delay=0, kind="s2tt"), dict(sec=[2.56], seed=[502], seg=640, k1=0, delay=0, kind="s2st"),
             dict(sec=[3.3], seed=[503], seg=320, k1=2, delay=1, kind="s2tt"), dict(sec=[2.9], seed=[504], seg=320, k1=0, delay=0, kind="s2st")]
    wavs = [[synth.make_audio(sec, seed=sd) for sec, sd in zip(s["sec"], s["seed"])] for s in specs]
    refs = []
    for s, ws in zip(specs, wavs):
        if s["kind"] == "s2tt":
            refs.append(single_refs(agent, [s], [ws])[0])
            continue
        c = s["seg"] // 40
        s2st.engine.set_chunk(c, 16 if c >= 16 else 8)
        s2st.whole_word = s["seg"] >= 640
        s2st.lagging_k1 = s["k1"]
        s2st.reset()
        refs.append(_s2st_calls(s2st, ws[0], s["seg"]))
    agents = [PooledS2TTAgent(pool, agent.dict["target_unigram"], s2tt_args(s["seg"], s["k1"])) if s["kind"] == "s2tt"
              else PooledS2STAgent(pool, s2st.dict, s2tt_args(s["seg"], s["k1"])) for s in specs]
    assert set(pool.s2st) == {a.slot for a in agents if isinstance(a, PooledS2STAgent)}
    got = run_pooled(agents, wavs, specs, record_s2st=_s2st_record)
    worst, writes = 0.0, 0
    for j, s in enumerate(specs):
        assert len(got[j]) == len(refs[j]), j
        for ci, (g, r) in enumerate(zip(got[j], refs[j])):
            if s["kind"] == "s2tt":
                assert g == r, (j, ci, g, r)
                continue
            assert g[:3] == r[:3] and g[3].shape == r[3].shape, (j, ci, g[:3], r[:3])
            if g[3].size:
                worst = max(worst, float(np.abs(g[3] - r[3]).max()))
            writes += g[0]
    report("pool_s2st_s2tt_mixed", s2st_wav_maxdiff=worst, s2st_writes=writes)
    assert writes >= 2 and worst < 1e-3, (writes, worst)
    s2st.engine.close()


def _s2st_record(seg, agent):
    import numpy as np

    return (not seg.is_empty, bool(seg.finished), dict((k, agent.trace.get(k)) for k in ("mt_tokens", "units", "dur")),
            np.asarray(seg.content if not seg.is_empty else [], dtype=np.float32))


def _s2st_calls(agent, wav, seg_ms):
    from streamspeech_b200.simuleval_compat import SpeechSegment

    n = 16 * seg_ms
    return [_s2st_record(agent.pushpop(SpeechSegment(content=wav[i:i + n].tolist(), sample_rate=16000, finished=i + n >= len(wav))), agent)
            for i in range(0, len(wav), n)]


@gpu
def test_incremental_launches_do_not_grow_with_streams(single):
    """the incremental MT call of 16 writing streams takes no more launches than that of 4"""
    agent, pool = single
    eng = pool.engine
    slots = [pool.acquire() for _ in range(16)]
    wavs = [synth.make_audio(3.0, seed=550 + j) for j in range(len(slots))]
    counts = {}
    for n in (4, 16):
        for sl in slots:
            pool.reset(sl)
        _step(pool, slots, wavs, 0, len(wavs[0]))
        torch.cuda.synchronize()
        l0 = eng.launch_count()
        eng.pool_mt_greedy_incremental(slots[:n], [None] * n, [3] * n, [100] * n)
        counts[n] = eng.launch_count() - l0
    report("pool_s2tt_launches", mt_4=counts[4], mt_16=counts[16])
    assert counts[16] <= counts[4], counts
    for sl in slots:
        pool.release(sl)


@gpu
def test_incremental_errors_leave_the_slots_unchanged(single):
    """every error code comes before any launch and leaves the slot's state as it was; the owner rule holds in both directions; after
    ss_pool_reset a second utterance on a slot equals a fresh one"""
    agent, pool = single
    eng = pool.engine
    lib, h, st = eng.lib, eng._h, eng._stream()
    a, b, empty = (pool.acquire() for _ in range(3))
    wa, wb = synth.make_audio(2.0, seed=601), synth.make_audio(2.0, seed=602)
    enc1 = _step(pool, [a, b], [wa, wb], 0, 16000)
    I32, I64 = ctypes.c_int32, ctypes.c_int64
    cap = 1024
    out, n_out = (I64 * cap)(), (I32 * 1)()
    h1 = eng.pool_mt_greedy_incremental([a], [None], [2], [100])[0]

    def inc(slot=a, prefix=tuple(h1), max_new=2, max_len=100, max_out=cap, null=None):
        sl = (I32 * 1)(slot)
        pf = (I64 * max(len(prefix), 1))(*prefix)
        args = [h, st, 1, sl, pf, (I32 * 1)(len(prefix)), (I32 * 1)(max_new), (I32 * 1)(max_len), out, max_out, n_out]
        if null is not None:
            args[null] = None
        return lib.ss_pool_mt_greedy_incremental(*args)

    vocab = eng.cfg.tgt_vocab
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    cases = [(inc(slot=99), SS_ERR_INVALID), (inc(slot=-1), SS_ERR_INVALID), (inc(slot=empty), SS_ERR_INVALID),
             (inc(prefix=tuple(h1) + (vocab,)), SS_ERR_INVALID), (inc(prefix=(-3,) + tuple(h1)[1:]), SS_ERR_INVALID),
             (inc(max_new=-1, max_len=0), SS_ERR_INVALID), (inc(max_new=-1, max_len=len(h1) - 1), SS_ERR_INVALID),
             (inc(max_new=-2 - len(h1)), SS_ERR_INVALID)]
    cases += [(inc(null=k), SS_ERR_INVALID) for k in (3, 4, 5, 6, 7, 8, 10)]
    two = (I32 * 2)(a, a)
    cases.append((lib.ss_pool_mt_greedy_incremental(h, st, 2, two, (I64 * 1)(), (I32 * 2)(0, 0), (I32 * 2)(1, 1), (I32 * 2)(9, 9),
                                                   (I64 * 2048)(), cap, (I32 * 2)()), SS_ERR_INVALID))
    cases.append((inc(prefix=tuple(h1) + (5, 6)), SS_ERR_STATE))  # a prefix longer than the state: kv_off < 0
    cases.append((inc(max_new=-1, max_len=1023), SS_ERR_CAPACITY))
    cases.append((inc(max_out=len(h1) + 1), SS_ERR_CAPACITY))
    eng.set_option("persistent_mt", 0)
    cases.append((inc(), SS_ERR_STATE))
    eng.set_option("persistent_mt", 1)
    assert eng.launch_count() == l0  # nothing was launched
    # the owner rule: a slot of ss_pool_mt_greedy refuses the incremental search and vice versa
    eng.pool_mt_greedy([b], [None], [2])
    torch.cuda.synchronize()
    l1 = eng.launch_count()
    cases.append((inc(slot=b, prefix=()), SS_ERR_STATE))
    feats = torch.empty(128, eng.cfg.mt_dim, device="cuda")
    cases.append((lib.ss_pool_mt_greedy(h, st, 1, (I32 * 1)(a), (I64 * 1)(), (I32 * 1)(0), (I32 * 1)(2), 100, out, cap, n_out,
                                        feats.data_ptr(), 128), SS_ERR_STATE))
    assert eng.launch_count() == l1
    for k, (rc, want) in enumerate(cases):
        assert rc == want, (k, rc, want)
    # the refused calls left slot a as it was: its next call equals the replay of the two valid calls
    enc2 = _step(pool, [a], [wa], 1, 16000)
    h2 = eng.pool_mt_greedy_incremental([a], [h1], [3], [100])[0]
    eng.mt_incremental_reset()
    assert eng.mt_greedy_incremental(enc1[0], None, 2, 100) == h1
    assert eng.mt_greedy_incremental(enc2[0], h1, 3, 100) == h2
    # after ss_pool_reset: a second utterance on both slots equals a fresh one (and slot b now takes the incremental search)
    for sl in (a, b):
        pool.reset(sl)
    enc3 = _step(pool, [a, b], [wb, wa], 0, 16000)
    h3 = eng.pool_mt_greedy_incremental([a, b], [None, None], [3, 3], [100, 100])
    for e, hh in zip(enc3, h3):
        eng.mt_incremental_reset()
        assert eng.mt_greedy_incremental(e, None, 3, 100) == hh
    eng.mt_incremental_reset()
    for sl in (a, b, empty):
        pool.release(sl)


def test_pooled_s2tt_agent_binds_its_slot():
    """without a device: the slot takes the S2TT chunk rule (conv chunk min(c, 16)), and a one-head pool is refused"""
    from streamspeech_b200.scheduler import PooledS2TTAgent, StreamPool

    class _Eng:
        cfg = ModelConfig()
        device = torch.device("cpu")

        def __init__(self):
            self.calls = []

        def __getattr__(self, name):
            if not name.startswith("pool_"):
                raise AttributeError(name)
            return lambda *a: self.calls.append((name,) + a)

    for seg, chunk in ((320, (8, 8)), (480, (12, 12)), (640, (16, 16)), (800, (20, 16))):
        eng = _Eng()
        pool = StreamPool(eng, n_slots=2, ctc_heads=2)
        a = PooledS2TTAgent(pool, {}, s2tt_args(seg))
        assert [c for c in eng.calls if c[0] == "pool_set_chunk"] == [("pool_set_chunk", a.slot) + chunk]
        assert pool.decoders[a.slot] is a and a.slot not in pool.s2st
        assert ("pool_reset", a.slot) in eng.calls  # reset() at construction clears the slot (and its incremental state)
    with pytest.raises(ValueError, match="ctc_heads=2"):
        PooledS2TTAgent(StreamPool(_Eng(), n_slots=1, ctc_heads=1), {}, s2tt_args(320))
