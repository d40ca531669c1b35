"""Simultaneous S2ST streams in one stream pool (PooledS2STAgent): one pool step, one batched MT search (ss_pool_mt_greedy) and one
T2U + unit-decoder call over ragged lengths (ss_t2u_unit_decode_ragged) per flush.  Every pooled stream must give what the single
StreamSpeechS2STAgent gives on that stream alone -- actions, flags, CTC / MT tokens, units and durations identical, waveform within
1e-3 -- and the two new entry points must equal their single-stream counterparts."""
import argparse
import ctypes
import json

import numpy as np
import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)
gpu = pytest.mark.gpu
WAV_TOL = 1e-3
FP_TOL = 2e-4
TRACE_KEYS = ("asr_tokens", "st_tokens", "mt_tokens", "units", "dur")


def report(name, **kw):
    """the measured maxima of a test as one JSON line on stdout (shown with `pytest -s`)"""
    print(json.dumps({"test": name, **kw}))


def s2st_args(seg_ms=320, lagging_k1=0, sample_rate=16000):
    return argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, global_stats=None,
                              tgt_splitter_type="SentencePiece", tgt_splitter_path=None, user_dir="", agent_dir="", max_len=200,
                              force_finish=False, shift_size=10, window_size=25, sample_rate=sample_rate, feature_dim=80, vocoder="synthetic",
                              vocoder_cfg=None, dur_prediction=True, lagging_k1=lagging_k1, lagging_k2=0, segment_size=seg_ms, stride_n=1,
                              stride_n2=1, unit_per_subword=15, extra_output_dir=None, output_asr_translation=False, source_segment_size=seg_ms,
                              vocoder_context="receptive-field", device_index=0, device="gpu")


def configure_single(agent, seg_ms, lagging_k1):
    """the single agent as if built with source_segment_size = seg_ms and this lagging_k1 (agent:207-210, 395-413)"""
    c = seg_ms // 40
    agent.engine.set_chunk(c, 16 if c >= 16 else 8)
    agent.whole_word = seg_ms >= 640
    agent.lagging_k1 = lagging_k1
    agent.reset()


def record(seg, agent):
    """one call's observable output: (is write, SpeechSegment.finished, WriteAction.finished seen through the states, trace, wav)"""
    return (not seg.is_empty, bool(seg.finished), dict((k, agent.trace.get(k)) for k in TRACE_KEYS),
            np.asarray(seg.content if not seg.is_empty else [], dtype=np.float32))


def run_single(agent, wav, seg_ms, rate=16000):
    from streamspeech_b200.simuleval_compat import SpeechSegment

    n = rate // 1000 * seg_ms
    out = []
    for i in range(0, len(wav), n):
        seg = agent.pushpop(SpeechSegment(content=wav[i:i + n].tolist(), sample_rate=rate, finished=i + n >= len(wav)))
        out.append(record(seg, agent))
    return out


def compare(got, ref, tag):
    assert len(got) == len(ref), (tag, len(got), len(ref))
    worst = 0.0
    for ci, (g, r) in enumerate(zip(got, ref)):
        assert g[:3] == r[:3], (tag, ci, g[:3], r[:3])
        assert g[3].shape == r[3].shape, (tag, ci, g[3].shape, r[3].shape)
        if g[3].size:
            worst = max(worst, float(np.abs(g[3] - r[3]).max()))
    return worst


def run_pooled(pool, agents, wavs, specs, rate=16000, between_rounds=None):
    """rounds of 320 ms; agent j pushes its own segment on the rounds it is due (a 640 ms agent every second round), starting
    `delay` rounds late, and optionally a second utterance on the same agent once the first is done.  Returns each agent's calls."""
    from streamspeech_b200.scheduler import pushpop_many
    from streamspeech_b200.simuleval_compat import SpeechSegment

    queues = [list(w) for w in wavs]  # per agent: utterances still to play
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
            n = rate // 1000 * s["seg"]
            fin = pos[j] + n >= len(w)
            segs.append(SpeechSegment(content=w[pos[j]:pos[j] + n].tolist(), sample_rate=rate, finished=fin))
            due.append(j)
            pos[j] += n
            if fin:
                queues[j].pop(0)
                pos[j] = 0
        if due:
            for j, seg in zip(due, pushpop_many([agents[j] for j in due], segs)):
                got[j].append(record(seg, agents[j]))
        if between_rounds is not None:
            between_rounds(rnd)
        rnd += 1
    return got


@pytest.fixture(scope="module")
def single():
    """one single-stream S2ST agent and, on its engine, a 40-slot pool with both CTC heads"""
    from streamspeech_b200.agent import StreamSpeechS2STAgent
    from streamspeech_b200.scheduler import StreamPool

    agent = StreamSpeechS2STAgent(s2st_args(320))
    pool = StreamPool(agent.engine, n_slots=40, max_seconds=11, ctc_heads=2)
    yield agent, pool
    agent.engine.close()


# ragged lengths (one shorter than its 320 ms chunk), two late joiners, 320 / 640 ms (whole-word) mixed, lagging_k1 0 / 2, and one
# agent that plays a second utterance after the first one's reset quirk
SPECS = [dict(sec=[4.0, 2.2], seed=[101, 102], seg=320, k1=0, delay=0), dict(sec=[2.6], seed=[103], seg=320, k1=2, delay=0),
         dict(sec=[0.25], seed=[104], seg=320, k1=0, delay=1), dict(sec=[5.12], seed=[105], seg=640, k1=0, delay=0),
         dict(sec=[3.84], seed=[106], seg=640, k1=2, delay=3), dict(sec=[3.3], seed=[107], seg=320, k1=0, delay=4),
         dict(sec=[4.4], seed=[108], seg=320, k1=2, delay=0)]


@gpu
def test_pooled_s2st_agents_equal_single_agent(single):
    from streamspeech_b200.scheduler import PooledS2STAgent

    agent, pool = single
    wavs = [[synth.make_audio(sec, seed=sd) for sec, sd in zip(s["sec"], s["seed"])] for s in SPECS]
    refs = []
    for s, ws in zip(SPECS, wavs):
        calls = []
        for w in ws:
            configure_single(agent, s["seg"], s["k1"])
            calls += run_single(agent, w, s["seg"])
        refs.append(calls)
    agents = [PooledS2STAgent(pool, agent.dict, s2st_args(s["seg"], s["k1"])) for s in SPECS]
    steps0 = pool.steps
    got = run_pooled(pool, agents, wavs, SPECS)
    assert max(pool.rows_per_step[steps0:]) >= 4  # the streams really shared flushes (640 ms ones every second round)
    worst = max(compare(g, r, j) for j, (g, r) in enumerate(zip(got, refs)))
    writes = sum(c[0] for calls in got for c in calls)
    report("pool_s2st_vs_single", wav_maxdiff=worst, writes=writes, calls=sum(len(c) for c in got))
    assert writes >= 10 and worst < WAV_TOL, (writes, worst)
    for a in agents:
        pool.release(a.slot)


@gpu
def test_single_agent_interleaved_with_pooled_flushes(single):
    """the single agent's MT / unit / vocoder state on the handle survives pooled flushes in between its calls"""
    from streamspeech_b200.scheduler import PooledS2STAgent
    from streamspeech_b200.simuleval_compat import SpeechSegment

    agent, pool = single
    w = synth.make_audio(4.2, seed=201)
    configure_single(agent, 320, 0)
    ref = run_single(agent, w, 320)
    configure_single(agent, 320, 0)
    specs = [dict(seg=320, delay=0), dict(seg=640, delay=0), dict(seg=320, delay=0)]
    others = [PooledS2STAgent(pool, agent.dict, s2st_args(s["seg"])) for s in specs]
    pw = [[synth.make_audio(4.5, seed=202 + j)] for j in range(len(specs))]
    got, n = [], 5120

    def single_call(rnd):
        i = rnd * n
        if i < len(w):
            seg = agent.pushpop(SpeechSegment(content=w[i:i + n].tolist(), sample_rate=16000, finished=i + n >= len(w)))
            got.append(record(seg, agent))

    run_pooled(pool, others, pw, specs, between_rounds=single_call)
    worst = compare(got, ref, "single")
    report("pool_s2st_single_interleaved", wav_maxdiff=worst)
    assert worst < WAV_TOL
    for a in others:
        pool.release(a.slot)


@gpu
def test_pooled_agents_reproduce_reference_policy_fixture(single, gold):
    """the c320 / c640 utterances of the reference's own policy() fixture share one pool with three other streams; each reproduces the
    fixture as test_s2st_agent_vs_reference_policy_fixture checks it, and one more pooled stream equals the oracle agent call by call"""
    from oracle.agent_oracle import OracleS2STAgent
    from oracle.streamspeech_oracle import StreamSpeechOracle
    from streamspeech_b200.dictionary import Dictionary
    from streamspeech_b200.scheduler import PooledS2STAgent

    agent, pool = single
    g = gold["agent_policy"]
    tags = ["c320", "c640"]
    specs = [dict(seg=int(g[f"{t}_segment_ms"]), delay=0) for t in tags]
    wavs = [[synth.make_audio(float(g[f"{t}_seconds"]), seed=int(g[f"{t}_seed"]))] for t in tags]
    specs += [dict(seg=320, delay=1), dict(seg=640, delay=0), dict(seg=320, delay=0)]
    wavs += [[synth.make_audio(3.0, seed=301)], [synth.make_audio(2.56, seed=302)], [synth.make_audio(3.5, seed=303)]]
    agents = [PooledS2STAgent(pool, agent.dict, s2st_args(s["seg"])) for s in specs]
    got = run_pooled(pool, agents, wavs, specs)
    worst, writes = 0.0, 0
    for j, t in enumerate(tags):
        kinds = g[f"{t}_kinds"].tolist()
        assert len(got[j]) == len(kinds), t
        for ci, (is_write, seg_fin, tr, wav) in enumerate(got[j]):
            assert is_write == bool(kinds[ci]), (t, ci)
            if kinds[ci]:
                ref = g[f"{t}_call{ci}_wav"]
                assert len(wav) == len(ref), (t, ci, len(wav), len(ref))
                assert seg_fin == bool(g[f"{t}_call{ci}_flags"][1]), (t, ci)
                if len(ref):
                    assert tr["units"] == g[f"{t}_call{ci}_units"].tolist(), (t, ci)
                    assert tr["dur"] == g[f"{t}_call{ci}_dur"].tolist(), (t, ci)
                    worst = max(worst, float(np.abs(wav - ref).max()))
                    writes += 1
    # stream 2 against the oracle agent (the CPU reference implementation of the policy)
    cfg = ModelConfig()
    o = StreamSpeechOracle(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    d = Dictionary.synthetic(cfg.tgt_vocab)
    oracle = OracleS2STAgent(o, 320, is_word_start=lambda t: d[t].startswith("▁"))
    w, n = wavs[2][0], 5120
    worst_o = 0.0
    for ci, i in enumerate(range(0, len(w), n)):
        oracle.push(w[i:i + n].tolist(), finished=i + n >= len(w))
        a_ref = oracle.policy()
        is_write, seg_fin, tr, wav = got[2][ci]
        assert is_write == (a_ref.kind == "write"), ci
        for k in ("asr_tokens", "st_tokens", "mt_tokens", "units", "dur"):
            assert tr.get(k) == a_ref.trace.get(k), (ci, k)
        if is_write:
            assert len(wav) == len(a_ref.wav) and seg_fin == a_ref.seg_finished, ci
            if len(wav):
                worst_o = max(worst_o, float(np.abs(wav - np.asarray(a_ref.wav, dtype=np.float32)).max()))
    report("pool_s2st_reference_fixture", wav_maxdiff=worst, writes=writes, oracle_wav_maxdiff=worst_o)
    assert writes >= 2 and worst < WAV_TOL and worst_o < WAV_TOL, (writes, worst, worst_o)
    for a in agents:
        pool.release(a.slot)


def _fill(pool, slots, seconds, seed0, steps):
    """push `seconds` of audio to every slot (a new, still open utterance) in `steps` equal pieces, one pool step each; returns the
    slots' encoder rows and T_final"""
    eng = pool.engine
    wavs = [synth.make_audio(seconds, seed=seed0 + j) for j in range(len(slots))]
    for sl in slots:
        pool.reset(sl)
    n = len(wavs[0]) // steps
    for k in range(steps):
        for sl, w in zip(slots, wavs):
            pool.push(sl, w[k * n:(k + 1) * n if k + 1 < steps else len(w)])
        pool.flush()
    return [(pool.results[sl]["T"], pool.results[sl]["T_final"]) for sl in slots]


@gpu
def test_pool_mt_greedy_equals_mt_greedy_per_stream(single):
    """33 streams (two groups: 32 on the batched kernel, 1 on the per-stream path), then 1 stream alone; empty and non-empty prefixes,
    max_new_tokens -1 / 1 / 3, a second call on the slots' cached cross K / V after another step, and fresh slots"""
    agent, pool = single
    eng = pool.engine
    slots = [pool.acquire() for _ in range(33)]
    g = torch.Generator().manual_seed(5)
    worst, checked = 0.0, 0
    for rnd, (steps, seconds) in enumerate([(1, 2.0), (2, 3.2)]):
        for part in range(2 if rnd == 1 else 1):  # round 1 calls again after its second step: rows below T_final come from the cache
            if part == 0:
                rows = _fill(pool, slots, seconds, 400 + 50 * rnd, steps)
            prefixes, limits = [], []
            for j in range(len(slots)):
                k = int(torch.randint(1, 6, (1,), generator=g)) if j % 2 else 0
                prefixes.append(torch.randint(4, eng.cfg.tgt_vocab, (k,), generator=g).tolist() if k else None)
                limits.append([-1, 1, 3][j % 3])
            for sel in (list(range(33)), [7]):
                hyps, feats = eng.pool_mt_greedy([slots[j] for j in sel], [prefixes[j] for j in sel], [limits[j] for j in sel])
                for q, j in enumerate(sel):
                    T, t_final = rows[j]
                    enc = eng.pool_encoder_rows(slots[j], T).clone()
                    for stable in (0, t_final):
                        eng.encoder_stream_reset()
                        ref, ref_f = eng.mt_greedy(enc, prefixes[j], limits[j], max_len_b=100, stable_rows=stable)
                        if stable:  # a second call on the same buffer takes the cached rows below the hint
                            ref, ref_f = eng.mt_greedy(enc, prefixes[j], limits[j], max_len_b=100)
                        assert hyps[q] == ref, (rnd, part, j, hyps[q], ref)
                        d = float((feats[q, :len(ref) + 1] - ref_f).abs().max())
                        worst = max(worst, d)
                        checked += 1
            if part == 0 and rnd == 1:
                for sl in slots:  # one more step on the same utterances before the second call
                    pool.push(sl, synth.make_audio(0.64, seed=sl + 900))
                pool.flush()
                rows = [(pool.results[sl]["T"], pool.results[sl]["T_final"]) for sl in slots]
    report("pool_mt_greedy_vs_mt_greedy", feats_maxdiff=worst, checked=checked)
    assert worst < FP_TOL, worst
    for sl in slots:
        pool.release(sl)


@gpu
def test_t2u_unit_decode_ragged(single):
    agent, pool = single
    eng = pool.engine
    g = torch.Generator().manual_seed(11)
    S = 14
    x = torch.randn(6, S, eng.cfg.mt_dim, generator=g).cuda().contiguous()
    lengths, pads = [14, 7, 3, 14, 1, 9], [0, 1, 0, 2, 0, 1]
    units, am, dev = eng.t2u_unit_decode_ragged(x, lengths, pads)
    R = eng.cfg.ctc_upsample_rate
    for b in range(6):
        r = eng.t2u_unit_decode(x[b, :lengths[b]].contiguous(), n_pad_tail=pads[b])
        assert units[b] == eng.units_to_host(r), b
        assert am[b] == r["argmax"].tolist(), b
        assert len(am[b]) == lengths[b] * R
    # equal lengths: bit-identical to ss_t2u_unit_decode_batch (same positional rows)
    rows = torch.stack([eng.unit_position_row(b) for b in range(6)]).cuda().contiguous()
    ub, amb, devb = eng.t2u_unit_decode_batch(x, pads)
    ur, amr, devr = eng.t2u_unit_decode_ragged(x, [S] * 6, pads, pos_rows=rows)
    assert ub == ur and amb == amr
    assert torch.equal(devb["argmax"], devr["argmax"]) and torch.equal(devb["packed"][:, :1].view(torch.int32)[:, :1], devr["packed"][:, :1].view(torch.int32)[:, :1])  # counts (+ units above)


@gpu
def test_flush_launches_do_not_grow_with_streams(single):
    """the MT search and the T2U + unit-decoder call of 16 writing streams take no more launches than those of 4"""
    agent, pool = single
    eng = pool.engine
    slots = [pool.acquire() for _ in range(16)]
    _fill(pool, slots, 3.0, 500, 1)
    g = torch.Generator().manual_seed(3)
    counts = {}
    for n in (4, 16):
        sel = slots[:n]
        prefixes = [torch.randint(4, eng.cfg.tgt_vocab, (20,), generator=g).tolist() for _ in sel]
        torch.cuda.synchronize()
        l0 = eng.launch_count()
        hyps, feats = eng.pool_mt_greedy(sel, prefixes, [3] * n)
        l1 = eng.launch_count()
        x = feats[:, :24].contiguous()
        eng.t2u_unit_decode_ragged(x, [len(h) + 1 for h in hyps], [0] * n)
        l2 = eng.launch_count()
        counts[n] = (l1 - l0, l2 - l1)
    report("pool_s2st_launches", mt_4=counts[4][0], t2u_4=counts[4][1], mt_16=counts[16][0], t2u_16=counts[16][1])
    assert counts[16][0] <= counts[4][0] and counts[16][1] <= counts[4][1], counts
    for sl in slots:
        pool.release(sl)


@gpu
def test_invalid_arguments(single):
    agent, pool = single
    eng = pool.engine
    lib, h, st = eng.lib, eng._h, eng._stream()
    slots = [pool.acquire() for _ in range(2)]
    _fill(pool, slots[:1], 1.0, 600, 1)
    empty = slots[1]
    I32, I64 = ctypes.c_int32, ctypes.c_int64
    cap, ld = 1024, 128
    out, n_out = (I64 * cap)(), (I32 * 1)()
    feats = torch.empty(ld, eng.cfg.mt_dim, device="cuda")

    def mt(slot=slots[0], prefix=(5, 6), max_new=3, max_len_b=100, null=None):
        sl = (I32 * 1)(slot)
        pf = (I64 * max(len(prefix), 1))(*prefix)
        npf, mn = (I32 * 1)(len(prefix)), (I32 * 1)(max_new)
        a = [h, st, 1, sl, pf, npf, mn, max_len_b, out, cap, n_out, feats.data_ptr(), ld]
        if null is not None:
            a[null] = None
        return lib.ss_pool_mt_greedy(*a)

    assert mt() == 0
    for rc in (mt(slot=99), mt(slot=-1), mt(slot=empty), mt(prefix=(5, 6, 7), max_new=-2), mt(prefix=(5,) * 6, max_new=-1, max_len_b=4),
               mt(prefix=(5, eng.cfg.tgt_vocab)), mt(prefix=(-3,)), mt(null=3), mt(null=4), mt(null=5), mt(null=6), mt(null=8), mt(null=10),
               mt(null=11)):
        assert rc == -1, rc
    two = (I32 * 2)(slots[0], slots[0])
    assert lib.ss_pool_mt_greedy(h, st, 2, two, (I64 * 1)(), (I32 * 2)(0, 0), (I32 * 2)(1, 1), 100, (I64 * 2048)(), cap, (I32 * 2)(),
                                 feats.data_ptr(), 64) == -1  # a slot listed twice
    x = torch.randn(2, 5, eng.cfg.mt_dim, device="cuda")
    rows = eng.unit_position_row(0).cuda().expand(2, -1).contiguous()
    L = 5 * eng.cfg.ctc_upsample_rate
    am, packed = torch.empty(2, L, dtype=torch.int64, device="cuda"), torch.empty(2, L + 1, dtype=torch.int64, device="cuda")

    def t2u(lens=(5, 3), pads=(0, 1), B=2, S=5, null=None):
        a = [h, st, x.data_ptr(), B, S, (I32 * 2)(*lens), (I32 * 2)(*pads), rows.data_ptr(), 0, am.data_ptr(), packed.data_ptr()]
        if null is not None:
            a[null] = None
        return lib.ss_t2u_unit_decode_ragged(*a)

    assert t2u() == 0
    for rc in (t2u(lens=(6, 3)), t2u(lens=(0, 3)), t2u(pads=(0, 3)), t2u(pads=(-1, 0)), t2u(B=0), t2u(S=0), t2u(null=2), t2u(null=6),
               t2u(null=7), t2u(null=9), t2u(null=10)):
        assert rc == -1, rc
    for sl in slots:
        pool.release(sl)


@gpu
def test_pooled_s2st_agents_48k_pool_equal_single_48k_agent():
    from streamspeech_b200.agent import StreamSpeechS2STAgent
    from streamspeech_b200.scheduler import PooledS2STAgent, StreamPool

    agent = StreamSpeechS2STAgent(s2st_args(320, sample_rate=48000))
    pool = StreamPool(agent.engine, n_slots=4, max_seconds=6, ctc_heads=2, sample_rate=48000)
    specs = [dict(sec=[3.0], seed=[701], seg=320, k1=0, delay=0), dict(sec=[2.56], seed=[702], seg=640, k1=0, delay=0),
             dict(sec=[2.2], seed=[703], seg=320, k1=2, delay=1)]
    wavs = [[synth.make_audio(sec, seed=sd, sample_rate=48000) for sec, sd in zip(s["sec"], s["seed"])] for s in specs]
    refs = []
    for s, ws in zip(specs, wavs):
        configure_single(agent, s["seg"], s["k1"])
        refs.append(run_single(agent, ws[0], s["seg"], rate=48000))
    agents = [PooledS2STAgent(pool, agent.dict, s2st_args(s["seg"], s["k1"], sample_rate=48000)) for s in specs]
    got = run_pooled(pool, agents, wavs, specs, rate=48000)
    worst = max(compare(g, r, j) for j, (g, r) in enumerate(zip(got, refs)))
    report("pool_s2st_48k_vs_single", wav_maxdiff=worst)
    assert worst < WAV_TOL, worst
    agent.engine.close()


def test_pooled_s2st_agent_binds_its_slot():
    """without a device: the slot takes the S2ST chunk rule (conv chunk 16 if c >= 16 else 8), and a one-head pool is refused"""
    from streamspeech_b200.scheduler import PooledS2STAgent, StreamPool

    class _Eng:
        cfg = ModelConfig()
        device = torch.device("cpu")

        def __init__(self):
            self.calls = []

        def __getattr__(self, name):
            if not name.startswith("pool_"):
                raise AttributeError(name)
            return lambda *a: self.calls.append((name,) + a)

    for seg, chunk in ((320, (8, 8)), (480, (12, 8)), (640, (16, 16)), (800, (20, 16))):
        eng = _Eng()
        pool = StreamPool(eng, n_slots=2, ctc_heads=2)
        a = PooledS2STAgent(pool, {}, s2st_args(seg))
        assert [c for c in eng.calls if c[0] == "pool_set_chunk"] == [("pool_set_chunk", a.slot) + chunk]
        assert a.whole_word == (seg >= 640) and pool.s2st[a.slot] is a
    with pytest.raises(ValueError, match="ctc_heads=2"):
        PooledS2STAgent(StreamPool(_Eng(), n_slots=1, ctc_heads=1), {}, s2st_args(320))
