"""Streams of different latencies in one stream pool (ss_pool_set_chunk): every slot runs at its own attention / conv chunk, all
slots share one batched step and ONE pass of the encoder layer stack per step (only the subsampler runs per geometry group).  Each
pooled stream must give what the single-stream agent gives at that stream's latency -- tokens bit-exact at every call, encoder rows
within the fp32 tolerance -- whatever the handle's own chunk setting is."""
import argparse

import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)
gpu = pytest.mark.gpu


def asr_args(seg_ms, sample_rate=16000):
    return argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, sample_rate=sample_rate,
                              max_len=200, force_finish=False, vocoder="synthetic", vocoder_cfg=None, dur_prediction=True, lagging_k1=0,
                              lagging_k2=0, segment_size=seg_ms, stride_n=1, stride_n2=1, unit_per_subword=15, source_segment_size=seg_ms,
                              vocoder_context="receptive-field", device_index=0)


def _alias(ptr, numel):
    """float32 CUDA tensor over existing device memory (test helper)"""
    class _Arr:
        __cuda_array_interface__ = {"shape": (numel,), "typestr": "<f4", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_Arr(), device="cuda")


def _reference(single, chunk, wav, n, heads, rate):
    """one utterance alone through the single-stream ASR path with the handle at `chunk`: tokens per call, final encoder rows"""
    from streamspeech_b200.simuleval_compat import SpeechSegment

    single.engine.set_chunk(*chunk)
    single.reset()
    calls, last_enc = [], None
    for i in range(0, len(wav), n):
        single.push(SpeechSegment(content=wav[i:i + n].tolist(), sample_rate=rate, finished=i + n >= len(wav)))
        feat = single._features()
        if feat.size(0) > 0:
            enc = single._encode(feat)
            if heads == 1:
                calls.append(single._ctc(0, enc)[0])
            else:
                pair = single._ctc_pair(enc)
                calls.append((pair[0][0], pair[1][0]))
            last_enc = enc.clone()
        else:
            calls.append(None)
    return calls, last_enc


def _run_pooled(eng, specs, wavs, heads, rate):
    """all streams in one pool, slot j at specs[j]'s chunk; rounds of 160 ms, stream j pushes its own segment (chunk * 40 ms) on the
    rounds it is due, starting `delay` rounds late.  The handle is the offline model meanwhile: no slot may read it.  Returns the
    pool, slots and the result of every call per stream."""
    from streamspeech_b200.scheduler import StreamPool

    pool = StreamPool(eng, n_slots=8, max_seconds=6, ctc_heads=heads, sample_rate=rate)
    slots = [pool.acquire() for _ in specs]
    for sl, spec in zip(slots, specs):
        pool.set_chunk(sl, *spec["chunk"])
    eng.set_chunk(None)
    pos, got = [0] * len(specs), [[] for _ in specs]
    rnd = 0
    while any(p < len(w) for p, w in zip(pos, wavs)):
        due = []
        for j, s in enumerate(specs):
            every = s["chunk"][0] // 4  # rounds per segment
            if rnd >= s["delay"] and (rnd - s["delay"]) % every == 0 and pos[j] < len(wavs[j]):
                n = rate // 1000 * 40 * s["chunk"][0]
                pool.push(slots[j], wavs[j][pos[j]:pos[j] + n], finished=pos[j] + n >= len(wavs[j]))
                pos[j] += n
                due.append(j)
        if due:
            pool.flush()
        for j in due:
            r = pool.results[slots[j]]
            got[j].append(None if r["T"] == 0 else (r["ctc"][0][0] if heads == 1 else (r["ctc"][0][0], r["ctc"][1][0])))
        rnd += 1
    return pool, slots, got


def _check(eng, slots, got, refs):
    cfg = ModelConfig()
    torch.cuda.synchronize()
    worst = 0.0
    for j, (calls, enc) in enumerate(refs):
        assert got[j] == calls, j  # tokens at every call (None: no encoder rows yet)
        if enc is None:
            continue
        T = enc.shape[0]
        rows = _alias(eng.pool_info(slots[j])["enc_out_ptr"], T * cfg.enc_dim).view(T, cfg.enc_dim).clone()
        worst = max(worst, float((rows - enc).abs().max()))
    assert worst < 2e-4, worst


# (4,4) / (8,8) / (16,16): the agents' 160 / 320 / 640 ms; (12,8) is an explicit setting whose grids do not nest.  Ragged lengths,
# two late joiners, and a 640 ms stream shorter than one of its chunks.
SPECS = [dict(sec=3.1, seed=11, delay=0, chunk=(4, 4)), dict(sec=2.0, seed=12, delay=0, chunk=(8, 8)),
         dict(sec=4.05, seed=13, delay=2, chunk=(16, 16)), dict(sec=0.5, seed=14, delay=1, chunk=(16, 16)),
         dict(sec=2.72, seed=15, delay=0, chunk=(12, 8)), dict(sec=3.3, seed=16, delay=3, chunk=(4, 4))]


@gpu
@pytest.mark.parametrize("heads", [1, 2])
def test_mixed_latencies_equal_single_stream_agent(heads):
    from streamspeech_b200.agent import StreamSpeechASRAgent

    single = StreamSpeechASRAgent(asr_args(160))
    wavs = [synth.make_audio(s["sec"], seed=s["seed"]) for s in SPECS]
    refs = [_reference(single, s["chunk"], w, 16 * 40 * s["chunk"][0], heads, 16000) for s, w in zip(SPECS, wavs)]
    pool, slots, got = _run_pooled(single.engine, SPECS, wavs, heads, 16000)
    assert max(pool.rows_per_step) >= 4  # streams of different latencies really shared steps
    _check(single.engine, slots, got, refs)
    single.engine.close()


@gpu
def test_mixed_latencies_48k_pool_equal_single_48k_agent():
    from streamspeech_b200.agent import StreamSpeechASRAgent

    single = StreamSpeechASRAgent(asr_args(160, 48000))
    specs = [dict(n=148801, seed=31, delay=0, chunk=(4, 4)), dict(n=96002, seed=32, delay=0, chunk=(8, 8)),
             dict(n=130561, seed=33, delay=2, chunk=(8, 8)), dict(n=5000, seed=34, delay=1, chunk=(4, 4))]
    wavs = [synth.make_audio(s["n"] / 48000 + 0.001, seed=s["seed"], sample_rate=48000)[:s["n"]].contiguous() for s in specs]
    refs = [_reference(single, s["chunk"], w, 48 * 40 * s["chunk"][0], 1, 48000) for s, w in zip(specs, wavs)]
    pool, slots, got = _run_pooled(single.engine, specs, wavs, 1, 48000)
    assert max(pool.rows_per_step) >= 3
    _check(single.engine, slots, got, refs)
    single.engine.close()


def _pool_geom_key(F, T_final, half=2):
    T1 = (F - 1) // 2 + 1
    T = (T1 - 1) // 2 + 1
    a0 = min(T_final, T)
    t1_lo = max(0, 2 * a0 - half)
    f_lo = max(0, 2 * t1_lo - half)
    return (a0 == 0, T - a0, T1 - t1_lo, F - f_lo)


@gpu
def test_one_encoder_pass_per_step():
    """A step whose 4 streams fall into 4 subsampler geometry groups (a first step, a second step, a steady step and a short final
    chunk) costs few more launches than a step of 4 streams of one geometry: only the subsampler runs per group."""
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    eng = Engine(cfg, synth.make_model_state_dict(cfg, 0), None, synth.make_gcmvn(cfg))
    eng.set_chunk(4, 4)
    eng.pool_create(8, 4)
    w = synth.make_audio(3.0, seed=7)
    seg = 2560

    def push(slot, n_chunks, last=seg):
        info = eng.pool_info(slot)
        start = info["n_audio"]
        for k in range(n_chunks):
            size = seg if k < n_chunks - 1 else last
            eng.pool_push_audio(slot, w[start:start + size].contiguous())
            start += size

    # history: slots 0-3 (lockstep) and 6, 7 get three chunks in three steps; slot 4 one chunk; slot 5 nothing
    for _ in range(3):
        for sl in (0, 1, 2, 3, 6, 7):
            push(sl, 1)
        eng.pool_step([0, 1, 2, 3, 6, 7], 1)
    push(4, 1)
    eng.pool_step([4], 1)
    # the measured steps: one more chunk everywhere, slot 7 a short final one
    for sl in (0, 1, 2, 3, 4, 5, 6):
        push(sl, 1)
    push(7, 1, last=700)
    keys = {}
    for sl in range(8):
        info = eng.pool_info(sl)
        keys[sl] = _pool_geom_key(eng.num_fbank_frames(info["n_audio"]), info["T_final"])
    assert len({keys[s] for s in (0, 1, 2, 3)}) == 1
    assert len({keys[s] for s in (4, 5, 6, 7)}) == 4
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    eng.pool_step([0, 1, 2, 3], 1)
    l1 = eng.launch_count()
    eng.pool_step([4, 5, 6, 7], 1)
    l2 = eng.launch_count()
    one, four = l1 - l0, l2 - l1
    assert one > 50  # the whole encoder ran
    assert four < 1.5 * one, (one, four)
    eng.close()


@gpu
def test_pooled_agents_with_args_run_at_their_own_latency():
    """PooledASRAgents built with args at 160 and 640 ms share one pool; driven by pushpop_many on their own cadences (a 640 ms agent
    every fourth 160 ms round), each returns the text of a single agent at its latency."""
    from streamspeech_b200.agent import StreamSpeechASRAgent
    from streamspeech_b200.scheduler import PooledASRAgent, StreamPool, pushpop_many
    from streamspeech_b200.simuleval_compat import SpeechSegment

    single = {seg: StreamSpeechASRAgent(asr_args(seg)) for seg in (160, 640)}
    eng = single[160].engine
    pool = StreamPool(eng, n_slots=4, max_seconds=5, ctc_heads=1)
    segs = [160, 640, 160, 640]
    agents = [PooledASRAgent(pool, single[160].dict["source_unigram"], asr_args(s)) for s in segs]
    eng.set_chunk(None)  # the agents' slots carry their own latency
    total = 40960  # 2.56 s: a whole number of 640 ms segments
    wavs = [synth.make_audio(total / 16000, seed=s)[:total] for s in (41, 42, 43, 44)]
    texts = [[] for _ in agents]
    pos = [0] * len(agents)
    rounds = 0
    while any(p < total for p in pos):
        due = [j for j, s in enumerate(segs) if rounds % (s // 160) == 0 and pos[j] < total]
        chunks = []
        for j in due:
            n = 16 * segs[j]
            chunks.append(SpeechSegment(content=wavs[j][pos[j]:pos[j] + n].tolist(), sample_rate=16000, finished=pos[j] + n >= total))
            pos[j] += n
        for j, o in zip(due, pushpop_many([agents[j] for j in due], chunks)):
            texts[j].append("" if o.is_empty else o.content)
        rounds += 1
    assert pool.steps == rounds
    eng.set_chunk(4, 4)  # the 160 ms single agent's own setting again
    for j, w in enumerate(wavs):
        ref_agent, n = single[segs[j]], 16 * segs[j]
        ref_agent.reset()
        ref = []
        for i in range(0, total, n):
            o = ref_agent.pushpop(SpeechSegment(content=w[i:i + n].tolist(), sample_rate=16000, finished=i + n >= total))
            ref.append("" if o.is_empty else o.content)
        assert texts[j] == ref, j
    for a in single.values():
        a.engine.close()


@gpu
def test_pool_set_chunk_errors_reset_and_release():
    from streamspeech_b200.engine import Engine, EngineError
    from streamspeech_b200.scheduler import StreamPool

    cfg = ModelConfig()
    eng = Engine(cfg, synth.make_model_state_dict(cfg, 0), None, synth.make_gcmvn(cfg))
    eng.set_chunk(4, 4)
    pool = StreamPool(eng, n_slots=2, max_seconds=2, ctc_heads=1)
    a, b = pool.acquire(), pool.acquire()
    x = synth.make_audio(1.0, seed=5)  # 98 fbank frames, 25 encoder rows

    def t_final(slot):
        pool.reset(slot)
        pool.push(slot, x)
        pool.flush()
        return pool.results[slot]["T_final"]

    assert t_final(a) == 24  # handle (4, 4): period 4 -> (98 // 16) * 4
    with pytest.raises(EngineError, match="holds samples"):
        pool.set_chunk(a, 8, 8)
    for bad in ((4, 3), (4, -2), (-4, 4), (4, 0), (0, 4)):
        with pytest.raises(EngineError, match="even conv chunk"):
            pool.set_chunk(b, *bad)
    with pytest.raises(EngineError, match="bad pool slot"):
        eng.pool_set_chunk(2, 4, 4)
    pool.set_chunk(b, 16, 16)
    assert t_final(b) == 16  # period 16 -> (98 // 64) * 16
    assert t_final(b) == 16  # the setting survived the reset
    eng.set_chunk(None)  # offline handle: only slots that follow it fail
    with pytest.raises(EngineError, match="needs a chunked model"):
        eng.pool_step([a, b], 1)
    assert t_final(b) == 16
    eng.set_chunk(4, 4)
    pool.release(b)
    b2 = pool.acquire()
    assert b2 == b and t_final(b2) == 24  # released: follows the handle again
    eng.close()


class _RecordingEngine:
    """the Engine calls a StreamPool / PooledASRAgent make, recorded (no device)"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("pool_"):
            raise AttributeError(name)
        return lambda *a: self.calls.append((name,) + a)


@pytest.mark.parametrize("seg_ms,chunk", [(160, (4, 4)), (320, (8, 8)), (640, (16, 16)), (800, (20, 16))])
def test_pooled_agent_binds_its_slot_to_the_segment_size(seg_ms, chunk):
    from streamspeech_b200.scheduler import PooledASRAgent, StreamPool

    eng = _RecordingEngine()
    pool = StreamPool(eng, n_slots=2)
    agent = PooledASRAgent(pool, ["x"], asr_args(seg_ms))
    agent.reset()  # between utterances: the binding is not repeated (it survives pool_reset)
    set_calls = [c for c in eng.calls if c[0] == "pool_set_chunk"]
    assert set_calls == [("pool_set_chunk", agent.slot) + chunk]
    plain = PooledASRAgent(pool, ["x"])
    plain.reset()
    assert [c for c in eng.calls if c[0] == "pool_set_chunk"] == set_calls  # without args: follows the engine's set_chunk
    assert plain.slot != agent.slot
