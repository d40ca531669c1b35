"""48 kHz sources in the multi-stream pool (ss_pool_create_rate): each slot's 16 kHz signal is produced inside the batched step with
the single-stream agents' rule (ss_resample_out_len) and arithmetic (resample_3to1), so a pooled 48 kHz stream must give exactly what
the single-stream 48 kHz agent gives -- tokens bit-exact at every call, encoder rows within the fp32 tolerance, fbank frames
bit-identical to those of a 16 kHz pool fed ss_resample_48k_to_16k's output."""
import argparse

import pytest
import torch

pytestmark = pytest.mark.gpu

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402

torch.set_grad_enabled(False)


def asr_args(seg_ms, sample_rate=48000):
    return argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, sample_rate=sample_rate,
                              max_len=200, force_finish=False, vocoder="synthetic", vocoder_cfg=None, dur_prediction=True, lagging_k1=0,
                              lagging_k2=0, segment_size=seg_ms, stride_n=1, stride_n2=1, unit_per_subword=15, source_segment_size=seg_ms,
                              vocoder_context="receptive-field", device_index=0)


def _alias(ptr, numel):
    """float32 CUDA tensor over existing device memory (test helper)"""
    class _Arr:
        __cuda_array_interface__ = {"shape": (numel,), "typestr": "<f4", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_Arr(), device="cuda")


def _wav48(n, seed):
    """n samples of a 48 kHz test signal (any length, not only whole milliseconds)"""
    return synth.make_audio(n / 48000 + 0.001, seed=seed, sample_rate=48000)[:n].contiguous()


# ragged on purpose: lengths that are not multiples of 3, a late joiner, a stream of fewer than 22 samples (no 16 kHz sample is
# final before it finishes), one that joins late and is shorter than a chunk
SPECS = [(148801, 11, 0), (96002, 12, 0), (194400, 13, 2), (20, 14, 1), (130561, 15, 0), (5000, 16, 3)]


@pytest.mark.parametrize("seg_ms,conv,heads", [(160, 4, 1), (320, 8, 2)])
def test_pool_48k_streams_equal_single_stream_48k_agents(seg_ms, conv, heads):
    from streamspeech_b200.agent import StreamSpeechASRAgent
    from streamspeech_b200.scheduler import StreamPool
    from streamspeech_b200.simuleval_compat import SpeechSegment

    single = StreamSpeechASRAgent(asr_args(seg_ms))
    eng = single.engine
    eng.set_chunk(seg_ms // 40, conv)
    wavs = [_wav48(n, seed) for n, seed, _ in SPECS]
    n = 3 * 16 * seg_ms
    # reference: every utterance alone through the single-stream 48 kHz agent; tokens per call and final encoder rows
    ref_tokens, ref_enc = [], []
    for w in wavs:
        single.reset()
        calls, last_enc = [], None
        for i in range(0, len(w), n):
            single.push(SpeechSegment(content=w[i:i + n].tolist(), sample_rate=48000, finished=i + n >= len(w)))
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
        ref_tokens.append(calls)
        ref_enc.append(last_enc)
    # pooled run: all streams concurrently at 48 kHz, stream j starts `delay` rounds late
    pool = StreamPool(eng, n_slots=8, max_seconds=5, ctc_heads=heads, sample_rate=48000)
    slots = [pool.acquire() for _ in SPECS]
    pos = [0] * len(SPECS)
    call_idx = [0] * len(SPECS)
    rnd = 0
    while any(p < len(w) for p, w in zip(pos, wavs)):
        active = [j for j, (_, _, delay) in enumerate(SPECS) if rnd >= delay and pos[j] < len(wavs[j])]
        for j in active:
            pool.push(slots[j], wavs[j][pos[j]:pos[j] + n], finished=pos[j] + n >= len(wavs[j]))
            pos[j] += n
        pool.flush()
        for j in active:
            r = pool.results[slots[j]]
            want = ref_tokens[j][call_idx[j]]
            if want is None:
                assert r["T"] == 0, (j, call_idx[j])
            elif heads == 1:
                assert r["ctc"][0][0] == want, (j, call_idx[j])
            else:
                assert (r["ctc"][0][0], r["ctc"][1][0]) == want, (j, call_idx[j])
            call_idx[j] += 1
        rnd += 1
    assert call_idx == [len(c) for c in ref_tokens]
    assert max(pool.rows_per_step) >= 4  # streams really were batched
    cfg = ModelConfig()
    worst = 0.0
    torch.cuda.synchronize()
    for j, (length, _, _) in enumerate(SPECS):
        info = eng.pool_info(slots[j])
        assert info["n_audio"] == eng.resample_out_len(length, True)  # the whole 16 kHz signal, ceil(n48 / 3)
        if ref_enc[j] is None:
            assert info["n_feat"] == 0
            continue
        T = ref_enc[j].shape[0]
        got = _alias(info["enc_out_ptr"], T * cfg.enc_dim).view(T, cfg.enc_dim).clone()
        worst = max(worst, float((got - ref_enc[j]).abs().max()))
    assert worst < 2e-4, worst
    eng.close()


def test_pool_48k_fbank_frames_equal_16k_pool_on_resampled_samples():
    """Through fbank: a 16 kHz pool on a second handle, fed at every step (the finishing step included) what ss_resample_48k_to_16k
    produces from the same 48 kHz prefix, holds bit-identical fbank frames -- the same ms_fbank reading bit-identical samples.  The
    48 kHz pool's step costs exactly one launch more (the resampler, for all slots) whenever some slot has new 16 kHz samples."""
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    sd, gcmvn = synth.make_model_state_dict(cfg, 0), synth.make_gcmvn(cfg)
    e48, e16 = Engine(cfg, sd, None, gcmvn), Engine(cfg, sd, None, gcmvn)
    for e in (e48, e16):
        e.set_chunk(4, 4)
    e48.pool_create(4, 3, sample_rate=48000)
    e16.pool_create(4, 3)
    specs = [(90001, 7001, 0), (64000, 7680, 0), (43211, 4999, 2), (17, 7001, 1)]  # 48 kHz length, push size, first round
    wavs = [_wav48(n, 40 + j) for j, (n, _, _) in enumerate(specs)]
    x48 = [w.cuda() for w in wavs]
    out16 = [torch.zeros(e16.resample_out_len(n, True), device="cuda") for n, _, _ in specs]
    pos, done16 = [0] * len(specs), [0] * len(specs)

    def step_both(active, any_new, rnd):
        l0 = e48.launch_count()
        r48 = e48.pool_step(active, 0)
        l1 = e48.launch_count()
        r16 = e16.pool_step(active, 0)
        l2 = e48.launch_count()
        assert (l1 - l0) - (l2 - l1) == int(any_new), rnd
        assert [r["T"] for r in r48] == [r["T"] for r in r16], rnd
        torch.cuda.synchronize()
        for j in active:
            i48, i16 = e48.pool_info(j), e16.pool_info(j)
            assert i48["n_audio"] == i16["n_audio"] == done16[j], (rnd, j)
            assert i48["n_feat"] == i16["n_feat"] == e16.num_fbank_frames(done16[j]), (rnd, j)
            nf = i48["n_feat"] * cfg.feat_dim
            if nf:
                assert torch.equal(_alias(i48["feats_ptr"], nf), _alias(i16["feats_ptr"], nf)), (rnd, j)

    rnd = 0
    while any(p < n for p, (n, _, _) in zip(pos, specs)):
        active = [j for j, (n, _, r0) in enumerate(specs) if rnd >= r0 and pos[j] < n]
        any_new = False
        for j in active:
            n, step, _ = specs[j]
            end = min(pos[j] + step, n)
            fin = end == n
            e48.pool_push_audio(j, wavs[j][pos[j]:end].contiguous())
            if fin:
                e48.pool_finish(j)
            want = e16.resample_out_len(end, fin)
            if want > done16[j]:
                e16.resample_48k_to_16k(x48[j][:end], out16[j], done16[j], want - done16[j])
                e16.pool_push_audio(j, out16[j][done16[j]:want].cpu().contiguous())
                done16[j] = want
                any_new = True
            pos[j] = end
        step_both(active, any_new, rnd)
        rnd += 1
    assert rnd >= 10
    assert done16 == [e16.resample_out_len(n, True) for n, _, _ in specs]
    step_both([0, 1, 2, 3], False, rnd)  # nothing new anywhere: no resample launch, nothing changes
    e48.close()
    e16.close()


def test_pooled_48k_agents_batch_behind_push_pop():
    """pushpop_many with 48 kHz SpeechSegments: the single 48 kHz agent's text, one engine step per round; a 16 kHz segment pushed
    into a 48 kHz pool raises before it touches the stream."""
    from streamspeech_b200.agent import StreamSpeechASRAgent
    from streamspeech_b200.scheduler import PooledASRAgent, StreamPool, pushpop_many
    from streamspeech_b200.simuleval_compat import SpeechSegment

    single = StreamSpeechASRAgent(asr_args(160))
    pool = StreamPool(single.engine, n_slots=4, max_seconds=5, ctc_heads=1, sample_rate=48000)
    agents = [PooledASRAgent(pool, single.dict["source_unigram"]) for _ in range(3)]
    total, n = 115202, 7680  # 2.4 s + 2 samples: the last chunk is short and not a multiple of 3
    wavs = [_wav48(total, s) for s in (21, 22, 23)]
    texts = [[] for _ in agents]
    rounds = 0
    for i in range(0, total, n):
        fin = i + n >= total
        segs = [SpeechSegment(content=w[i:i + n].tolist(), sample_rate=48000, finished=fin) for w in wavs]
        for j, o in enumerate(pushpop_many(agents, segs)):
            texts[j].append("" if o.is_empty else o.content)
        rounds += 1
    assert pool.steps == rounds and all(r == 3 for r in pool.rows_per_step)
    for j, w in enumerate(wavs):
        single.reset()
        ref = []
        for i in range(0, total, n):
            o = single.pushpop(SpeechSegment(content=w[i:i + n].tolist(), sample_rate=48000, finished=i + n >= total))
            ref.append("" if o.is_empty else o.content)
        assert texts[j] == ref, j
    with pytest.raises(ValueError, match="16000 Hz segment"):
        agents[0].push(SpeechSegment(content=[0.0] * 160, sample_rate=16000, finished=False))
    assert agents[0].states.source == []
    single.engine.close()


def test_pool_48k_errors_and_finish_flag():
    """A bad rate, capacity counted in 48 kHz samples, a push after ss_pool_finish, and a reset that clears the flag; on a 16 kHz pool
    ss_pool_finish only sets the flag."""
    from streamspeech_b200.engine import Engine, EngineError

    cfg = ModelConfig()
    sd, gcmvn = synth.make_model_state_dict(cfg, 0), synth.make_gcmvn(cfg)
    e48, e16 = Engine(cfg, sd, None, gcmvn), Engine(cfg, sd, None, gcmvn)
    for e in (e48, e16):
        e.set_chunk(4, 4)
    with pytest.raises(EngineError, match="16000 or 48000"):
        e48.pool_create(2, 1, sample_rate=44100)
    e48.pool_create(2, 1, sample_rate=48000)  # the refused rate left no pool behind
    w = _wav48(49200, 3)
    # capacity in 48 kHz samples: 1 s -> 48000 + 1200 (a 16 kHz count would refuse anything beyond 16400)
    e48.pool_push_audio(0, w[:30000].contiguous())
    with pytest.raises(EngineError, match="capacity"):
        e48.pool_push_audio(0, torch.zeros(19201))
    e48.pool_push_audio(0, w[30000:].contiguous())
    e48.pool_step([0], 0)
    assert e48.pool_info(0)["n_audio"] == e48.resample_out_len(49200, False) == 16393
    e48.pool_finish(0)
    e48.pool_step([0], 0)
    assert e48.pool_info(0)["n_audio"] == 16400  # the tail, ceil(49200 / 3)
    with pytest.raises(EngineError, match="finished"):
        e48.pool_push_audio(0, torch.zeros(10))
    with pytest.raises(EngineError, match="bad pool slot"):
        e48.pool_finish(2)
    e48.pool_reset(0)
    assert e48.pool_info(0)["n_audio"] == 0
    e48.pool_push_audio(0, w[:100].contiguous())  # the reset cleared the flag
    e48.pool_step([0], 0)
    assert e48.pool_info(0)["n_audio"] == e48.resample_out_len(100, False) == 27
    # 16 kHz pool: finishing changes nothing the step computes, pushes still fail until the reset
    e16.pool_create(2, 1)
    x = synth.make_audio(0.5, seed=4)
    e16.pool_push_audio(0, x)
    e16.pool_push_audio(1, x)
    e16.pool_finish(1)
    ra, rb = e16.pool_step([0, 1], 1)
    assert ra == rb and ra["T"] > 0
    assert e16.pool_info(0)["n_audio"] == e16.pool_info(1)["n_audio"] == x.numel()
    with pytest.raises(EngineError, match="finished"):
        e16.pool_push_audio(1, x)
    e16.pool_reset(1)
    e16.pool_push_audio(1, x)
    e48.close()
    e16.close()
