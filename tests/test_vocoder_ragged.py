"""The vocoder of n sequences in one call (ss_vocoder_durations_ragged / ss_vocoder_generate_ragged): every sequence must give
what the single-sequence calls give on it alone, bit for bit, in a number of launches that does not grow with n; the pooled S2ST
flush and the offline generator use it."""
import argparse
import ctypes

import numpy as np
import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
TRACE_KEYS = ("asr_tokens", "st_tokens", "mt_tokens", "units", "dur")


def s2st_args(seg_ms=320):
    return argparse.Namespace(model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, global_stats=None,
                              tgt_splitter_type="SentencePiece", tgt_splitter_path=None, user_dir="", agent_dir="", max_len=200,
                              force_finish=False, shift_size=10, window_size=25, sample_rate=16000, feature_dim=80, vocoder="synthetic",
                              vocoder_cfg=None, dur_prediction=True, lagging_k1=0, lagging_k2=0, segment_size=seg_ms, stride_n=1,
                              stride_n2=1, unit_per_subword=15, extra_output_dir=None, output_asr_translation=False, source_segment_size=seg_ms,
                              vocoder_context="receptive-field", device_index=0, device="gpu")


@pytest.fixture(scope="module")
def single():
    """one single-stream S2ST agent (its engine carries the synthetic vocoder) and a 16-slot pool on that engine"""
    from streamspeech_b200.agent import StreamSpeechS2STAgent
    from streamspeech_b200.scheduler import StreamPool

    agent = StreamSpeechS2STAgent(s2st_args(320))
    pool = StreamPool(agent.engine, n_slots=16, max_seconds=8, ctc_heads=2)
    yield agent, pool
    agent.engine.close()


def random_codes(eng, lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, eng.cfg.vocoder.num_embeddings, (U,), generator=g).tolist() for U in lengths]


def singles(eng, codes, dp, args):
    """per sequence: durations, cumsum and the waveform of the single-sequence calls"""
    out = []
    for c, (t, f0, nf, lc) in zip(codes, args):
        dur, cum = eng.vocoder_durations(torch.tensor(c, dtype=torch.long, device="cuda"), dp)
        out.append((dur.tolist(), cum.tolist(), eng.vocoder_generate(t, f0, nf, lc).clone()))
    return out


@pytest.mark.parametrize("dp", [True, False])
def test_durations_equal_single_calls(single, dp):
    eng = single[0].engine
    lengths = [1, 2, 7, 40, 300, 2, 1]  # U = 1, 2 next to long sequences: each one's zero padding at its own end
    codes = random_codes(eng, lengths, 11)
    durs, cums, dev = eng.vocoder_durations_ragged(codes, dp)
    for c, d, cs in zip(codes, durs, cums):
        dur1, cum1 = eng.vocoder_durations(torch.tensor(c, dtype=torch.long, device="cuda"), dp)
        assert d == dur1.tolist() and cs == cum1.tolist()
        if not dp:
            assert d == [1] * len(c)
    assert dev["dur"].numel() == sum(lengths) and dev["cumsum"].numel() == sum(lengths) + len(lengths)
    eng.check_async_error()


def streaming_args(cums, rng, explicit=False):
    """(total, frame0, n_frames, left_context) per sequence: the tail of its frames, some new frames starting inside the receptive
    field, the receptive field (-1) or an explicit context as left context"""
    out = []
    for cs in cums:
        total = cs[-1]
        new = int(rng.integers(1, min(total, 40) + 1))
        out.append((total, total - new, new, int(rng.integers(0, 30)) if explicit else -1))
    return out


def check_generate(eng, codes, args, dp=True):
    eng.vocoder_durations_ragged(codes, dp)
    got = [w.clone() for w in eng.vocoder_generate_ragged(*zip(*args))]
    again = eng.vocoder_generate_ragged(*zip(*args))
    ref = singles(eng, codes, dp, args)
    for s, (g, a, (_, _, w)) in enumerate(zip(got, again, ref)):
        assert g.numel() == args[s][2] * eng.hop
        assert torch.equal(g, w), (s, float((g - w).abs().max()))
        assert torch.equal(g, a), s  # repeated calls: the schedule does not change a sum
    eng.check_async_error()
    return got


def test_generate_bit_identical_mixes(single):
    eng = single[0].engine
    rng = np.random.default_rng(5)
    # one stream
    codes = random_codes(eng, [30], 1)
    _, cums, _ = eng.vocoder_durations_ragged(codes, True)
    check_generate(eng, codes, streaming_args(cums, rng))
    # 32 streaming-shape streams, receptive-field context; short ones start inside the receptive field
    codes = random_codes(eng, rng.integers(2, 60, 32).tolist(), 2)
    _, cums, _ = eng.vocoder_durations_ragged(codes, True)
    check_generate(eng, codes, streaming_args(cums, rng))
    # explicit contexts
    check_generate(eng, codes[:9], streaming_args(cums[:9], rng, explicit=True))
    # frame0 = 0 full passes, and 750-frame streams (one frame per code)
    codes = random_codes(eng, [3, 17, 750, 64, 750], 3)
    _, cums, _ = eng.vocoder_durations_ragged(codes, False)
    check_generate(eng, codes, [(cs[-1], 0, cs[-1], 0) for cs in cums], dp=False)


def test_generate_fallback_and_group_split(single):
    eng = single[0].engine
    rng = np.random.default_rng(6)
    # a stream over the fused kernel's 1024-frame limit among short ones: it takes the multi-launch path
    codes = random_codes(eng, [20, 1100, 8], 4)
    _, cums, _ = eng.vocoder_durations_ragged(codes, False)
    check_generate(eng, codes, [(cums[0][-1], cums[0][-1] - 5, 5, -1), (1100, 0, 1100, 0), (cums[2][-1], 0, cums[2][-1], -1)], dp=False)
    # 40 streams: more than one group (32 streams per generator kernel)
    codes = random_codes(eng, rng.integers(2, 30, 40).tolist(), 5)
    _, cums, _ = eng.vocoder_durations_ragged(codes, True)
    check_generate(eng, codes, streaming_args(cums, rng))
    # 12 offline-shape streams of 750 frames: more frames than one group holds
    codes = random_codes(eng, [750] * 12, 6)
    _, cums, _ = eng.vocoder_durations_ragged(codes, False)
    check_generate(eng, codes, [(750, 0, 750, 0)] * 12, dp=False)


def test_generate_close_to_multi_launch_path(single):
    eng = single[0].engine
    rng = np.random.default_rng(8)
    codes = random_codes(eng, rng.integers(2, 60, 8).tolist(), 7)
    _, cums, _ = eng.vocoder_durations_ragged(codes, True)
    args = streaming_args(cums, rng)
    fused = [w.clone() for w in eng.vocoder_generate_ragged(*zip(*args))]
    try:
        eng.set_option("vocoder_fused", 0)
        multi = eng.vocoder_generate_ragged(*zip(*args))
    finally:
        eng.set_option("vocoder_fused", -1)
    worst = max(float((f - m).abs().max()) for f, m in zip(fused, multi))
    print("ragged fused vs multi-launch max-abs:", worst)
    assert worst <= 1e-4, worst


def test_launches_do_not_grow_with_streams(single):
    eng = single[0].engine
    counts = {}
    for n in (4, 32):
        codes = random_codes(eng, [20 + j % 7 for j in range(n)], 9)
        l0 = eng.launch_count()
        _, cums, _ = eng.vocoder_durations_ragged(codes, True)
        l1 = eng.launch_count()
        args = [(cs[-1], cs[-1] - 10, 10, -1) for cs in cums]
        eng.vocoder_generate_ragged(*zip(*args))  # first use of this shape: tables and packed weights
        l2 = eng.launch_count()
        eng.vocoder_generate_ragged(*zip(*args))
        counts[n] = (l1 - l0, eng.launch_count() - l2)
    print("vocoder launches (durations, generate) by streams:", counts)
    assert counts[32][0] == counts[4][0], counts
    assert counts[4][1] == counts[32][1] == 2, counts  # frame expansion + the generator kernel


def record(seg, agent):
    return (not seg.is_empty, bool(seg.finished), dict((k, agent.trace.get(k)) for k in TRACE_KEYS),
            np.asarray(seg.content if not seg.is_empty else [], dtype=np.float32))


@pytest.mark.parametrize("n", [4, 16])
def test_pooled_flush_one_vocoder_call(single, n):
    """n writing PooledS2STAgents: one durations and one generate call per flush, launches of the vocoder stage independent of n,
    and every call's action, trace and waveform equal to the single agent's, bit for bit"""
    from streamspeech_b200.agent import StreamSpeechS2STAgent
    from streamspeech_b200.scheduler import PooledS2STAgent, pushpop_many
    from streamspeech_b200.simuleval_compat import SpeechSegment

    agent, pool = single
    eng = agent.engine
    wavs = [synth.make_audio(2.4 + 0.3 * (j % 3), seed=700 + j) for j in range(n)]
    step = 16 * 320
    refs = []
    agent.engine.set_chunk(8, 8)
    for w in wavs:
        agent.reset()
        refs.append([record(agent.pushpop(SpeechSegment(content=w[i:i + step].tolist(), sample_rate=16000, finished=i + step >= len(w))), agent)
                     for i in range(0, len(w), step)])
    agents = [PooledS2STAgent(pool, agent.dict, s2st_args(320)) for _ in range(n)]
    stage = []  # per vocoder stage of a flush: (streams, launches, engine vocoder calls)
    vocode = StreamSpeechS2STAgent._vocode
    calls = {"n": 0}
    orig = {k: getattr(eng, k) for k in ("vocoder_durations", "vocoder_generate", "vocoder_durations_ragged", "vocoder_generate_ragged")}

    def counted(f):
        def g(*a, **kw):
            calls["n"] += 1
            return f(*a, **kw)
        return g

    def timed_vocode(e, ags, units):
        c0, l0 = calls["n"], eng.launch_count()
        out = vocode(e, ags, units)
        stage.append((len(ags), eng.launch_count() - l0, calls["n"] - c0))
        return out

    try:
        for k, f in orig.items():
            setattr(eng, k, counted(f))
        StreamSpeechS2STAgent._vocode = staticmethod(timed_vocode)
        got = [[] for _ in agents]
        for i in range(0, max(len(w) for w in wavs), step):
            due = [j for j in range(n) if i < len(wavs[j])]
            segs = [SpeechSegment(content=wavs[j][i:i + step].tolist(), sample_rate=16000, finished=i + step >= len(wavs[j])) for j in due]
            for j, seg in zip(due, pushpop_many([agents[j] for j in due], segs)):
                got[j].append(record(seg, agents[j]))
    finally:
        StreamSpeechS2STAgent._vocode = staticmethod(vocode)
        for k in orig:
            delattr(eng, k)
        for a in agents:
            pool.release(a.slot)
    for j in range(n):
        assert len(got[j]) == len(refs[j])
        for g, r in zip(got[j], refs[j]):
            assert g[:3] == r[:3], j
            assert np.array_equal(g[3], r[3]), j
    multi = [s for s in stage if s[0] > 1]
    assert multi, stage  # some flush vocoded several streams at once
    assert all(c == 2 for _, _, c in stage), stage  # one durations call (one host read) and one generate call (a batch of one: the
    # single-sequence calls)
    assert len({l for _, l, _ in multi}) == 1, stage  # launches independent of the streams vocoded
    assert all(l <= multi[0][1] for _, l, _ in stage), stage
    print(f"pooled vocoder stages at n={n} (streams, launches, calls):", stage)


def test_offline_synthesize_batch_and_waveform_script(single, tmp_path):
    from streamspeech_b200 import generate_waveform_from_code as gw
    from streamspeech_b200.offline import OfflineS2STGenerator

    eng = single[0].engine
    gen = OfflineS2STGenerator.__new__(OfflineS2STGenerator)
    gen.engine = eng
    codes = random_codes(eng, [5, 120, 1, 37, 260], 12)
    batch = gen.synthesize_batch(codes)
    for c, w in zip(codes, batch):
        assert torch.equal(w, gen.synthesize(c))
    # the script's per-group vocoder call against its per-line one, on the engine of a VocoderOnly
    voc = gw.VocoderOnly.__new__(gw.VocoderOnly)
    voc.engine = eng
    lines = random_codes(eng, [9, 31, 4, 70, 1, 18, 50], 13)
    lines[1] = lines[1][:5] + [-1] + lines[1][5:]  # an invalid code the script drops
    path = tmp_path / "units.txt"
    path.write_text("\n".join(" ".join(map(str, l)) for l in lines) + "\n")
    (tmp_path / "cfg.json").write_text("{}")  # (read by main; the engine comes from VocoderOnly below)
    old = gw.LINES_PER_CALL, gw.VocoderOnly
    try:
        gw.LINES_PER_CALL = 3  # groups of 3, 3 and 1 lines
        gw.VocoderOnly = lambda *a, **kw: voc
        ns = argparse.Namespace(cpu=False, vocoder_cfg=str(tmp_path / "cfg.json"), vocoder="synthetic", in_code_file=str(path),
                                results_path=str(tmp_path / "out"), dur_prediction=True, speaker_id=-1)
        assert gw.main(ns) == len(lines)
    finally:
        gw.LINES_PER_CALL, gw.VocoderOnly = old
    for i, line in enumerate(lines):
        ref_dir = tmp_path / "ref"
        ref_dir.mkdir(exist_ok=True)
        gw.write_wav(str(ref_dir / f"{i}.wav"), voc(line, True).cpu().numpy())
        assert (tmp_path / "out" / f"{i}_pred.wav").read_bytes() == (ref_dir / f"{i}.wav").read_bytes(), i


def test_invalid_arguments(single):
    eng = single[0].engine
    lib, h, st = eng.lib, eng._h, eng._stream()
    I32 = ctypes.c_int32
    codes = torch.randint(0, 100, (10,), dtype=torch.int64, device="cuda")
    dur = torch.empty(10, dtype=torch.int64, device="cuda")
    cum = torch.empty(12, dtype=torch.int32, device="cuda")
    wav = torch.empty(64 * eng.hop, device="cuda")

    def durs(n=2, U=(4, 6), null=None):
        a = [h, st, n, codes.data_ptr(), (I32 * 2)(*U), 1, dur.data_ptr(), cum.data_ptr()]
        if null is not None:
            a[null] = None
        return lib.ss_vocoder_durations_ragged(*a)

    def gen(n=2, t=(4, 6), f0=(0, 2), nf=(4, 4), lc=(-1, -1), null=None):
        a = [h, st, n, (I32 * 2)(*t), (I32 * 2)(*f0), (I32 * 2)(*nf), (I32 * 2)(*lc), wav.data_ptr()]
        if null is not None:
            a[null] = None
        return lib.ss_vocoder_generate_ragged(*a)

    for rc in (durs(n=0), durs(n=-1), durs(U=(4, 0)), durs(U=(-2, 6)), durs(null=3), durs(null=4), durs(null=6)):
        assert rc == -1, rc
    assert durs() == 0
    torch.cuda.synchronize()
    cs = cum.tolist()
    T0, T1 = cs[4], cs[-1]
    ok = dict(t=(T0, T1), f0=(0, T1 - 4), nf=(T0, 4))
    assert gen(**ok) == 0
    for rc in (gen(**dict(ok, n=0)), gen(**dict(ok, f0=(1, T1 - 4))), gen(**dict(ok, nf=(T0, 0), f0=(0, T1))), gen(**dict(ok, f0=(-1, T1 - 4))),
               gen(**dict(ok, f0=(0, T1 - 3))), gen(**dict(ok, null=3)), gen(**dict(ok, null=7))):
        assert rc == -1, rc
    assert gen(**dict(ok, n=1)) == -4  # n differs from the durations call's
    eng.check_async_error()
    # an engine without vocoder weights
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig().tiny()
    e2 = Engine(cfg, synth.make_model_state_dict(cfg, 0), None, None)
    try:
        assert e2.lib.ss_vocoder_durations_ragged(e2._h, e2._stream(), 1, codes.data_ptr(), (I32 * 1)(4), 1, dur.data_ptr(), None) == -4
        assert e2.lib.ss_vocoder_generate_ragged(e2._h, e2._stream(), 1, (I32 * 1)(4), (I32 * 1)(0), (I32 * 1)(4), (I32 * 1)(-1),
                                                 wav.data_ptr()) == -4
        e2.check_async_error()
    finally:
        e2.close()
