"""GPU: the vocoder (duration predictor and HiFi-GAN generator) against a float64 reference of the same operation.

The references are the oracle's own `dur_predict` and `hifigan` (oracle/streamspeech_oracle.py) run in float64, the arithmetic that
test_oracle_golden.py::test_vocoder_fixture pins to the reference's fixture.  The vocoder weights are built without weight norm, so
the engine and the oracle start from the same fp32 weights.  The generator's input frames are exact: `dict.weight` rows repeated by
the engine's own integer durations (one frame per code without duration prediction), so a duration near-tie cannot shift frames.
The float64 generator runs as torch / cuDNN float64 convolutions on the GPU (the CPU is too slow for 1000-frame passes); one small
case checks that it agrees with the CPU float64 result.

Every generator case runs on every route of the generator (ROUTES): the fused persistent kernel (`vocoder_fused_kernel`, bf16x3
wgmma), the multi-launch bf16x3 path on three streams and on one, the multi-launch bf16x6 path and the fp32 CUDA-core path.  Frame
counts put each stage's rows (N x 1, 5, 20, 80, 160, 320) on both sides of the 128-row tile.  The fused kernel's tile width is 32
columns in a phase when that phase's 32-column items reach the SM count (`vocoder_fused_fill`).  On a 132-SM H100, N <= 33 runs
16-column tiles in every phase; 52 switches the resblocks of stages 2 and 3 to 32 columns; 127 and 128 every phase from the stage-1
resblocks to the last 32-channel one (stage 3); 129 the stage-0 resblocks too; 750 every phase but conv_pre; and 1025
(vocoder_fused = 1) conv_pre as well.  The 16-channel last stage always runs 16-column tiles.

Errors are max-abs on the waveform.  Every reference is asserted to stay clear of tanh's saturation, which would hide errors.
Cases are chosen pairwise over the edges rather than as a full cross product; the measured maxima are printed as JSON lines
(`pytest -s`) before the bars are asserted, so a failing run still says which route drifted and by how much.
"""
import contextlib
import copy
import json
import time

import numpy as np
import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

pytestmark = pytest.mark.gpu

torch.set_grad_enabled(False)
F64 = torch.float64
MARGIN = 1e-4  # an engine duration may differ from the float64 one only where exp(ld) - 1 lies this close to a k + 0.5 boundary
RF_TOL = 1e-10  # float64 window vs float64 full pass: the same arithmetic on the same frames
SAT, SAT_SHARE = 0.95, 0.01

# route: engine options (all three set, so that a route does not depend on the environment's defaults)
ROUTES = {
    "fused": dict(umma_vocoder=12, vocoder_fused=-1, vocoder_streams=1),
    "fused_forced": dict(umma_vocoder=12, vocoder_fused=1, vocoder_streams=1),
    "multi_bf16x3": dict(umma_vocoder=12, vocoder_fused=0, vocoder_streams=1),
    "multi_bf16x3_1stream": dict(umma_vocoder=12, vocoder_fused=0, vocoder_streams=0),
    "multi_bf16x6": dict(umma_vocoder=13, vocoder_fused=-1, vocoder_streams=1),
    "multi_fp32": dict(umma_vocoder=0, vocoder_fused=-1, vocoder_streams=1),
}
DEFAULTS = ROUTES["fused"]
# Bars: max-abs waveform error against float64, by route.  About 10x the largest error measured on an H100 80GB HBM3 (700 W) over
# every case of this file, given in the comments.  bf16x6 measures only 2x below bf16x3, the fp32 CUDA-core convs 14x.
TOL = {
    "fused": 1e-4,  # 1.08e-5 (twelve 750-frame ragged passes), 9.8e-6 (streaming windows), 9.5e-6 (full passes)
    "fused_forced": 1e-4,  # 9.5e-6 (1025 frames)
    "multi_bf16x3": 1e-4,  # 1.09e-5 (full passes), 8.9e-6 (the 1100-frame fallback inside a fused call)
    "multi_bf16x3_1stream": 1e-4,  # 1.09e-5
    "multi_bf16x6": 6e-5,  # 5.8e-6
    "multi_fp32": 8e-6,  # 7.8e-7
}

FULL_N = [1, 2, 3, 4, 5, 8, 9, 25, 26, 32, 33, 52, 127, 128, 129, 750, 1025]
N_CODES = 1200


def report(name, **kw):
    print(json.dumps({"test": name, **kw}))


class Voc:
    """engine, float64 oracle on the GPU, the fixed code sequence and a cache of float64 full passes over its prefixes"""

    def __init__(self):
        from oracle.streamspeech_oracle import StreamSpeechOracle
        from streamspeech_b200.engine import Engine

        cfg = ModelConfig()
        cfg.enc_layers = 3
        vsd = synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=False)
        self.eng = Engine(cfg, synth.make_model_state_dict(cfg, 0), vsd, None)
        self.oracle_cpu = StreamSpeechOracle(cfg, {}, vsd, None, dtype=F64)
        self.oracle = copy.copy(self.oracle_cpu)
        self.oracle.vsd = {k: v.cuda() for k, v in self.oracle_cpu.vsd.items()}
        self.dict64 = self.oracle.vsd["dict.weight"]
        self.hop = self.eng.hop
        assert self.hop == cfg.vocoder.hop
        self.codes = torch.randint(0, cfg.vocoder.num_embeddings, (N_CODES,), generator=torch.Generator().manual_seed(1)).cuda()
        self._full = {}

    def frames(self, codes, dur=None):
        """float64 generator input [N, 128]: dict rows repeated by the durations (one frame per code without)"""
        x = self.dict64[torch.as_tensor(codes, device="cuda")]
        return x if dur is None else x.repeat_interleave(torch.as_tensor(dur, device="cuda"), dim=0)

    def hifigan(self, frames, oracle=None):
        """float64 waveform [B, N * hop] of frames [B, N, 128] (or [N, 128] -> [N * hop]); the reference is asserted unsaturated"""
        squeeze = frames.dim() == 2
        x = frames.unsqueeze(0) if squeeze else frames
        w = (oracle or self.oracle).hifigan(x.transpose(1, 2).contiguous())[:, 0]
        assert float((w.abs() > SAT).double().mean()) <= SAT_SHARE, "saturated reference: tanh would hide errors"
        return w[0] if squeeze else w

    def full(self, N):
        """float64 full pass over the first N codes, one frame per code"""
        if N not in self._full:
            self._full[N] = self.hifigan(self.frames(self.codes[:N]))
        return self._full[N]

    def one_frame_per_code(self, N):
        """the engine's durations call over the first N codes, no duration prediction: frames = those codes"""
        dur, cum = self.eng.vocoder_durations(self.codes[:N].contiguous(), False)
        assert int(cum[-1].item()) == N

    def generate(self, total, frame0, n, ctx):
        """(waveform, launches) of one vocoder_generate call, after a first call of the same shape (tables and packed weights)"""
        self.eng.vocoder_generate(total, frame0, n, ctx)
        l0 = self.eng.launch_count()
        w = self.eng.vocoder_generate(total, frame0, n, ctx)
        launches = self.eng.launch_count() - l0
        assert w.numel() == n * self.hop
        return w, launches


@pytest.fixture(scope="module")
def voc():
    v = Voc()
    yield v
    v.eng.close()


@contextlib.contextmanager
def route(eng, name):
    try:
        for k, val in ROUTES[name].items():
            eng.set_option(k, val)
        yield
    finally:
        for k, val in DEFAULTS.items():
            eng.set_option(k, val)


def err(got, ref):
    return float((got.double() - ref).abs().max())


def expect_fused(name, N):
    """whether route `name` runs an N-frame window as the fused kernel (2 launches: frame expansion + the kernel)"""
    return name == "fused_forced" or (name == "fused" and N <= 1024)


def check_bars(errs):
    """errs: (case, route, error); asserted after the report"""
    bad = [(c, r, e) for c, r, e in errs if not e < TOL[r]]
    assert not bad, bad[:10]


def worst_by_route(errs, prefix=""):
    """{prefix + route: largest error, prefix + route + "_at": its case}"""
    w = {}
    for c, r, e in errs:
        if e >= w.get(prefix + r, -1.0):
            w[prefix + r], w[prefix + r + "_at"] = e, str(c)
    return w


# ------------------------------------------------------------------------------------------ float64 reference
def test_fp64_reference_on_gpu_matches_cpu(voc):
    """the GPU float64 generator and duration predictor (cuDNN) against the same float64 ops on the CPU"""
    x = voc.frames(voc.codes[:9])
    w_gpu = voc.hifigan(x)
    w_cpu = voc.hifigan(x.cpu(), oracle=voc.oracle_cpu)
    e = float((w_gpu.cpu() - w_cpu).abs().max())
    ld_gpu = voc.oracle.dur_predict(voc.frames(voc.codes[:40]).unsqueeze(0))
    ld_cpu = voc.oracle_cpu.dur_predict(voc.frames(voc.codes[:40]).cpu().unsqueeze(0))
    e_ld = float((ld_gpu.cpu() - ld_cpu).abs().max())
    report("vocoder_fp64_gpu_vs_cpu", wav=e, log_dur=e_ld)
    assert e < 1e-10 and e_ld < 1e-10, (e, e_ld)


# ------------------------------------------------------------------------------------------ 1. durations
DUR_SINGLE = [1, 2, 3, 40, 300]


def fp64_durations(voc, codes):
    """float64 exp(log-duration) - 1 of one sequence alone (zero padding at both of its ends)"""
    ld = voc.oracle.dur_predict(voc.frames(codes).unsqueeze(0))[0]
    return (torch.exp(ld) - 1).cpu()


def check_durations(got, v, label):
    """got: the engine's integer durations of sequence `label`; v: float64 exp(ld) - 1.  Returns (near-ties where they differ, smallest distance of v to
    a k + 0.5 boundary)"""
    want = torch.clamp(torch.round(v).long(), min=1)  # torch.round: half to even, as the reference
    dist = (v - torch.floor(v) - 0.5).abs()
    bad = torch.as_tensor(got, dtype=torch.long) != want
    far = bad & (dist >= MARGIN)
    assert not bool(far.any()), (label, [(int(i), got[int(i)], int(want[int(i)]), float(v[int(i)])) for i in torch.nonzero(far).flatten()[:10]])
    return int(bad.sum()), float(dist.min())


def test_durations_vs_fp64(voc):
    t0 = time.time()
    eng = voc.eng
    g = torch.Generator().manual_seed(2)
    near, closest, units = 0, 1.0, 0
    for U in DUR_SINGLE:  # U = 1, 2, 3: the kernel-3 convs pad at both ends of the sequence
        codes = torch.randint(0, eng.cfg.vocoder.num_embeddings, (U,), generator=g).cuda()
        dur, _ = eng.vocoder_durations(codes, True)
        n, c = check_durations(dur.tolist(), fp64_durations(voc, codes), ("single", U))
        near, closest, units = near + n, min(closest, c), units + U
    # one ragged call of 40 sequences: long ones (2500, 3000 units) among short ones, so that the zero-padded [count, U_max] blocks
    # form several groups and most sequences are padded to a longer one of their block
    rng = np.random.default_rng(3)
    lengths = [1, 2, 3, 40, 300, 2500] + rng.integers(1, 60, 14).tolist() + [3000, 1, 2] + rng.integers(1, 300, 17).tolist()
    assert len(lengths) == 40
    seqs = [torch.randint(0, eng.cfg.vocoder.num_embeddings, (U,), generator=g).cuda() for U in lengths]
    durs, cums, _ = eng.vocoder_durations_ragged(seqs, True)
    near_r = 0
    for s, (c, d, cs) in enumerate(zip(seqs, durs, cums)):
        assert cs == [0] + np.cumsum(d).tolist(), s
        n, cl = check_durations(d, fp64_durations(voc, c), ("ragged", s, len(d)))
        near_r, closest, units = near_r + n, min(closest, cl), units + len(d)
    eng.check_async_error()
    report("vocoder_durations_fp64", units=units, near_ties_single=near, near_ties_ragged=near_r, closest_to_boundary=closest,
           seconds=round(time.time() - t0, 1))


# ------------------------------------------------------------------------------------------ 2. generator full passes
def test_generator_full_pass_vs_fp64(voc):
    """frame0 = 0, context 0: the whole waveform of N frames on every route"""
    t0 = time.time()
    errs = []
    for N in FULL_N:
        ref = voc.full(N)
        voc.one_frame_per_code(N)
        for name in ROUTES:
            if name == "fused_forced" and N <= 1024:
                continue  # the default already runs these as the fused kernel
            with route(voc.eng, name):
                w, launches = voc.generate(N, 0, N, 0)
            assert (launches == 2) == expect_fused(name, N), (N, name, launches)
            errs.append((N, name, err(w, ref)))
    voc.eng.check_async_error()
    report("vocoder_full_pass_fp64", cases=len(errs), seconds=round(time.time() - t0, 1), **worst_by_route(errs))
    check_bars(errs)


# ------------------------------------------------------------------------------------------ 3. streaming windows
# (total, new frames n): receptive-field context; totals are frame counts of FULL_N, so the full passes are shared.  (25, 4) and
# (9, 4) start below the receptive field (context clipped to frame0: the full pass); (52, 28) starts right at it.
RF_WINDOWS = [(129, 1), (128, 4), (52, 28), (750, 156), (25, 4), (9, 4)]
# (total, n, explicit context below the receptive field)
CTX_WINDOWS = [(128, 4, 0), (129, 1, 1), (52, 28, 7), (750, 156, 0), (750, 28, 7), (33, 4, 1)]
WINDOW_ROUTES = ["fused", "multi_bf16x3"]


def test_streaming_windows_vs_fp64(voc):
    """vocoder_generate(total, frame0, n, ctx): with ctx = -1 the last n * hop samples of the float64 full pass; with an explicit ctx
    below the receptive field, the last n * hop samples of the float64 generator over frames [frame0 - ctx, total) alone (the
    zero-padded window the engine computes)"""
    t0 = time.time()
    rf = voc.eng.vocoder_receptive_field
    errs = []
    for total, n in RF_WINDOWS:
        ref = voc.full(total)[-n * voc.hop:]
        voc.one_frame_per_code(total)
        for name in WINDOW_ROUTES:
            with route(voc.eng, name):
                w, launches = voc.generate(total, total - n, n, -1)
            assert (launches == 2) == expect_fused(name, n + min(rf, total - n)), (total, n, name, launches)
            errs.append((("rf", total, n), name, err(w, ref)))
    for total, n, ctx in CTX_WINDOWS:
        f0 = total - n
        ref = voc.hifigan(voc.frames(voc.codes[f0 - ctx:total]))[-n * voc.hop:]
        voc.one_frame_per_code(total)
        for name in WINDOW_ROUTES:
            with route(voc.eng, name):
                w, _ = voc.generate(total, f0, n, ctx)
            errs.append((("ctx", total, n, ctx), name, err(w, ref)))
    voc.eng.check_async_error()
    report("vocoder_windows_fp64", cases=len(errs), receptive_field=rf, seconds=round(time.time() - t0, 1),
           **{kv: e for k in ("rf", "ctx") for kv, e in worst_by_route([x for x in errs if x[0][0] == k], k + "_").items()})
    check_bars(errs)


# ------------------------------------------------------------------------------------------ 4. receptive field (float64 only)
RF_N = 120


def test_receptive_field_fp64(voc):
    """the engine's receptive field (the host formula of engine_weights.cu) as left context: the float64 generator over frames
    [frame0 - rf, total) alone reproduces the float64 full pass's last n * hop samples.  Only the engine's number is read; the rest
    is float64, so the check has no fp32 noise.  The smallest context that still does (the formula's slack) is printed, not
    asserted: measured 18 frames against the formula's 24 (the error one frame below it, 2e-9, is over RF_TOL)."""
    t0 = time.time()
    rf = voc.eng.vocoder_receptive_field
    x = voc.frames(voc.codes[:RF_N])
    full = voc.full(RF_N)
    at_rf, smallest, below = {}, {}, {}
    for n in (1, 4, 28):
        f0 = RF_N - n
        tail = full[-n * voc.hop:]

        def window(c):
            return err(voc.hifigan(x[f0 - c:])[-n * voc.hop:], tail)

        at_rf[n] = window(rf)
        c = rf
        while c > 0 and window(c - 1) < RF_TOL:
            c -= 1
        smallest[n] = c
        below[n] = window(c - 1) if c > 0 else 0.0
    report("vocoder_receptive_field_fp64", receptive_field=rf, error_at_receptive_field=max(at_rf.values()),
           smallest_context=max(smallest.values()), slack=rf - max(smallest.values()), error_one_below_smallest=min(below.values()),
           seconds=round(time.time() - t0, 1))
    assert max(at_rf.values()) < RF_TOL, at_rf


# ------------------------------------------------------------------------------------------ 5. ragged generate
def test_ragged_generate_vs_fp64(voc):
    """vocoder_generate_ragged, every sequence against its own float64 reference"""
    t0 = time.time()
    eng, hop = voc.eng, voc.hop
    errs = []
    # 32 streaming-shape windows with duration prediction (receptive-field context; the short ones start inside it), on the fused
    # kernel and the multi-launch path
    rng = np.random.default_rng(4)
    g = torch.Generator().manual_seed(5)
    seqs = [torch.randint(0, eng.cfg.vocoder.num_embeddings, (U,), generator=g).cuda() for U in rng.integers(2, 20, 32).tolist()]
    durs, cums, _ = eng.vocoder_durations_ragged(seqs, True)
    args = []
    for cs in cums:
        new = int(rng.integers(1, min(cs[-1], 40) + 1))
        args.append((cs[-1], cs[-1] - new, new, -1))
    refs = [voc.hifigan(voc.frames(c, d))[-a[2] * hop:] for c, d, a in zip(seqs, durs, args)]
    for name in WINDOW_ROUTES:
        with route(eng, name):
            got = eng.vocoder_generate_ragged(*zip(*args))
            errs += [(("stream", s), name, err(w, r)) for s, (w, r) in enumerate(zip(got, refs))]
    # an 1100-frame sequence among short ones: it takes the multi-launch path inside a fused call
    eng.vocoder_durations_ragged([voc.codes[:20], voc.codes[:1100], voc.codes[:8]], False)
    args = [(20, 15, 5, -1), (1100, 0, 1100, 0), (8, 0, 8, -1)]
    l0 = eng.launch_count()
    got = eng.vocoder_generate_ragged(*zip(*args))
    assert eng.launch_count() - l0 > 2
    refs = [voc.full(20)[-5 * hop:], voc.full(1100), voc.full(8)]
    errs += [(("mix", s), r, err(w, ref)) for s, (w, ref, r) in enumerate(zip(got, refs, ("fused", "multi_bf16x3", "fused")))]
    # twelve distinct 750-frame sequences: three groups of four (3072 frames per group), one fused launch each
    seqs = [voc.codes[37 * k:37 * k + 750] for k in range(12)]
    eng.vocoder_durations_ragged(seqs, False)
    args = [(750, 0, 750, 0)] * 12
    eng.vocoder_generate_ragged(*zip(*args))  # first use of this shape: tables and packed weights
    l0 = eng.launch_count()
    got = eng.vocoder_generate_ragged(*zip(*args))
    assert eng.launch_count() - l0 == 6, eng.launch_count() - l0  # per group: frame expansion + the generator kernel
    refs = voc.hifigan(torch.stack([voc.frames(c) for c in seqs]))
    errs += [(("offline", s), "fused", err(w, r)) for s, (w, r) in enumerate(zip(got, refs))]
    eng.check_async_error()
    report("vocoder_ragged_fp64", cases=len(errs), seconds=round(time.time() - t0, 1),
           **{kv: e for k in ("stream", "mix", "offline") for kv, e in worst_by_route([x for x in errs if x[0][0] == k], k + "_").items()})
    check_bars(errs)


# ------------------------------------------------------------------------------------------ routing state across handles
def test_op_linear_ignores_routing_left_by_other_handles(voc):
    """ss_op_linear is the plain linear (skinny / fp32 kernels) whatever entry point of whichever handle ran before it on the thread.
    It used to take the tensor-core routing, and its weight cache, that the last handle's entry point had left in thread-local
    state: once this module's engine was closed, op_linear on the next engine read that engine's freed cache and crashed."""
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig().tiny()
    other = Engine(cfg, synth.make_model_state_dict(cfg, 0), None, None)
    g = torch.Generator().manual_seed(6)
    x, w, b = torch.randn(250, 256, generator=g).cuda(), (torch.randn(768, 256, generator=g) / 16).cuda(), torch.randn(768, generator=g).cuda()
    outs = []
    try:
        for umma_linear in (0, 13):
            voc.eng.set_option("umma_linear", umma_linear)
            voc.eng.op_linear_umma(x, w, b)  # an entry point of another handle with the tensor-core routing on or off
            outs.append(other.op_linear(x, w, b))
    finally:
        voc.eng.set_option("umma_linear", 13)
        other.close()
    assert torch.equal(outs[0], outs[1])


def test_t2u_batch_routing_stays_with_its_handle():
    """ss_t2u_unit_decode_batch alternating on one thread between two live handles with different tensor-core routing: each handle's
    units and arg-max equal its run with the other handle absent (a call reads the routing of its own handle only)."""
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig().tiny()
    sd = synth.make_model_state_dict(cfg, 0)
    feats = torch.randn(3, 20, cfg.unit_dim, generator=torch.Generator().manual_seed(6)).cuda()
    pads = [0, 2, 5]
    routes = [dict(umma_linear=13, umma_min_rows=64), dict(umma_linear=0, umma_min_rows=128)]

    def make(r):
        e = Engine(cfg, sd, None, None)
        for k, v in r.items():
            e.set_option(k, v)
        return e

    def decode(e):  # (units, arg-max) per sample: the rows the call writes
        units, argmax, _ = e.t2u_unit_decode_batch(feats, pads)
        return units, argmax

    alone = []
    for r in routes:
        e = make(r)
        try:
            alone.append(decode(e))
        finally:
            e.close()
    engines = [make(r) for r in routes]
    try:
        for _ in range(2):
            for i, e in enumerate(engines):
                assert decode(e) == alone[i], routes[i]
    finally:
        for e in engines:
            e.close()
