"""GPU: the attention and depthwise-conv kernels against a float64 reference of the same operation.

The references are the oracle's own attention / depthwise cores (oracle/streamspeech_oracle.py: rel_attention_core, mha_core,
depthwise_bn_silu_core) run in float64, so they are the arithmetic that the float64-oracle-vs-fixture tests pin
(test_oracle_golden.py).  Every attention case runs on the row kernel (kernel = 1), the tile kernel (kernel = 2) and the engine's
own choice (kernel = 0), which must be bit-identical to the forced kernel the shape rule of kernels_attn.cu picks.

Position rows and keys are random, not the smooth sinusoid, so an off-by-one relative index or key limit moves the result by O(1).
Cases are chosen pairwise over the edges (lengths around the 16-query and 64-key tiles, chunk sizes, windows that start inside a
16-query tile, ragged lengths, the first and last position-table rows) rather than as a full cross product.  Errors are max-abs over
max|V| (attention) or over max|reference| (depthwise conv); the measured maxima are printed as JSON lines (`pytest -s`).
"""
import ctypes
import json

import pytest
import torch

from oracle.streamspeech_oracle import chunk_mask, depthwise_bn_silu_core, mha_core, rel_attention_core

pytestmark = pytest.mark.gpu

torch.set_grad_enabled(False)
F64 = torch.float64
SS_ERR_INVALID = -1
HD = 64

# Bars: error / max|V| (attention), error / max|reference| (depthwise), by score mode ("unit": scores of unit scale; "spread": +-50
# with the maximum in the last 64-key tile; "equal": all scores equal; "dominant": one key 30 above the rest).  Each is about 10x the
# largest error of the row and tile kernels measured on an H100 80GB HBM3 (700 W), given in the comments.
RELPOS_TOL = {"unit": 5e-6, "spread": 1.5e-5, "equal": 2.5e-7, "dominant": 3e-7}  # 9.0e-7, 1.7e-6, 2.7e-8, 3.1e-8
MHA_TOL = {"unit": 3e-6, "spread": 4e-5, "equal": 3e-7, "dominant": 4e-7}  # 3.3e-7, 4.3e-6, 3.4e-8, 4.3e-8
GROUPED_TOL = 2.5e-6  # 2.7e-7
MS_RELPOS_TOL = 3e-6  # 3.5e-7
DW_TOL = 1.5e-6  # 1.7e-7 (single-stream kernel), 1.6e-7 (multi-stream kernel)


def report(name, **kw):
    print(json.dumps({"test": name, **kw}))


@pytest.fixture(scope="module")
def eng():
    from streamspeech_b200 import synth
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig().tiny()
    e = Engine(cfg, synth.make_model_state_dict(cfg, 0), None, None, max_enc_frames=64)
    yield e
    e.close()


def dev(x):
    return x.float().cuda().contiguous()


def rule_kernel(nQ, H, B_choice, T):
    """the row / tile choice of launch_attn (kernels_attn.cu) for kernel = 0"""
    return 1 if ((nQ + 15) // 16) * H * B_choice < 96 and T * 4 <= 160 * 1024 else 2


def rel_err(got, ref, denom):
    return float((got.double().cpu() - ref).abs().max()) / denom


# ------------------------------------------------------------------------------------------ inputs
def attn_inputs(g, B, Tq, Tk, H, mode, relpos=False, scale=0.125):
    """q [B,Tq,H,64], k / v [B,Tk,H,64] (+ bias_u / bias_v [H,64], position rows drawn by the caller) in float64 (fp32-representable).
    mode: "unit" (scores of unit scale), "spread" (scores rising from -50 to +50 with the key index, so the maximum of every query is
    its last visible key, in its last 64-key tile), "equal" (every score equal), "dominant" (one key 30 above the rest)."""
    D = H * HD
    v = torch.randn(B, Tk, H, HD, generator=g, dtype=F64)
    if mode == "unit":
        q = torch.randn(B, Tq, H, HD, generator=g, dtype=F64)
        k = torch.randn(B, Tk, H, HD, generator=g, dtype=F64)
    else:
        u = torch.randn(H, HD, generator=g, dtype=F64)
        u = u / u.norm(dim=-1, keepdim=True)
        q = (u / scale).expand(B, Tq, H, HD).clone()
        if mode == "spread":
            s = torch.linspace(-50.0, 50.0, Tk, dtype=F64) if Tk > 1 else torch.tensor([50.0], dtype=F64)
            k = s.view(1, Tk, 1, 1) * u + 0.02 * torch.randn(B, Tk, H, HD, generator=g, dtype=F64)
        elif mode == "equal":
            k = (0.5 * u).expand(B, Tk, H, HD).clone()
        else:
            k = 0.02 * torch.randn(B, Tk, H, HD, generator=g, dtype=F64)
            k[:, (Tk * 2) // 3] = 30.0 * u
    bias = [torch.randn(H, HD, generator=g, dtype=F64) * (1.0 if mode == "unit" else 0.0) for _ in range(2)] if relpos else None
    r = lambda t: t.float().double()  # the kernels see the fp32 values
    return r(q), r(k), r(v), ([r(b) for b in bias] if relpos else None)


# ------------------------------------------------------------------------------------------ rel-pos attention
REL_T = [1, 15, 16, 17, 63, 64, 65, 79, 80, 129, 383, 384, 1000, 1024]
REL_CHUNK = [0, 1, 2, 4, 8, 12, 16, 24, 40, 64, 65, -1]  # -1: a chunk >= T


def relpos_cases():
    """(T, chunk, Tpos, B, lengths, q_offset, nQ, mode): every T twice (two chunks, both table sizes, B = 1 and 3), streaming
    windows that start at the open chunk group with nQ in {1, 15, 16, 17, 400}, and the score stress cases on both kernels."""
    cases = []
    for i, T in enumerate(REL_T):
        for j in range(2):
            chunk = REL_CHUNK[(i + 5 * j) % len(REL_CHUNK)]
            chunk = T + 3 if chunk == -1 else chunk
            Tpos = 1024 if (i + j) % 2 == 0 else T
            B = 3 if j == 1 and T <= 400 else 1
            lengths = None if B == 1 else [T, 1, max(1, min(17, T)) if i % 2 == 0 else max(1, T - 1)]
            cases.append((T, chunk, Tpos, B, lengths, 0, T, "unit"))
    # windows: q_offset = start of the open chunk group (not a multiple of 16), nQ queries from there
    for T, chunk, q_offset, nQ, Tpos, B in ((383, 12, 360, 17, 1024, 1), (129, 8, 120, 1, 129, 3), (80, 4, 52, 15, 1024, 1),
                                             (1000, 40, 600, 400, 1000, 1), (1024, 24, 600, 16, 1024, 3), (384, 64, 320, 17, 384, 1),
                                             (65, 65, 0, 17, 65, 1), (1024, 65, 390, 400, 1024, 1), (17, 1, 5, 1, 1024, 1),
                                             (1000, 2, 998, 1, 1024, 3)):
        lengths = None if B == 1 else [T, T - 1, 17]
        cases.append((T, chunk, Tpos, B, lengths, q_offset, nQ, "unit"))
    for mode in ("spread", "equal", "dominant"):
        cases.append((1000, 0, 1000, 1, None, 0, 1000, mode))
        cases.append((383, 12, 1024, 1, None, 360, 17, mode))
        cases.append((129, 64, 129, 3, [129, 65, 1], 0, 129, mode))
    return cases


def relpos_reference(q, k, v, pos_rows, bu, bv, T, Tpos, chunk, lengths):
    """rel_attention_core over all T queries.  pos_rows [2*Tpos-1, D] is in the kernels' order (row r + Tpos - 1 holds relative
    position r, the engine's flipped copy of the reference table), the core takes the reference's order (row k holds relative
    position T-1-k): the slice [Tpos - T, Tpos + T - 1), reversed."""
    B, _, H, _ = q.shape
    pp = pos_rows[Tpos - T:Tpos + T - 1].flip(0).view(1, 2 * T - 1, H, HD).transpose(1, 2)
    mask = chunk_mask(T, chunk) if chunk > 0 else None
    kpm = None if lengths is None else torch.arange(T).unsqueeze(0) >= torch.tensor(lengths).unsqueeze(1)
    return rel_attention_core(q, k.transpose(1, 2), v.transpose(1, 2), pp, bu, bv, mask, kpm)  # [B, T, D]


def test_relpos_attention_vs_fp64(eng):
    g = torch.Generator().manual_seed(1)
    H = 4
    D = H * HD
    worst = {}
    for case in relpos_cases():
        T, chunk, Tpos, B, lengths, q_offset, nQ, mode = case
        q, k, v, (bu, bv) = attn_inputs(g, B, T, T, H, mode, relpos=True)
        pos = torch.randn(2 * Tpos - 1, D, generator=g, dtype=F64).float().double() * (1.0 if mode == "unit" else 0.0)
        ref = relpos_reference(q, k, v, pos, bu, bv, T, Tpos, chunk, lengths)[:, q_offset:q_offset + nQ].reshape(B * nQ, D)
        vmax = float(v.abs().max())
        # fused q | k | v rows (the encoder's layout, row stride 3D) when the queries are all T rows, else a separate query buffer
        if q_offset == 0 and nQ == T:
            qkv = dev(torch.cat([q.reshape(B * T, D), k.reshape(B * T, D), v.reshape(B * T, D)], dim=1))
            qd, kd, vd = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        else:
            qd = dev(q[:, q_offset:q_offset + nQ].reshape(B * nQ, D))
            kv = dev(torch.cat([k.reshape(B * T, D), v.reshape(B * T, D)], dim=1))
            kd, vd = kv[:, :D], kv[:, D:]
        args = (qd, kd, vd, dev(pos), dev(bu.reshape(D)), dev(bv.reshape(D)), B, nQ, q_offset, T, H, chunk, lengths)
        outs = {kn: eng.op_relpos_attention(*args, kernel=kn) for kn in (1, 2, 0)}
        assert torch.equal(outs[0], outs[rule_kernel(nQ, H, B, T)]), case
        tol = RELPOS_TOL[mode]
        for kn in (1, 2):
            e = rel_err(outs[kn], ref, vmax)
            key = f"{'row' if kn == 1 else 'tile'}_{mode}"
            worst[key] = max(worst.get(key, 0.0), e)
            assert e < tol, (case, kn, e)
    report("relpos_attention_fp64", cases=len(relpos_cases()), **worst)


# ------------------------------------------------------------------------------------------ plain multi-head attention
def mha_cases():
    """(B, Tq, Tk, H, layout, causal_offset or None, kv_len, mode).  layout "fused": q | k | v rows of one [B*T][3D] buffer (self-attention,
    Tq == Tk); "cross": separate q rows and k | v rows of one [B*Tk][2D] buffer (cross-attention and the incremental-cache form
    causal_offset = past, Tk = past + Tq)."""
    c = []
    for Tq, Tk in ((1, 1), (2, 2), (16, 16), (17, 17), (64, 64), (65, 65), (175, 175), (176, 176), (1000, 1000)):
        c.append((1, Tq, Tk, 8, "fused", 0, None, "unit"))
    c += [(3, 65, 65, 4, "fused", 0, [65, 1, 64], "unit"), (3, 176, 176, 8, "fused", 0, [176, 175, 1], "unit"),
          (1, 1000, 1000, 4, "fused", None, None, "unit"), (3, 17, 17, 8, "fused", None, [1, 17, 16], "unit")]
    for Tq, Tk in ((1, 3000), (2, 1000), (16, 175), (17, 176), (64, 65), (65, 64), (175, 2), (176, 1), (1000, 17), (3000, 16),
                   (3000, 65)):
        c.append((1, Tq, Tk, 8 if Tq % 2 else 4, "cross", None, None, "unit"))
    c += [(3, 17, 3000, 8, "cross", None, [3000, 1, 1000], "unit"), (3, 176, 65, 4, "cross", None, [65, 64, 1], "unit")]
    # incremental-cache form: past keys already cached, Tq new queries
    for past, Tq in ((0, 1), (1, 1), (15, 1), (63, 2), (64, 16), (111, 65), (999, 1), (2000, 1000), (159, 17)):
        c.append((1, Tq, past + Tq, 8, "cross", past, None, "unit"))
    c.append((3, 17, 176, 8, "cross", 159, [176, 1, 170], "unit"))
    for mode in ("spread", "equal", "dominant"):
        c += [(1, 1000, 1000, 8, "fused", 0, None, mode), (1, 1, 3000, 8, "cross", None, None, mode),
              (3, 65, 130, 4, "cross", 65, [130, 66, 1], mode)]
    return c


def mha_reference(q, k, v, scale, causal_offset, kv_len):
    B, Tq, H, _ = q.shape
    Tk = k.shape[1]
    t = lambda x: x.reshape(B, x.shape[1], H * HD).transpose(0, 1)
    mask = None if causal_offset is None else torch.arange(Tk).unsqueeze(0) > torch.arange(Tq).unsqueeze(1) + causal_offset
    kpm = None if kv_len is None else torch.arange(Tk).unsqueeze(0) >= torch.tensor(kv_len).unsqueeze(1)
    return mha_core(t(q) * scale, t(k), t(v), H, mask, kpm).transpose(0, 1).reshape(B * Tq, H * HD)


def test_mha_attention_vs_fp64(eng):
    g = torch.Generator().manual_seed(2)
    worst = {}
    for case in mha_cases():
        B, Tq, Tk, H, layout, coff, kv_len, mode = case
        D = H * HD
        scale = 0.125
        q, k, v, _ = attn_inputs(g, B, Tq, Tk, H, mode, scale=scale)
        ref = mha_reference(q, k, v, scale, coff, kv_len)
        if layout == "fused":
            qkv = dev(torch.cat([q.reshape(B * Tq, D), k.reshape(B * Tk, D), v.reshape(B * Tk, D)], dim=1))
            qd, kd, vd = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        else:
            qd = dev(q.reshape(B * Tq, D))
            kv = dev(torch.cat([k.reshape(B * Tk, D), v.reshape(B * Tk, D)], dim=1))
            kd, vd = kv[:, :D], kv[:, D:]
        args = (qd, kd, vd, B, Tq, Tk, H, scale, coff is not None, coff or 0, kv_len)
        outs = {kn: eng.op_mha_attention(*args, kernel=kn) for kn in (1, 2, 0)}
        assert torch.equal(outs[0], outs[rule_kernel(Tq, H, 1, Tk)]), case
        tol = MHA_TOL[mode]
        vmax = float(v.abs().max())
        for kn in (1, 2):
            e = rel_err(outs[kn], ref, vmax)
            key = f"{'row' if kn == 1 else 'tile'}_{mode}"
            worst[key] = max(worst.get(key, 0.0), e)
            assert e < tol, (case, kn, e)
    report("mha_attention_fp64", cases=len(mha_cases()), **worst)


# ------------------------------------------------------------------------------------------ grouped causal attention
def grouped_cases():
    """(S, R, kv_len per sample): B = 1 over S x R (S * R <= 3000 rows for the expanded reference) with the valid group count cycling
    through S, 1, S-1, S/2, and one B = 3 case per S"""
    c = []
    for i, S in enumerate((1, 2, 7, 16, 17, 120, 1024)):
        lens = [S, 1, max(1, S - 1), max(1, S // 2)]
        for j, R in enumerate((1, 2, 25)):
            if S * R <= 3000:
                c.append((S, R, [lens[(i + j) % 4]]))
        c.append((S, 25 if S <= 120 else 2, [lens[i % 4], lens[(i + 1) % 4], lens[(i + 2) % 4]]))
    return c


def test_grouped_causal_attention_vs_fp64(eng):
    """the reference is mha_core over the S*R expanded rows (every group's row repeated R times) with the causal mask and key padding over
    the padded groups' copies"""
    g = torch.Generator().manual_seed(3)
    H = 8
    D = H * HD
    scale = 0.125
    worst = 0.0
    for S, R, kv_len in grouped_cases():
        B = len(kv_len)
        q, k, v, _ = attn_inputs(g, B, S, S, H, "unit", scale=scale)
        qkv = dev(torch.cat([q.reshape(B * S, D), k.reshape(B * S, D), v.reshape(B * S, D)], dim=1))
        got = eng.op_grouped_causal_attention(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], B, S, R, H, scale, kv_len).double().cpu()
        L = S * R
        causal = torch.triu(torch.ones(L, L, dtype=torch.bool), 1)
        for b in range(B):
            kpm = (torch.arange(S) >= kv_len[b]).repeat_interleave(R).unsqueeze(0)
            ex = lambda x: x[b].repeat_interleave(R, dim=0).unsqueeze(1)  # [L, 1, H, 64]
            for h in range(H):  # one head at a time: [L, L] scores
                ref = mha_core(ex(q)[:, :, h] * scale, ex(k)[:, :, h], ex(v)[:, :, h], 1, causal, kpm)[:, 0]
                e = float((got[b * L:(b + 1) * L, h * HD:(h + 1) * HD] - ref).abs().max()) / float(v.abs().max())
                worst = max(worst, e)
                assert e < GROUPED_TOL, (S, R, kv_len, b, h, e)
    report("grouped_causal_attention_fp64", cases=len(grouped_cases()), worst=worst)


# ------------------------------------------------------------------------------------------ depthwise conv + BN + SiLU
def depthwise_cases():
    """(T, k, chunk, t0, n)"""
    c = []
    Ts = (1, 7, 8, 9, 100, 1000)
    for i, T in enumerate(Ts):
        for j, kk in enumerate((1, 3, 15, 31)):
            chunk = (0, 8, 16, 12)[(i + j) % 4]
            b = chunk if chunk and chunk < T else T // 2
            t0 = max(0, min(T - 1, (b, b - 1, b + 1, 0)[(i + 2 * j) % 4]))
            n = T - t0 if (i + j) % 2 == 0 else max(1, min(T - t0, 9))
            c.append((T, kk, chunk, t0, n))
    return c


def depthwise_reference(x, w, gamma, beta, chunk):
    """x [B,T,C] float64, w [k,C] -> [B,T,C]; BatchNorm with mean 0 and var + eps = 1, so that its folded scale / shift are gamma / beta"""
    C = x.shape[2]
    y = depthwise_bn_silu_core(x.transpose(1, 2), w.t().unsqueeze(1), torch.zeros(C, dtype=F64), torch.full((C,), 1.0 - 1e-5, dtype=F64),
                               gamma, beta, chunk if chunk > 0 else None)
    return y.transpose(1, 2)


def test_depthwise_bn_silu_vs_fp64(eng):
    g = torch.Generator().manual_seed(4)
    B, C, ldx = 2, 256, 264
    worst = 0.0
    for T, kk, chunk, t0, n in depthwise_cases():
        x = torch.randn(B, T, ldx, generator=g).double()
        w = (torch.randn(kk, C, generator=g) / kk ** 0.5).double()
        gamma, beta = torch.randn(C, generator=g).double(), torch.randn(C, generator=g).double()
        ref = depthwise_reference(x[:, :, :C], w, gamma, beta, chunk)[:, t0:t0 + n].reshape(B * n, C)
        got = eng.op_depthwise_bn_silu(dev(x.reshape(B * T, ldx)), dev(w), dev(gamma), dev(beta), B, T, t0, n, chunk)
        e = rel_err(got, ref, float(ref.abs().max()))
        worst = max(worst, e)
        assert e < DW_TOL, (T, kk, chunk, t0, n, e)
    report("depthwise_bn_silu_fp64", cases=len(depthwise_cases()), worst=worst)


# ------------------------------------------------------------------------------------------ multi-stream kernels
MS_STREAMS = [  # 4 streams with their own slot, chunk, a0 and T; the third has no active rows (rows 91.. would be its next ones)
    dict(slot=3, a0=40, nA=9, T=49, attn_chunk=8, conv_chunk=8, row0=0),
    dict(slot=0, a0=372, nA=17, T=389, attn_chunk=12, conv_chunk=12, row0=9),
    dict(slot=2, a0=77, nA=0, T=77, attn_chunk=16, conv_chunk=16, row0=91),
    dict(slot=1, a0=0, nA=65, T=65, attn_chunk=40, conv_chunk=0, row0=26),
]
SENTINEL = 12345.0


def test_multistream_kernels_vs_fp64(eng):
    """ms_relpos_attn_kernel / ms_depthwise_kernel with per-stream chunk sizes and slot strides in one launch; rows of no stream (and
    the stream with nA = 0 owns none) keep their sentinel"""
    g = torch.Generator().manual_seed(5)
    H, n_slots, cap, Tpos = 4, 4, 400, 512
    D = H * HD
    rows = 91 + 65
    kc = torch.randn(n_slots, cap, D, generator=g).double()
    vc = torch.randn(n_slots, cap, D, generator=g).double()
    qf = torch.randn(n_slots, cap, D, generator=g).double()  # the queries of every position a stream could have
    pos = torch.randn(2 * Tpos - 1, D, generator=g).double()
    bu, bv = torch.randn(H, HD, generator=g).double(), torch.randn(H, HD, generator=g).double()
    q = torch.zeros(rows, D, dtype=F64)
    for s in MS_STREAMS:
        q[s["row0"]:s["row0"] + s["nA"]] = qf[s["slot"], s["a0"]:s["a0"] + s["nA"]]
    out = torch.full((rows, D), SENTINEL, device="cuda")
    eng.op_ms_relpos_attention(dev(q), dev(kc), dev(vc), dev(pos), dev(bu.reshape(D)), dev(bv.reshape(D)), out, H, MS_STREAMS)
    C, kk = 256, 31
    xc = torch.randn(n_slots, cap, C, generator=g).double()
    w = (torch.randn(kk, C, generator=g) / kk ** 0.5).double()
    gamma, beta = torch.randn(C, generator=g).double(), torch.randn(C, generator=g).double()
    y = torch.full((rows, C), SENTINEL, device="cuda")
    eng.op_ms_depthwise(dev(xc), dev(w), dev(gamma), dev(beta), y, MS_STREAMS)
    out, y = out.double().cpu(), y.double().cpu()
    owned = torch.zeros(rows, dtype=torch.bool)
    worst_a = worst_d = 0.0
    for s in MS_STREAMS:
        sl, a0, nA, T, r0 = s["slot"], s["a0"], s["nA"], s["T"], s["row0"]
        owned[r0:r0 + nA] = True
        if nA == 0:
            continue
        ra = relpos_reference(qf[sl, :T].view(1, T, H, HD), kc[sl, :T].view(1, T, H, HD), vc[sl, :T].view(1, T, H, HD), pos, bu, bv, T,
                              Tpos, s["attn_chunk"], None)[0, a0:a0 + nA]
        ea = float((out[r0:r0 + nA] - ra).abs().max()) / float(vc[sl, :T].abs().max())
        rd = depthwise_reference(xc[sl, :T].unsqueeze(0), w, gamma, beta, s["conv_chunk"])[0, a0:a0 + nA]
        ed = float((y[r0:r0 + nA] - rd).abs().max()) / float(rd.abs().max())
        worst_a, worst_d = max(worst_a, ea), max(worst_d, ed)
        assert ea < MS_RELPOS_TOL and ed < DW_TOL, (s, ea, ed)
    assert bool((out[~owned] == SENTINEL).all()) and bool((y[~owned] == SENTINEL).all())
    report("multistream_fp64", relpos=worst_a, depthwise=worst_d)


# ------------------------------------------------------------------------------------------ argument checks
def test_op_hooks_reject_bad_arguments(eng):
    """every hook returns SS_ERR_INVALID for a shape its kernels do not take, before launching anything; the handle stays usable"""
    lib, h, st = eng.lib, eng._h, eng._stream()
    H, D, T = 4, 256, 64
    buf = torch.zeros(4 * T, 3 * D, device="cuda")  # inputs of the accepted calls (which stay inside it)
    outbuf = torch.zeros(4 * T, 3 * D, device="cuda")
    p, o = buf.data_ptr(), outbuf.data_ptr()
    i32 = lambda *xs: (ctypes.c_int32 * len(xs))(*xs)

    def relpos(Tpos=T, nQ=T, q_offset=0, T_=T, D_=D, lengths=None, kernel=0, ldq=3 * D, chunk=8, B=1):
        return lib.ss_op_relpos_attention(h, st, p, ldq, p, 3 * D, p, 3 * D, p, Tpos, p, p, o, B, nQ, q_offset, T_, H, D_, chunk, lengths, kernel)

    assert relpos() == 0
    for bad in (dict(Tpos=T - 1), dict(q_offset=1), dict(nQ=0), dict(D_=D + 64), dict(lengths=i32(0)), dict(lengths=i32(T + 1)),
                dict(B=2, lengths=i32(T, 0)), dict(kernel=3), dict(kernel=1, T_=40961, Tpos=40961, nQ=1), dict(ldq=D - 4), dict(ldq=D + 2),
                dict(chunk=-1)):
        assert relpos(**bad) == SS_ERR_INVALID, bad

    def mha(Tq=T, Tk=T, kv_len=None, kernel=0, causal=0, coff=0, ldo=D, H_=H):
        return lib.ss_op_mha_attention(h, st, p, 3 * D, p, 3 * D, p, 3 * D, o, ldo, 1, Tq, Tk, H_, ctypes.c_float(0.125), causal, coff, kv_len, kernel)

    assert mha() == 0
    for bad in (dict(Tq=0), dict(Tk=0), dict(kv_len=i32(0)), dict(kv_len=i32(T + 1)), dict(kernel=-1), dict(kernel=1, Tk=40961, Tq=1),
                dict(causal=1, coff=-1), dict(ldo=D - 4), dict(H_=0)):
        assert mha(**bad) == SS_ERR_INVALID, bad

    def grouped(S=T, R=25, kv_len=None, B=1):
        return lib.ss_op_grouped_causal_attention(h, st, p, 3 * D, p, 3 * D, p, 3 * D, o, 3 * D, S, R, H, ctypes.c_float(0.125), B, kv_len)

    assert grouped(S=16, R=2) == 0
    for bad in (dict(S=0), dict(R=0), dict(B=0), dict(kv_len=i32(0)), dict(kv_len=i32(T + 1)), dict(S=12 * 1024 + 1)):
        assert grouped(**bad) == SS_ERR_INVALID, bad

    def dw(T_=T, t0=0, n=T, k=31, chunk=8, ldx=D):
        return lib.ss_op_depthwise_bn_silu(h, st, p, ldx, p, p, p, o, D, 1, T_, t0, n, D, k, chunk)

    assert dw() == 0
    for bad in (dict(t0=1), dict(n=0), dict(t0=-1, n=1), dict(k=4), dict(k=0), dict(chunk=-1), dict(ldx=D - 1)):
        assert dw(**bad) == SS_ERR_INVALID, bad

    def ms(which, slot=0, a0=0, nA=8, T_=8, chunk=8, row0=0, n_slots=2, rows=8, stride=T * D):
        arrs = (i32(slot), i32(a0), i32(nA), i32(T_), i32(chunk), i32(row0))
        if which == "attn":
            return lib.ss_op_ms_relpos_attention(h, st, p, D, p, p, stride, n_slots, p, T, p, p, o, D, rows, H, 1, *arrs)
        return lib.ss_op_ms_depthwise(h, st, p, stride, n_slots, p, p, p, o, D, rows, D, 31, 1, *arrs)

    for which in ("attn", "conv"):
        assert ms(which) == 0
        for bad in (dict(slot=2), dict(slot=-1), dict(nA=9), dict(a0=1), dict(a0=-1), dict(nA=-1), dict(T_=0), dict(row0=1),
                    dict(chunk=-1), dict(T_=T + 1, a0=T, nA=1) if which == "attn" else dict(T_=T * 2, a0=T * 2 - 1, nA=1, stride=T * D)):
            assert ms(which, **bad) == SS_ERR_INVALID, (which, bad)
    # still usable
    x = torch.randn(T * 2, D, device="cuda")
    got = eng.op_depthwise_bn_silu(x, torch.ones(1, D, device="cuda"), torch.ones(D, device="cuda"), torch.zeros(D, device="cuda"), 2, T,
                                   0, T, 0)
    assert torch.allclose(got, torch.nn.functional.silu(x), atol=1e-6)
