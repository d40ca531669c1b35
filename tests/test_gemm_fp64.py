"""GPU: the GEMM kernel layer (gemm_conv, skinny_gemm, umma2_conv) and layer_norm against a float64 restatement of the launch contract in
kernels.h (ConvA, Epilogue), through the ss_op_gemm / ss_op_layer_norm hooks: every tile shape and template variant, M / N / K tails,
split-K, every epilogue field, the ASR and streaming-encoder conv shapes, the batch-invariance identities the engine relies on, and the
refusals of shapes the kernels cannot take.

Bars.  S = sum_k |a_k w_k| per output element (fp64).  A GEMM output may differ from fp64 by c * sqrt(K) * 2^-24 * S (c per kernel class),
plus 2^-22 of the magnitudes the epilogue adds; the activation's slope (<= 1.13) and GLU's gate (|v| / 4 per unit of gate error) carry
it through.  Every case also asserts that its bar is smaller than the fp64 change from dropping one tap, one input row or one channel,
so a kernel that skips a term cannot pass.  The constants are about 4x the worst ratios measured on an H100 80GB HBM3 (SXM, 700 W);
test_route_coverage prints them per route."""
import math

import pytest
import torch

from streamspeech_b200.engine import EngineError, GemmArgs

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
# c per kernel class: fp32 CUDA-core kernels and umma2 with 3 pieces, umma2 with 2 pieces (bf16x3: ~2^-16 relative per product)
C_FP32 = 6.0      # measured worst 1.6 (gemm_conv 128x64, umma2 NP3)
C_BF16X3 = 75.0   # measured worst 18 (umma2 NP2 BN32)
RATIOS = {}  # route name -> worst err / (sqrt(K) 2^-24 S) seen
ROUTES = set()  # route names exercised


@pytest.fixture(scope="module")
def eng():
    from streamspeech_b200 import synth
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    e = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    yield e
    e.close()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale).cuda()


# ------------------------------------------------------------------------------------------------ the float64 restatement
def im2col(x, c):
    """A [M][ksize * C_in] in fp64 by explicit index: x is [B * x_rows][ldx] (buffer rows of each batch element from logical row x_row0)"""
    B, L_rows, C_in, k = c["B"], c["L_rows"], c["C_in"], c["ksize"]
    xr = c["x_rows"] or c["L_in"]
    t = torch.arange(L_rows, device="cuda").view(1, L_rows, 1) + c["t_offset"]
    tap = torch.arange(k, device="cuda").view(1, 1, k)
    b = torch.arange(B, device="cuda").view(B, 1, 1)
    center = t * c["stride"]
    pos = center + tap * c["dil"] - c["pad_left"]
    ok = (pos >= 0) & (pos < c["L_in"])
    if c["chunk"] > 0:
        ok = ok & (pos < (center // c["chunk"] + 1) * c["chunk"])
    if c.get("lengths") is not None:
        ok = ok & (pos < torch.tensor(c["lengths"], device="cuda").view(B, 1, 1))
    pr = pos - c["x_row0"]
    ok = ok & (pr >= 0) & (pr < xr)
    row = torch.where(ok, b * xr + pr, torch.zeros_like(pr))
    A = x[row.reshape(-1)][:, :C_in].view(B, L_rows, k, C_in) * ok.unsqueeze(-1)
    if c["pre_lrelu"] != 1.0:
        A = torch.where(A > 0, A, A * c["pre_lrelu"])
    return A.reshape(B * L_rows, k * C_in)


def act64(y, act):
    if act == 1:
        return torch.relu(y)
    if act == 2:
        return y * torch.sigmoid(y)
    if act == 3:
        return torch.tanh(y)
    if act == 4:
        return 0.5 * y * (1.0 + torch.erf(y / math.sqrt(2.0)))
    return y


def reference(c, x, w):
    """(values, bars) of every written output element: dict (buffer name, flat index) tensors"""
    A = im2col(x, c)
    if c.get("ln_gamma") is not None:
        mu = A.mean(1, keepdim=True)
        var = ((A - mu) ** 2).mean(1, keepdim=True)
        A = (A - mu) / torch.sqrt(var + 1e-5) * c["ln_gamma"] + c["ln_beta"]
    K = A.shape[1]
    acc = A @ w.T
    S = A.abs() @ w.abs().T
    bias = c.get("bias")
    pre = acc + (bias if bias is not None else 0.0)
    e_pre = c["cls"] * math.sqrt(K) * EPS * S + 2 * EPS * (acc.abs() + (bias.abs() if bias is not None else 0.0))
    if c["glu"]:
        v, gt = pre[:, 0::2], pre[:, 1::2]
        y = v * torch.sigmoid(gt)
        e = e_pre[:, 0::2] * torch.sigmoid(gt) + v.abs() * 0.25 * e_pre[:, 1::2] + 4 * EPS * y.abs()
    else:
        y = act64(pre, c["act"])
        e = 1.13 * e_pre + 4 * EPS * y.abs()
    y = c["alpha"] * y
    e = abs(c["alpha"]) * e
    return A, y, e, S


def out_rows(c):
    M = c["B"] * c["L_rows"]
    m = torch.arange(M, device="cuda")
    if c["out_L"] > 0:
        b, t = m // c["L_rows"], m % c["L_rows"]
        return b * c["out_L"] + t * c["out_row_stride"] + c["out_row_offset"]
    return m


def expected(c, y, e, prev, res):
    """scatter y (and its bar) into the output buffers; prev / res: the buffers' previous contents and the residual buffers"""
    rows = out_rows(c)
    ncols = y.shape[1]
    outs = {}
    split = c["split_n"] or ncols
    for p, name in enumerate(("out", "out2", "out3")):
        lo, hi = p * split, min(ncols, (p + 1) * split)
        if lo >= hi:
            break
        ref = prev[name].clone()
        bar = torch.zeros_like(ref)
        ld = c["ld"][name]
        idx = rows.view(-1, 1) * ld + torch.arange(hi - lo, device="cuda").view(1, -1)
        val, eb = y[:, lo:hi].clone(), e[:, lo:hi].clone()
        if c["residual"]:
            r = res[name].view(-1)[idx]
            val = val + c["res_scale"] * r
            eb = eb + 4 * EPS * (abs(c["res_scale"]) * r.abs() + val.abs())
        if c["accumulate"]:
            q = prev[name].view(-1)[idx]
            val = val + q
            eb = eb + 4 * EPS * (q.abs() + val.abs())
        ref.view(-1)[idx.reshape(-1)] = val.reshape(-1)
        bar.view(-1)[idx.reshape(-1)] = eb.reshape(-1)
        outs[name] = (ref, bar, idx)
    return outs


# ------------------------------------------------------------------------------------------------ one case through ss_op_gemm
BASE = dict(B=1, stride=1, dil=1, pad_left=0, chunk=0, pre_lrelu=1.0, t_offset=0, x_row0=0, x_rows=0, k_tiles_per_split=0, ksize=1, act=0,
            glu=0, alpha=1.0, res_scale=1.0, accumulate=0, out_L=0, out_row_stride=1, out_row_offset=0, split_n=0, kernel=1, splitk=1,
            bias=True, residual=False, ln=False, x_off=0, ldx=None, lengths=None)


def route_name(a):
    k = a.route_kernel
    if k == 1:
        return f"gemm_conv {a.route_bm}x{a.route_bn}" + (" split" if a.route_splits > 1 else "")
    if k == 2:
        return f"skinny MR{a.route_mr} KS{a.route_ks} CPT{a.route_cpt}"
    return f"umma2 NP{k - 1} BN{a.route_u_bn} CK{a.route_u_ck} UPT{a.route_u_upt} SB{a.route_u_sb}" + (" split" if a.route_splits > 1 else "")


def make_case(g, **kw):
    c = dict(BASE)
    c.update(kw)
    c.setdefault("L_rows", c.get("L_in"))
    c.setdefault("L_in", c["L_rows"])
    ldx = c["ldx"] or c["C_in"]
    c["ldx"] = ldx
    xr = c["x_rows"] or c["L_in"]
    K = c["ksize"] * c["C_in"]
    N = c["N"]
    x_full = rnd(g, c["B"] * xr * ldx + c["x_off"], scale=1.0)
    x = x_full[c["x_off"]:].view(c["B"] * xr, ldx)
    w = rnd(g, N, K, scale=1.0 / math.sqrt(K))
    c["bias"] = rnd(g, N) if c["bias"] else None
    if c["ln"]:
        c["ln_gamma"], c["ln_beta"] = 1.0 + 0.3 * rnd(g, K), 0.3 * rnd(g, K)
        x = x * 2.0 + 0.5
        x_full[c["x_off"]:] = x.reshape(-1)
    return c, x_full, x, w


def run_case(eng, g, check_sensitivity=True, **kw):
    c, x_full, x, w = make_case(g, **kw)
    c["cls"] = C_BF16X3 if c["kernel"] == 3 else C_FP32
    M, N = c["B"] * c["L_rows"], c["N"]
    ncols = N // 2 if c["glu"] else N
    split = c["split_n"] or ncols
    nbuf = 3 if c["split_n"] else 1
    rows_out = (c["B"] * c["out_L"]) if c["out_L"] > 0 else M
    ld = {}
    prev, res, bufs = {}, {}, {}
    for p, name in enumerate(("out", "out2", "out3")[:nbuf]):
        width = min(ncols, split) + (3 if p else 0)  # ldo2 / ldo3 wider than a block: the gaps must stay untouched
        ld[name] = c.get("ldo", width) if p == 0 else width
        buf = torch.full((rows_out + 2, ld[name]), float("nan"), dtype=torch.float64, device="cuda")  # + 2 rows past the last one
        prev[name] = buf
        res[name] = rnd(g, rows_out + 2, ld[name]) if c["residual"] else None
    c["ld"] = ld
    A, y, e, S = reference(c, x, w)
    if c["accumulate"]:  # written positions hold previous values, the rest stays NaN
        for name in prev:
            idx = expected(c, y, e, prev, res)[name][2]
            prev[name].view(-1)[idx.reshape(-1)] = rnd(g, idx.numel())
    exp = expected(c, y, e, prev, res)
    dev = {n: prev[n].float().contiguous() for n in prev}
    xf = x_full.float()
    wf = w.float().contiguous()
    keep = [xf, wf]
    a = GemmArgs()
    a.x = xf.data_ptr() + 4 * c["x_off"]
    for f in ("B", "L_in", "L_rows", "C_in", "ldx", "ksize", "stride", "dil", "pad_left", "chunk", "t_offset", "x_row0", "x_rows",
              "k_tiles_per_split", "N", "act", "glu", "accumulate", "out_L", "out_row_stride", "out_row_offset", "split_n", "kernel", "splitk"):
        setattr(a, f, int(c[f]))
    a.pre_lrelu, a.alpha, a.res_scale = c["pre_lrelu"], c["alpha"], c["res_scale"]
    if c["lengths"] is not None:
        lens = torch.tensor(c["lengths"], dtype=torch.int32, device="cuda")
        keep.append(lens)
        a.lengths = lens.data_ptr()
    a.w = wf.data_ptr()
    if c["bias"] is not None:
        bf = c["bias"].float()
        keep.append(bf)
        a.bias = bf.data_ptr()
    if c["residual"]:
        rf = {n: res[n].float().contiguous() for n in res}
        keep.append(rf)
        a.residual = rf["out"].data_ptr()
        assert nbuf == 1
    if c["ln"]:
        gf, bf2 = c["ln_gamma"].float(), c["ln_beta"].float()
        keep += [gf, bf2]
        a.ln_gamma, a.ln_beta = gf.data_ptr(), bf2.data_ptr()
    a.out, a.ldo = dev["out"].data_ptr(), ld["out"]
    if nbuf == 3:
        a.out2, a.ldo2, a.out3, a.ldo3 = dev["out2"].data_ptr(), ld["out2"], dev["out3"].data_ptr(), ld["out3"]
    eng.op_gemm(a)
    torch.cuda.synchronize()
    name = route_name(a)
    ROUTES.add(name)
    K = A.shape[1]
    unit = math.sqrt(K) * EPS * S  # the bar's GEMM term per unit of c
    worst = 0.0
    for n in dev:
        ref, bar, idx = exp[n]
        got = dev[n].double()
        nan_ref = torch.isnan(ref)
        assert torch.equal(torch.isnan(got), nan_ref), (name, n, "an element outside the output was written, or one inside was not")
        err = (got - ref).abs()[~nan_ref]
        over = err > bar[~nan_ref] + 1e-30
        assert not bool(over.any()), (name, n, float((err / (bar[~nan_ref] + 1e-30)).max()))
        # the GEMM term's measured ratio: error per unit of c of this block's columns
        p = ("out", "out2", "out3").index(n)
        u = (unit[:, 0::2] if c["glu"] else unit)[:, p * split:p * split + idx.shape[1]]
        gerr = (got.view(-1)[idx.reshape(-1)] - ref.view(-1)[idx.reshape(-1)]).abs().view_as(u)
        big = u > 1e-3 * float(u.max())  # where the GEMM term is not negligible (masked rows have S = 0)
        if bool(big.any()):
            worst = max(worst, float((gerr[big] / (abs(c["alpha"]) * u[big])).max()))
    RATIOS[name] = max(RATIOS.get(name, 0.0), worst)
    if check_sensitivity:
        assert_bar_sees_missing_terms(c, x, w, y, e)
    del keep
    return a, dev


def assert_bar_sees_missing_terms(c, x, w, y, e):
    """the fp64 output changes by more than the bar somewhere when one channel, one tap or one input row is dropped"""
    C_in, k = c["C_in"], c["ksize"]
    drops = []
    w1 = w.clone()
    w1[:, C_in - 1::C_in] = 0  # the last channel of every tap
    drops.append(("channel", x, w1))
    if k > 1:
        w2 = w.clone()
        w2[:, (k - 1) * C_in:] = 0
        drops.append(("tap", x, w2))
    xr = c["x_rows"] or c["L_in"]
    x3 = x.clone()
    x3[min(xr - 1, xr // 2)] = 0  # a middle buffer row of the first batch element
    drops.append(("row", x3, w))
    for what, xx, ww in drops:
        _, y2, _, _ = reference(c, xx, ww)
        ratio = float(((y2 - y).abs() / (e * 1.0 + 1e-300)).max())
        assert ratio > 2.0, (what, ratio)


# ------------------------------------------------------------------------------------------------ gemm_conv
def test_gemm_conv_tiles_and_tails(eng, sms):
    g = torch.Generator().manual_seed(1)
    seen = set()
    plain = [  # (M, N, K): each tile choice from both sides of its threshold, M / N tails at 1 and tile - 1
        (128 * sms, 16, 20), (128 * sms + 1, 13, 28), (128 * sms - 128, 16, 4),                   # 128x16 | 32x16
        (33, 15, 12), (63, 1, 4),                                                                  # 32x16 tails
        (64 * sms, 32, 28), (64 * sms + 63, 17, 20), (64 * sms - 64, 32, 12), (65, 31, 4),        # 64x32 | 32x32
        (128 * sms, 128, 20), (128 * sms + 127, 65, 12),                                           # 128x64
        (64 * sms, 64, 60), (64 * sms + 1, 127, 28),                                               # 64x64
        (32 * sms, 64, 60), (32 * sms + 31, 64, 4),                                                 # 32x64
        (32 * 4, 64, 44), (31, 200, 12),                                                           # 32x32 (few CTAs, short K)
    ]
    for M, N, K in plain:
        a, _ = run_case(eng, g, L_rows=M, C_in=K, N=N, kernel=1, splitk=0)
        seen.add((a.route_bm, a.route_bn))
    # conv mode (implicit im2col) on the same tiles: ksize 3, padding 1
    for M, N, K in plain:
        a, _ = run_case(eng, g, L_rows=M, C_in=K, N=N, ksize=3, pad_left=1, kernel=1, splitk=0)
        seen.add((a.route_bm, a.route_bn, "conv"))
    tiles = {(128, 16), (32, 16), (64, 32), (32, 32), (128, 64), (64, 64), (32, 64)}
    assert tiles <= {s[:2] for s in seen if len(s) == 2}, seen
    assert tiles <= {s[:2] for s in seen if len(s) == 3}, seen


@pytest.mark.parametrize("ep", ["plain", "act", "glu_res_acc", "scatter", "alpha_res"])
def test_gemm_conv_split_k_epilogues(eng, ep):
    g = torch.Generator().manual_seed(2)
    kw = dict(L_rows=40, C_in=1024, N=64, kernel=1, splitk=1)
    if ep == "act":
        for act in (1, 2, 3, 4):
            a, _ = run_case(eng, g, act=act, **kw)
            assert a.route_splits > 1
        return
    if ep == "glu_res_acc":
        kw.update(glu=1, residual=True, accumulate=1, alpha=0.7, res_scale=-1.3)
    if ep == "scatter":  # transposed-conv polyphase rows: the odd rows of a twice-as-long output, even rows untouched
        kw.update(B=2, L_rows=20, out_L=41, out_row_stride=2, out_row_offset=1, accumulate=1)
    if ep == "alpha_res":
        kw.update(alpha=-0.5, residual=True, res_scale=0.25, act=2, pre_lrelu=0.1)
    a, _ = run_case(eng, g, **kw)
    assert a.route_splits > 1, route_name(a)


def test_gemm_conv_fixed_k_tiles_per_split(eng, sms):
    g = torch.Generator().manual_seed(3)
    for M in (1, 7, 64 * sms):
        a, _ = run_case(eng, g, L_rows=M, C_in=256, N=64, k_tiles_per_split=4, kernel=1, splitk=1)
        assert a.route_splits == 4


def test_gemm_conv_asr_shapes(eng):
    g = torch.Generator().manual_seed(4)
    # the extractor's stride-2 layers (k 3 and k 2) over ragged utterances
    for k in (3, 2):
        L_in = 77
        lengths = [77, 50, 9]
        run_case(eng, g, B=3, L_in=L_in, L_rows=(L_in - k) // 2 + 1, C_in=64, N=64, ksize=k, stride=2, lengths=lengths, kernel=1, splitk=0)
    # the grouped positional conv: k 128, pad 64, x and out offset by g * cg inside rows of D, GELU + residual
    D, cg, T = 256, 64, 90
    for grp in (0, 3):
        run_case(eng, g, B=2, L_in=T, C_in=cg, ldx=D, x_off=grp * cg, N=cg, ksize=128, pad_left=64, lengths=[T, 61], act=4, residual=True,
                 kernel=1, splitk=0)
    # an odd positional kernel
    run_case(eng, g, B=2, L_in=T, C_in=cg, ldx=D, N=cg, ksize=15, pad_left=7, lengths=[T, 40], act=4, residual=True, kernel=1, splitk=0)


def test_gemm_conv_dilation_chunks_and_windows(eng):
    g = torch.Generator().manual_seed(5)
    for dil in (3, 5):
        run_case(eng, g, L_in=150, C_in=32, N=48, ksize=5, dil=dil, pad_left=2 * dil, kernel=1, splitk=1)
    for chunk in (8, 16):  # chunk-causal subsampling conv (stride 2, k 3)
        run_case(eng, g, B=2, L_in=100, L_rows=50, C_in=80, N=96, ksize=3, stride=2, pad_left=1, chunk=chunk, kernel=1, splitk=1)
    # the streaming encoder's windowed conv: output rows are logical positions t_offset.., x holds logical rows x_row0 .. x_row0 + x_rows
    run_case(eng, g, B=2, L_in=60, L_rows=9, t_offset=20, x_row0=35, x_rows=12, C_in=80, N=64, ksize=3, stride=2, pad_left=1, chunk=8,
             kernel=1, splitk=0)
    run_case(eng, g, B=1, L_in=40, L_rows=6, t_offset=8, x_row0=13, x_rows=10, C_in=32, N=40, ksize=3, stride=2, pad_left=1, kernel=1, splitk=1)


# ------------------------------------------------------------------------------------------------ skinny_gemm
@pytest.mark.parametrize("M", [1, 2, 8, 9, 16, 17, 33, 64])
def test_skinny_rows_and_slices(eng, M):
    g = torch.Generator().manual_seed(10 + M)
    seen = set()
    for K, N, kw in ((128, 256, {}), (256, 256, {}), (512, 252, {}), (1024, 256, dict(act=4)), (256, 254, {}), (512, 256, dict(glu=1))):
        a, _ = run_case(eng, g, L_rows=M, C_in=K, N=N, kernel=2, **kw)
        seen.add((a.route_ks, a.route_cpt))
    assert {1, 2, 4, 8} <= {s[0] for s in seen} and {1, 2, 4} <= {s[1] for s in seen}, seen


def test_skinny_epilogues(eng):
    g = torch.Generator().manual_seed(20)
    for act in (0, 1, 2, 3, 4):
        run_case(eng, g, L_rows=5, C_in=256, N=128, act=act, alpha=0.8, kernel=2)
    run_case(eng, g, L_rows=12, C_in=256, N=128, residual=True, res_scale=0.5, accumulate=1, kernel=2)
    for K in (128, 512, 1024):  # fused LayerNorm with lda > K
        run_case(eng, g, L_rows=9, C_in=K, ldx=K + 12, N=96, ln=True, kernel=2)
    run_case(eng, g, L_rows=3, C_in=512, N=3 * 64, split_n=64, ln=True, kernel=2)  # Q|K|V routing, split_n % 4 == 0: CPT 4
    a, _ = run_case(eng, g, L_rows=3, C_in=256, N=3 * 6, split_n=6, kernel=2)  # split_n % 4 != 0: CPT 1
    assert a.route_cpt == 1


def test_skinny_grid_cap(eng, sms):
    g = torch.Generator().manual_seed(21)
    for ln, cap in ((False, 8 * sms), (True, 2 * sms)):
        N = 4 * 8 * (cap + 3)  # CPT 4, KS 1 (K = 128): more tasks than cap CTAs hold, so the CTAs loop
        a, _ = run_case(eng, g, L_rows=4, C_in=128, N=N, ln=ln, kernel=2, check_sensitivity=False)
        assert a.route_grid == cap and a.route_ks == 1 and a.route_cpt == 4


# ------------------------------------------------------------------------------------------------ umma2_conv
@pytest.mark.parametrize("pieces", [2, 3])
def test_umma2_tiles_halo_and_epilogues(eng, pieces):
    g = torch.Generator().manual_seed(30 + pieces)
    kern = pieces + 1
    seen = set()

    def run(**kw):
        eng.set_option("umma2_cache_clear", 1)  # packed weights are keyed by pointer and torch reuses addresses
        a, dev = run_case(eng, g, kernel=kern, **kw)
        seen.add((a.route_u_bn, a.route_u_ck, a.route_u_upt, a.route_splits > 1))
        return a

    for N in (16, 24, 48, 64, 200, 128):  # BN 16 / 32 / 64 / 128 with N tails
        run(L_rows=300, C_in=64, N=N, splitk=0)
    run(L_rows=129, C_in=48, N=40, splitk=0)  # CK 16, M tail
    run(L_rows=255, L_in=250, C_in=64, N=64, ksize=33, dil=2, pad_left=32, splitk=0)  # halo 64, L_rows != L_in
    run(L_rows=200, C_in=32, N=32, ksize=65, pad_left=32, splitk=1)  # halo 64, split
    run(L_rows=300, C_in=64, ldx=100, x_off=12, N=96, ksize=3, pad_left=1, pre_lrelu=0.1, splitk=0)  # ldx > C_in, offset x
    run(L_rows=150, C_in=256, N=64, ksize=3, pad_left=1, splitk=1)  # split over (chunk, tap) units
    run(L_rows=150, C_in=256, N=64, ksize=3, pad_left=1, glu=1, residual=True, accumulate=1, res_scale=0.5, splitk=1)
    run(L_rows=300, C_in=64, N=128, glu=1, splitk=0)
    run(L_rows=140, C_in=64, N=64, ksize=5, pad_left=2, residual=True, accumulate=1, alpha=0.5, act=4, splitk=0)
    run(L_rows=140, C_in=64, N=48, ksize=3, pad_left=1, out_L=281, out_row_stride=2, out_row_offset=1, splitk=0)  # scatter
    for act in (1, 2, 3):
        run(L_rows=130, C_in=32, N=32, act=act, splitk=0)
    assert {16, 32, 64, 128} <= {s[0] for s in seen} and {16, 32} <= {s[1] for s in seen}, seen
    assert {4, 6} <= {s[2] for s in seen} and {True, False} <= {s[3] for s in seen}, seen


# ------------------------------------------------------------------------------------------------ identities the engine relies on
def gemm_rows(eng, x, w, kernel, splitk, k_tiles_per_split=0):
    M, K = x.shape
    out = torch.empty(M, w.shape[0], dtype=torch.float32, device="cuda")
    a = GemmArgs()
    a.x, a.B, a.L_in, a.L_rows, a.C_in, a.ldx, a.ksize, a.stride, a.dil = x.data_ptr(), 1, M, M, K, K, 1, 1, 1
    a.pre_lrelu, a.alpha, a.res_scale, a.out_row_stride = 1.0, 1.0, 1.0, 1
    a.k_tiles_per_split, a.w, a.N, a.out, a.ldo, a.kernel, a.splitk = k_tiles_per_split, w.data_ptr(), w.shape[0], out.data_ptr(), w.shape[0], kernel, splitk
    eng.op_gemm(a)
    torch.cuda.synchronize()
    return out, a


def test_batch_invariance_and_determinism(eng):
    g = torch.Generator().manual_seed(40)
    x = torch.randn(3000, 256, generator=g).cuda()
    w = (torch.randn(64, 256, generator=g) / 16).cuda()
    # fixed k_tiles_per_split (the vocoder's duration predictor): row 0 alone equals row 0 among 3000
    one, a1 = gemm_rows(eng, x[:1].contiguous(), w, 1, 1, 4)
    many, a2 = gemm_rows(eng, x, w, 1, 1, 4)
    assert a1.route_splits == a2.route_splits == 4
    assert torch.equal(one[0], many[0])
    # no scratch (the ASR handle): a row does not depend on M or its neighbours, on gemm_conv and on umma2
    for kern in (1, 4):
        eng.set_option("umma2_cache_clear", 1)
        ref, _ = gemm_rows(eng, x[:700].contiguous(), w, kern, 0)
        for M in (130, 333, 3000):
            y = torch.randn(M, 256, generator=g).cuda()
            y[17] = x[17]
            got, a = gemm_rows(eng, y, w, kern, 0)
            assert a.route_splits == 1 and torch.equal(got[17], ref[17]), (kern, M)
    # split-K is bit-identical from run to run
    wk = (torch.randn(64, 2048, generator=g) / 45).cuda()
    xs = torch.randn(40, 2048, generator=g).cuda()
    r1, a = gemm_rows(eng, xs, wk, 1, 1)
    r2, _ = gemm_rows(eng, xs, wk, 1, 1)
    assert a.route_splits > 1 and torch.equal(r1, r2)
    eng.set_option("umma2_cache_clear", 1)
    r1, a = gemm_rows(eng, xs, wk, 4, 1)
    r2, _ = gemm_rows(eng, xs, wk, 4, 1)
    assert a.route_splits > 1 and torch.equal(r1, r2)


def test_engine_route_is_reported(eng):
    """kernel 0 takes the engine's own routing: skinny for a small plain matrix, gemm_conv or wgmma by the handle's options otherwise"""
    g = torch.Generator().manual_seed(41)
    x = torch.randn(8, 256, generator=g).cuda()
    w = (torch.randn(64, 256, generator=g) / 16).cuda()
    _, a = gemm_rows(eng, x, w, 0, 1)
    assert a.route_kernel == 2
    x = torch.randn(300, 256, generator=g).cuda()
    _, a = gemm_rows(eng, x, w, 0, 1)
    assert a.route_kernel == 4  # umma_linear = 13 on a fresh Engine (3 pieces)


# ------------------------------------------------------------------------------------------------ layer_norm
def test_layer_norm_every_width(eng):
    g = torch.Generator().manual_seed(50)
    worst = 0.0
    for C in range(32, 1025, 32):
        rows = 37
        x = torch.randn(rows, C + 8, generator=g, dtype=torch.float64)
        x[3] = 0.75  # a constant row: variance 0
        x[5] = x[5] + 1e3  # mean 1e3
        x[6] = x[6] * 1e-3 - 7.0
        gam = 1.0 + 0.5 * torch.randn(C, generator=g, dtype=torch.float64)
        bet = torch.randn(C, generator=g, dtype=torch.float64)
        xf = x.float().cuda()
        out = torch.full((rows, C + 4), float("nan"), device="cuda")
        eng.op_layer_norm(xf, gam.float().cuda(), bet.float().cuda(), out)
        x64 = xf.double()[:, :C]
        mu = x64.mean(1, keepdim=True)
        var = ((x64 - mu) ** 2).mean(1, keepdim=True)
        rstd = 1 / torch.sqrt(var + 1e-5)
        ref = (x64 - mu) * rstd * gam.cuda() + bet.cuda()
        # fp32 statistics: the centred value carries ~ulp(|x| + |mu|) times a few, scaled by rstd and gamma
        bar = 16 * EPS * ((x64.abs() + mu.abs()) * rstd * gam.cuda().abs() + bet.cuda().abs()) + 1e-30
        got = out.double()
        assert torch.isnan(got[:, C:]).all(), C
        ratio = float(((got[:, :C] - ref).abs() / bar).max())
        worst = max(worst, ratio)
        assert ratio < 1.0, (C, ratio)
        # the bar sees a dropped column: LayerNorm over C - 1 columns moves some output by more than the bar
        mu2 = x64[:, :-1].mean(1, keepdim=True)
        var2 = ((x64[:, :-1] - mu2) ** 2).mean(1, keepdim=True)
        ref2 = (x64[:, :-1] - mu2) / torch.sqrt(var2 + 1e-5) * gam.cuda()[:-1] + bet.cuda()[:-1]
        assert float(((ref2 - ref[:, :-1]).abs() / bar[:, :-1]).max()) > 2.0, C
    print(f"layer_norm worst err / bar over 32 widths: {worst:.3f}")


def test_refusals_before_any_launch(eng):
    """shapes the kernels cannot take return SS_ERR_INVALID with a message, and nothing is launched"""
    g = torch.Generator().manual_seed(60)
    x = torch.randn(64, 64, generator=g).cuda()
    w = torch.randn(64, 64, generator=g).cuda()
    out = torch.zeros(64, 64, device="cuda")
    before = eng.launch_count()

    def refused(match, **kw):
        a = GemmArgs()
        base = dict(x=x.data_ptr(), B=1, L_in=16, L_rows=16, C_in=8, ldx=8, ksize=1, stride=1, dil=1, w=w.data_ptr(), N=16, out=out.data_ptr(),
                    ldo=16, out_row_stride=1, kernel=1, splitk=1)
        base.update(kw)
        for k, v in base.items():
            setattr(a, k, v)
        a.pre_lrelu, a.alpha, a.res_scale = 1.0, 1.0, 1.0
        with pytest.raises(EngineError, match=match) as e:
            eng.op_gemm(a)
        assert e.value.code == -1

    refused("multiples of 4", C_in=6, ldx=6)                       # K = 6: a float4 would cross rows
    refused("multiples of 4", C_in=8, ldx=10)                      # ldx % 4 != 0
    refused("16-byte aligned", x=x.data_ptr() + 4)                 # misaligned x
    refused("16-byte aligned", w=w.data_ptr() + 8)                 # misaligned w
    refused("even N", N=15, glu=1)
    refused("ln_gamma / split_n", ln_gamma=w.data_ptr(), ln_beta=w.data_ptr())
    refused("skinny_gemm needs", kernel=2, L_in=65, L_rows=65, C_in=128, ldx=128)  # M > 64
    refused("skinny_gemm needs", kernel=2, C_in=96, ldx=96)                        # K % 128 != 0
    refused("skinny_gemm needs", kernel=2, C_in=128, ldx=128, ksize=3)             # not a plain matrix
    refused("wgmma", kernel=4, C_in=16, ldx=16, stride=2)
    refused("wgmma", kernel=3, C_in=8, ldx=8)                                      # C_in % 16 != 0
    refused("bad epilogue", act=5)
    refused(r"kernel must be in \[0, 4\]", kernel=5)
    with pytest.raises(EngineError, match="K % 4 == 0") as e:
        eng.op_linear(torch.randn(4, 6).cuda(), torch.randn(8, 6).cuda(), None)
    assert e.value.code == -1
    with pytest.raises(EngineError, match="C_in % 4 == 0"):
        eng.op_conv1d(torch.randn(10, 6).cuda(), torch.randn(8, 18).cuda(), None, 3, pad_left=1)
    for C in (48, 1056, 16):
        with pytest.raises(EngineError, match="multiple of 32"):
            eng.op_layer_norm(torch.randn(4, C).cuda(), torch.ones(C).cuda(), torch.zeros(C).cuda())
    assert eng.launch_count() == before


# ------------------------------------------------------------------------------------------------ coverage
def test_route_coverage():
    """every tile shape and template variant above was exercised (run with the rest of the module)"""
    if not ROUTES:
        pytest.skip("run with the rest of test_gemm_fp64.py")
    print("GEMM routes exercised:", len(ROUTES))
    for r in sorted(RATIOS):
        print(f"  {r:48s} worst err / (sqrt(K) 2^-24 S) = {RATIOS[r]:.3f}")
    tiles = {"128x16", "32x16", "64x32", "32x32", "128x64", "64x64", "32x64"}
    assert tiles <= {r.split()[1] for r in ROUTES if r.startswith("gemm_conv")}
    assert any(r.startswith("gemm_conv") and r.endswith("split") for r in ROUTES)
    sk = [r.split()[1:] for r in ROUTES if r.startswith("skinny")]
    assert {"MR1", "MR8", "MR16"} <= {s[0] for s in sk} and {"KS1", "KS2", "KS4", "KS8"} <= {s[1] for s in sk}
    assert {"CPT1", "CPT2", "CPT4"} <= {s[2] for s in sk}
    u2 = [r.split() for r in ROUTES if r.startswith("umma2")]
    assert {"NP2", "NP3"} <= {s[1] for s in u2} and {"BN16", "BN32", "BN64", "BN128"} <= {s[2] for s in u2}
    assert {"CK16", "CK32"} <= {s[3] for s in u2} and {"UPT4", "UPT6"} <= {s[4] for s in u2} and {"SB3", "SB4"} <= {s[5] for s in u2}
    assert any(s[-1] == "split" for s in u2) and any(s[-1] != "split" for s in u2)
