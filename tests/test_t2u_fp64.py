"""GPU: the T2U encoder -> CTC unit decoder -> unit arg-max / collapse call (t2u_unit_decode, engine_run.cu) against a float64
reference of the same operation, at the shapes where the call switches kernels.

Three entry points reach it: ss_t2u_unit_decode (one sample, the S2ST agent), ss_t2u_unit_decode_batch (the offline generator) and
ss_t2u_unit_decode_ragged (the pooled S2ST flush).  With S T2U positions, R = 25 upsampled rows per position and H = 8 heads:
- linears run on the skinny kernel (LayerNorm fused) for <= 64 rows in the whole call, on the fp32 tiled GEMM above that, and on the
  bf16x6 wgmma GEMM (umma_linear = 13, the default) from umma_min_rows = 128 rows per sample.  The T2U linears have S rows per sample,
  the unit decoder's R * S (skinny for S <= 2, fp32 for S = 3 .. 5, wgmma from S = 6); its grouped layer-1 QKV projection and its
  cross-attention K | V projection have S rows;
- attention takes the row kernel while ceil(rows / 16) * H < 96 (launch_attn, decided from one sample): unit self- and
  cross-attention switch between S = 7 and 8 (175 -> 200 query rows), T2U self-attention between S = 176 and 177;
- unit layer 1 runs grouped_causal_attention (unit_grouped = 1) or the full R * S causal attention (0);
- a call runs in groups of G = max(1, 32768 / (R * S_stride)) samples, every per-sample array indexed from the group's first sample;
- the T2U encoder is causal for the agent model (uni_encoder = True) and bidirectional for the offline one;
- the arg-max never selects pad, unk (and eos with mask_eos); the collapse drops blank = unit_vocab - 1 and, in ragged calls, reads only
  each sample's S_b * R rows;
- sample b's positional row is added only where the T2U output's channel 0 is not exactly 1.0 (N1: the reference derives the position
  from that value).

The reference is StreamSpeechOracle.t2u_encoder / unit_decoder_logits (oracle/streamspeech_oracle.py, pinned to the reference's
fixtures by test_oracle_golden.py) restated as float64 torch operations on the GPU with an arbitrary positional row per sample, a key
length per sample and causal or bidirectional T2U attention; attention runs in query blocks so that S = 1024 (25 600 rows) fits.
test_reference_matches_the_cpu_oracle checks it against the oracle's own float64 functions on the CPU once.  Both sides get the same fp32
MT features: ss_mt_features of random token sequences over one engine encoder output (the real final-LayerNorm scale, rms ~65), pad
tokens' features at pad-tail positions.  An arg-max may differ from the float64 one only where the float64 top-2 margin of the masked
log-probs is below MARGIN (near ties, counted and reported); it must be the masked arg-max of the fp32 log-softmax of the engine's own
logits (up to the rounding of that log-softmax, check_own_argmax), and the units must equal the oracle's ctc_collapse of the engine's
arg-max exactly.  The measured maxima, the case of each maximum and the near-tie counts are printed as one JSON line per test
(`pytest -s`) before the bars are asserted.
"""
import ctypes
import json

import pytest
import torch
import torch.nn.functional as F

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

pytestmark = pytest.mark.gpu

torch.set_grad_enabled(False)
F64 = torch.float64
MARGIN = 1e-4
# Max-abs bars against float64, about ten times the largest error measured on an H100 80GB HBM3 (700 W) over every case of this file
# (in the comments).  "fp32": every linear of the stage on the fp32 kernels (skinny or tiled); "tc": some linear of the stage on the
# bf16x6 wgmma GEMM (umma_linear = 13 and >= umma_min_rows rows per sample).
T2U_TOL = {
    "fp32": 1e-5,  # 9.1e-7 (offline, S = 1024, pad tail 1)
    "tc": 1e-5,  # 8.4e-7 (agent, S = 1024)
}
LOGIT_TOL = {
    "fp32": 2e-5,  # 2.2e-6 (offline, S = 1024, pad tail 1)
    "tc": 5e-5,  # 5.3e-6 (agent, S = 1024); 3.2e-6 at S = 120
}
LINEAR_ROUTINGS = {"tc": 13, "fp32": 0}  # umma_linear
UMMA_MIN_ROWS = 128
UNIT_BATCH_ROWS = 32768  # SS_UNIT_BATCH_ROWS (include/streamspeech_b200.h)
QUERY_BLOCK = 1024  # query rows per block of the float64 attention: [H, 1024, 25 600] float64 scores are 1.7 GB

# ss_t2u_unit_decode: every S runs twice, with complementary settings of (model, mask_eos, unit_grouped, umma_linear); the pattern of
# the first run cycles so that every pair of settings of every two options occurs (a pairwise design), and the two runs take two
# different pad tails out of {0, 1, S - 1}
SINGLE_S = [1, 2, 3, 5, 6, 7, 8, 16, 17, 64, 65, 127, 128, 176, 177, 1024]
PATTERNS = ["0000", "0011", "0101", "0110"]  # bits: offline model, mask_eos, unit_grouped = 0, umma_linear = 0
RANDOM_ROW_S = (8, 65, 177)  # the first run of these S sets a random positional row (ss_unit_position_row)


def report(name, **kw):
    print(json.dumps({"test": name, **kw}))


def maxdiff(a, b):
    """max-abs difference; a NaN counts as infinite"""
    d = float((a.double() - b.to(a.device).double()).abs().max()) if a.numel() else 0.0
    return float("inf") if d != d else d


class Worst:
    """the largest error per key and the case it came from"""

    def __init__(self):
        self.v = {}

    def add(self, key, err, case):
        if key not in self.v or err > self.v[key][0]:
            self.v[key] = (err, case)

    def get(self, key):
        return self.v.get(key, (0.0, None))[0]

    def as_dict(self):
        return {k: {"max_abs": v, "case": c} for k, (v, c) in sorted(self.v.items())}


class Ref64:
    """StreamSpeechOracle.t2u_encoder + unit_decoder_logits (2 pre-LN T2U layers, 2 unit decoder layers) in float64 on the GPU, for one
    sample: the weights are the fp32 checkpoint's, converted"""

    def __init__(self, cfg, sd):
        self.cfg = cfg
        self.w = {k: v.float().to("cuda", F64) for k, v in sd.items()
                  if k.startswith(("synthesizer_encoder.", "decoder.")) and v.is_floating_point()}

    def _lin(self, x, name):
        return F.linear(x, self.w[name + ".weight"], self.w.get(name + ".bias"))

    def _ln(self, x, name):
        return F.layer_norm(x, (x.shape[-1],), self.w[name + ".weight"], self.w[name + ".bias"], 1e-5)

    def _mha(self, x, kv, name, n_keys, causal):
        """mha: x [Tq, C] attends to the first n_keys rows of kv [Tk, C] (key_padding_mask), causal: query i to keys <= i"""
        H = self.cfg.unit_heads
        Tq, C = x.shape
        hd = C // H
        q = (self._lin(x, name + ".q_proj") * hd ** -0.5).view(Tq, H, hd).transpose(0, 1)
        k = self._lin(kv[:n_keys], name + ".k_proj").view(-1, H, hd).transpose(0, 1)
        v = self._lin(kv[:n_keys], name + ".v_proj").view(-1, H, hd).transpose(0, 1)
        o = torch.empty(H, Tq, hd, dtype=F64, device="cuda")
        for q0 in range(0, Tq, QUERY_BLOCK):
            q1 = min(Tq, q0 + QUERY_BLOCK)
            nk = min(n_keys, q1) if causal else n_keys  # keys beyond the block's last query are masked for all of it
            w = q[:, q0:q1] @ k[:, :nk].transpose(1, 2)
            if causal:
                w.masked_fill_(torch.arange(nk, device="cuda")[None, :] > torch.arange(q0, q1, device="cuda")[:, None], float("-inf"))
            o[:, q0:q1] = torch.softmax(w, dim=-1) @ v[:, :nk]
        return self._lin(o.transpose(0, 1).reshape(Tq, C), name + ".out_proj")

    def t2u_encoder(self, x, n_keys, causal):
        """UniTransformerEncoderNoEmb.forward: x [S, 512] (fp32 MT features) -> [S, 512]"""
        x = x.to("cuda", F64)
        for i in range(self.cfg.t2u_layers):
            p = f"synthesizer_encoder.layers.{i}"
            y = self._ln(x, p + ".self_attn_layer_norm")
            x = x + self._mha(y, y, p + ".self_attn", n_keys, causal)
            x = x + self._lin(F.relu(self._lin(self._ln(x, p + ".final_layer_norm"), p + ".fc1")), p + ".fc2")
        return self._ln(x, "synthesizer_encoder.layer_norm")

    def unit_logits(self, t2u, n_keys, pos_row):
        """CTCTransformerUnitDecoder: t2u [S, 512] -> logits [R * S, unit_vocab]; pos_row [512] is added to the rows whose channel 0 is
        not 1.0 (N1: make_positions of that value gives pad, the zero row, where it equals pad = 1)"""
        R = self.cfg.ctc_upsample_rate
        x = t2u.repeat_interleave(R, dim=0)
        x = x + torch.where(x[:, :1] != 1.0, pos_row.to("cuda", F64)[None, :], 0.0)
        for i in range(self.cfg.unit_layers):
            p = f"decoder.layers.{i}"
            y = self._ln(x, p + ".self_attn_layer_norm")
            x = x + self._mha(y, y, p + ".self_attn", n_keys * R, True)
            x = x + self._mha(self._ln(x, p + ".encoder_attn_layer_norm"), t2u, p + ".encoder_attn", n_keys, False)
            x = x + self._lin(F.relu(self._lin(self._ln(x, p + ".final_layer_norm"), p + ".fc1")), p + ".fc2")
        return F.linear(self._ln(x, "decoder.layer_norm"), self.w["decoder.output_projection.weight"])

    def forward(self, x, n_pad, pos_row, causal):
        t2u = self.t2u_encoder(x, x.shape[0] - n_pad, causal)
        return t2u, self.unit_logits(t2u, x.shape[0] - n_pad, pos_row)


def masked_lprobs(cfg, logits, mask_eos):
    """CTCSequenceGenerator: never pad, unk (agent) [+ eos, offline]"""
    lp = F.log_softmax(logits.double(), dim=-1)
    lp[:, masked_cols(cfg, mask_eos)] = float("-inf")
    return lp


def masked_cols(cfg, mask_eos):
    return [cfg.pad, cfg.unk] + ([cfg.eos] if mask_eos else [])


def check_argmax(got, lp, what):
    """got [N] int, lp [N, V] float64 masked log-probs: got must be the arg-max wherever the top-2 margin is at least MARGIN; returns
    the number of near-tie positions where it is not"""
    top = lp.topk(2, dim=-1)
    bad = torch.as_tensor(got, device=lp.device).long() != top.indices[:, 0]
    hard = bad & (top.values[:, 0] - top.values[:, 1] >= MARGIN)
    assert not bool(hard.any()), (what, torch.nonzero(hard).flatten()[:10].tolist())
    return int(bad.sum())


def check_own_argmax(cfg, am, logits, mask_eos, what):
    """am must be the masked arg-max of the fp32 log-softmax of the engine's own logits.  The engine ranks log-probs (x - max) - lse in
    fp32 (block_masked_argmax256), which can round two logits closer than an ulp of lse to one value and then takes the lower index, so
    where am differs from torch's arg-max its log-prob must equal the maximum to within that rounding.  Returns the number of such rows."""
    lp = torch.log_softmax(logits, dim=-1)
    lp[:, masked_cols(cfg, mask_eos)] = float("-inf")
    want = lp.argmax(-1)
    rows = torch.nonzero(am != want).flatten()
    best, got = lp[rows, want[rows]], lp[rows, am[rows]]
    assert bool(((best - got).abs() <= 4 * torch.finfo(torch.float32).eps * best.abs()).all()), (what, rows[:10].tolist())
    return int(rows.numel())


def check_units(cfg, units, argmax, what):
    """the engine's units equal the oracle's collapse of the engine's own arg-max"""
    from oracle.streamspeech_oracle import ctc_collapse

    want, _ = ctc_collapse([int(t) for t in argmax], blank=cfg.unit_blank, pad=cfg.pad)
    assert [int(u) for u in units] == want, (what, len(units), len(want))


def wgmma_ran(e, fn):
    """(fn(), whether some wgmma GEMM ran in it): the umma2 kernels stamp a zeroed debug buffer when they start (option umma2_debug)"""
    e.set_option("umma2_debug", 1)
    stamps = (ctypes.c_uint64 * 16)()
    try:
        r = fn()
        torch.cuda.synchronize()
        e._check(e.lib.ss_debug_copy(e._h, b"umma2_ts", ctypes.cast(stamps, ctypes.c_void_p), ctypes.sizeof(stamps)))
    finally:
        e.set_option("umma2_debug", 0)
    return r, any(stamps)


def offline_cfg():
    cfg = ModelConfig()
    cfg.uni_encoder = False  # offline model: bidirectional T2U encoder
    return cfg


class Setup:
    """both engines (agent: causal T2U, offline: bidirectional), the float64 reference, the encoder rows the MT features are computed
    over, and caches of features and float64 results.

    The synthetic checkpoint's unit decoder never ranks eos first, so mask_eos would change nothing.  Its eos output row (tied with the
    input embedding, which the unit decoder does not read) becomes 1.02 times the row of the unit it picks most often on a probe: eos
    then takes that unit's rows wherever its logit is positive, by a margin of 2 % of the logit, and only the eos mask gives them back."""

    def __init__(self):
        from streamspeech_b200.engine import Engine

        c = self.cfg = ModelConfig()
        sd = synth.make_model_state_dict(c, 0)
        gc = synth.make_gcmvn(c)
        probe = Engine(c, sd, None, gc)
        try:
            self.enc = probe.encoder(probe.fbank(synth.make_audio(3.0, seed=29).cuda().contiguous()).unsqueeze(0).contiguous())[0].clone()
            g = torch.Generator().manual_seed(5)
            x = probe.mt_features(self.enc, [c.eos] + torch.randint(c.unk + 1, c.tgt_vocab, (63,), generator=g).tolist())
            am = probe.t2u_unit_decode(x.contiguous())["argmax"]
        finally:
            probe.close()
        units = am[(am > c.unk) & (am < c.unit_blank)]
        top = int(torch.bincount(units, minlength=c.unit_vocab).argmax())
        emb = sd["decoder.embed_tokens.weight"].clone()
        emb[c.eos] = 1.02 * emb[top]
        self.sd = {**sd, "decoder.embed_tokens.weight": emb, "decoder.output_projection.weight": emb}
        self.eng = {"agent": Engine(c, self.sd, None, gc), "offline": Engine(offline_cfg(), self.sd, None, gc)}
        self.eng["agent"].set_chunk(8)
        self.eng["offline"].set_chunk(None, None)
        for e in self.eng.values():
            e.set_option("umma_min_rows", UMMA_MIN_ROWS)
        self.ref = Ref64(c, self.sd)
        self._feats, self._ref = {}, {}

    def close(self):
        for e in self.eng.values():
            e.close()

    def feats(self, S, n_pad, seed=0):
        """fp32 MT features [S, mt_dim] of [eos] + S - 1 - n_pad random tokens + n_pad pads"""
        key = (S, n_pad, seed)
        if key not in self._feats:
            c = self.cfg
            g = torch.Generator().manual_seed(1000 * S + 10 * n_pad + seed)
            toks = [c.eos] + torch.randint(c.unk + 1, c.tgt_vocab, (S - 1 - n_pad,), generator=g).tolist() + [c.pad] * n_pad
            self._feats[key] = self.eng["agent"].mt_features(self.enc, toks).contiguous()
        return self._feats[key]

    def f64(self, model, S, n_pad, row, row_key, seed=0):
        """float64 (t2u_out, logits) of feats(S, n_pad, seed) with positional row `row` (cached under row_key)"""
        key = (model, S, n_pad, seed, row_key)
        if key not in self._ref:
            self._ref[key] = self.ref.forward(self.feats(S, n_pad, seed), n_pad, row, model == "agent")
        return self._ref[key]


@pytest.fixture(scope="module")
def t2u():
    s = Setup()
    yield s
    s.close()


def test_reference_matches_the_cpu_oracle(t2u):
    """the GPU float64 restatement against StreamSpeechOracle(dtype=float64).t2u_encoder / unit_decoder_logits on the CPU, for both T2U
    encoders, with and without a pad tail, with the oracle's own positional row (B = 1: position pad + 1); and the engine's row of
    batch index b is the oracle table's row pad + 1 + b"""
    from oracle.streamspeech_oracle import StreamSpeechOracle, sinusoidal_table

    c = t2u.cfg
    table = sinusoidal_table(max(1200, c.pad + 1 + 64 + 1), c.unit_dim, c.pad)
    for b in (0, 1, 9, 39):
        assert torch.equal(t2u.eng["agent"].unit_position_row(b), table[c.pad + 1 + b]), b
    res = {}
    for model, cfg in (("agent", t2u.cfg), ("offline", offline_cfg())):
        o = StreamSpeechOracle(cfg, t2u.sd, None, None, dtype=F64)
        for S, n_pad in ((9, 0), (9, 3)):
            x = t2u.feats(S, n_pad)
            pm = torch.zeros(1, S, dtype=torch.bool)
            pm[0, S - n_pad:] = True
            want_t2u = o.t2u_encoder(x.double().cpu().unsqueeze(1), pm if n_pad else None)
            want_logits = o.unit_decoder_logits(want_t2u, pm if n_pad else None)[0]
            got_t2u, got_logits = t2u.ref.forward(x, n_pad, table[c.pad + 1], cfg.uni_encoder)
            res[f"{model} S={S} pad={n_pad}"] = {"t2u": maxdiff(got_t2u.cpu(), want_t2u[:, 0]),
                                                 "logits": maxdiff(got_logits.cpu(), want_logits)}
    report("t2u_fp64_reference_vs_cpu_oracle", **res)
    for k, v in res.items():
        assert v["t2u"] < 1e-12 and v["logits"] < 1e-12, (k, v)


def single_cases():
    """(S, n_pad, model, mask_eos, unit_grouped, umma_linear, random row)"""
    out = []
    for i, S in enumerate(SINGLE_S):
        pads = sorted({0, 1, S - 1} & set(range(S)))
        first = PATTERNS[i % len(PATTERNS)]
        for half, bits in enumerate((first, "".join("1" if ch == "0" else "0" for ch in first))):
            out.append((S, pads[(i + half) % len(pads)], "offline" if bits[0] == "1" else "agent", int(bits[1]), 1 - int(bits[2]),
                        LINEAR_ROUTINGS["fp32" if bits[3] == "1" else "tc"], half == 0 and S in RANDOM_ROW_S))
    return out


def test_single_sample_vs_fp64(t2u):
    """ss_t2u_unit_decode over the pairwise design single_cases(): T2U output and unit logits within their bars, arg-max by the margin
    rule and the masked arg-max of the fp32 log-softmax of the engine's own logits, units exactly the collapse of the arg-max.  Below
    umma_min_rows rows per sample umma_linear 13 and 0 must run the same kernels: bit-identical T2U output (S < 128) and logits
    (25 * S < 128); a wgmma GEMM runs exactly when umma_linear = 13 and 25 * S >= umma_min_rows."""
    c = t2u.cfg
    R = c.ctc_upsample_rate
    cases = single_cases()
    g = torch.Generator().manual_seed(31)
    worst, near, eos_rows, same_routes, tc_seen, lp_ties = Worst(), {}, {0: 0, 1: 0}, 0, False, 0
    for S, n_pad, model, mask_eos, grouped, umma, random_row in cases:
        e = t2u.eng[model]
        what = f"{model} S={S} pad={n_pad} mask_eos={mask_eos} grouped={grouped} umma={umma}{' random_row' if random_row else ''}"
        x = t2u.feats(S, n_pad)
        row = torch.randn(c.unit_dim, generator=g) if random_row else e.unit_position_row(0)
        e.set_option("unit_grouped", grouped)
        e.set_option("umma_linear", umma)
        try:
            if random_row:
                e._check(e.lib.ss_unit_position_row(e._h, row.data_ptr()))
            r, ran = wgmma_ran(e, lambda: e.t2u_unit_decode(x, n_pad_tail=n_pad, mask_eos=bool(mask_eos), debug=True))
            assert ran == (umma == 13 and R * S >= UMMA_MIN_ROWS), (what, ran)
            tc_seen |= ran
            if S < UMMA_MIN_ROWS:  # the other routing runs the same kernels on every linear that has fewer rows
                e.set_option("umma_linear", LINEAR_ROUTINGS["fp32"] if umma == 13 else LINEAR_ROUTINGS["tc"])
                r2 = e.t2u_unit_decode(x, n_pad_tail=n_pad, mask_eos=bool(mask_eos), debug=True)
                assert torch.equal(r2["t2u_out"], r["t2u_out"]), what
                if R * S < UMMA_MIN_ROWS:
                    assert torch.equal(r2["logits"], r["logits"]), what
                same_routes += 1
        finally:
            e.set_unit_batch_index(0)
            e.set_option("umma_linear", LINEAR_ROUTINGS["tc"])
            e.set_option("unit_grouped", 1)
        t2u64, logits64 = t2u.f64(model, S, n_pad, row, f"random{S}" if random_row else 0)
        t2u_route = "tc" if umma == 13 and S >= UMMA_MIN_ROWS else "fp32"
        unit_route = "tc" if umma == 13 and R * S >= UMMA_MIN_ROWS else "fp32"
        worst.add(f"t2u_{t2u_route}", maxdiff(r["t2u_out"], t2u64), what)
        worst.add(f"logits_{unit_route}", maxdiff(r["logits"], logits64), what)
        am = r["argmax"]
        near[what] = check_argmax(am, masked_lprobs(c, logits64, mask_eos), what)
        eos_rows[mask_eos] += int((r["logits"].argmax(-1) == c.eos).sum())  # rows where only the eos mask keeps eos out
        lp_ties += check_own_argmax(c, am, r["logits"], mask_eos, what)
        n = int(r["count"][0])
        check_units(c, r["units"][:n].tolist(), am.tolist(), what)
    report("t2u_single_sample_fp64", cases=len(cases), bit_identical_routings=same_routes, rows_with_eos_on_top=eos_rows,
           log_softmax_ties=lp_ties, **worst.as_dict(), near_ties={k: v for k, v in near.items() if v})
    assert tc_seen and eos_rows[0] > 0 and eos_rows[1] > 0, eos_rows  # the routes and the eos mask were exercised
    for stage, tol in (("t2u", T2U_TOL), ("logits", LOGIT_TOL)):
        for route in LINEAR_ROUTINGS:
            assert worst.get(f"{stage}_{route}") < tol[route], worst.as_dict()


# ss_t2u_unit_decode_batch on the offline engine: (S_stride, B, mask_eos), each sample with positional row unit_position_row(b)
BATCH_CASES = [(120, 23, 1), (1024, 2, 0), (2, 40, 1)]


def test_batch_vs_fp64(t2u):
    """S = 120 at B = 23 (groups of 10, 10 and 3, pad tails in every group), S = 1024 at B = 2 (groups of one), S = 2 at B = 40 (80 T2U
    rows: no skinny kernel; no linear reaches umma_min_rows rows per sample, so no wgmma GEMM may run).  Every sample's arg-max against
    the float64 pass of that sample alone with its own row, its units against the collapse of its arg-max."""
    c = t2u.cfg
    e = t2u.eng["offline"]
    R = c.ctc_upsample_rate
    near, ran_wgmma = {}, {}
    for S, B, mask_eos in BATCH_CASES:
        G = max(1, UNIT_BATCH_ROWS // (R * S))
        pads = [(b % 4) % S for b in range(B)]
        assert G == 1 or all(any(pads[g0:g0 + G]) for g0 in range(0, B, G))
        x = torch.stack([t2u.feats(S, pads[b], b) for b in range(B)]).contiguous()
        (units, argmax, _), ran_wgmma[f"S={S} B={B}"] = wgmma_ran(e, lambda: e.t2u_unit_decode_batch(x, pads, mask_eos=bool(mask_eos)))
        assert ran_wgmma[f"S={S} B={B}"] == (R * S >= UMMA_MIN_ROWS), (S, B)  # routing by one sample's rows, not the batch's
        nt = 0
        for b in range(B):
            what = f"S={S} B={B} G={G} b={b} pad={pads[b]}"
            _, logits64 = t2u.f64("offline", S, pads[b], e.unit_position_row(b), b, b)
            nt += check_argmax(argmax[b], masked_lprobs(c, logits64, mask_eos), what)
            check_units(c, units[b], argmax[b], what)
        near[f"S={S} B={B} G={G}"] = nt
    report("t2u_batch_fp64", near_ties=near, wgmma_ran=ran_wgmma)


def ragged_inputs(t2u, S_stride, lengths, pads, fill):
    x = torch.full((len(lengths), S_stride, t2u.cfg.mt_dim), fill, device="cuda")
    for b, (Sb, p) in enumerate(zip(lengths, pads)):
        x[b, :Sb] = t2u.feats(Sb, p, 100 + b)
    return x.contiguous()


def test_ragged_vs_fp64(t2u):
    """ss_t2u_unit_decode_ragged on the agent engine: 45 samples of S_stride = 64 (groups of 20, 20 and 5) with lengths 1 .. 64, short
    samples and pad tails in every group and a distinct random positional row per sample; the rows beyond each sample's length are NaN.
    Every sample against the float64 pass of that sample alone; its first S_b * 25 arg-max rows and its units must not change when the
    NaN rows are zeros.  Then the long-utterance case S = 120 / 97 (pad tail 4) with both unit_grouped settings, single-sample logits
    included."""
    c = t2u.cfg
    e = t2u.eng["agent"]
    R = c.ctc_upsample_rate
    g = torch.Generator().manual_seed(37)
    S_stride, B = 64, 45
    G = UNIT_BATCH_ROWS // (R * S_stride)
    assert (G, -(-B // G)) == (20, 3)
    lengths = torch.randint(1, S_stride + 1, (B,), generator=g).tolist()
    for g0 in range(0, B, G):
        lengths[g0], lengths[min(B, g0 + G) - 1] = S_stride, 1
        lengths[g0 + 1] = 2 + g0 // G
    pads = [min(b % 5, Sb - 1) for b, Sb in enumerate(lengths)]
    rows = torch.randn(B, c.unit_dim, generator=g)
    near, res, out = {}, {}, {}
    for fill, value in (("nan", float("nan")), ("zero", 0.0)):
        x = ragged_inputs(t2u, S_stride, lengths, pads, value)
        out[fill] = e.t2u_unit_decode_ragged(x, lengths, pads, rows.cuda().contiguous(), mask_eos=False)
    units, argmax, _ = out["nan"]
    nt = 0
    for b in range(B):
        what = f"ragged b={b} S_b={lengths[b]} pad={pads[b]}"
        assert len(argmax[b]) == lengths[b] * R
        _, logits64 = t2u.f64("agent", lengths[b], pads[b], rows[b], f"ragged{b}", 100 + b)
        nt += check_argmax(argmax[b], masked_lprobs(c, logits64, False), what)
        check_units(c, units[b], argmax[b], what)
        assert out["zero"][1][b] == argmax[b] and out["zero"][0][b] == units[b], what
    near["S_stride=64 B=45"] = nt
    # the long-utterance case: two samples of one ragged call, and each alone with its logits
    S, pads2 = (120, 97), (0, 4)
    x = ragged_inputs(t2u, 120, S, pads2, 0.0)
    worst = Worst()
    for grouped in (1, 0):
        e.set_option("unit_grouped", grouped)
        try:
            units, argmax, _ = e.t2u_unit_decode_ragged(x, list(S), list(pads2))
            singles = [e.t2u_unit_decode(x[b, :S[b]].contiguous(), n_pad_tail=pads2[b], debug=True) for b in range(2)]
        finally:
            e.set_option("unit_grouped", 1)
        nts = []
        for b in range(2):
            what = f"long S={S[b]} pad={pads2[b]} grouped={grouped}"
            t2u64, logits64 = t2u.f64("agent", S[b], pads2[b], e.unit_position_row(0), 0, 100 + b)
            lp = masked_lprobs(c, logits64, False)
            worst.add("t2u_fp32", maxdiff(singles[b]["t2u_out"], t2u64), what)
            worst.add("logits_tc", maxdiff(singles[b]["logits"], logits64), what)
            nts.append(check_argmax(argmax[b], lp, what))
            nts.append(check_argmax(singles[b]["argmax"], lp, what))
            check_units(c, units[b], argmax[b], what)
        res[f"grouped{grouped}"] = nts
    report("t2u_ragged_fp64", lengths=lengths, near_ties=near, long_near_ties=res, **worst.as_dict())
    assert worst.get("t2u_fp32") < T2U_TOL["fp32"] and worst.get("logits_tc") < LOGIT_TOL["tc"], worst.as_dict()


def test_position_row_skipped_where_channel_0_is_one(t2u):
    """N1: with synthesizer_encoder.layer_norm gain 0 and bias 1.0 on channel 0, every T2U output row has channel 0 exactly 1.0, so the
    reference adds the pad (zero) row and the engine must add none: one sample (S = 17, pad tail 1) against float64 within the bars, and
    a batch of 3 (S = 8) whose rows b > 0 are not zero"""
    from streamspeech_b200.engine import Engine

    c = t2u.cfg
    sd = dict(t2u.sd)
    for k, v in (("weight", 0.0), ("bias", 1.0)):
        sd[f"synthesizer_encoder.layer_norm.{k}"] = sd[f"synthesizer_encoder.layer_norm.{k}"].clone()
        sd[f"synthesizer_encoder.layer_norm.{k}"][0] = v
    e = Engine(c, sd, None, synth.make_gcmvn(c))
    ref = Ref64(c, sd)
    try:
        S, n_pad = 17, 1
        x = t2u.feats(S, n_pad)
        r = e.t2u_unit_decode(x, n_pad_tail=n_pad, debug=True)
        t2u64, logits64 = ref.forward(x, n_pad, e.unit_position_row(0), True)
        assert bool((t2u64[:, 0] == 1.0).all()) and bool((r["t2u_out"][:, 0] == 1.0).all())
        d_t2u, d_logits = maxdiff(r["t2u_out"], t2u64), maxdiff(r["logits"], logits64)
        near = [check_argmax(r["argmax"], masked_lprobs(c, logits64, False), "single")]
        check_units(c, r["units"][:int(r["count"][0])].tolist(), r["argmax"].tolist(), "single")
        S, B = 8, 3
        pads = [0, 2, 1]
        xb = torch.stack([t2u.feats(S, pads[b], b) for b in range(B)]).contiguous()
        units, argmax, _ = e.t2u_unit_decode_batch(xb, pads)
        for b in range(B):
            assert float(e.unit_position_row(b).abs().max()) > 0.5
            _, logits64 = ref.forward(xb[b], pads[b], e.unit_position_row(b), True)
            near.append(check_argmax(argmax[b], masked_lprobs(c, logits64, False), f"batch b={b}"))
            check_units(c, units[b], argmax[b], f"batch b={b}")
    finally:
        e.close()
    report("t2u_n1_channel0_fp64", t2u_max_abs=d_t2u, logits_max_abs=d_logits, near_ties=near)
    assert d_t2u < T2U_TOL["fp32"] and d_logits < LOGIT_TOL["tc"], (d_t2u, d_logits)  # (25 * 17 unit rows: wgmma linears)
