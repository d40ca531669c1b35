"""The MT search with the reference's incremental states (ss_mt_greedy_incremental on the handle, ss_pool_mt_greedy_incremental per
pool slot) against a float64 reference of the same state, read back after every call.

The state lives across calls and keeps two quirks of the reference on purpose (include/streamspeech_b200.h, SURVEY.md N12):
- every call feeds the last prefix token again, so the self-attention cache holds one duplicate entry per call: the entry of position p
  sits at p + kv_off (kv_off = entries - prefix length), while its positional row stays pad + 1 + p;
- cross-attention K / V are projected only for encoder rows no earlier call saw and never refreshed, so early rows keep the projections
  of a provisional encoder output.

IncRef64 restates StreamSpeechOracle._mt_step_incremental (oracle/streamspeech_oracle.py) in float64 on any device, teacher-forced on the
engine's tokens: per call it projects the encoder rows beyond the cached ones, then feeds the last prefix token at position start and
each engine token after it, appending one self-attention entry per step.  test_reference_matches_the_cpu_oracle pins it to the oracle's
own float64 mt_greedy_incremental on the CPU.  After every call of every case:
- tokens follow the margin rule of test_long_utterance_fp64.py: each new token is the float64 arg-max unless the float64 top-2 margin is
  below MARGIN (such near ties are counted and reported); the prefix comes back unchanged;
- the read-back (ss_debug_copy "mt_inc_state" / "pool_mt_inc_state:<slot>") holds exactly the reference's entries and cross rows;
- self K, self V and cross K | V are within a bar of the reference, as max-abs error over max |reference| per tensor.
Each case also shows that the quirks are observable: its stale cross rows differ from a fresh projection of the call's rows by at least
STALE_FACTOR times the cross bar, and its duplicate entries differ from their first entry beyond the self bar in layers >= 1.  An engine
that refreshed stale rows or deduplicated entries would fail the state check.

Stale rows are real (the provisional tail of ss_encoder_stream_step / ss_pool_step changes between calls) and forced: before a call the
test adds O(1) noise to rows an earlier call saw, in the handle's enc argument or, in the pool, through pool_encoder_rows, a view of the
pool's own encoder rows (the search reads them from there).  Routes are proved from the single-token kernel's launch count (mt_time)
and the library launch counter.  The measured maxima, the case of each and the near-tie counts are printed as one JSON line per test
(`pytest -s`), with the card's name and power limit.
"""
import ctypes
import json
import math
import subprocess

import pytest
import torch
import torch.nn.functional as F

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

torch.set_grad_enabled(False)
gpu = pytest.mark.gpu
F64 = torch.float64
MARGIN = 1e-4
SS_ERR_STATE, SS_ERR_CAPACITY = -4, -5
# Bars: max |engine - float64| / max |float64| per tensor (every layer, every entry or row), about ten times the largest error measured
# on an H100 80GB HBM3 (700 W) over every case of this file (in the comments).
SELF_TOL = {"single": 3e-6, "batched": 3e-6}  # self K / V: 2.5e-7 single-token kernel, 3.0e-7 batched kernel (stream 160 ms, pool groups)
CROSS_TOL = 1.5e-5  # cross K | V over every GEMM route: 1.3e-6 (500 new rows on the wgmma kernel, forced-stale case, T = 700)
STALE_FACTOR = 100
MAX_LEN = 200  # the generator's max_len of the finishing calls
BATCH_ROWS = 32  # MT_BATCH_MAX_ROWS
# commit rules: the prefix of the next call from the last hypothesis
RULES = {"full": lambda h: list(h), "minus1": lambda h: list(h[:-1]), "minus2": lambda h: list(h[:-2]), "empty": lambda h: []}


def report(name, **kw):
    print(json.dumps({"test": name, **kw}))


def card():
    """the GPU's name and power limit (part of every number this file measures)"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def rel(a, b):
    """max |a - b| / max |b| (b the float64 reference)"""
    if b.numel() == 0:
        return 0.0
    return float((a.to(b.device, F64) - b).abs().max() / b.abs().max().clamp_min(1e-300))


class Worst:
    """the largest value per key and the case it came from"""

    def __init__(self):
        self.v = {}

    def add(self, key, err, case):
        if key not in self.v or err > self.v[key][0]:
            self.v[key] = (err, case)

    def get(self, key):
        return self.v.get(key, (0.0, None))[0]

    def as_dict(self):
        return {k: {"max": v, "case": c} for k, (v, c) in self.v.items()}


class IncRef64:
    """StreamSpeechOracle._mt_step_incremental (pre-LN TransformerDecoderBase with incremental states) in float64 on `device`: the weights
    are the fp32 checkpoint's, converted; the position table is the oracle's.  A state is per-layer K / V tensors that only grow."""

    def __init__(self, cfg, sd, device):
        from oracle.streamspeech_oracle import sinusoidal_table

        self.cfg, self.dev = cfg, torch.device(device)
        pfx = "target_unigram_decoder."
        self.w = {k[len(pfx):]: v.float().to(self.dev, F64) for k, v in sd.items() if k.startswith(pfx) and v.is_floating_point()}
        self.table = sinusoidal_table(4096 + cfg.pad + 2, cfg.mt_dim, cfg.pad).to(self.dev, F64)
        self.emb = self.w["embed_tokens.weight"]

    def state(self):
        L, D = self.cfg.mt_layers, self.cfg.mt_dim
        z = lambda: [torch.zeros(0, D, dtype=F64, device=self.dev) for _ in range(L)]  # noqa: E731
        return {"k": z(), "v": z(), "ck": z(), "cv": z(), "pos": [], "tok": [], "stale": 0.0}

    @staticmethod
    def entries(st):
        return st["k"][0].shape[0]

    @staticmethod
    def rows(st):
        return st["ck"][0].shape[0]

    def _lin(self, x, name):
        return F.linear(x, self.w[name + ".weight"], self.w.get(name + ".bias"))

    def _ln(self, x, name):
        return F.layer_norm(x, (x.shape[-1],), self.w[name + ".weight"], self.w[name + ".bias"], 1e-5)

    def _attn(self, q, k, v, name, mask):
        H = self.cfg.mt_heads
        hd = q.shape[-1] // H
        q = (q * hd ** -0.5).view(-1, H, hd).transpose(0, 1)
        w = q @ k.view(-1, H, hd).permute(1, 2, 0)
        if mask is not None:
            w = w.masked_fill(mask, float("-inf"))
        o = (torch.softmax(w, dim=-1) @ v.view(-1, H, hd).transpose(0, 1)).transpose(0, 1).reshape(q.shape[1], -1)
        return self._lin(o, name + ".out_proj")

    def cross(self, enc, l):
        p = f"layers.{l}.encoder_attn"
        return self._lin(enc, p + ".k_proj"), self._lin(enc, p + ".v_proj")

    def call(self, st, enc, prefix, new_tokens, max_len):
        """one incremental call teacher-forced on the engine's new tokens (eos excluded): returns the masked log-probs [steps, vocab] of
        positions start .. start + len(new_tokens); the state gains the new cross rows and one entry per step"""
        c = self.cfg
        enc = enc.to(self.dev, F64)
        start = len(prefix)
        toks = [c.eos] + list(prefix) + list(new_tokens)
        steps = list(range(start, len(toks)))
        have = self.rows(st)
        if have and enc.shape[0]:  # the stale rows against a fresh projection of this call's rows (the quirk's size)
            n = min(have, enc.shape[0])
            for l in range(c.mt_layers):
                k, v = self.cross(enc[:n], l)
                scale = torch.cat([st["ck"][l], st["cv"][l]], -1).abs().max()
                st["stale"] = max(st["stale"], float(torch.cat([st["ck"][l][:n] - k, st["cv"][l][:n] - v], -1).abs().max() / scale))
        if enc.shape[0] > have:  # only rows beyond the cached ones are projected (transformer_layer.py:492-505)
            for l in range(c.mt_layers):
                k, v = self.cross(enc[have:], l)
                st["ck"][l] = torch.cat([st["ck"][l], k])
                st["cv"][l] = torch.cat([st["cv"][l], v])
        t = torch.tensor([toks[s] for s in steps], device=self.dev)
        pos = torch.tensor([c.pad if toks[s] == c.pad else c.pad + 1 + s for s in steps], device=self.dev)
        x = math.sqrt(c.mt_dim) * self.emb[t] + self.table[pos]
        E0, m = self.entries(st), len(steps)
        mask = torch.arange(E0 + m, device=self.dev)[None, :] > (E0 + torch.arange(m, device=self.dev))[:, None]  # step i sees E0 + i + 1
        for l in range(c.mt_layers):
            p = f"layers.{l}"
            y = self._ln(x, p + ".self_attn_layer_norm")
            st["k"][l] = torch.cat([st["k"][l], self._lin(y, p + ".self_attn.k_proj")])
            st["v"][l] = torch.cat([st["v"][l], self._lin(y, p + ".self_attn.v_proj")])
            x = x + self._attn(self._lin(y, p + ".self_attn.q_proj"), st["k"][l], st["v"][l], p + ".self_attn", mask)
            y = self._ln(x, p + ".encoder_attn_layer_norm")
            x = x + self._attn(self._lin(y, p + ".encoder_attn.q_proj"), st["ck"][l], st["cv"][l], p + ".encoder_attn", None)
            x = x + self._lin(F.relu(self._lin(self._ln(x, p + ".final_layer_norm"), p + ".fc1")), p + ".fc2")
        st["pos"] += steps
        st["tok"] += [toks[s] for s in steps]
        lp = F.log_softmax(self._ln(x, "layer_norm") @ self.w["output_projection.weight"].T, dim=-1)
        lp[:, c.pad] = float("-inf")
        for i, s in enumerate(steps):
            if s == 0:
                lp[i, c.eos] = float("-inf")  # min_len = 1
            if s >= max_len:  # eos forced
                keep = lp[i, c.eos].clone()
                lp[i] = float("-inf")
                lp[i, c.eos] = keep
        return lp

    def dup_diff(self, st):
        """max over the entries that repeat an earlier (position, token) of |entry - first entry| / max |K or V|, layers >= 1"""
        first, pairs = {}, []
        for j, key in enumerate(zip(st["pos"], st["tok"])):
            if key in first:
                pairs.append((first[key], j))
            else:
                first[key] = j
        if not pairs:
            return None
        a, b = torch.tensor([p[0] for p in pairs]), torch.tensor([p[1] for p in pairs])
        d = 0.0
        for l in range(1, self.cfg.mt_layers):
            for kv in (st["k"][l], st["v"][l]):
                d = max(d, float((kv[b] - kv[a]).abs().max() / kv.abs().max()))
        return d


def check_tokens(ref, lp, prefix, hyp, max_len, what):
    """the engine's hypothesis of one call against the float64 log-probs of its steps; returns the near ties"""
    c = ref.cfg
    start, n = len(prefix), len(hyp)
    assert list(hyp[:start]) == list(prefix), what
    assert start <= n <= max_len, (what, start, n, max_len)
    got = list(hyp[start:]) + ([c.eos] if n < max_len else [])
    if not got:
        return 0
    top = lp[:len(got)].topk(2, dim=-1)
    want, margin = top.indices[:, 0].cpu(), (top.values[:, 0] - top.values[:, 1]).cpu()
    bad = torch.tensor(got) != want
    hard = bad & (margin >= MARGIN)
    assert not bool(hard.any()), (what, [start + int(i) for i in torch.nonzero(hard).flatten()[:10]])
    return int(bad.sum())


def check_state(ref, st, got, kernel, worst, what):
    """a read-back against the reference's state: exact counts, values within the bars"""
    assert (got["entries"], got["cross_rows"]) == (ref.entries(st), ref.rows(st)), (what, got["entries"], got["cross_rows"], ref.entries(st), ref.rows(st))
    errs = {"self_k": rel(got["self_k"], torch.stack(st["k"])), "self_v": rel(got["self_v"], torch.stack(st["v"])),
            "cross_kv": rel(got["cross_kv"], torch.stack([torch.cat([k, v], -1) for k, v in zip(st["ck"], st["cv"])]))}
    for name, err in errs.items():
        worst.add(f"{kernel}:{name}", err, what)
    assert errs["self_k"] < SELF_TOL[kernel] and errs["self_v"] < SELF_TOL[kernel], (what, kernel, errs)
    assert errs["cross_kv"] < CROSS_TOL, (what, errs)


def check_quirks(ref, st, kernel, worst, what, stale=True, dup=True):
    """the case's stale rows and duplicate entries are large enough for the state check to tell a refresh or a deduplication (the
    report's stale_min / dup_min are the smallest case values, negated)"""
    d = ref.dup_diff(st)
    worst.add("stale_min", -st["stale"], what)
    if stale:
        assert st["stale"] >= STALE_FACTOR * CROSS_TOL, (what, st["stale"])
    if dup:
        assert d is not None and d > SELF_TOL[kernel], (what, d)
        worst.add("dup_min", -d, what)


def mt_launches(e, fn):
    """(result, library launches, single-token kernel launches that produced a token) of fn()"""
    torch.cuda.synchronize()
    e.mt_time()
    l0 = e.launch_count()
    r = fn()
    torch.cuda.synchronize()
    return r, e.launch_count() - l0, e.mt_time()[1]


def call_max_len(prefix, max_new, max_len):
    return max_len if max_new == -1 else len(prefix) + max_new


# ---------------------------------------------------------------------------------------------------------------- reference (CPU)
def test_reference_matches_the_cpu_oracle():
    """IncRef64 on the CPU against StreamSpeechOracle(dtype=float64).mt_greedy_incremental over five calls (kv_off 0 .. 4): T grows,
    stays, drops below the cached rows; earlier rows change between calls (stale); the prefix is the full hypothesis, one token less and
    empty.  Tokens, every state tensor and the count of entries and rows must agree."""
    from oracle.streamspeech_oracle import StreamSpeechOracle

    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    o = StreamSpeechOracle(cfg, sd, None, None, dtype=F64)
    ref = IncRef64(cfg, sd, "cpu")
    g = torch.Generator().manual_seed(7)
    base = torch.randn(40, cfg.enc_dim, generator=g, dtype=F64)
    ost, st = o.mt_incremental_state(), ref.state()
    hyp, n_calls = None, 0
    for T, rule, max_new in ((3, None, 2), (12, "full", 2), (12, "minus1", 3), (7, "full", 1), (30, "empty", -1)):
        enc = base[:T].clone()
        enc[:min(T, ref.rows(st))] += torch.randn(min(T, ref.rows(st)), cfg.enc_dim, generator=g, dtype=F64)
        prefix = RULES[rule](hyp) if rule else []
        ml = call_max_len(prefix, max_new, 9)
        out = o.mt_greedy_incremental(ost, enc.unsqueeze(1), prefix, max_new, 9)
        assert out[-1] == cfg.eos
        hyp = out[:-1]
        lp = ref.call(st, enc, prefix, hyp[len(prefix):], ml)
        want = list(hyp[len(prefix):]) + ([cfg.eos] if len(hyp) < ml else [])
        assert lp[:len(want)].argmax(-1).tolist() == want, (T, rule)
        n_calls += 1
    for name, a, b in (("self_k", st["k"], ost["self_k"]), ("self_v", st["v"], ost["self_v"]), ("cross_k", st["ck"], ost["cross_k"]),
                       ("cross_v", st["cv"], ost["cross_v"])):
        for l in range(cfg.mt_layers):
            assert a[l].shape == b[l].shape, (name, l, a[l].shape, b[l].shape)
            assert float((a[l] - b[l]).abs().max()) < 1e-10, (name, l)
    assert ref.rows(st) == 30 and st["stale"] > 0.1
    assert ref.dup_diff(st) > 1e-3
    report("mt_incremental_reference_vs_cpu_oracle", calls=n_calls, entries=ref.entries(st), rows=ref.rows(st))


# ---------------------------------------------------------------------------------------------------------------- GPU fixtures
N_SLOTS = 34  # 33 streams for the split groups, and one slot no test uses before the slot-reuse check
FRESH_SLOT = 33


@pytest.fixture(scope="module")
def inc():
    """engine (1024 MT positions, room for 1025 encoder rows, a 34-slot pool of 7 s streams), the float64 reference on the GPU and
    1025 encoder rows of a 41 s utterance"""
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    e = Engine(cfg, sd, None, synth.make_gcmvn(cfg), max_enc_frames=1280)
    e.set_option("persistent_time", 1)  # mt_time counts the single-token kernel's launches
    e.set_chunk(8)
    feats = e.fbank(synth.make_audio(41.0, seed=41).cuda().contiguous())
    enc = e.encoder(feats.unsqueeze(0).contiguous())[0]
    assert enc.shape[0] > 1024
    e.pool_create(N_SLOTS, max_seconds=7)
    yield cfg, sd, e, IncRef64(cfg, sd, "cuda"), enc[:1025].clone()
    e.close()


class HandleCase:
    """one utterance's calls on the handle's incremental state, each checked against the float64 reference"""

    def __init__(self, e, ref, name, worst):
        self.e, self.ref, self.name, self.worst = e, ref, name, worst
        self.st, self.hyp, self.calls, self.near = ref.state(), None, 0, 0
        e.mt_incremental_reset()
        assert e.mt_incremental_state()["entries"] == 0

    def cached(self):
        return self.ref.rows(self.st)

    def call(self, enc, rule, max_new, max_len=MAX_LEN):
        prefix = RULES[rule](self.hyp) if rule and self.hyp is not None else []
        what = f"{self.name} call={self.calls} T={enc.shape[0]} prefix={len(prefix)} max_new={max_new}"
        hyp, _, n_v2 = mt_launches(self.e, lambda: self.e.mt_greedy_incremental(enc, prefix, max_new, max_len))
        assert n_v2 >= 1, what  # the single-token kernel
        ml = call_max_len(prefix, max_new, max_len)
        lp = self.ref.call(self.st, enc, prefix, hyp[len(prefix):], ml)
        self.near += check_tokens(self.ref, lp, prefix, hyp, ml, what)
        check_state(self.ref, self.st, self.e.mt_incremental_state(), "single", self.worst, what)
        self.hyp = hyp
        self.calls += 1
        return hyp


def perturb(x, n, seed):
    """O(1) noise on rows [0, n) of x, in place"""
    if n > 0:
        g = torch.Generator(device=x.device).manual_seed(seed)
        x[:n] += torch.randn(n, x.shape[1], generator=g, device=x.device)


def stream_encoder_calls(e, wav, seg_ms):
    """the handle's streaming encoder over wav in seg_ms segments: yields the encoder rows [0, T) of each step (a copy)"""
    c = seg_ms // 40
    e.set_chunk(c, min(c, 16))
    e.encoder_stream_reset()
    n = 16 * seg_ms
    buf = torch.zeros(e.encoder_out_frames(e.num_fbank_frames(len(wav))) + 8, e.cfg.enc_dim, device="cuda")
    wd = wav.cuda().contiguous()
    for i in range(n, len(wav) + n, n):
        feats = e.fbank(wd[:min(i, len(wav))].contiguous())
        T, _ = e.encoder_stream_step(feats, buf)
        if T > 0:
            yield buf[:T].clone()


@gpu
@pytest.mark.parametrize("seg_ms,seconds,rules,max_news", [
    (160, 6.9, ("full",), (1, 2, 5)),  # the agent's rule: kv_off + 1 per call, >= 40 calls
    (320, 5.1, ("minus1", "full", "minus2", "empty", "full"), (2, 5, 1)),
])
def test_handle_on_streaming_encoder_rows_vs_fp64(inc, seg_ms, seconds, rules, max_news):
    """ss_mt_greedy_incremental on the provisional rows of ss_encoder_stream_step, one call per segment, the last with
    max_new_tokens = -1: the provisional tail changes between calls, so early cross rows are really stale"""
    cfg, sd, e, ref, _ = inc
    worst = Worst()
    case = HandleCase(e, ref, f"stream {seg_ms} ms", worst)
    encs = list(stream_encoder_calls(e, synth.make_audio(seconds, seed=500 + seg_ms), seg_ms))
    for i, enc in enumerate(encs):
        last = i == len(encs) - 1
        case.call(enc, None if i == 0 else rules[i % len(rules)], -1 if last else max_news[i % len(max_news)])
    e.set_chunk(8)
    if seg_ms == 160:
        assert case.calls >= 41
    check_quirks(ref, case.st, "single", worst, case.name)
    report("mt_incremental_stream_fp64", seg_ms=seg_ms, calls=case.calls, entries=ref.entries(case.st), rows=ref.rows(case.st),
           stale=case.st["stale"], dup=ref.dup_diff(case.st), near_ties=case.near, **worst.as_dict(), card=card())
    e.mt_incremental_reset()


# (T, commit rule, max_new_tokens) of the forced-staleness case on the handle: a first call at T = 1, a call without new rows, calls with
# T below the cached rows, the empty prefix on a non-empty state, calls at Tk = 1024
HANDLE_SCHEDULE = [(1, None, 2), (40, "full", 1), (40, "full", 5), (25, "minus1", 2), (200, "minus2", 5), (200, "empty", 2),
                   (700, "full", 1), (1024, "full", 5), (1000, "minus1", 2), (1024, "full", -1)]


@gpu
def test_handle_forced_staleness_edges_and_refusals_vs_fp64(inc):
    """The schedule above with O(1) noise on every row an earlier call saw; then the refusals, each with the read-back and the launch
    counter unchanged: Tk = 1025 (SS_ERR_STATE: the single-token kernel keeps at most 1024 cross scores), max_len + kv_off + 2 =
    max_mt_positions + 1 (SS_ERR_CAPACITY) and a prefix longer than the state (SS_ERR_STATE); then the largest search that fits."""
    cfg, sd, e, ref, enc = inc
    worst = Worst()
    case = HandleCase(e, ref, "forced stale", worst)
    for i, (T, rule, max_new) in enumerate(HANDLE_SCHEDULE):
        x = enc[:T].clone()
        perturb(x, min(T, case.cached()), 100 + i)
        case.call(x, rule, max_new)
    check_quirks(ref, case.st, "single", worst, case.name)
    lib, h, st = e.lib, e._h, e._stream()
    I32, I64 = ctypes.c_int32, ctypes.c_int64
    P = e.max_mt_positions
    before = e.mt_incremental_state()
    hyp = case.hyp
    kv_off = before["entries"] - len(hyp)
    assert kv_off > 0
    out, n_one = (I64 * P)(), I32(0)
    pf = (I64 * (before["entries"] + 1))(*(hyp + [cfg.unk + 1] * (before["entries"] + 1 - len(hyp))))
    x = enc[:1025].contiguous()
    refusals = [(x, len(hyp), -1, MAX_LEN, SS_ERR_STATE, b"persistent MT kernel"),
                (enc[:1024].contiguous(), len(hyp), -1, P - 1 - kv_off, SS_ERR_CAPACITY, b"needs %d self-attention entries" % (P + 1)),
                (enc[:1024].contiguous(), before["entries"] + 1, -1, before["entries"] + 1, SS_ERR_STATE, b"shorter than the prefix")]
    for xx, n_pf, mn, ml, code, msg in refusals:
        torch.cuda.synchronize()
        l0 = e.launch_count()
        rc = lib.ss_mt_greedy_incremental(h, st, xx.data_ptr(), xx.shape[0], pf, n_pf, mn, ml, out, P, ctypes.byref(n_one))
        assert rc == code and msg in lib.ss_last_error(h), (rc, code, lib.ss_last_error(h))
        assert e.launch_count() == l0
        after = e.mt_incremental_state()
        assert all(torch.equal(after[k], before[k]) for k in ("self_k", "self_v", "cross_kv")) and after["entries"] == before["entries"]
    # one entry less is accepted, and continues the state as the reference does
    case.call(enc[:1024].contiguous(), "full", -1, P - 2 - kv_off)
    report("mt_incremental_handle_forced_stale_fp64", calls=case.calls, entries=ref.entries(case.st), kv_off=kv_off, stale=case.st["stale"],
           dup=ref.dup_diff(case.st), near_ties=case.near, **worst.as_dict(), card=card())
    e.mt_incremental_reset()


class PoolCase:
    """pool slots driven through ss_pool_step and ss_pool_mt_greedy_incremental, every stream checked against its own float64 state"""

    def __init__(self, e, ref, worst):
        self.e, self.ref, self.worst = e, ref, worst
        self.st, self.hyp, self.T, self.calls, self.wav, self.pushed = {}, {}, {}, {}, {}, {}
        self.near, self.routes = 0, {"batched": 0, "single": 0}

    def start(self, slot, wav, chunk):
        self.e.pool_reset(slot)
        assert self.e.mt_incremental_state(slot)["entries"] == 0 and self.e.mt_incremental_state(slot)["cross_rows"] == 0
        self.e.pool_set_chunk(slot, chunk, chunk)
        self.st[slot], self.hyp[slot], self.T[slot], self.calls[slot] = self.ref.state(), None, 0, 0
        self.wav[slot], self.pushed[slot] = wav, 0

    def push(self, slots, seconds):
        """push the next `seconds` of each slot's utterance, then one ss_pool_step over them"""
        slots = [s for s in slots if self.pushed[s] < len(self.wav[s])]
        for s in slots:
            n = min(int(seconds * 16000), len(self.wav[s]) - self.pushed[s])
            self.e.pool_push_audio(s, self.wav[s][self.pushed[s]:self.pushed[s] + n].contiguous())
            self.pushed[s] += n
        if slots:
            for s, r in zip(slots, self.e.pool_step(slots, ctc_heads=0)):
                self.T[s] = r["T"]

    def call(self, slots, rules, max_news, min_rows=2, stale_seed=None, max_lens=None):
        """one ss_pool_mt_greedy_incremental over `slots`; stale_seed: O(1) noise on the rows each slot's earlier calls saw first"""
        e, ref = self.e, self.ref
        max_lens = max_lens or [MAX_LEN] * len(slots)
        prefixes = [RULES[r](self.hyp[s]) if r and self.hyp[s] is not None else [] for s, r in zip(slots, rules)]
        encs = []
        for i, s in enumerate(slots):
            if stale_seed is not None:
                perturb(e.pool_encoder_rows(s, self.T[s]), min(self.T[s], ref.rows(self.st[s])), stale_seed + s)  # (pool memory)
            encs.append(e.pool_encoder_rows(s, self.T[s]).clone())
        e.set_option("mt_batch_min_rows", min_rows)
        out, _, n_v2 = mt_launches(e, lambda: e.pool_mt_greedy_incremental(slots, prefixes, max_news, max_lens))
        e.set_option("mt_batch_min_rows", 2)
        groups = [slots[g:g + BATCH_ROWS] for g in range(0, len(slots), BATCH_ROWS)]
        single = [s for g in groups if len(g) < min_rows for s in g]
        assert (n_v2 > 0) == bool(single) and n_v2 >= len(single), (len(slots), min_rows, n_v2)  # the route of every group
        for i, s in enumerate(slots):
            kernel = "single" if s in single else "batched"
            self.routes[kernel] += 1
            what = f"slot={s} call={self.calls[s]} T={self.T[s]} prefix={len(prefixes[i])} max_new={max_news[i]} group={len(slots)} {kernel}"
            ml = call_max_len(prefixes[i], max_news[i], max_lens[i])
            lp = ref.call(self.st[s], encs[i], prefixes[i], out[i][len(prefixes[i]):], ml)
            self.near += check_tokens(ref, lp, prefixes[i], out[i], ml, what)
            check_state(ref, self.st[s], e.mt_incremental_state(s), kernel, self.worst, what)
            self.hyp[s] = out[i]
            self.calls[s] += 1
        return out


RULE_CYCLE = ("full", "full", "minus1", "minus2", "empty", "full")
NEW_CYCLE = (1, 2, 5)
GROUP_SIZES = (2, 5, 17, 32, 1, 9, 24, 33, 3)  # 33: a group of 32 and a tail group of 1


@gpu
def test_pool_groups_routes_vs_fp64(inc):
    """33 streams of 2.6 .. 4.6 s (160 ms and 320 ms chunks) that start in four waves, 160 ms per round.  Each round one group of
    GROUP_SIZES decodes: groups of 2 .. 32 on the batched kernel mix slots on different calls (kv_off 0 .. k), fresh slots, slots not
    stepped this round (no new rows) and different T; a group of 1 runs on the single-token kernel, 33 streams as 32 + 1; one round runs
    all 33 with mt_batch_min_rows = 33 (every stream on the single-token kernel).  Every other round forces stale rows through the pool
    view.  The last round finishes every stream (max_new_tokens = -1)."""
    cfg, sd, e, ref, _ = inc
    worst = Worst()
    pc = PoolCase(e, ref, worst)
    slots = list(range(33))
    for s in slots:
        pc.start(s, synth.make_audio(2.6 + 0.25 * (s % 9), seed=700 + s), 4 if s % 2 == 0 else 8)
    rounds = 0
    for r in range(len(GROUP_SIZES) + 4):
        started = [s for s in slots if s % 4 <= r]
        pc.push([s for s in started if (s + r) % 5 != 0], 0.16)  # (s + r) % 5 == 0: no new rows this round
        ready = [s for s in started if pc.T[s] > 0]
        size = GROUP_SIZES[r % len(GROUP_SIZES)] if r < len(GROUP_SIZES) else (33 if r == len(GROUP_SIZES) else 6)
        k = (5 * r) % len(ready)
        group = (ready[k:] + ready[:k])[:size]
        min_rows = 33 if r == len(GROUP_SIZES) else 2
        pc.call(group, [RULE_CYCLE[(s + pc.calls[s]) % len(RULE_CYCLE)] for s in group], [NEW_CYCLE[(s + r) % 3] for s in group], min_rows,
                stale_seed=1000 * r if r % 2 else None)
        rounds += 1
    pc.push(slots, 10.0)  # the rest of every utterance, then the finishing call of all 33 (32 + 1)
    pc.call(slots, ["full"] * 33, [-1] * 33, stale_seed=99000)
    kv = [pc.calls[s] for s in slots]
    assert max(kv) >= 6 and min(kv) >= 2
    for s in slots:  # (the finishing call forced stale rows and fed a duplicate entry on every slot)
        check_quirks(ref, pc.st[s], "batched", worst, f"slot {s}")
    assert pc.routes["batched"] > 0 and pc.routes["single"] >= 33
    report("mt_incremental_pool_groups_fp64", rounds=rounds + 1, calls=sum(kv), routes=pc.routes, near_ties=pc.near, **worst.as_dict(),
           card=card())


def gemm_route(M, rows_per_sample, umma, min_rows=128):
    """the cross-K/V projection's GEMM (linear() in engine_run.cu): the skinny kernel up to 64 rows, the wgmma kernel (umma_linear >= 12)
    at >= umma_min_rows rows per sample, the fp32 kernel otherwise"""
    if M <= 64:
        return "skinny"
    return "wgmma" if umma >= 12 and rows_per_sample >= min_rows else "fp32"


@gpu
def test_pool_cross_projection_gemm_routes_vs_fp64(inc):
    """Bg * max_new new encoder rows on every route of the group's cross-K/V projection (<= 64 rows skinny, 65 .. 127 fp32, >= 128 rows
    per stream wgmma) under umma_linear 13 and 0: pairs of fresh slots whose first call projects 30, 50 or 140 rows, then a second call
    after more audio, with forced stale rows, projects 8 .. 50 more"""
    cfg, sd, e, ref, _ = inc
    worst, seen = Worst(), {}
    for umma in (13, 0):
        e.set_option("umma_linear", umma)
        for first_s, more_s in ((1.25, 2.0), (2.05, 0.5), (5.65, 0.3)):
            pc = PoolCase(e, ref, worst)
            pair = [0, 1]
            for s in pair:
                pc.start(s, synth.make_audio(first_s + more_s, seed=800 + s + int(10 * first_s)), 8)
            pc.push(pair, first_s)
            for step in range(2):
                news = [pc.T[s] - ref.rows(pc.st[s]) for s in pair]
                M = len(pair) * max(news)
                seen.setdefault(umma, {}).setdefault(gemm_route(M, max(news), umma), []).append(M)
                pc.call(pair, ["full", "full"], [2, 5], stale_seed=500 + step if step else None)
                pc.push(pair, more_s)
        e.set_option("umma_linear", 13)
    assert set(seen[13]) == {"skinny", "fp32", "wgmma"} and set(seen[0]) == {"skinny", "fp32"}, seen
    report("mt_incremental_cross_gemm_routes_fp64", rows_per_route=seen, **worst.as_dict(), card=card())


@gpu
def test_pool_slot_reuse_equals_a_fresh_slot(inc):
    """a slot reused after ss_pool_reset reads back {0, 0}, and its next utterance (three calls, in one group with a slot no call has
    used) gives the fresh slot's tokens and state"""
    cfg, sd, e, ref, _ = inc
    worst = Worst()
    used = 3
    e.pool_reset(used)
    got = e.mt_incremental_state(used)
    assert (got["entries"], got["cross_rows"]) == (0, 0)
    pc = PoolCase(e, ref, worst)
    wav = synth.make_audio(1.9, seed=901)
    for s in (used, FRESH_SLOT):
        pc.start(s, wav, 8)
    for k in range(3):
        pc.push([used, FRESH_SLOT], 0.64)
        pc.call([used, FRESH_SLOT], ["full", "full"], [2, 2] if k < 2 else [-1, -1])
        assert pc.hyp[used] == pc.hyp[FRESH_SLOT]
        a, b = e.mt_incremental_state(used), e.mt_incremental_state(FRESH_SLOT)
        assert (a["entries"], a["cross_rows"]) == (b["entries"], b["cross_rows"])
        for key in ("self_k", "self_v", "cross_kv"):
            assert rel(a[key], b[key].double()) < 1e-6, key
    report("mt_incremental_slot_reuse", **worst.as_dict())


# ---------------------------------------------------------------------------------------------------------------- long caches (no-eos checkpoint)
LONG_POSITIONS = 2304
BOUNDARY_ENTRIES = (1023, 1024, 1025, 2 * 1024 + 1)


@pytest.fixture(scope="module")
def noeos():
    """an engine with room for 2049 entries on the checkpoint whose eos row is zero (its searches fill max_len), an 8-slot pool and the
    float64 reference"""
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    for k in ("target_unigram_decoder.embed_tokens.weight", "target_unigram_decoder.output_projection.weight"):
        sd[k] = sd[k].clone()
        sd[k][cfg.eos] = 0.0
    e = Engine(cfg, sd, None, synth.make_gcmvn(cfg), max_mt_positions=LONG_POSITIONS)
    e.set_option("persistent_time", 1)
    e.set_chunk(8, 8)
    e.pool_create(8, max_seconds=3)
    yield cfg, e, IncRef64(cfg, sd, "cuda")
    e.close()


@gpu
def test_long_caches_with_kv_off_vs_fp64(noeos):
    """Three calls per stream ((2 new tokens), (3 more), then -1) with kv_off = 2 at the finishing call, whose cache ends at 1023, 1024,
    1025 and 2049 entries (attend_head_long above 1024), on the single-token kernel (handle) and the batched kernel (pool: the four
    lengths and four short streams in one group); stale rows forced before the second and third call"""
    cfg, e, ref = noeos
    worst = Worst()
    pc = PoolCase(e, ref, worst)
    slots = list(range(8))
    for s in slots:
        pc.start(s, synth.make_audio(1.6 + 0.08 * s, seed=950 + s), 8)
    pc.push(slots, 3.0)
    mls = [E - 3 for E in BOUNDARY_ENTRIES] + [40 + 3 * s for s in range(4)]
    for k, (rule, mn) in enumerate(((None, 2), ("full", 3), ("full", -1))):
        pc.call(slots, [rule] * 8, [mn] * 8, stale_seed=300 * k if k else None, max_lens=mls)
    for i, E in enumerate(BOUNDARY_ENTRIES):
        assert ref.entries(pc.st[i]) == E and e.mt_incremental_state(i)["entries"] == E
        check_quirks(ref, pc.st[i], "batched", worst, f"pool E={E}")
    # the same four lengths on the handle (single-token kernel), on the slots' rows
    near_handle = 0
    x0 = e.pool_encoder_rows(0, pc.T[0]).clone()
    for E in BOUNDARY_ENTRIES:
        case = HandleCase(e, ref, f"handle E={E}", worst)
        for k, (rule, mn) in enumerate(((None, 2), ("full", 3), ("full", -1))):
            x = x0.clone()
            perturb(x, min(x.shape[0], case.cached()), 400 * k + E)
            case.call(x, rule, mn, E - 3)
        assert ref.entries(case.st) == E and e.mt_incremental_state()["entries"] == E
        check_quirks(ref, case.st, "single", worst, case.name)
        near_handle += case.near
    e.mt_incremental_reset()
    report("mt_incremental_long_caches_fp64", entries=list(BOUNDARY_ENTRIES), near_ties={"pool": pc.near, "handle": near_handle},
           **worst.as_dict(), card=card())


# ---------------------------------------------------------------------------------------------------------------- isolation of the state
def same_state(a, b):
    return (a["entries"], a["cross_rows"]) == (b["entries"], b["cross_rows"]) and all(torch.equal(a[k], b[k]) for k in ("self_k", "self_v", "cross_kv"))


@gpu
def test_state_is_isolated_from_the_other_searches(inc):
    """Between two incremental calls on the handle: ss_mt_greedy_batch, ss_mt_features_batch, ss_mt_beam_batch, ss_pool_mt_greedy and
    ss_pool_mt_greedy_incremental on other slots leave the handle's read-back bit-identical, and its next call matches the reference.
    Between two calls on a pool slot, incremental calls on other slots and on the handle leave the slot's read-back bit-identical."""
    cfg, sd, e, ref, enc = inc
    worst = Worst()
    case = HandleCase(e, ref, "isolation", worst)
    case.call(enc[:60].contiguous(), None, 3)
    pc = PoolCase(e, ref, worst)
    for s in range(6):
        pc.start(s, synth.make_audio(1.5, seed=600 + s), 8)
    pc.push(list(range(6)), 1.2)
    pc.call([4], [None], [2])  # the pool slot whose state is watched below (a group of 1: the single-token kernel over the slot)
    held, held_slot = e.mt_incremental_state(), e.mt_incremental_state(4)
    batch = torch.zeros(2, 120, cfg.enc_dim, device="cuda")
    batch[0], batch[1, :80] = enc[:120], enc[200:280]
    others = {
        "ss_mt_greedy_batch": lambda: e.mt_greedy_batch(batch, [120, 80], 30),
        "ss_mt_features_batch": lambda: e.mt_features_batch(batch, [120, 80], [[cfg.eos, 11, 12], [cfg.eos, 13, cfg.pad]]),
        "ss_mt_beam_batch": lambda: e.mt_beam_batch(batch, [120, 80], 2, 30),
        "ss_pool_mt_greedy": lambda: e.pool_mt_greedy([0, 1], [None, [15, 16]], [3, 2], 30),
        "ss_pool_mt_greedy_incremental": lambda: pc.call([2, 3], [None, None], [2, 3]),
    }
    for name, fn in others.items():
        fn()
        torch.cuda.synchronize()
        assert same_state(e.mt_incremental_state(), held), name
        assert same_state(e.mt_incremental_state(4), held_slot), name
    case.call(enc[:90].contiguous(), "full", 2)  # the handle continues its own state
    assert same_state(e.mt_incremental_state(4), held_slot)
    pc.call([5], [None], [2])
    assert same_state(e.mt_incremental_state(4), held_slot)
    pc.push([4], 0.3)
    pc.call([4], ["full"], [3])  # and the slot its own
    check_quirks(ref, case.st, "single", worst, case.name, stale=False)
    e.mt_incremental_reset()
    report("mt_incremental_isolation", checked=list(others), **worst.as_dict())


@gpu
def test_mt_greedy_between_incremental_calls_is_refused(inc):
    """ss_mt_greedy and ss_mt_features write the caches the handle's incremental state lives in: after either, on a non-empty state, the
    next ss_mt_greedy_incremental is SS_ERR_STATE before any launch, naming ss_mt_incremental_reset; the reset clears it.  On an empty
    state they are harmless."""
    cfg, sd, e, ref, enc = inc
    lib, h, st = e.lib, e._h, e._stream()
    x = enc[:50].contiguous()
    out, n_one = (ctypes.c_int64 * e.max_mt_positions)(), ctypes.c_int32(0)
    for name, other in (("ss_mt_greedy", lambda: e.mt_greedy(x, None, 3)), ("ss_mt_features", lambda: e.mt_features(x, [cfg.eos, 21, 22]))):
        e.mt_incremental_reset()
        other()  # an empty state: nothing to lose
        h1 = e.mt_greedy_incremental(x, None, 2, MAX_LEN)
        small = (ctypes.c_int32 * 4)()  # the read-back refuses a buffer below the whole state, and a slot outside the pool
        assert lib.ss_debug_copy(h, b"mt_inc_state", small, ctypes.sizeof(small)) == -1 and b"needs" in lib.ss_last_error(h)
        assert lib.ss_debug_copy(h, b"pool_mt_inc_state:%d" % N_SLOTS, small, 8) == -1 and b"bad pool slot" in lib.ss_last_error(h)
        other()
        pf = (ctypes.c_int64 * len(h1))(*h1)
        torch.cuda.synchronize()
        l0 = e.launch_count()
        rc = lib.ss_mt_greedy_incremental(h, st, x.data_ptr(), 50, pf, len(h1), 2, MAX_LEN, out, e.max_mt_positions, ctypes.byref(n_one))
        assert rc == SS_ERR_STATE and b"ss_mt_incremental_reset" in lib.ss_last_error(h), (name, rc, lib.ss_last_error(h))
        assert e.launch_count() == l0, name
        e.mt_incremental_reset()
        assert e.mt_greedy_incremental(x, None, 2, MAX_LEN) == h1
    e.mt_incremental_reset()
