"""GPU: every route of the MT decoder against a float64 reference of the same operation, at the shapes where its kernels split work.

Five code paths compute MT tokens and features:
- `mt_prefix_persistent_kernel` (kernels_persist_mtp.cu) teacher-forces a prefix of up to 64 rows: GEMMs in 16-row blocks, attention
  in tasks of 8 query rows, values in rounds of 32 keys;
- `mt_decode_persistent_kernel_v2` (kernels_persist_mt.cu) runs the single-token steps: values in rounds of 128 keys, at most 1024
  cross-attention scores;
- `mt_decode_batch_kernel` (kernels_persist_mtb.cu) runs groups of up to 32 searches (ss_mt_greedy_batch, ss_pool_mt_greedy);
- the per-op decoder (mt_forward / dec_layer) serves ss_mt_features, prefixes longer than 64 and persistent_mt = 0;
- the per-op teacher-forced pass with a sample axis serves ss_mt_features_batch and ss_pool_mt_greedy's prefix rows (ragged prefixes
  as masked pad tails).

The reference is the decoder of StreamSpeechOracle (oracle/streamspeech_oracle.py, pinned to the reference's fixtures by
test_oracle_golden.py) restated as float64 torch operations on the GPU; test_reference_matches_the_cpu_oracle checks it against the
oracle's own float64 mt_features on the CPU once.  Both sides get the same fp32 encoder rows: prefixes of one engine encoder output of a
41 s utterance, so T reaches 1024.  The float64 side teacher-forces [eos] + hypothesis in one pass and gives the features of every
position and the masked log-probs (pad always masked, eos banned at step 0, eos forced at max_len).  Tokens follow the margin rule of
test_long_utterance_fp64.py, generalised to searches with a prefix: at every position >= n_prefix an engine token may differ from the
float64 arg-max only where the float64 top-2 margin is below MARGIN; such near ties are counted and reported.

Cases follow a covering design rather than the full product: every prefix length runs at two to four encoder lengths and every encoder
length with two to four prefix lengths.  The route that ran is proved from the launch counter (ss_launch_count) and the single-token
kernel's launch count (mt_time): the prefix kernel is one launch, the per-op prefix dozens.  The measured maxima, the case of each
maximum and the near-tie counts are printed as one JSON line per test (`pytest -s`) before the bars are asserted.
"""
import json
import math

import pytest
import torch
import torch.nn.functional as F

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

pytestmark = pytest.mark.gpu

torch.set_grad_enabled(False)
F64 = torch.float64
MARGIN = 1e-4
# Max-abs bars against float64, from the largest error measured on an H100 80GB HBM3 (700 W) over every case of this file (in the
# comments).  The features are the final LayerNorm's output with the synthetic checkpoint's gain of 64 (rms 65, up to 244), so fp32
# arithmetic alone leaves ~1e-4: ten times the measured error would exceed the project's 2e-4 bar on every route.  Routes that measure
# <= 1.5e-4 keep that bar; the three that measure above it get about 2.5x their maximum.  Linears of >= umma_min_rows rows per sample
# run on the bf16x6 tensor-core GEMM by default (umma_linear = 13), which raises the error of ss_mt_features at 1024 rows fivefold.
FEAT_TOL = {
    "prefix_kernel": 2e-4,  # 1.04e-4 (prefix 48, T = 1000)
    "per_op_prefix": 2e-4,  # 9.5e-5 (prefix 65, T = 1024)
    "per_op": 2e-4,  # 9.5e-5 (prefix 65, T = 1024)
    "whole_table": 2e-4,  # 1.05e-4 (1023 rows, prefix 64, T = 1000)
    "pool": 2e-4,  # 1.39e-4 (prefix 70, T = 30)
    "features_fp32": 2e-4,  # 1.52e-4 (S = 1024, T = 1000)
    "features_tc": 2e-3,  # 8.0e-4 (S = 1024, T = 129)
    "features_batch_fp32": 5e-4,  # 1.86e-4 (T = 988, pad tail 3)
    "features_batch_tc": 6e-4,  # 2.38e-4 (T = 988, pad tail 3)
}
LOGIT_TOL = 5e-5  # ss_mt_features' last-row logits: 5.0e-6 (fp32 linears), 3.4e-6 (tensor-core linears)
# umma_linear: the engine's default (13: linears of >= umma_min_rows rows per sample on the bf16x6 tensor-core GEMM) and 0 (fp32 kernels)
LINEAR_ROUTINGS = {"tc": 13, "fp32": 0}
MAX_LEN_B = 200
UTTERANCE_S = 41.0
UNIT_BATCH_ROWS = 32768  # SS_UNIT_BATCH_ROWS (include/streamspeech_b200.h): samples per ss_mt_features_batch group = that / (S * rate)
BATCH_ROWS = 32  # MT_BATCH_MAX_ROWS: rows per launch of the batched search kernel
PREFIX_KERNEL_ROWS = 64  # the prefix kernel takes [eos] + prefix[:-1], at most 64 rows
PER_OP_PREFIX_LAUNCHES = 20  # the per-op prefix pass is an embedding, about ten launches per layer and a final LayerNorm

# ss_mt_greedy: (prefix length, encoder rows T, max_new_tokens, ending) with ending "eos" or "max_len" (eos forced)
GREEDY_CASES = [
    (0, 1, -1, "eos"), (0, 1000, -1, "eos"), (0, 128, 5, "max_len"),
    (1, 2, 1, "max_len"), (1, 1024, -1, "eos"),
    (2, 15, -1, "eos"), (2, 257, 0, "max_len"),
    (7, 16, 5, "max_len"), (7, 1023, -1, "eos"),
    (8, 17, -1, "eos"), (8, 129, 1, "max_len"),
    (9, 31, 0, "max_len"), (9, 255, -1, "eos"),
    (15, 33, -1, "eos"), (15, 1024, 5, "max_len"),
    (16, 127, -1, "eos"), (16, 1, 1, "max_len"), (16, 1023, 0, "max_len"),
    (17, 128, -1, "eos"), (17, 2, 5, "max_len"),
    (31, 129, 5, "max_len"), (31, 15, -1, "eos"),
    (32, 255, 1, "max_len"), (32, 16, -1, "eos"), (32, 1000, 5, "max_len"),
    (33, 257, -1, "eos"), (33, 17, 0, "max_len"),
    (48, 1000, 1, "max_len"), (48, 31, -1, "eos"),
    (63, 1023, -1, "eos"), (63, 33, 5, "max_len"),
    (64, 1024, 0, "max_len"), (64, 127, -1, "eos"), (64, 1, 5, "max_len"),
    (65, 1, -1, "eos"), (65, 128, 5, "max_len"), (65, 1024, 1, "max_len"),
    (100, 2, 5, "max_len"), (100, 255, -1, "eos"),
]
OWN_PREFIX_T = 1000  # one more case continues the first half of the engine's own hypothesis at this T
# route: engine options (both set, so that a route does not depend on the environment's defaults)
ROUTES = {
    "prefix_kernel": dict(persistent_mt=1, persistent_mt_prefix=1),
    "per_op_prefix": dict(persistent_mt=1, persistent_mt_prefix=0),
    "per_op": dict(persistent_mt=0, persistent_mt_prefix=1),
}


def report(name, **kw):
    print(json.dumps({"test": name, **kw}))


def maxdiff(a, b):
    return float((a.double() - b.to(a.device).double()).abs().max()) if a.numel() else 0.0


def set_route(e, route):
    for k, v in ROUTES[route].items():
        e.set_option(k, v)


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
        return {k: {"max_abs": v, "case": c} for k, (v, c) in self.v.items()}


class Ref64:
    """StreamSpeechOracle.mt_features (TransformerDecoderBase, pre-LN, 4 layers) in float64 on the GPU: the weights are the fp32
    checkpoint's, converted; the position table is the oracle's fp32 table, converted"""

    def __init__(self, cfg, sd):
        from oracle.streamspeech_oracle import sinusoidal_table

        self.cfg = cfg
        pfx = "target_unigram_decoder."
        self.w = {k[len(pfx):]: v.float().to("cuda", F64) for k, v in sd.items() if k.startswith(pfx) and v.is_floating_point()}
        self.table = sinusoidal_table(2048 + cfg.pad + 2, cfg.mt_dim, cfg.pad).to("cuda", F64)
        self.out_w = self.w["output_projection.weight"]

    def _lin(self, x, name):
        return F.linear(x, self.w[name + ".weight"], self.w.get(name + ".bias"))

    def _ln(self, x, name):
        return F.layer_norm(x, (x.shape[-1],), self.w[name + ".weight"], self.w[name + ".bias"], 1e-5)

    def _attn(self, x, kv, name, mask):
        H = self.cfg.mt_heads
        hd = x.shape[-1] // H
        q = (self._lin(x, name + ".q_proj") * hd ** -0.5).view(-1, H, hd).transpose(0, 1)
        k = self._lin(kv, name + ".k_proj").view(-1, H, hd).transpose(0, 1)
        v = self._lin(kv, name + ".v_proj").view(-1, H, hd).transpose(0, 1)
        w = q @ k.transpose(1, 2)
        if mask is not None:
            w = w.masked_fill(mask, float("-inf"))
        o = (torch.softmax(w, dim=-1) @ v).transpose(0, 1).reshape(x.shape)
        return self._lin(o, name + ".out_proj")

    def features(self, tokens, enc):
        """tokens [L] (pads only as a tail), enc [T, enc_dim] -> final-LN features [L, mt_dim] (float64)"""
        c = self.cfg
        t = torch.as_tensor(list(tokens), dtype=torch.long, device="cuda")
        L = t.numel()
        keep = t.ne(c.pad)
        pos = torch.cumsum(keep.long(), 0) * keep.long() + c.pad  # make_positions
        x = math.sqrt(c.mt_dim) * self.w["embed_tokens.weight"][t] + self.table[pos]
        mask = torch.triu(torch.ones(L, L, dtype=torch.bool, device="cuda"), 1) | ~keep[None, :]
        enc = enc.to("cuda", F64)
        for i in range(c.mt_layers):
            p = f"layers.{i}"
            y = self._ln(x, p + ".self_attn_layer_norm")
            x = x + self._attn(y, y, p + ".self_attn", mask)
            x = x + self._attn(self._ln(x, p + ".encoder_attn_layer_norm"), enc, p + ".encoder_attn", None)
            x = x + self._lin(F.relu(self._lin(self._ln(x, p + ".final_layer_norm"), p + ".fc1")), p + ".fc2")
        return self._ln(x, "layer_norm")

    def lprobs(self, feats, max_len=None):
        """masked log-probs of the search (sequence_generator): pad never, eos not at step 0, only eos at step max_len"""
        c = self.cfg
        lp = F.log_softmax(feats @ self.out_w.T, dim=-1)
        lp[:, c.pad] = float("-inf")
        lp[0, c.eos] = float("-inf")
        if max_len is not None and max_len < lp.shape[0]:
            keep = lp[max_len, c.eos].clone()
            lp[max_len] = float("-inf")
            lp[max_len, c.eos] = keep
        return lp


def check_search(ref, enc, hyp, n_prefix, max_len, what):
    """hyp = the engine's hypothesis (prefix included, eos excluded) of a search with this prefix length and max_len.  Every token at
    positions >= n_prefix, and the eos after the last one unless it was forced at max_len, must be the float64 arg-max wherever the
    float64 top-2 margin is at least MARGIN.  Returns (float64 features of [eos] + hyp, near ties)."""
    c = ref.cfg
    n = len(hyp)
    assert n_prefix <= n <= max_len, (what, n_prefix, n, max_len)
    f64 = ref.features([c.eos] + list(hyp), enc)
    lp = ref.lprobs(f64, max_len)
    got = list(hyp[n_prefix:]) + ([c.eos] if n < max_len else [])
    if not got:
        return f64, 0
    top = lp[n_prefix:n_prefix + len(got)].topk(2, dim=-1)
    want, margin = top.indices[:, 0].cpu(), (top.values[:, 0] - top.values[:, 1]).cpu()
    bad = torch.tensor(got) != want
    hard = bad & (margin >= MARGIN)
    assert not bool(hard.any()), (what, [n_prefix + int(i) for i in torch.nonzero(hard).flatten()[:10]])
    return f64, int(bad.sum())


def random_tokens(cfg, n, g):
    return torch.randint(cfg.unk + 1, cfg.tgt_vocab, (n,), generator=g).tolist()


def launches(e, fn):
    """(result, library launches, single-token kernel launches that produced a token) of fn()"""
    torch.cuda.synchronize()
    e.mt_time()
    l0 = e.launch_count()
    r = fn()
    torch.cuda.synchronize()
    return r, e.launch_count() - l0, e.mt_time()[1]


def v2_launches(start, max_new, max_len, n_out, fed):
    """launches of the single-token kernel in ss_mt_greedy's burst loop (engine_run.cu) for a search that fed `fed` rows before the
    loop (the prefix kernel's rows, else 0) and returned n_out tokens (eos produced at step n_out when n_out < max_len)"""
    burst = max(1, max_new) if max_new >= 0 else 16
    step, count, done = start, 0, False
    while not done:
        first, enq = step, 0
        while step <= max_len and enq < burst:
            if step + 1 - fed == 1:
                cnt = min(max_len - step + 1, burst - enq)
                count += 1
                fed = step + cnt
                done = step + cnt - 1 >= max_len
                step, enq = step + cnt, enq + cnt
                break
            fed = step + 1  # the per-op pass over rows fed .. step
            if step >= max_len:
                done, step = True, step + 1
                break
            step, enq = step + 1, enq + 1
        produced = step - first - (1 if done else 0)
        if produced > 0 and first <= n_out < first + produced and n_out < max_len:
            done = True
        done = done or step > max_len
    return count


@pytest.fixture(scope="module")
def mt():
    """engine, float64 reference and the fp32 encoder rows [1024, enc_dim] both sides get (the first 1024 rows of a 41 s utterance)"""
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    gc = synth.make_gcmvn(cfg)
    e = Engine(cfg, sd, None, gc, max_enc_frames=1280)  # 41 s are 1025 encoder rows
    e.set_chunk(8)
    e.set_option("persistent_time", 1)  # mt_time counts the single-token kernel's launches
    wav = synth.make_audio(UTTERANCE_S, seed=41)
    feats = e.fbank(wav.cuda().contiguous())
    enc = e.encoder(feats.unsqueeze(0).contiguous())[0]
    assert enc.shape[0] > 1024
    enc = enc[:1024].clone()
    assert bool(torch.isfinite(enc).all())
    yield cfg, sd, e, Ref64(cfg, sd), enc
    e.close()


def test_reference_matches_the_cpu_oracle(mt):
    """the GPU float64 decoder against StreamSpeechOracle(dtype=float64).mt_features on the CPU: a pad tail and 37 encoder rows"""
    from oracle.streamspeech_oracle import StreamSpeechOracle

    cfg, sd, e, ref, enc = mt
    g = torch.Generator().manual_seed(3)
    toks = [cfg.eos] + random_tokens(cfg, 9, g) + [cfg.pad] * 2
    o = StreamSpeechOracle(cfg, sd, None, None, dtype=F64)
    want = o.mt_features(torch.tensor([toks]), enc[:37].double().cpu().unsqueeze(1))[0]
    got = ref.features(toks, enc[:37])
    d = maxdiff(got.cpu(), want)
    report("mt_fp64_reference_vs_cpu_oracle", max_abs=d)
    assert d < 1e-10, d


def test_mt_greedy_routes_vs_fp64(mt):
    """ss_mt_greedy on its three routes: the prefix kernel + the single-token kernel, the per-op prefix + the single-token kernel, and
    the per-op decoder throughout, over the covering design GREEDY_CASES and one prefix that is the engine's own earlier hypothesis"""
    cfg, sd, e, ref, enc = mt
    g = torch.Generator().manual_seed(11)
    cases = [(p, T, mn, end, random_tokens(cfg, p, g)) for p, T, mn, end in GREEDY_CASES]
    set_route(e, "prefix_kernel")
    own, _ = e.mt_greedy(enc[:OWN_PREFIX_T].contiguous(), None, -1, max_len_b=MAX_LEN_B)
    assert len(own) >= 8
    cases.append((len(own) // 2, OWN_PREFIX_T, -1, "eos", own[:len(own) // 2]))
    cross = {}  # T -> launches of the cross K / V projection (a search without prefix: projection + 2 single-token launches)
    for T in sorted({c[1] for c in cases}):
        _, n, _ = launches(e, lambda: e.mt_greedy(enc[:T].contiguous(), None, 1, max_len_b=MAX_LEN_B))
        cross[T] = n - 2
    worst, near, ends, ref_cache, wrong_end = Worst(), {r: 0 for r in ROUTES}, {"eos": 0, "max_len": 0}, {}, []
    for route in ROUTES:
        set_route(e, route)
        for p, T, mn, end, prefix in cases:
            what = f"{route} prefix={p} T={T} max_new={mn}"
            x = enc[:T].contiguous()
            (hyp, feats), n, n_v2 = launches(e, lambda: e.mt_greedy(x, prefix, mn, max_len_b=MAX_LEN_B))
            max_len = min(MAX_LEN_B, e.max_mt_positions - 1) if mn == -1 else p + mn
            kernel_prefix = route == "prefix_kernel" and 1 <= p <= PREFIX_KERNEL_ROWS
            single = 0 if route == "per_op" else v2_launches(p, mn, max_len, len(hyp), p if kernel_prefix else 0)
            other = n - cross[T] - single  # the prefix pass: one launch of the prefix kernel, dozens per-op (every step on per_op)
            if kernel_prefix or (p == 0 and route != "per_op"):
                assert other == int(kernel_prefix), (what, n, cross[T], single)  # the prefix kernel, not the per-op fallback
            else:
                assert other >= PER_OP_PREFIX_LAUNCHES, (what, n, cross[T], single)
            assert n_v2 <= single, (what, n_v2, single)  # (mt_time counts the launches that produced a token)
            assert hyp[:p] == prefix, what
            ended = "max_len" if len(hyp) == max_len else "eos"
            if ended != end:
                wrong_end.append((what, ended, len(hyp)))
            ends[ended] += 1
            key = (T, tuple(hyp), p, max_len)
            if key not in ref_cache:
                ref_cache[key] = check_search(ref, x, hyp, p, max_len, what)
            f64, nt = ref_cache[key]
            near[route] += nt
            worst.add(route, maxdiff(feats, f64), what)
    e.set_option("persistent_mt", 1)
    e.set_option("persistent_mt_prefix", 1)
    report("mt_greedy_routes_fp64", cases=len(cases), endings=ends, feat=worst.as_dict(), near_ties=near, wrong_endings=wrong_end)
    assert not wrong_end and ends["eos"] and ends["max_len"], wrong_end
    for route in ROUTES:
        assert worst.get(route) < FEAT_TOL[route], (route, worst.as_dict()[route])


@pytest.fixture(scope="module")
def noeos(mt):
    """an engine with the default 1024 MT positions on the checkpoint whose eos row is zero (its searches never end on eos), and its
    float64 reference"""
    from streamspeech_b200.engine import Engine

    cfg, sd, _, _, enc = mt
    sd = dict(sd)
    for k in ("target_unigram_decoder.embed_tokens.weight", "target_unigram_decoder.output_projection.weight"):
        sd[k] = sd[k].clone()
        sd[k][cfg.eos] = 0.0
    e = Engine(cfg, sd, None, synth.make_gcmvn(cfg))
    e.set_option("persistent_time", 1)
    yield e, Ref64(cfg, sd), enc
    e.close()


def test_mt_greedy_whole_position_table_vs_fp64(noeos):
    """the longest search the default capacity admits (max_len + 2 = max_mt_positions): 1023 feature rows, every position of the table,
    with no prefix (single-token kernel throughout) and with a 64-token prefix (prefix kernel, then the single-token kernel)"""
    e, ref, enc = noeos
    cfg = ref.cfg
    max_len = e.max_mt_positions - 2
    g = torch.Generator().manual_seed(5)
    worst, near = Worst(), {}
    for p, T in ((0, 1024), (PREFIX_KERNEL_ROWS, 1000)):
        prefix = random_tokens(cfg, p, g)
        what = f"prefix={p} T={T} max_len={max_len}"
        x = enc[:T].contiguous()
        (hyp, feats), n, n_v2 = launches(e, lambda: e.mt_greedy(x, prefix, -1, max_len_b=max_len))
        assert len(hyp) == max_len and feats.shape[0] == max_len + 1, (what, len(hyp))
        assert n_v2 >= (max_len - p) // 16
        f64, near[what] = check_search(ref, x, hyp, p, max_len, what)
        worst.add("whole_table", maxdiff(feats, f64), what)
    report("mt_greedy_whole_position_table_fp64", max_len=max_len, feat=worst.as_dict(), near_ties=near)
    assert worst.get("whole_table") < FEAT_TOL["whole_table"], worst.as_dict()


# ss_mt_features: (sequence length S including [eos], pad tail, encoder rows T); S = 1024 is the capacity limit
FEATURE_CASES = [(1, 0, 1024), (2, 1, 1), (16, 0, 17), (16, 3, 1000), (17, 1, 128), (17, 0, 1023), (64, 3, 33), (64, 0, 257),
                 (65, 0, 1023), (65, 1, 2), (300, 3, 255), (300, 0, 1024), (1024, 1, 129), (1024, 3, 1000)]


def test_mt_features_vs_fp64(mt):
    """ss_mt_features (per-op decoder) with pad tails, and the logits of its last row (want_logits), with the engine's default linear
    routing (linears of >= umma_min_rows rows per sample on the bf16x6 tensor-core GEMM) and with every linear on the fp32 kernels"""
    cfg, sd, e, ref, enc = mt
    worst = Worst()
    for routing, umma in LINEAR_ROUTINGS.items():
        e.set_option("umma_linear", umma)
        g = torch.Generator().manual_seed(13)
        for S, npad, T in FEATURE_CASES:
            toks = [cfg.eos] + random_tokens(cfg, S - 1 - npad, g) + [cfg.pad] * npad
            what = f"S={S} pad={npad} T={T}"
            x = enc[:T].contiguous()
            feats, logits = e.mt_features(x, toks, want_logits=True)
            f64 = ref.features(toks, x)
            worst.add(f"features_{routing}", maxdiff(feats, f64), what)
            worst.add(f"logits_{routing}", maxdiff(logits, f64[-1] @ ref.out_w.T), what)
    e.set_option("umma_linear", LINEAR_ROUTINGS["tc"])
    report("mt_features_fp64", cases=len(FEATURE_CASES), **worst.as_dict())
    for routing in LINEAR_ROUTINGS:
        assert worst.get(f"features_{routing}") < FEAT_TOL[f"features_{routing}"], worst.as_dict()
        assert worst.get(f"logits_{routing}") < LOGIT_TOL, worst.as_dict()


def test_mt_features_batch_vs_fp64(mt):
    """ss_mt_features_batch: 45 samples of S = 64 rows with ragged T (1 .. 1024) and ragged pad tails form three launch groups of
    UNIT_BATCH_ROWS / (S * ctc_upsample_rate) = 20, 20 and 5 samples; each sample against its own float64 pass"""
    cfg, sd, e, ref, enc = mt
    S, B = 64, 45
    G = max(1, UNIT_BATCH_ROWS // (S * cfg.ctc_upsample_rate))
    assert (G, -(-B // G)) == (20, 3)
    g = torch.Generator().manual_seed(17)
    Ts = [1, 1024] + torch.randint(1, 1025, (B - 2,), generator=g).tolist()
    Ts[G - 1], Ts[G], Ts[2 * G] = 1024, 1, 129  # both ends of the group boundaries
    pads = [(7 * b) % 6 for b in range(B)]
    toks = [[cfg.eos] + random_tokens(cfg, S - 1 - pads[b], g) + [cfg.pad] * pads[b] for b in range(B)]
    batch = torch.zeros(B, 1024, cfg.enc_dim, device="cuda")
    for b, T in enumerate(Ts):
        batch[b, :T] = enc[:T]
    feats = {}
    for routing, umma in LINEAR_ROUTINGS.items():
        e.set_option("umma_linear", umma)
        feats[routing] = e.mt_features_batch(batch, Ts, toks).clone()
    e.set_option("umma_linear", LINEAR_ROUTINGS["tc"])
    _, n_all, _ = launches(e, lambda: e.mt_features_batch(batch, Ts, toks))
    # the launches of the whole call are those of its three groups called one by one: it really ran as 20 + 20 + 5
    _, n_full, _ = launches(e, lambda: e.mt_features_batch(batch[:G].contiguous(), Ts[:G], toks[:G]))
    _, n_tail, _ = launches(e, lambda: e.mt_features_batch(batch[2 * G:].contiguous(), Ts[2 * G:], toks[2 * G:]))
    assert n_all == 2 * n_full + n_tail, (n_all, n_full, n_tail)
    worst = Worst()
    for b in range(B):
        f64 = ref.features(toks[b], enc[:Ts[b]])
        for routing in LINEAR_ROUTINGS:
            worst.add(f"features_batch_{routing}", maxdiff(feats[routing][b], f64), f"b={b} T={Ts[b]} pad={pads[b]}")
    report("mt_features_batch_fp64", B=B, S=S, group=G, **worst.as_dict())
    for routing in LINEAR_ROUTINGS:
        assert worst.get(f"features_batch_{routing}") < FEAT_TOL[f"features_batch_{routing}"], worst.as_dict()


def test_mt_greedy_batch_vs_fp64(mt):
    """ss_mt_greedy_batch: B = 2 (one launch group), 32 (a full group) and 33 (a full group and a single sample, which runs on the
    single-token kernel), ragged T with 1 and 1024; then B = 33 with mt_batch_min_rows above the group size, so every sample runs on
    the single-token kernel.  Every hypothesis against its own float64 pass."""
    cfg, sd, e, ref, enc = mt
    g = torch.Generator().manual_seed(19)
    max_len = MAX_LEN_B
    near, n_checked, ref_cache = {}, 0, {}
    for B, min_rows in ((2, 2), (32, 2), (33, 2), (33, BATCH_ROWS + 1)):
        Ts = [1024, 1] + torch.randint(1, 1025, (B - 2,), generator=g).tolist()
        if B > BATCH_ROWS:
            Ts[-1] = 1  # the second group's lone sample
        batch = torch.zeros(B, 1024, cfg.enc_dim, device="cuda")
        for b, T in enumerate(Ts):
            batch[b, :T] = enc[:T]
        e.set_option("mt_batch_min_rows", min_rows)
        hyps, _, n_v2 = launches(e, lambda: e.mt_greedy_batch(batch, Ts, max_len))
        # the single-token kernel runs only the samples of groups below mt_batch_min_rows
        fallback = sum(min(BATCH_ROWS, B - g0) for g0 in range(0, B, BATCH_ROWS) if min(BATCH_ROWS, B - g0) < min_rows)
        assert (n_v2 >= fallback) and (n_v2 == 0) == (fallback == 0), (B, min_rows, n_v2, fallback)
        nt = 0
        for b, (T, hyp) in enumerate(zip(Ts, hyps)):
            key = (T, tuple(hyp))
            if key not in ref_cache:
                ref_cache[key] = check_search(ref, enc[:T], hyp, 0, max_len, f"B={B} min_rows={min_rows} b={b} T={T}")[1]
            nt += ref_cache[key]
            n_checked += 1
        near[f"B={B} min_rows={min_rows}"] = nt
    e.set_option("mt_batch_min_rows", 2)
    report("mt_greedy_batch_fp64", hypotheses=n_checked, near_ties=near)


# ss_pool_mt_greedy: per slot (utterance seconds, prefix length, max_new_tokens)
POOL_CASES = [(2.1, 0, -1), (0.5, 1, 5), (6.3, 16, -1), (3.7, 17, 1), (9.8, 64, -1), (1.2, 70, 0), (12.4, 5, -1), (4.4, 33, 5)]


def test_pool_mt_greedy_vs_fp64(mt):
    """ss_pool_mt_greedy on 8 slots of ragged length: the prefix pass teacher-forces ragged prefixes (0, 1, 5, 16, 17, 33, 64, 70) as
    masked pad tails, then the batched kernel searches with mixed max_new_tokens.  Tokens and features of every slot against the float64
    pass over the slot's own pool encoder rows."""
    cfg, sd, e, ref, enc = mt
    g = torch.Generator().manual_seed(23)
    n = len(POOL_CASES)
    e.pool_create(n, max_seconds=13)
    slots = list(range(n))
    for sl, (sec, _, _) in enumerate(POOL_CASES):
        e.pool_reset(sl)
        e.pool_push_audio(sl, synth.make_audio(sec, seed=300 + sl).contiguous())
    res = e.pool_step(slots, ctc_heads=0)
    rows = [e.pool_encoder_rows(sl, r["T"]).clone() for sl, r in zip(slots, res)]
    prefixes = [random_tokens(cfg, p, g) for _, p, _ in POOL_CASES]
    max_new = [mn for _, _, mn in POOL_CASES]
    (hyps, feats), _, n_v2 = launches(e, lambda: e.pool_mt_greedy(slots, prefixes, max_new, MAX_LEN_B))
    assert n_v2 == 0  # one group on the batched kernel, no stream on the single-token kernel
    worst, near, ends = Worst(), {}, []
    for sl, ((sec, p, mn), prefix, hyp) in enumerate(zip(POOL_CASES, prefixes, hyps)):
        what = f"slot={sl} T={rows[sl].shape[0]} prefix={p} max_new={mn}"
        max_len = MAX_LEN_B if mn == -1 else p + mn
        assert hyp[:p] == prefix, what
        f64, near[what] = check_search(ref, rows[sl], hyp, p, max_len, what)
        worst.add("pool", maxdiff(feats[sl, :len(hyp) + 1], f64), what)
        ends.append("max_len" if len(hyp) == max_len else "eos")
    report("pool_mt_greedy_fp64", T=[r.shape[0] for r in rows], endings=ends, feat=worst.as_dict(), near_ties=near)
    assert worst.get("pool") < FEAT_TOL["pool"], worst.as_dict()
