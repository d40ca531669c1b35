"""GPU: the beam instantiation of the batched decoder kernel (mt_decode_batch_kernel<kMtbBeam>, kernels_persist_mtb.cu) behind its
two front doors, and the T2U encoder that feeds the second, against float64 restatements of the same operations:

- ss_mt_beam_batch (the offline generator's `--beam-mt K`) against oracle/mt_beam_oracle.mt_beam on a float64 StreamSpeechOracle:
  every width at launch splits with a partial last group, T = 1 and 1024 in one launch, samples bit-identical when searched alone,
  finalization edges (the K-hypothesis cap, eos at ranks K .. 2K - 1, samples done while their launch searches on, hypotheses
  finalized at step 1), the length penalty, exact ties decided by the flat index, and buffers grown or shared between calls;
- ss_unit_search_batch (UnitY's unit search, the same kernel at K = 1) against UnitYOracle.unit_search in float64: max_len at the
  16-step burst edges, the length penalty, launch splits with S = 1 and 1024 in one launch, duplicated unit rows;
- ss_t2u_encode_batch against UnitYOracle.t2u_encode at S and B that reach every GEMM class and both attention kernels.

Decisions.  A search may take another decision than float64 only where float64's gap between the candidates is below the error
fp32 can make.  For the MT beam that bar grows with the step: MT_BASE (the log-probability's own error) plus |score| * (step + 1) *
2^-23 (one ulp of the cumulative score per step, on both candidates), taken per pair of neighbouring distinct scores.  The oracle reports the smallest gap between distinct scores
among the 2K + 1 best candidates of each step (exactly equal scores are ordered by the flat index, not by arithmetic), and every MT
case asserts that its encoder rows clear the bar at every step: then tokens, order, scores and positional scores must match.  The
seeds of the rows were chosen so that they do.  Unit-search rows follow the rule of tests/test_unity_gpu.py (tokens up to the first
step whose top-2 gap is below UNIT_MARGIN; the whole row where none is).

Every case asserts that the event it exists for happened in the oracle's trace.  Errors and margins are printed as one JSON line per
test (`pytest -s`).
"""
import json
import math

import numpy as np
import pytest
import torch

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

# the bar of an MT beam decision at step s between neighbouring distinct scores a > b: MT_BASE + |b| * (s + 1) * 2^-23, the base
# above the fp32 errors measured on an H100 80GB HBM3 (700 W): positional scores (differences of cumulative scores, so with their
# rounding) within 7.5e-6 of float64 on the synthetic checkpoints and 1.4e-5 on the sharpened one (sharp_sd), final scores within
# 8.5e-6.  Every decision of every case below matched float64 there.
MT_BASE = 2e-5
UNIT_MARGIN = 1e-4
ENC_DIM = 256
LEAK = 1e3  # encoder / T2U rows beyond a sample's length are filled with values of this size: any leak would show


def report(name, **kw):
    print(json.dumps({"test": name, **kw}, default=float))


def offline_cfg():
    cfg = ModelConfig()
    cfg.uni_encoder = False
    return cfg


def mt_oracle(sd):
    from oracle.streamspeech_oracle import StreamSpeechOracle

    cfg = offline_cfg()
    return StreamSpeechOracle(cfg, sd, None, synth.make_gcmvn(cfg), chunk_size=None, conv_chunk_size=None, dtype=torch.float64)


def mt_engine(sd):
    from streamspeech_b200.engine import Engine

    cfg = offline_cfg()
    e = Engine(cfg, sd, synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    e.set_chunk(None, None)
    return e


@pytest.fixture(scope="module")
def base_sd():
    return synth.make_model_state_dict(offline_cfg(), 0)


@pytest.fixture(scope="module")
def eng(base_sd):
    e = mt_engine(base_sd)
    yield e
    e.close()


@pytest.fixture(scope="module")
def o64(base_sd):
    return mt_oracle(base_sd)


def enc_rows(seed, T):
    return torch.randn(T, ENC_DIM, generator=torch.Generator().manual_seed(seed))


def pad_batch(rows, T=None):
    """[B, T, C] on the device, rows beyond each sample's length LEAK-sized"""
    T = T or max(r.shape[0] for r in rows)
    g = torch.Generator().manual_seed(7)
    x = LEAK * torch.randn(len(rows), T, ENC_DIM, generator=g)
    for b, r in enumerate(rows):
        x[b, : r.shape[0]] = r
    return x.cuda().contiguous()


def mt_clearance(want):
    """the smallest margin by which the float64 gap between two neighbouring distinct scores among a step's 2K + 1 best exceeds the
    bar of that step (positive: every decision of the search is clear of fp32 error)"""
    return min((a - b - mt_bar(b, s) for s, t in enumerate(want["tops"]) for a, b in zip(t, t[1:])), default=math.inf)


def mt_bar(score, step):
    return MT_BASE + abs(score) * (step + 1) * 2.0 ** -23


class Worst:
    def __init__(self):
        self.v = {}

    def add(self, key, err, case):
        if key not in self.v or err > self.v[key][0]:
            self.v[key] = (err, case)

    def as_dict(self):
        return {k: {"max": v, "case": c} for k, (v, c) in sorted(self.v.items())}


def check_mt(got, want, what, worst):
    """the engine's K hypotheses of one sample against the float64 oracle's: tokens and order exactly, scores and positional scores
    within bars that grow with the cumulative score (each step adds about one ulp of it)"""
    eos = offline_cfg().eos
    clear = mt_clearance(want)
    worst.add("-clearance", -clear, what)
    worst.add("min_margin_inv", 1.0 / max(want["margin"], 1e-30), what)
    assert clear > 0, (what, "float64 margin below the bar", want["margin"], clear)
    hyps = want["hyps"]
    assert len(got) == len(hyps), what
    for i, (h, w) in enumerate(zip(got, hyps)):
        assert h["tokens"] + [eos] == w["tokens"], (what, i)
        n = len(w["tokens"])
        raw = abs(sum(w["positional_scores"]))
        e_s = abs(h["score"] - w["score"])
        e_p = max(abs(x - y) for x, y in zip(h["positional_scores"], w["positional_scores"]))
        worst.add("score", e_s, what)
        worst.add("positional", e_p, what)
        assert e_s < 1e-5 + 2.0 ** -22 * raw * n, (what, i, h["score"], w["score"])
        assert e_p < 1e-5 + 2.0 ** -22 * raw * n, (what, i, e_p)


# ---- widths and launch splits: K -> (B, max_len_b, len_penalty, seed offsets of the samples' encoder rows).  B gives at least two
# launch groups of 32 // K samples and a partial last one (K = 31, 32: one sample per launch, 1 and 0 idle rows).  Sample 0 has one
# encoder row, sample 1 has 1024; the others WIDTH_T.  Sample b's rows are enc_rows(10000 K + 100 b + offset).
WIDTHS = {
    2: (33, 8, 1.0),
    3: (21, 8, 0.6),
    4: (17, 6, 2.0),
    5: (13, 5, 0.0),
    7: (9, 4, 1.0),
    8: (9, 4, 0.6),
    11: (5, 3, 2.0),
    16: (5, 2, 0.0),
    31: (2, 2, 1.0),
    32: (2, 2, 0.6),
}
WIDTH_SEEDS = {
    2: [0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 2, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0],
    3: [1, 1, 2, 4, 0, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0],
    4: [1, 0, 1, 0, 0, 0, 1, 1, 2, 0, 1, 0, 0, 0, 0, 0, 0],
    5: [0, 2, 1, 0, 2, 0, 0, 0, 0, 0, 1, 3, 0],
    7: [2, 0, 0, 0, 1, 0, 1, 0, 1],
    8: [2, 1, 0, 1, 0, 1, 2, 0, 2],
    11: [0, 6, 0, 0, 2],
    16: [0, 1, 0, 0, 1],
    31: [11, 30],
    32: [12, 13],
}


def width_T(K, b):
    return 1 if b == 0 else 1024 if b == 1 else 2 + (37 * b + 11 * K) % 90


@pytest.mark.parametrize("K", sorted(WIDTHS))
def test_mt_beam_widths_and_launch_splits(eng, o64, K):
    from oracle.mt_beam_oracle import mt_beam

    B, ml, lp = WIDTHS[K]
    seeds = WIDTH_SEEDS[K]
    Ts = [width_T(K, b) for b in range(B)]
    rows = [enc_rows(10000 * K + 100 * b + seeds[b], Ts[b]) for b in range(B)]
    enc = pad_batch(rows)
    got = eng.mt_beam_batch(enc, Ts, K, ml, lp)
    per = 32 // K
    assert B > 2 * per or (per == 1 and B >= 2)
    assert B % per != 0 or per == 1  # a partial last launch group
    worst = Worst()
    for b in range(B):
        want = mt_beam(o64, rows[b].unsqueeze(1), K, ml, lp)
        check_mt(got[b], want, f"K={K} b={b} T={Ts[b]}", worst)
        alone = eng.mt_beam_batch(pad_batch([rows[b]]), [Ts[b]], K, ml, lp)[0]
        assert alone == got[b], (K, b)  # bit for bit
    report(f"widths K={K}", **worst.as_dict())


def dup_row_sd(sd, key_emb, keys, a, b):
    """a copy of sd whose tied embedding row a is row b's (both tokens then get bit-identical logits in fp32 and in float64)"""
    out = dict(sd)
    e = sd[key_emb].clone()
    e[a] = e[b]
    for k in keys:
        out[k] = e
    return out


MT_EMB = "target_unigram_decoder.embed_tokens.weight"
MT_TIED = (MT_EMB, "target_unigram_decoder.output_projection.weight")
# the early-eos checkpoint (its eos row scaled by -0.2, as tests/golden/mt_beam.npz's early cases): samples finalize hypotheses at
# step 1, fill the K-th slot at step 8 with more eos in the first K than slots left, and rank eos at K .. 2K - 1; the sample with 5
# encoder rows finalizes one hypothesis at step 1 and then searches on to the forced eos at step 40, past two burst boundaries.  Over
# 40 steps of this checkpoint's flat distributions its float64 gaps fall below the bar, so it is held bit-identical to its search
# alone but not compared with float64 (test_mt_beam_burst_edges compares K >= 2 searches across bursts on a sharper checkpoint).
# (seed, T) of enc_rows per sample
EARLY_SAMPLES = [(2, 19), (4, 33), (5, 40), (0, 5), (1, 12)]
EARLY_RUN_ON = 3  # the index of the sample that searches on


@pytest.fixture(scope="module")
def early_sd(base_sd):
    from oracle.mt_beam_oracle import early_eos_state_dict

    return early_eos_state_dict(base_sd, offline_cfg().eos, -0.2)


def test_mt_beam_finalization_edges_and_len_penalty(early_sd):
    """the cap on finalized hypotheses, eos outside the top K, a sample done while its launch searches on across two burst
    boundaries, step-1 hypotheses; len_penalty in {0, 0.6, 1, 2} on the same searches, reordering the finalized hypotheses"""
    from oracle.mt_beam_oracle import mt_beam

    eng = mt_engine(early_sd)
    o = mt_oracle(early_sd)
    worst = Worst()
    try:
        for K in (3, 4):
            rows = [enc_rows(s, T) for s, T in EARLY_SAMPLES]
            Ts = [T for _, T in EARLY_SAMPLES]
            enc = pad_batch(rows)
            ev = {"capped": 0, "eos_out": 0, "fin_step1": 0, "reordered": 0}
            for lp in (0.0, 0.6, 1.0, 2.0):
                got = eng.mt_beam_batch(enc, Ts, K, 40, lp)
                steps = []
                for b, r in enumerate(rows):
                    want = mt_beam(o, r.unsqueeze(1), K, 40, lp, trace=True)
                    tr = want["trace"]
                    steps.append(len(tr))
                    what = f"early K={K} lp={lp} b={b}"
                    if b != EARLY_RUN_ON:
                        check_mt(got[b], want, what, worst)
                        ev["capped"] += sum(s["capped"] for s in tr)
                        ev["eos_out"] += sum(s["eos_out"] for s in tr)
                        ev["fin_step1"] += tr[1]["new_fin"] if len(tr) > 1 else 0
                        raw = [sum(h["positional_scores"]) for h in want["hyps"]]
                        ev["reordered"] += raw != sorted(raw, reverse=True)
                    alone = eng.mt_beam_batch(pad_batch([r]), [Ts[b]], K, 40, lp)[0]
                    assert alone == got[b], (what, "differs from the sample searched alone")
                # a sample done before the first burst boundary while the run-on sample searches past the second
                assert min(steps) <= 16 and steps[EARLY_RUN_ON] > 33, steps
            report(f"finalization K={K}", events=ev)
            assert ev["capped"] > 0 and ev["eos_out"] > 0 and ev["fin_step1"] > 0 and ev["reordered"] > 0, ev
    finally:
        eng.close()
    report("finalization", **worst.as_dict())


def test_mt_beam_exact_ties(base_sd, early_sd):
    """token 4's tied embedding row set to token 1338's (the early-eos search's first token): the two get bit-identical
    candidates, and so do the beams that differ only by them.  The lower flat index must win every such tie, in the candidates of a
    row and in the selection of a sample, and equal finalized scores keep their finalization order"""
    from oracle.mt_beam_oracle import mt_beam

    worst = Worst()
    for name, sd, samples, widths in (("early", early_sd, [(2, 19), (4, 33), (1, 12)], (3, 4, 6)),
                                      ("plain", base_sd, [(2, 19), (1, 12)], (3, 4))):
        sd = dup_row_sd(sd, MT_EMB, MT_TIED, 4, 1338)
        eng = mt_engine(sd)
        o = mt_oracle(sd)
        try:
            rows = [enc_rows(s, T) for s, T in samples]
            Ts = [T for _, T in samples]
            enc = pad_batch(rows)
            for K in widths:
                got = eng.mt_beam_batch(enc, Ts, K, 12)
                ties = fin_ties = 0
                for b, r in enumerate(rows):
                    want = mt_beam(o, r.unsqueeze(1), K, 12, trace=True)
                    check_mt(got[b], want, f"ties {name} K={K} b={b}", worst)
                    ties += sum(s["ties"] for s in want["trace"])
                    fin_ties += want["fin_ties"]
                report(f"ties {name} K={K}", ties=ties, fin_ties=fin_ties)
                assert ties > 0 and fin_ties > 0, (name, K, ties, fin_ties)
        finally:
            eng.close()
    report("ties", **worst.as_dict())


def test_mt_beam_buffer_growth_and_sharing(base_sd):
    """a fresh handle: a short search, then T = 1000 rows and a longer max_len (cross and self K / V buffers grow between calls);
    then a UnitY handle alternating unit searches (beam 1: one self K / V buffer) and MT beam searches (the second buffer), which
    share the buffers"""
    from oracle.mt_beam_oracle import mt_beam
    from oracle.unity_oracle import UnitYOracle
    from streamspeech_b200.engine import Engine

    worst = Worst()
    eng = mt_engine(base_sd)
    o = mt_oracle(base_sd)
    try:
        for K, ml, s, T in ((2, 3, 20003, 7), (3, 8, 2, 1000), (2, 8, 20000, 33)):
            r = enc_rows(s, T)
            want = mt_beam(o, r.unsqueeze(1), K, ml)
            check_mt(eng.mt_beam_batch(pad_batch([r]), [T], K, ml)[0], want, f"growth K={K} T={T} ml={ml}", worst)
    finally:
        eng.close()
    cfg = ModelConfig.unity_default()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    ue = Engine(cfg, sd, None, None, device=0)
    u64 = UnitYOracle(cfg, sd, torch.float64)
    try:
        lens = [9, 4, 1]
        x = unit_states(3, 9, lens, 5)
        want_units = u64.unit_search(x, lens, 40)
        for K, ml, s, T in ((2, 3, 20003, 7), (3, 8, 3, 1000)):
            assert check_rows(ue.unit_search_batch(x.cuda().contiguous(), lens, 40), want_units, cfg, worst, "shared units") == 3
            r = enc_rows(s, T)
            want = mt_beam(u64.o, r.unsqueeze(1), K, ml, max_decoder_positions=cfg.max_target_positions)
            check_mt(ue.mt_beam_batch(pad_batch([r]), [T], K, ml)[0], want, f"shared K={K} T={T}", worst)
        assert check_rows(ue.unit_search_batch(x.cuda().contiguous(), lens, 40), want_units, cfg, worst, "shared units") == 3
    finally:
        ue.close()
    report("buffers", **worst.as_dict())


def sharp_sd(sd, gain=8.0):
    """a copy of sd whose MT final LayerNorm (weight and bias) is multiplied by `gain`: every logit scales by it, so the float64 gaps
    between a step's best candidates grow while the decoder below is unchanged, and beams clear the bar over 33 steps"""
    out = dict(sd)
    for k in ("target_unigram_decoder.layer_norm.weight", "target_unigram_decoder.layer_norm.bias"):
        out[k] = sd[k] * gain
    return out


# burst edges: max_len_b on either side of the first and second 16-step bursts.  name -> (early-eos scale or None, K, (seed, T) of
# enc_rows per sample), all on sharp_sd.  "sharp": every beam runs to the forced eos at max_len_b; "early15": the sample finalizes
# one hypothesis at step 16 (the first step of the second burst) and searches on with the cap applying later; "early17": one sample
# finalizes both hypotheses at steps 9 and 15 (done within the first burst) while the other searches on to the forced eos
BURSTS = {
    "sharp2": (None, 2, [(0, 10), (1, 23)]),
    "sharp4": (None, 4, [(2, 36)]),
    "early15": (-0.15, 3, [(1, 23)]),
    "early17": (-0.17, 2, [(0, 10), (3, 49)]),
}


@pytest.mark.parametrize("name", sorted(BURSTS))
def test_mt_beam_burst_edges(base_sd, name):
    """K >= 2 searches across burst boundaries: the alternating self-attention caches gathered through parent rows, cumulative
    scores, tokens and finalized hypotheses carried from one launch into the next, a forced eos on a burst's first or last step"""
    from oracle.mt_beam_oracle import early_eos_state_dict, mt_beam

    scale, K, samples = BURSTS[name]
    sd = sharp_sd(base_sd if scale is None else early_eos_state_dict(base_sd, offline_cfg().eos, scale))
    eng = mt_engine(sd)
    o = mt_oracle(sd)
    worst = Worst()
    ends = set()
    try:
        rows = [enc_rows(s, T) for s, T in samples]
        Ts = [T for _, T in samples]
        enc = pad_batch(rows)
        for ml in (15, 16, 17, 31, 32, 33):
            got = eng.mt_beam_batch(enc, Ts, K, ml)
            for b, r in enumerate(rows):
                want = mt_beam(o, r.unsqueeze(1), K, ml, trace=True)
                check_mt(got[b], want, f"{name} ml={ml} b={b}", worst)
                steps = [len(h["tokens"]) - 1 for h in want["hyps"]]  # the step each hypothesis was finalized at
                ends |= {(ml, b, s) for s in steps}
                if scale is None:
                    assert steps == [ml] * K  # every beam to the forced eos
    finally:
        eng.close()
    report(f"burst edges {name}", ends=sorted(ends), **worst.as_dict())
    if name == "early15":  # a hypothesis finalized on the first step of the second burst, the others later
        assert all((ml, 0, 16) in ends for ml in (17, 31, 32, 33)) and (33, 0, 33) in ends, ends
    if name == "early17":  # sample 1 done within the first burst, sample 0 searching on to the forced eos
        assert all((ml, 1, 15) in ends and (ml, 0, ml) in ends for ml in (31, 32, 33)), ends


# ---- end to end


@pytest.mark.parametrize("beam_mt", [1, 4])
def test_unity_generator_end_to_end(beam_mt):
    """offline.UnitYGenerator on a ragged batch of random CMVN-scale features against unity_generate on a float64 UnitYOracle: the
    MT hypotheses exactly where every float64 MT decision clears E2E_MT_BASE + |score| * (step + 1) * 2^-23 (the fp32 encoder adds
    its error to the decoder's), the units by the margin rule"""
    from oracle.mt_beam_oracle import mt_beam
    from oracle.unity_oracle import UnitYOracle, unity_generate
    from streamspeech_b200.engine import Engine
    from streamspeech_b200.offline import UnitYGenerator

    cfg = ModelConfig.unity_default()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    u64 = UnitYOracle(cfg, sd, torch.float64)
    lens = E2E_LENGTHS
    g = torch.Generator().manual_seed(E2E_SEED)
    x = torch.zeros(len(lens), max(lens), cfg.feat_dim)
    for b, n in enumerate(lens):
        x[b, :n] = torch.randn(n, cfg.feat_dim, generator=g)
    want = unity_generate(u64, x, lens, beam_mt, 1.0, 10, E2E_MAX_LEN_B_MT)
    enc = u64.o.encoder(x, torch.tensor(lens))
    worst = Worst()
    for b in range(len(lens)):
        Tb = int(enc["out_lengths"][b])
        m = mt_beam(u64.o, enc["encoder_out"][0][:Tb, b:b + 1], beam_mt, E2E_MAX_LEN_B_MT, max_decoder_positions=cfg.max_target_positions)
        assert [t for t in m["hyps"][0]["tokens"] if t != cfg.eos] == want["mt_hyps"][b]  # (beam 1: the greedy search)
        clear = min((a - c - (E2E_MT_BASE + abs(c) * (s + 1) * 2.0 ** -23) for s, t in enumerate(m["tops"]) for a, c in zip(t, t[1:])),
                    default=math.inf)
        worst.add("-mt_clearance", -clear, f"b={b}")
        assert clear > 0, (b, clear)
    eng = Engine(cfg, sd, None, None, device=0)
    try:
        res = UnitYGenerator(eng, beam_size_mt=beam_mt, max_len_a=1.0, max_len_b=10, max_len_b_mt=E2E_MAX_LEN_B_MT).generate(x.cuda(), lens)
    finally:
        eng.close()
    assert [r["mt_tokens"] for r in res] == want["mt_hyps"]
    got = [{"tokens": r["units"], "score": r["unit_score"], "positional_scores": torch.as_tensor(r["unit_positional_scores"])} for r in res]
    whole = check_rows(got, want["units"], cfg, worst, f"e2e beam_mt={beam_mt}")
    report(f"e2e beam_mt={beam_mt}", whole=whole, mt=[len(h) for h in want["mt_hyps"]], **worst.as_dict())
    assert whole == len(lens)


E2E_LENGTHS = [96, 61, 80]
E2E_SEED = 8
E2E_MAX_LEN_B_MT = 4
E2E_MT_BASE = 1e-4


# ---- unit search


@pytest.fixture(scope="module")
def unity():
    from oracle.unity_oracle import UnitYOracle
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig.unity_default()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    eng = Engine(cfg, sd, None, None, device=0)
    yield cfg, sd, eng, UnitYOracle(cfg, sd, torch.float64)
    eng.close()


def zero_eos_sd(cfg):
    """the synthetic UnitY weights (seed 1) with eos's output row zero: its logit is 0 at every step, below the best unit's"""
    sd = synth.make_unity_state_dict(cfg, seed=1)
    e = sd["decoder.embed_tokens.weight"].clone()
    e[cfg.eos] = 0.0
    sd["decoder.embed_tokens.weight"] = sd["decoder.output_projection.weight"] = e
    return sd


def unit_states(B, S, lens, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, S, 512, generator=g)
    for b, n in enumerate(lens):
        x[b, n:] = LEAK * torch.randn(S - n, 512, generator=g)
    return x


def check_rows(got, want, cfg, worst, what):
    """tokens up to the first step whose float64 top-2 gap is below UNIT_MARGIN; rows without one whole, with score and positional
    scores (tests/test_unity_gpu.py's bars).  Returns the number of rows checked whole."""
    whole = 0
    for b, (a, r) in enumerate(zip(got, want)):
        n = next((i for i, m in enumerate(r["margins"]) if m < UNIT_MARGIN), len(r["margins"]))
        worst.add("unit_min_margin_inv", 1.0 / max(r["margin"], 1e-30), f"{what} b={b}")
        assert a["tokens"][:n] == r["tokens"][:n], (what, b, n)
        if n == len(r["margins"]):
            whole += 1
            assert a["tokens"] == r["tokens"], (what, b)
            e_s = abs(a["score"] - r["score"])
            worst.add("unit_score", e_s, f"{what} b={b}")
            assert e_s < 2e-4 * max(1.0, abs(r["score"])), (what, b, a["score"], r["score"])
            pos = a["positional_scores"].double().numpy()
            e_p = float(np.abs(pos - np.array(r["positional_scores"])).max())
            worst.add("unit_positional", e_p, f"{what} b={b}")
            assert e_p < 2e-4 + 2.4e-7 * abs(r["score"]) * len(r["tokens"]), (what, b)
            assert a["tokens"][-1] == cfg.eos
    return whole


@pytest.mark.parametrize("zero_eos", [False, True])
def test_unit_search_burst_edges(unity, zero_eos):
    """max_len in {1, 2, 15, 16, 17, 31, 32, 33}: the forced eos on either side of a 16-step burst; len_penalty 0.5, 1, 2"""
    from oracle.unity_oracle import UnitYOracle
    from streamspeech_b200.engine import Engine

    cfg, sd, eng, u64 = unity
    if zero_eos:
        sd = zero_eos_sd(cfg)
        eng = Engine(cfg, sd, None, None, device=0)
        u64 = UnitYOracle(cfg, sd, torch.float64)
    worst = Worst()
    try:
        S = 14
        lens = [S - (b * 5) % S for b in range(6)]
        x = unit_states(6, S, lens, 30 + zero_eos)
        whole = rows = 0
        forced = set()
        for ml in (1, 2, 15, 16, 17, 31, 32, 33):
            for lp in (0.5, 1.0, 2.0):
                got = eng.unit_search_batch(x.cuda().contiguous(), lens, ml, lp)
                want = u64.unit_search(x, lens, ml, lp)
                whole += check_rows(got, want, cfg, worst, f"zero_eos={zero_eos} ml={ml} lp={lp}")
                rows += len(want)
                forced |= {ml for r in want if len(r["tokens"]) == ml + 1}
                if ml == 1:
                    for a in got:  # exactly one unit and eos
                        assert len(a["tokens"]) == 2 and a["tokens"][-1] == cfg.eos and a["tokens"][0] != cfg.eos
        report(f"unit burst edges zero_eos={zero_eos}", whole=whole, rows=rows, forced=sorted(forced), **worst.as_dict())
        assert whole == rows, (whole, rows)  # every row clear of UNIT_MARGIN at every step
        if zero_eos:  # every row runs to the forced eos at every max_len
            assert forced == {1, 2, 15, 16, 17, 31, 32, 33}
    finally:
        if zero_eos:
            eng.close()


@pytest.mark.parametrize("B", [31, 32, 33, 64, 65])
def test_unit_search_launch_splits(unity, B):
    """ragged S with 1 and 1024 in one launch; B = 65: three launches, the last of one row"""
    cfg, _, eng, u64 = unity
    S = 1024
    lens = [1 if b == 0 else S if b == 1 else 1 + (97 * b) % S for b in range(B)]
    x = unit_states(B, S, lens, 201 if B == 64 else 40 + B)  # (seeds whose rows all clear UNIT_MARGIN)
    worst = Worst()
    got = eng.unit_search_batch(x.cuda().contiguous(), lens, 40)
    want = u64.unit_search(x, lens, 40)
    whole = check_rows(got, want, cfg, worst, f"B={B}")
    n = [len(r["tokens"]) for r in want]
    report(f"unit launch splits B={B}", whole=whole, lengths=sorted(set(n)), **worst.as_dict())
    assert whole == B and len(set(n)) > 2, (whole, n)


def test_unit_search_one_row_runs_on(unity):
    """every row but one finishes within the first burst (2, 2 and 3 tokens): the launch goes on for that row alone to the forced
    eos at step 40, the others stay put; every row compared whole"""
    cfg, sd, eng, u64 = unity
    lens = [6, 3, 1, 5]
    x = unit_states(4, 6, lens, 58)
    want = u64.unit_search(x, lens, 40)
    n = sorted(len(r["tokens"]) for r in want)
    assert n[-2] <= 16 and n[-1] == 41, n
    worst = Worst()
    assert check_rows(eng.unit_search_batch(x.cuda().contiguous(), lens, 40), want, cfg, worst, "one runs on") == 4
    report("unit one row runs on", lengths=[len(r["tokens"]) for r in want], **worst.as_dict())


def test_unit_search_refuses_1025_states(unity):
    from streamspeech_b200.engine import EngineError

    cfg, _, eng, _ = unity
    x = torch.zeros(2, 1025, 512, device="cuda")
    with pytest.raises(EngineError) as e:
        eng.unit_search_batch(x, [1025, 3], 10)
    assert e.value.code == -5  # SS_ERR_CAPACITY


def test_unit_search_duplicated_rows(unity):
    """unit rows 10 and 11 set to the row of the unit the search picks most: the lower index wins every exact tie"""
    from oracle.unity_oracle import UnitYOracle
    from streamspeech_b200.engine import Engine

    cfg, sd, _, u64 = unity
    lens = [14, 9, 4, 1]
    x = unit_states(4, 14, lens, 60)
    first = u64.unit_search(x, lens, 20)
    top = max(set(t for r in first for t in r["tokens"][:-1]), key=lambda t: sum(r["tokens"].count(t) for r in first))
    keys = ("decoder.embed_tokens.weight", "decoder.output_projection.weight")
    d = dup_row_sd(dup_row_sd(sd, keys[0], keys, 10, top), keys[0], keys, 11, top)
    eng = Engine(cfg, d, None, None, device=0)
    try:
        want = UnitYOracle(cfg, d, torch.float64).unit_search(x, lens, 20)
        ties = sum(r["ties"] for r in want)
        assert ties > 0 and any(10 in r["tokens"] for r in want) and not any(top in r["tokens"] or 11 in r["tokens"] for r in want)
        worst = Worst()
        check_rows(eng.unit_search_batch(x.cuda().contiguous(), lens, 20), want, cfg, worst, "duplicated rows")
        report("unit duplicated rows", ties=ties, **worst.as_dict())
    finally:
        eng.close()


# ---- T2U encoder: n = B * S rows per launch group (G = max(1, 32768 // S) samples); linears on the skinny kernel up to 64 rows, the
# fp32 tiled GEMM below 128, the wgmma GEMM from 128 (umma_linear 13, the default); (S, B) pairs over those classes and both attention
# kernels, S = 1024 with two launch groups
T2U_SHAPES = [(1, 1), (1, 40), (63, 1), (64, 1), (65, 1), (63, 3), (127, 1), (128, 1), (129, 2), (1024, 2), (1024, 33)]
# max-abs error relative to the sample's max |value|, per umma_linear, about five times the maxima measured on an H100 80GB HBM3
# (700 W): 4.2e-6 on the wgmma GEMM (S = 1024, B = 33, ragged), 3.2e-7 on the fp32 kernels (S = 1024, B = 33)
T2U_TOL = {13: 2e-5, 0: 2e-6}


@pytest.mark.parametrize("umma", [13, 0])
def test_t2u_encoder_shapes(unity, umma):
    cfg, _, eng, u64 = unity
    worst = Worst()
    eng.set_option("umma_linear", umma)
    try:
        for S, B in T2U_SHAPES:
            for ragged in (True, False):
                lens = [max(1, S - (b * 7) % S) for b in range(B)] if ragged else [S] * B
                if ragged and all(n == S for n in lens):
                    continue
                x = unit_states(B, S, lens, S * 131 + B)
                got = eng.t2u_encode_batch(x.cuda().contiguous(), lens).cpu().double()
                pick = sorted({0, B // 2, B - 1, min(32, B - 1)})  # (S = 1024: both launch groups)
                want = u64.t2u_encode(x[pick], [lens[b] for b in pick])
                for i, b in enumerate(pick):
                    n = lens[b]
                    err = float((got[b, :n] - want[i, :n]).abs().max() / want[i, :n].abs().max())
                    worst.add("t2u_rel", err, f"umma={umma} S={S} B={B} ragged={ragged} b={b}")
                    assert err < T2U_TOL[umma], (S, B, ragged, b, err)
    finally:
        eng.set_option("umma_linear", 13)
    report(f"t2u umma={umma}", **worst.as_dict())
