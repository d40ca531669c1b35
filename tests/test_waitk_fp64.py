"""GPU: the wait-k-stride-n agents (streamspeech_b200/waitk.py) on UnitY, Uni-UnitY and Chunk-UnitY against float64 restatements of
every stage they call, at the lengths and routes the fixture tests (tests/test_waitk_gpu.py, tests/test_unity_variants_gpu.py) do not
reach.

- Per-call stages, teacher-forced: the engine's agent runs call by call; at a compared call every stage's float64 reference gets the
  inputs the engine's stage had (the fbank rows of the source prefix, the engine's encoder rows, its previous hypothesis as prefix,
  its MT features, its T2U states, its units).  One near tie then excuses one decision and the run goes on.  Encoder rows within
  ENC_TOL of the route taken; MT tokens exact except at a step whose float64 top-2 margin is below MARGIN; MT features of
  [eos] + tokens and T2U states within relative bars; units by tests/test_search_fp64.py's UNIT_MARGIN rule, durations exact, the
  emitted samples within WAV_TOL of the float64 vocoder on the same units.  S2TT runs go to T = 1000 encoder rows; S2ST runs pass
  1024 unit positions; the S2TT default runs on UnitY and Uni-UnitY pass an MT prefix of 64 tokens; every finishing call's max_len
  is capped at max_decoder_positions - 1 = 1199.
- Chunk-UnitY's incremental encoder in the agent's call pattern on every STREAM_ROUTES entry, each call's route proven by
  cluster_steps() / launch_count(): all T rows against the float64 chunk encoder of the prefix, rows below the previous call's
  T_final bit-identical, and ss_mt_greedy with the stable-rows hint against a search that re-projects every row (the same tokens,
  features within HINT_REL) and, on the cluster route, against float64 with an MT prefix that grows past 64 tokens.
- The causal T2U encoder (Uni-UnitY) at tests/test_search_fp64.py's T2U_SHAPES, and the unit search on its output at launch splits.
- Uni-UnitY's whole-prefix re-encode (ss_encoder_forward, attention chunk 1, symmetric convolutions) on both sides of the wgmma switch.

Bars are about ten times the maxima measured on an H100 80GB HBM3 (700 W), given in the comments.  Every test prints one JSON line
(`pytest -s`) with its worst errors, near-tie counts and the edges it reached.
"""
import argparse
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.simuleval_compat import SpeechSegment

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
MARGIN = 1e-4  # float64 top-2 gap below which an MT decision may differ
# relative max-abs bars (error over the reference's max |value|), about ten times the maxima measured on an H100 80GB HBM3 (700 W)
MT_FEAT_REL = 1e-5  # 1.3e-6 (Chunk-UnitY, T = 1024, 128-token prefix); 5.1e-7 in the agents' runs
T2U_REL = 3e-6  # 2.3e-7 (Uni-UnitY S2ST k5n2)
WAV_TOL = 1e-4  # 8.4e-6 absolute (UnitY S2ST default, finishing call)
# the MT features of a search that reuses the cross K / V of final rows against those of one that projects every row: the two
# projections run the same rows as GEMMs of different row counts, which the engine may route to different kernels, so they agree
# to rounding, not bit for bit.  A hint that declares provisional rows final moves the features by about 1.0 (relative 1e-2).
HINT_REL = 1e-5  # 6.8e-7 (320 ms, T = 1016)
FILLER = 1338  # the token appended to an MT prefix whose search ended at once, so that the prefix keeps growing
UMMA_MIN_ROWS = 128


def _load(name):
    spec = importlib.util.spec_from_file_location(f"_wk_{name}", os.path.join(ROOT, "tests", f"{name}.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def enc64():
    return _load("test_encoder_fp64")


@pytest.fixture(scope="module")
def search64():
    return _load("test_search_fp64")


def checkpoint(variant):
    state = synth.make_unity_checkpoint(variant, seed=0)
    return ModelConfig.from_checkpoint(state), state["model"]


def engine(variant):
    """a handle as the wait-k agents make it: MT positions for the finishing call's max_len of max_decoder_positions - 1"""
    from streamspeech_b200.engine import Engine

    cfg, sd = checkpoint(variant)
    return cfg, sd, Engine(cfg, sd, None, synth.make_gcmvn(cfg), max_mt_positions=cfg.max_target_positions + 1)


def oracle_chunks(cfg):
    """(attention chunk, conv chunk) of the float64 encoder (Ref64.encoder) for the variant"""
    from oracle.unity_variant_oracle import oracle_geometry

    return oracle_geometry(cfg)


def rel(got, want):
    want = want.double()
    return float((got.double().to(want.device) - want).abs().max() / want.abs().max().clamp_min(1e-30))


# --------------------------------------------------------------------------------------------------------------------------------
# A. per-call stages of the agents, teacher-forced
# --------------------------------------------------------------------------------------------------------------------------------
# tag -> (kind, k1, k2, n, n2, segment ms, seconds, source seed, compare every k-th working call)
CASES = {
    "s2st_default": ("s2st", 3, 1, 1, 1, 320, 24.0, 71, 10),
    "s2st_k5n2": ("s2st", 5, 1, 2, 2, 640, 24.0, 72, 5),
    "s2tt_default": ("s2tt", 3, 1, 1, 1, 320, 40.0, 73, 8),
    "s2tt_k5n2": ("s2tt", 5, 1, 2, 2, 640, 40.0, 74, 4),
}
FIRST_SECONDS = 3.0  # every working call whose source is at most this long is compared
MAX_DECODER_POSITIONS = 1200


class Recorder:
    """the inputs and outputs of the engine stages one policy() call ran (instance attributes shadow the engine's methods)"""

    def __init__(self, eng):
        self.rec = {}
        for name in ("encoder", "encoder_stream_step", "mt_greedy", "t2u_encode_batch", "unit_search_batch"):
            setattr(eng, name, self._wrap(name, getattr(eng, name)))

    def _wrap(self, name, fn):
        def call(*args, **kw):
            out = fn(*args, **kw)
            if name == "encoder":
                self.rec["feats"], self.rec["enc"] = args[0][0].clone(), out[0].clone()
            elif name == "encoder_stream_step":
                T = out[0]
                self.rec["feats"], self.rec["enc"], self.rec["t_final"] = args[0].clone(), args[1][:T].clone(), out[1]
            elif name == "mt_greedy":
                self.rec["mt"] = dict(enc=args[0].clone(), prefix=list(args[1] or []), new=int(args[2]), max_len_b=int(kw["max_len_b"]),
                                      stable_rows=int(kw.get("stable_rows", 0)), tokens=list(out[0]), feats=out[1].clone())
            elif name == "t2u_encode_batch":
                self.rec["t2u"] = dict(x=args[0].clone(), lengths=list(args[1]), out=out.clone())
            else:
                self.rec["units"] = dict(t2u=args[0].clone(), lengths=list(args[1]), max_len=int(args[2]), out=out)
            return out
        return call


def make_agent(variant, kind, k1, k2, n, n2, seg):
    from streamspeech_b200.waitk import WaitkS2STAgent, WaitkS2TTAgent, add_waitk_args

    parser = argparse.ArgumentParser()
    add_waitk_args(parser)
    user_dir = "researches/ctc_unity" if variant == "unity" else f"researches/{variant}"
    args = parser.parse_args(["--model-path", "synthetic", "--user-dir", user_dir, "--data-bin", ".", "--vocoder", "synthetic", "--vocoder-cfg",
                              "none", "--dur-prediction", "--lagging-k1", str(k1), "--lagging-k2", str(k2), "--stride-n", str(n), "--stride-n2",
                              str(n2), "--unit-per-subword", "15", "--segment-size", str(seg)])
    return WaitkS2STAgent(args) if kind == "s2st" else WaitkS2TTAgent(args)


def check_mt(o64, mt, cfg, worst, what):
    """the engine's hypothesis against float64 logits of [eos] + tokens over the engine's encoder rows: every searched step's token
    (eos at the last) is the float64 arg-max unless that step's top-2 margin is below MARGIN.  Returns (near ties, excused)."""
    prefix, toks = mt["prefix"], mt["tokens"]
    start, n = len(prefix), len(toks)
    assert toks[:start] == prefix, (what, "the hypothesis does not extend its prefix")
    max_len = start + mt["new"] if mt["new"] != -1 else min(mt["max_len_b"], MAX_DECODER_POSITIONS - 1)
    assert start <= n <= max_len, (what, start, n, max_len)
    feats = o64.mt_features(torch.tensor([[cfg.eos] + toks]), mt["enc"].unsqueeze(1))[0]  # [n + 1, D]
    worst.add("mt_feat_rel", rel(mt["feats"], feats), what)
    lp = F.log_softmax(F.linear(feats[start:], o64.sd["target_unigram_decoder.output_projection.weight"]), dim=-1)
    lp[:, cfg.pad] = -float("inf")
    near = excused = 0
    for i, step in enumerate(range(start, n + 1)):
        row = lp[i].clone()
        if step >= max_len:
            keep = row[cfg.eos].clone()
            row[:] = -float("inf")
            row[cfg.eos] = keep
        elif step < 1:
            row[cfg.eos] = -float("inf")
        top = row.topk(2)
        margin = float(top.values[0] - top.values[1])
        want = toks[step] if step < n else cfg.eos
        near += margin < MARGIN
        if int(top.indices[0]) != want:
            assert margin < MARGIN, (what, "MT step", step, "differs away from a near tie", margin)
            excused += 1
    return near, excused


@pytest.mark.parametrize("variant", ["unity", "uni_unity", "chunk_unity"])
@pytest.mark.parametrize("tag", sorted(CASES))
def test_waitk_agent_stages_vs_fp64(enc64, search64, variant, tag):
    from oracle.streamspeech_oracle import StreamSpeechOracle
    from oracle.unity_variant_oracle import VariantUnitYOracle

    kind, k1, k2, n, n2, seg, seconds, seed, every = CASES[tag]
    agent = make_agent(variant, kind, k1, k2, n, n2, seg)
    cfg = agent.cfg
    assert cfg.unity_variant == variant and cfg.max_target_positions == MAX_DECODER_POSITIONS
    sd = checkpoint(variant)[1]
    ref = enc64.Ref64(cfg, sd, synth.make_gcmvn(cfg))
    u64 = VariantUnitYOracle(cfg, sd, F64, device="cuda")
    voc = StreamSpeechOracle(cfg, {}, synth.make_vocoder_state_dict(cfg.vocoder, 1), None, chunk_size=None, dtype=F64,
                             device="cuda") if kind == "s2st" else None
    ac, cc = oracle_chunks(cfg)
    rec = Recorder(agent.engine)
    wav = synth.make_audio(seconds, seed=seed)
    step = seg * 16
    worst, w_units = enc64.Worst(), search64.Worst()
    edges = {"max_prefix": 0, "max_T": 0, "max_unit_positions": 0, "capped_finish": 0}
    counts = {"calls": 0, "working": 0, "compared": 0, "mt_steps_near_tie": 0, "mt_excused": 0, "unit_rows_whole": 0, "unit_rows": 0}
    try:
        for i in range(0, len(wav), step):
            fin = i + step >= len(wav)
            rec.rec = {}
            agent.push(SpeechSegment(content=wav[i:i + step].tolist(), sample_rate=16000, finished=fin))
            action = agent.policy()
            counts["calls"] += 1
            r = rec.rec
            if "mt" not in r:
                continue
            w = counts["working"]
            counts["working"] += 1
            mt = r["mt"]
            T = mt["enc"].shape[0]
            edges["max_prefix"] = max(edges["max_prefix"], len(mt["prefix"]))
            edges["max_T"] = max(edges["max_T"], T)
            if mt["new"] == -1 and mt["max_len_b"] == MAX_DECODER_POSITIONS - 1:
                edges["capped_finish"] += 1
            if "units" in r:
                edges["max_unit_positions"] = max(edges["max_unit_positions"], len(r["units"]["out"][0]["tokens"]))
            if not (fin or w % every == 0 or (i + step) <= FIRST_SECONDS * 16000):
                continue
            counts["compared"] += 1
            what = f"{variant} {tag} call {counts['calls'] - 1} T={T}"
            # encoder: the route this call took
            F_ = r["feats"].shape[0]
            enc_want = ref.encoder(r["feats"], None, ac, cc)[0]
            route = "stream" if agent.incremental else "tc" if T >= UMMA_MIN_ROWS else "fp32"
            worst.add(f"enc_{route}", enc64.maxdiff(r["enc"], enc_want), what)
            assert torch.equal(r["enc"], mt["enc"]), what  # the MT search read the rows the encoder wrote
            near, excused = check_mt(u64.o, mt, cfg, worst, what)
            counts["mt_steps_near_tie"] += near
            counts["mt_excused"] += excused
            if kind == "s2tt":
                continue
            if "t2u" not in r:
                continue
            t = r["t2u"]
            S = t["lengths"][0]
            assert torch.equal(t["x"][0], mt["feats"][:S]), what
            worst.add("t2u_rel", rel(t["out"][0], u64.t2u_encode(t["x"].double(), t["lengths"])[0]), what)
            us = r["units"]
            want = u64.unit_search(us["t2u"], us["lengths"], us["max_len"])
            whole = search64.check_rows(us["out"], want, cfg, w_units, what)
            counts["unit_rows_whole"] += whole
            counts["unit_rows"] += 1
            if action.is_read() or not action.content.content:
                continue
            units = agent.trace["units"]
            w64, dur = voc.vocoder(units, True)
            assert dur.view(-1).tolist() == list(agent.trace["dur"]), (what, "durations")
            got = torch.tensor(action.content.content, dtype=F64)
            worst.add("wav", enc64.maxdiff(got, w64[-got.numel():]), what)
        agent.engine.check_async_error()
    finally:
        agent.engine.close()
    enc64.report(f"waitk_stages_fp64_{variant}_{tag}", edges=edges, **counts, **worst.as_dict(), **w_units.as_dict())
    assert counts["compared"] >= 5, counts
    worst.check({**enc64.ENC_TOL, **{f"enc_{k}": v for k, v in enc64.ENC_TOL.items()}, "mt_feat_rel": MT_FEAT_REL, "t2u_rel": T2U_REL,
                 "wav": WAV_TOL})
    # the edges these runs exist for
    assert edges["capped_finish"] == 1, edges
    if tag == "s2tt_default" and variant != "chunk_unity":  # (the synthetic Chunk-UnitY ends its hypotheses early on this source)
        assert edges["max_prefix"] > 64, edges
    if kind == "s2tt":
        assert edges["max_T"] >= 1000, edges
    else:
        assert edges["max_unit_positions"] > 1024, edges
        assert counts["unit_rows"] > 0 and counts["unit_rows_whole"] > 0, counts


# --------------------------------------------------------------------------------------------------------------------------------
# B. Chunk-UnitY's streaming step on every route, and the stable-rows hint
# --------------------------------------------------------------------------------------------------------------------------------
# segment ms -> seconds of source: the 320 ms case runs to F = 4094 fbank frames, T = 1024 (the engine's capacity)
STREAM_CASES = {320: (41.0, 4094), 640: (12.0, None)}


@pytest.mark.parametrize("seg", sorted(STREAM_CASES))
def test_chunk_unity_stream_routes_vs_fp64(enc64, seg):
    from streamspeech_b200.engine import Engine

    from oracle.unity_variant_oracle import VariantUnitYOracle

    seconds, f_cap = STREAM_CASES[seg]
    cfg, sd, e = engine("chunk_unity")
    u64 = VariantUnitYOracle(cfg, sd, F64, device="cuda")
    e2 = Engine(cfg, sd, None, synth.make_gcmvn(cfg), max_mt_positions=cfg.max_target_positions + 1)  # the unhinted searches: every row projected on every call
    worst, routes_seen, max_prefix, near = enc64.Worst(), {}, 0, 0
    try:
        ac, cc = cfg.encoder_chunk()
        G = enc64.lcm(ac, cc)
        e.set_chunk(ac, cc)
        ref = enc64.Ref64(cfg, sd, synth.make_gcmvn(cfg))
        wav = synth.make_audio(seconds, seed=81).cuda().contiguous()
        feats = e.fbank(wav)
        Fs = []
        for n in range(seg * 16, wav.numel() + seg * 16, seg * 16):
            F_ = e.num_fbank_frames(min(n, wav.numel()))
            Fs.append(min(F_, f_cap) if f_cap else F_)
        enc_want = {}
        hint_calls = 0
        for route, (pe, cl, ff) in enc64.STREAM_ROUTES.items():
            e.set_option("persistent_encoder", pe)
            e.set_option("persistent_encoder_cluster", cl)
            e.set_option("persistent_ffn_fused", ff)
            buf = torch.full((1024, cfg.enc_dim), float("nan"), device="cuda")
            prev, t_final, prefix = None, 0, None
            e.encoder_stream_reset()
            try:
                for k, F_ in enumerate(Fs):
                    nA = enc64.out_frames(F_) - min(t_final, enc64.out_frames(F_))
                    n_cl, n_l = e.cluster_steps(), e.launch_count()
                    T, tf = e.encoder_stream_step(feats[:F_].contiguous(), buf)
                    d_cl, d_l = e.cluster_steps() - n_cl, e.launch_count() - n_l
                    what = f"seg {seg} {route} call {k} F={F_} nA={nA}"
                    want_route = enc64.expected_route(route, nA)
                    got_route = ("cluster" if d_cl == 1 else "per_op" if d_l >= enc64.PER_OP_STEP
                                 else "persistent" if 0 < d_l <= enc64.ONE_LAUNCH_STEP else f"? ({d_l})")
                    if want_route == "none":
                        got_route = want_route if d_l == 0 and d_cl == 0 else got_route
                    assert got_route == want_route and d_cl == (want_route == "cluster"), (what, got_route, d_l, d_cl)
                    routes_seen.setdefault(route, {}).setdefault(want_route, 0)
                    routes_seen[route][want_route] += 1
                    assert tf % G == 0 and tf <= T and T == enc64.out_frames(F_), what
                    if prev is not None:
                        assert torch.equal(buf[:t_final], prev[:t_final]), (what, "a final row changed")
                    if F_ not in enc_want:
                        enc_want[F_] = ref.encoder(feats[:F_], None, ac, cc)[0]
                    worst.add("stream", enc64.maxdiff(buf[:T], enc_want[F_]), what)
                    # the agent's MT call (one new token, -1 once the source has ended) with the stable-rows hint, and the same search
                    # on a handle that projects every row
                    fin = k == len(Fs) - 1
                    new = -1 if fin else 1
                    max_len_b = min(F_ + 200, cfg.max_target_positions - 1)
                    toks, fts = e.mt_greedy(buf[:T], prefix, new, max_len_b=max_len_b, stable_rows=tf)
                    toks2, fts2 = e2.mt_greedy(buf[:T].clone(), prefix, new, max_len_b=max_len_b)
                    assert toks == toks2, (what, "the stable-rows hint changed the tokens")
                    worst.add("hint_rel", rel(fts, fts2), what)
                    hint_calls += t_final > 0
                    max_prefix = max(max_prefix, len(prefix or []))
                    if route == "cluster" and (k % 8 == 0 or fin):
                        mt = dict(enc=buf[:T].clone(), prefix=list(prefix or []), new=new, max_len_b=max_len_b, tokens=toks, feats=fts)
                        near += check_mt(u64.o, mt, cfg, worst, what)[0]
                    prefix = toks if len(toks) > len(prefix or []) else toks + [FILLER]
                    prev, t_final = buf[:T].clone(), tf
            finally:
                e.set_option("persistent_encoder", 1)
                e.set_option("persistent_encoder_cluster", 1)
                e.set_option("persistent_ffn_fused", 1)
        e.check_async_error()
        e2.check_async_error()
    finally:
        e.close()
        e2.close()
    enc64.report(f"chunk_unity_stream_routes_fp64_seg{seg}", calls=len(Fs), T_max=enc64.out_frames(Fs[-1]), routes=routes_seen,
                 hinted_calls=hint_calls, max_prefix=max_prefix, mt_steps_near_tie=near, **worst.as_dict())
    worst.check({**enc64.ENC_TOL, "hint_rel": HINT_REL, "mt_feat_rel": MT_FEAT_REL})
    assert routes_seen["cluster"].get("cluster", 0) > 0, routes_seen
    assert routes_seen["persistent_fused"].get("persistent", 0) > 0, routes_seen
    assert routes_seen["persistent_unfused"].get("persistent", 0) > 0, routes_seen
    assert set(routes_seen["per_op"]) == {"per_op"}, routes_seen
    assert hint_calls > 0
    if f_cap:
        assert enc64.out_frames(Fs[-1]) == 1024 and max_prefix > 64, (Fs[-1], max_prefix)


# --------------------------------------------------------------------------------------------------------------------------------
# C. the causal T2U encoder and the unit search on its output
# --------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def uni():
    from oracle.unity_variant_oracle import VariantUnitYOracle

    cfg, sd, e = engine("uni_unity")
    assert cfg.uni_encoder
    yield cfg, sd, e, VariantUnitYOracle(cfg, sd, F64, device="cuda")
    e.close()


# relative max-abs bars of the causal T2U encoder per umma_linear: 4.0e-6 on the wgmma GEMM, 2.9e-7 on the fp32 kernels (S = 1024,
# B = 33); rows before a changed position moved by exactly 0 on both
CAUSAL_T2U_TOL = {13: 4e-5, 0: 3e-6}


@pytest.mark.parametrize("umma", [13, 0])
def test_causal_t2u_encoder_shapes(search64, uni, umma):
    cfg, _, e, u64 = uni
    assert u64.o.cfg.uni_encoder
    worst = search64.Worst()
    e.set_option("umma_linear", umma)
    try:
        for S, B in search64.T2U_SHAPES:
            for ragged in (True, False):
                lens = [max(1, S - (b * 7) % S) for b in range(B)] if ragged else [S] * B
                if ragged and all(n == S for n in lens):
                    continue
                x = search64.unit_states(B, S, lens, S * 131 + B)
                got = e.t2u_encode_batch(x.cuda().contiguous(), lens)
                pick = sorted({0, B // 2, B - 1, min(32, B - 1)})
                want = u64.t2u_encode(x[pick], [lens[b] for b in pick])
                for i, b in enumerate(pick):
                    m = lens[b]
                    err = rel(got[b, :m], want[i, :m])
                    worst.add("t2u_rel", err, f"umma={umma} S={S} B={B} ragged={ragged} b={b}")
                    assert err < CAUSAL_T2U_TOL[umma], (S, B, ragged, b, err)
                # causality: row s of a sample does not move when later positions change
                if S > 1:
                    y = x.clone()
                    y[:, S // 2:] += 1.0
                    got2 = e.t2u_encode_batch(y.cuda().contiguous(), lens)
                    moved = rel(got2[0, :S // 2], got[0, :S // 2])
                    worst.add("prefix_rows_moved", moved, f"umma={umma} S={S} B={B} ragged={ragged}")
                    assert moved < CAUSAL_T2U_TOL[umma], (S, B, ragged, "a row moved when later positions changed", moved)
    finally:
        e.set_option("umma_linear", 13)
    search64.report(f"causal t2u umma={umma}", **worst.as_dict())


@pytest.mark.parametrize("B", [31, 32, 33, 65])
def test_unit_search_on_causal_t2u_launch_splits(search64, uni, B):
    """ragged S with 1 and 1024 in one launch, states from the engine's causal T2U encoder; the float64 search on the same states"""
    cfg, _, e, u64 = uni
    S = 1024
    lens = [1 if b == 0 else S if b == 1 else 1 + (97 * b) % S for b in range(B)]
    x = search64.unit_states(B, S, lens, 40 + B)
    t2u = e.t2u_encode_batch(x.cuda().contiguous(), lens)
    got = e.unit_search_batch(t2u, lens, 40)
    worst = search64.Worst()
    want = u64.unit_search(t2u, lens, 40)
    whole = search64.check_rows(got, want, cfg, worst, f"B={B}")
    n = [len(r["tokens"]) for r in want]
    search64.report(f"causal unit launch splits B={B}", whole=whole, lengths=sorted(set(n)), **worst.as_dict())
    assert whole == B, (whole, n)  # every row clear of UNIT_MARGIN at every step


# --------------------------------------------------------------------------------------------------------------------------------
# D. Uni-UnitY's re-encode across the wgmma switch
# --------------------------------------------------------------------------------------------------------------------------------
def test_uni_unity_reencode_across_wgmma_switch(enc64, uni):
    """ss_encoder_forward at chunk (1, 0) on prefixes of T = 127, 128, 129 and 1024 rows, umma_linear 13 and 0: a wgmma GEMM runs
    exactly when umma_linear = 13 and T >= umma_min_rows"""
    cfg, sd, e, _ = uni
    assert cfg.encoder_chunk() == (1, 0)
    e.set_chunk(1, 0)
    e.set_option("umma_min_rows", UMMA_MIN_ROWS)
    ref = enc64.Ref64(cfg, sd, synth.make_gcmvn(cfg))
    feats = e.fbank(synth.make_audio(41.0, seed=19).cuda().contiguous())[:4094].contiguous()
    worst = enc64.Worst()
    for F_ in (508, 512, 516, 4094):
        T = enc64.out_frames(F_)
        want = ref.encoder(feats[:F_], None, 1, None)[0]
        for umma in (13, 0):
            e.set_option("umma_linear", umma)
            try:
                out, ran = enc64.wgmma_ran(e, lambda: e.encoder(feats[:F_].unsqueeze(0).contiguous()))
            finally:
                e.set_option("umma_linear", 13)
            tc = umma == 13 and T >= UMMA_MIN_ROWS
            assert ran == tc, (F_, umma, ran)
            worst.add("tc" if tc else "fp32", enc64.maxdiff(out[0], want), f"T={T} umma={umma}")
    assert [enc64.out_frames(f) for f in (508, 512, 516, 4094)] == [127, 128, 129, 1024]
    enc64.report("uni_unity_reencode_wgmma_switch_fp64", **worst.as_dict())
    worst.check(enc64.ENC_TOL)
