"""Stage split of OfflineS2STGenerator.generate and the per-sample decoder stages against the batched ones.

For B padded utterances (synthetic weights and audio) the script times, with CUDA events, each stage of generate():
encoder, CTC prints, MT search, MT features, T2U + unit decoder.  The CTC / MT-features / T2U stages run in two arms, alternated
rep by rep: the per-sample loop generate() used before the batched calls existed (kept below as `per_sample_arm`) and the
batched calls (`batched_arm`, what generate() runs now).  Before timing it checks that both arms give identical integer outputs
(CTC prints, unit arg-max, units) and reports the mt_feats difference.  Per stage it reports the median time, kernel launches
(ss_launch_count) and host synchronisations (calls that block the host, counted here from the calls each arm makes), and it
prints the card name and power limit of the run.

    python tools/offline_units_bench.py --batch 8 32 --seconds 15 --max-len-b 100 --reps 5 --json out.json
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402
from streamspeech_b200.engine import Engine  # noqa: E402

STAGES = ("encoder", "ctc", "mt_search", "mt_features", "t2u_units")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def per_sample_arm(eng, enc, out_len, hyps, stage):
    """the per-sample loops of generate() before the batched calls; returns (outputs, host synchronisations)"""
    c = eng.cfg
    B, T = enc.shape[0], enc.shape[1]
    if stage == "ctc":
        res = []
        for b in range(B):
            eb = enc[b].contiguous()
            am = torch.zeros(T, dtype=torch.int64, device=eb.device)
            res.append((eng.ctc_greedy_rows(0, eb, 0, am), eng.ctc_greedy_rows(1, eb, 0, am)))
        return res, 2 * B  # one device->host copy per head and sample
    if stage == "t2u_units":  # `hyps` holds the per-sample features here
        units, argmax = [], []
        syncs = 0
        try:
            for b in range(B):
                eng.set_unit_batch_index(b)  # device synchronisation + copy
                r = eng.t2u_unit_decode(hyps[b].contiguous(), n_pad_tail=n_pad_of[b], mask_eos=True)
                units.append(eng.units_to_host(r))
                argmax.append(r["argmax"].tolist())
                syncs += 3 + (1 if n_pad_of[b] > 0 else 0)  # positional row, two device->host copies, key-length upload
        finally:
            eng.set_unit_batch_index(0)
        return (units, argmax), syncs
    max_tgt_len = max(len(h) for h in hyps) + 1
    n_pad = [max_tgt_len - (len(h) + 1) for h in hyps]
    prev = [[c.eos] + h + [c.pad] * n for h, n in zip(hyps, n_pad)]
    return [eng.mt_features(enc[b, : out_len[b]].contiguous(), prev[b]) for b in range(B)], B  # stage mt_features: token upload


n_pad_of = []  # pad tails of the current batch (the T2U stage of both arms)


def batched_arm(eng, enc, out_len, hyps, stage):
    c = eng.cfg
    if stage == "ctc":
        res, _ = eng.ctc_greedy_batch(enc)
        return res, 1
    if stage == "mt_features":
        max_tgt_len = max(len(h) for h in hyps) + 1
        prev = [[c.eos] + h + [c.pad] * (max_tgt_len - 1 - len(h)) for h in hyps]
        return eng.mt_features_batch(enc, out_len, prev), 1  # token / length upload
    units, argmax, _ = eng.t2u_unit_decode_batch(hyps, n_pad_of, mask_eos=True)
    # positional rows upload, one device->host copy, and the key-length upload when some sample has a pad tail
    return (units, argmax), 2 + (1 if any(n_pad_of) else 0)


def timed(eng, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n0 = eng.launch_count()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1), eng.launch_count() - n0


def run_batch(eng, B, seconds, max_len_b, reps):
    global n_pad_of
    feats = [eng.fbank(synth.make_audio(seconds, seed=7000 + b).cuda()) for b in range(B)]
    F = max(f.shape[0] for f in feats)
    src = torch.zeros(B, F, eng.cfg.feat_dim, device="cuda")
    for b, f in enumerate(feats):
        src[b, : f.shape[0]] = f
    lengths = [f.shape[0] for f in feats]
    out_len = [eng.encoder_out_frames(n) for n in lengths]
    arms = {"per_sample": per_sample_arm, "batched": batched_arm}
    times = {a: {s: [] for s in STAGES} for a in arms}
    launches = {a: {} for a in arms}
    syncs = {a: {} for a in arms}
    checked = None
    for rep in range(reps + 1):  # rep 0 warms up every shape and checks the outputs
        for arm_name in (("per_sample", "batched") if rep % 2 == 0 else ("batched", "per_sample")):
            arm = arms[arm_name]
            enc, t, n = timed(eng, lambda: eng.encoder(src, lengths))
            times[arm_name]["encoder"].append(t)
            launches[arm_name]["encoder"] = n
            ctc, t, n = timed(eng, lambda: arm(eng, enc, out_len, None, "ctc"))
            times[arm_name]["ctc"].append(t)
            launches[arm_name]["ctc"], syncs[arm_name]["ctc"] = n, ctc[1]
            hyps, t, n = timed(eng, lambda: eng.mt_greedy_batch(enc, out_len, max_len_b))
            times[arm_name]["mt_search"].append(t)
            launches[arm_name]["mt_search"] = n
            S = max(len(h) for h in hyps) + 1
            n_pad_of = [S - 1 - len(h) for h in hyps]
            mf, t, n = timed(eng, lambda: arm(eng, enc, out_len, hyps, "mt_features"))
            times[arm_name]["mt_features"].append(t)
            launches[arm_name]["mt_features"], syncs[arm_name]["mt_features"] = n, mf[1]
            fe = mf[0] if arm_name == "per_sample" else mf[0].contiguous()
            un, t, n = timed(eng, lambda: arm(eng, enc, out_len, fe, "t2u_units"))
            times[arm_name]["t2u_units"].append(t)
            launches[arm_name]["t2u_units"], syncs[arm_name]["t2u_units"] = n, un[1]
            if rep == 0:
                if checked is None:
                    checked = {"ctc": ctc[0], "units": un[0], "feats": [f.clone() for f in fe]}
                else:
                    assert ctc[0] == checked["ctc"], "CTC prints differ between the arms"
                    assert un[0] == checked["units"], "units / unit arg-max differ between the arms"
                    d = max(float((fe[b] - checked["feats"][b]).abs().max()) for b in range(B))
                    checked["mt_feats_max_abs"] = d
    med = {a: {s: statistics.median(v[1:]) for s, v in times[a].items()} for a in arms}
    return {"B": B, "seconds": seconds, "max_len_b": max_len_b, "reps": reps, "S": S, "median_ms": med, "launches": launches,
            "host_syncs": syncs, "mt_feats_max_abs": checked["mt_feats_max_abs"], "integer_outputs_identical": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--seconds", type=float, default=15.0)
    ap.add_argument("--max-len-b", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.set_grad_enabled(False)
    cfg = ModelConfig()
    cfg.uni_encoder = False
    eng = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1), synth.make_gcmvn(cfg))
    eng.set_chunk(None, None)
    res = {"card": card(), "runs": []}
    print(json.dumps(res["card"]))
    for B in a.batch:
        r = run_batch(eng, B, a.seconds, a.max_len_b, a.reps)
        res["runs"].append(r)
        print(f"B = {B} (S = {r['S']}), mt_feats max-abs {r['mt_feats_max_abs']:.2e}, integer outputs identical")
        print(f"  {'stage':<12} {'per-sample ms':>14} {'batched ms':>11} {'launches':>17} {'host syncs':>12}")
        for s in STAGES:
            p, b = r["median_ms"]["per_sample"][s], r["median_ms"]["batched"][s]
            lp, lb = r["launches"]["per_sample"][s], r["launches"]["batched"][s]
            sp, sb = r["host_syncs"]["per_sample"].get(s, "-"), r["host_syncs"]["batched"].get(s, "-")
            print(f"  {s:<12} {p:>14.2f} {b:>11.2f} {lp:>8} / {lb:<7} {str(sp):>5} / {str(sb):<5}")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
