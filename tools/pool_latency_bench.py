#!/usr/bin/env python
"""Streams of different latencies in one stream pool vs one pool per latency, and the one-pass batched step on staggered streams.

Workload: 32 concurrent 10 s streaming-ASR utterances with staggered starts (stream j starts j % 8 rounds late), 11 at 160 ms,
11 at 320 ms and 10 at 640 ms chunks.  A round is 160 ms of wall time; a stream pushes its own segment only on the rounds when it is
due (every chunk_ms / 160 rounds).  Every round's host->device copies, batched steps and token reads are inside the timed region, as
in bench.py's asr_streams_leg.

Arms (run alternately, --repeats times each):
  a  mixed:     one pool, every slot at its own latency (ss_pool_set_chunk)
  b  split:     three handles, one pool per latency (each handle's ss_set_chunk) -- three steps per round
  c  lockstep:  32 equal-length streams at 160 ms starting together (one geometry group per step)
  d  staggered: the same 32 streams at 160 ms with the staggered starts of arm a (several geometry groups per step)
Arms c and d use only the handle-wide chunk setting, so they also run against builds without per-slot latency.

Before timing, arms a and b must give identical tokens at every call of every stream.  Reported per arm: ms per round and audio-s/s
(best and median), kernel launches per round, and, from the step geometry of an untimed pass: encoder passes per step of this build
(one per step with active rows), the number of subsampler geometry groups per step (= encoder passes per step of a build that runs
the layer stack once per group), and encoder rows per step.  The card name, power limit and max SM clock are read in the same process.

  python tools/pool_latency_bench.py [--arms a,b,c,d] [--repeats 3] [--dump DIR]
  python tools/pool_latency_bench.py --compare DIR_A DIR_B    (dumps of arms c / d from two builds: bytewise / largest row difference)
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

RATE = 16000
N_STREAMS, SECONDS = 32, 10.0
MIX = [160] * 11 + [320] * 11 + [640] * 10
ONE_PASS = True


def card():
    """name, power limit and max SM clock of the device this process runs on"""
    p = torch.cuda.get_device_properties(0)
    info = {"name": p.name}
    try:
        bus = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
        out = subprocess.run(["nvidia-smi", f"--id={bus}", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60)
        limit, clock = (x.strip() for x in out.stdout.strip().split(","))
        info.update(power_limit=limit, max_sm_clock=clock)
    except Exception as e:  # the numbers are still reported, marked as measured on an unidentified power limit
        info.update(power_limit=f"not read ({type(e).__name__})", max_sm_clock=None)
    return info


def chunks(seg_ms):
    """(attention chunk, conv chunk) of a segment size: the ASR agent's rule (speech_to_text.asr agent :361-375)"""
    c = seg_ms // 40
    return c, min(c, 16)


def geometry_key(F, T_final, attn, conv, half):
    """the subsampler group key of one stream's step (engine_pool.inc pool_geom) and its number of active encoder rows"""
    T1 = (F - 1) // 2 + 1
    T = (T1 - 1) // 2 + 1
    a0 = min(T_final, T)
    t1_lo = max(0, 2 * a0 - half)
    f_lo = max(0, 2 * t1_lo - half)
    return (a0 == 0, T - a0, T1 - t1_lo, F - f_lo, attn, conv), T - a0, T


class Arm:
    """one or more (engine, pool) pairs fed the same per-stream schedule; streams[j] = (pool index, slot, seg_ms, start round)"""

    def __init__(self, name, pools, streams, wavs):
        self.name, self.pools, self.streams, self.wavs = name, pools, streams, wavs
        self.calls = [[] for _ in streams]  # tokens of every call, per stream (untimed record pass)
        self.groups, self.rows, self.passes = [], [], []

    def run(self, record=False, half=2):
        for p, sl, _, _ in self.streams:
            self.pools[p][1].reset(sl)
        pos = [0] * len(self.streams)
        T_final = [0] * len(self.streams)
        rounds = 0
        while any(q < w.numel() for q, w in zip(pos, self.wavs)):
            for p, (eng, pool) in enumerate(self.pools):
                due = []
                for j, (pj, sl, seg, start) in enumerate(self.streams):
                    every = seg // 160
                    if pj == p and rounds >= start and (rounds - start) % every == 0 and pos[j] < self.wavs[j].numel():
                        n = RATE * seg // 1000
                        pool.push(sl, self.wavs[j][pos[j]:pos[j] + n])
                        pos[j] = min(pos[j] + n, self.wavs[j].numel())
                        due.append(j)
                if not due:
                    continue
                if record:
                    keys, rows = set(), 0
                    for j in due:
                        attn, conv = chunks(self.streams[j][2])
                        key, nA, _ = geometry_key(eng.num_fbank_frames(pos[j]), T_final[j], attn, conv, half)
                        if nA > 0:
                            keys.add(key)
                            rows += nA
                    self.groups.append(len(keys))
                    self.rows.append(rows)
                    self.passes.append((1 if rows else 0) if ONE_PASS else len(keys))
                pool.flush()
                if record:
                    for j in due:
                        r = pool.results[self.streams[j][1]]
                        self.calls[j].append(r["ctc"][0][0])
                        T_final[j] = r["T_final"]
            rounds += 1
        return rounds

    def timed(self):
        torch.cuda.synchronize()
        l0 = self.pools[0][0].launch_count()  # process-wide counter
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        rounds = self.run()
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e)
        return ms, rounds, self.pools[0][0].launch_count() - l0

    def dump(self, out_dir, cfg):
        os.makedirs(out_dir, exist_ok=True)
        torch.cuda.synchronize()
        for j, (p, sl, _, _) in enumerate(self.streams):
            eng, pool = self.pools[p]
            info = eng.pool_info(sl)
            T = pool.results[sl]["T"]
            np.save(os.path.join(out_dir, f"{self.name}_{j:02d}_tokens.npy"), np.array(self.calls[j][-1], dtype=np.int64))
            np.save(os.path.join(out_dir, f"{self.name}_{j:02d}_enc.npy"), read_rows(info["enc_out_ptr"], T, cfg.enc_dim))


def read_rows(ptr, T, D):
    class _Arr:  # float32 CUDA tensor over the pool's encoder rows of one slot
        __cuda_array_interface__ = {"shape": (T * D,), "typestr": "<f4", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_Arr(), device="cuda").view(T, D).cpu().numpy().copy()


def compare(dir_a, dir_b):
    """arms c / d dumped by two builds: c bytewise, d tokens equal and the largest encoder-row difference"""
    out = {}
    for arm in ("c", "d"):
        files = sorted(f for f in os.listdir(dir_a) if f.startswith(arm + "_"))
        if not files:
            continue
        same_bytes, tok_equal, worst = True, True, 0.0
        for f in files:
            a, b = open(os.path.join(dir_a, f), "rb").read(), open(os.path.join(dir_b, f), "rb").read()
            same_bytes &= a == b
            x, y = np.load(os.path.join(dir_a, f)), np.load(os.path.join(dir_b, f))
            if f.endswith("_tokens.npy"):
                tok_equal &= x.shape == y.shape and bool((x == y).all())
            else:
                worst = max(worst, float(np.abs(x - y).max()) if x.shape == y.shape and x.size else (0.0 if x.shape == y.shape else math.inf))
        out[arm] = {"files": len(files), "bytewise_identical": same_bytes, "tokens_equal": tok_equal, "max_abs_enc_diff": worst}
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arms", default="a,b,c,d")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--dump", default=None, help="write every stream's final tokens and encoder rows of arms c and d here")
    ap.add_argument("--compare", nargs=2, default=None, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        return compare(*args.compare)
    if not torch.cuda.is_available():
        raise SystemExit("pool_latency_bench needs a CUDA device: nothing is measured without one")
    torch.set_grad_enabled(False)
    from streamspeech_b200 import synth
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.engine import Engine
    from streamspeech_b200.scheduler import StreamPool

    global ONE_PASS  # builds with per-slot latency run the encoder once per step; earlier ones once per geometry group
    ONE_PASS = hasattr(Engine, "pool_set_chunk")
    arms_wanted = args.arms.split(",")
    cfg = ModelConfig()
    sd, gcmvn = synth.make_model_state_dict(cfg, 0), synth.make_gcmvn(cfg)
    wavs = [synth.make_audio(SECONDS, seed=5000 + j).contiguous() for j in range(N_STREAMS)]
    starts = [j % 8 for j in range(N_STREAMS)]
    max_s = int(SECONDS) + 2

    def engine(seg_ms):
        e = Engine(cfg, sd, None, gcmvn)
        e.set_chunk(*chunks(seg_ms))
        return e

    arms = {}
    if "a" in arms_wanted:
        e = engine(160)
        pool = StreamPool(e, n_slots=N_STREAMS, max_seconds=max_s, ctc_heads=1)
        slots = [pool.acquire() for _ in range(N_STREAMS)]
        for sl, seg in zip(slots, MIX):
            pool.set_chunk(sl, *chunks(seg))
        arms["a"] = Arm("a", [(e, pool)], [(0, sl, seg, st) for sl, seg, st in zip(slots, MIX, starts)], wavs)
    if "b" in arms_wanted:
        pools, streams = [], [None] * N_STREAMS
        for p, seg in enumerate((160, 320, 640)):
            idx = [j for j in range(N_STREAMS) if MIX[j] == seg]
            e = engine(seg)
            pool = StreamPool(e, n_slots=len(idx), max_seconds=max_s, ctc_heads=1)
            pools.append((e, pool))
            for j in idx:
                streams[j] = (p, pool.acquire(), seg, starts[j])
        arms["b"] = Arm("b", pools, streams, wavs)
    for name, st in (("c", [0] * N_STREAMS), ("d", starts)):
        if name in arms_wanted:
            e = engine(160)
            pool = StreamPool(e, n_slots=N_STREAMS, max_seconds=max_s, ctc_heads=1)
            arms[name] = Arm(name, [(e, pool)], [(0, pool.acquire(), 160, s) for s in st], wavs)

    # untimed record pass: tokens of every call, step geometry (also the warm-up of every shape the timed runs use)
    for arm in arms.values():
        arm.run(record=True, half=cfg.conv_kernel // 2)
    if "a" in arms and "b" in arms:
        assert arms["a"].calls == arms["b"].calls, "mixed-latency pool and per-latency pools disagree"
    if args.dump:
        for name in ("c", "d"):
            if name in arms:
                arms[name].dump(args.dump, cfg)
    times = {name: [] for name in arms}
    launches = {}
    rounds = {}
    for _ in range(args.repeats):  # alternate the arms: the host and the GPU are shared
        for name, arm in arms.items():
            ms, r, nl = arm.timed()
            times[name].append(ms / r)
            rounds[name], launches[name] = r, nl / r
    audio_s = N_STREAMS * SECONDS
    result = {"workload": f"streaming ASR, {N_STREAMS} concurrent {SECONDS:g} s utterances, 160 ms rounds, one GPU", "card": card(),
              "one_pass_build": ONE_PASS, "tokens_a_equal_b": True if "a" in arms and "b" in arms else None, "arms": {}}
    for name, arm in arms.items():
        steps = len(arm.groups)
        result["arms"][name] = {
            "rounds": rounds[name],
            "ms_per_round": {"best": min(times[name]), "median": statistics.median(times[name]), "runs": times[name]},
            "audio_s_per_s": {"best": audio_s / (min(times[name]) * rounds[name] * 1e-3),
                              "median": audio_s / (statistics.median(times[name]) * rounds[name] * 1e-3)},
            "launches_per_round": launches[name],
            "steps_per_round": steps / rounds[name],
            "encoder_passes_per_step": sum(arm.passes) / steps,
            "geometry_groups_per_step": sum(arm.groups) / steps,
            "rows_per_step": sum(arm.rows) / steps,
            "tokens_final": sum(len(c[-1]) for c in arm.calls),
        }
    print(json.dumps(result))
    for arm in arms.values():
        for e, _ in arm.pools:
            e.close()


if __name__ == "__main__":
    main()
