"""Concurrent simultaneous S2TT streams: PooledS2TTAgents on one stream pool vs the same utterances through one single-stream
StreamSpeechS2TTAgent, one after another, on the same engine (synthetic 12-layer model).

Workloads: N in {1, 8, 16, 32} concurrent utterances of --seconds (default 6.4; synth.make_audio, seeds 9000 + j) at 320 ms segments,
and a mixed set of 16 streams, every other one at 640 ms.  The finishing call of an utterance reserves max_len = fbank frames + 200
self-attention entries plus one per earlier MT call, whatever the length of the hypothesis: 6.4 s fits the engine's default
max_mt_positions = 1024, a 10 s utterance needs --max-mt-positions 2048 (32 MB of incremental MT cache per pool slot instead of 16 MB).
The pool is sized from --seconds.  The pooled arm feeds all streams round by round through pushpop_many (a 640 ms stream every
second 320 ms round); the single arm plays each utterance to its end before the next.

Before timing, both arms must emit identical actions, text deltas and CTC / MT tokens on every call.  Then the two arms run
alternately (--reps times each); every run ends with a device synchronisation and is timed on the host clock.  Reported per
workload: audio seconds per wall second of both arms; the pooled arm's device time per flush stage (CUDA events at the stage
boundaries, so each stage includes the host work between its engine calls); kernel launches per flush; host synchronisations per
flush, counted from the engine calls the flush makes (one per upload or read-back, one per 16-step MT burst); the card's name, power
limit and max SM clock, read in the same run.

    python tools/pool_s2tt_bench.py [--streams 1 8 16 32] [--seconds 6.4] [--max-mt-positions 1024] [--reps 2] [--out results/pool_s2tt_bench.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.agent import StreamSpeechS2TTAgent  # noqa: E402
from streamspeech_b200.scheduler import PooledS2TTAgent, StreamPool, pushpop_many  # noqa: E402
from streamspeech_b200.simuleval_compat import SpeechSegment  # noqa: E402

KEYS = ("asr_tokens", "st_tokens", "mt_tokens")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def args_for(seg, max_mt_positions=1024):
    return argparse.Namespace(max_mt_positions=max_mt_positions, model_path="synthetic", data_bin=".", config_yaml=None, multitask_config_yaml=None, sample_rate=16000, max_len=200,
                              force_finish=False, lagging_k1=0, lagging_k2=0, segment_size=seg, stride_n=1, stride_n2=1, unit_per_subword=15,
                              source_segment_size=seg, device_index=0)


def obs(seg, agent):
    return (not seg.is_empty, seg.content if not seg.is_empty else None, bool(seg.finished), tuple(str(agent.trace.get(k)) for k in KEYS))


def run_single(single, wavs, segs):
    out = []
    for w, seg in zip(wavs, segs):
        c = seg // 40
        single.engine.set_chunk(c, min(c, 16))
        single.reset()
        n, calls = 16 * seg, []
        for i in range(0, len(w), n):
            calls.append(obs(single.pushpop(SpeechSegment(content=w[i:i + n].tolist(), sample_rate=16000, finished=i + n >= len(w))), single))
        out.append(calls)
    torch.cuda.synchronize()
    return out


def run_pooled(pool, agents, wavs, segs):
    out = [[] for _ in agents]
    pos = [0] * len(agents)
    rnd = 0
    while any(p < len(w) for p, w in zip(pos, wavs)):
        due = [j for j, s in enumerate(segs) if rnd % (s // 320) == 0 and pos[j] < len(wavs[j])]
        chunks = []
        for j in due:
            if pos[j] == 0 and agents[j].states.source_finished:  # its previous utterance ended on an unchanged hypothesis: no reset quirk
                agents[j].reset()
            n = 16 * segs[j]
            chunks.append(SpeechSegment(content=wavs[j][pos[j]:pos[j] + n].tolist(), sample_rate=16000, finished=pos[j] + n >= len(wavs[j])))
            pos[j] += n
        for j, seg in zip(due, pushpop_many([agents[j] for j in due], chunks)):
            out[j].append(obs(seg, agents[j]))
        rnd += 1
    torch.cuda.synchronize()
    return out


class SyncCounter:
    """counts the host synchronisations of the engine calls a flush makes (wraps the engine's methods on this instance)"""

    def __init__(self, eng):
        self.n = 0
        f_step = eng.pool_step

        def step(*a, **kw):
            self.n += 2  # descriptor staging + CTC read-back
            return f_step(*a, **kw)
        eng.pool_step = step
        f = eng.pool_mt_greedy_incremental

        def mt(slots, prefixes, limits, max_lens):
            hyps = f(slots, prefixes, limits, max_lens)
            for g0 in range(0, len(slots), 32):
                steps = [len(h) - len(p or []) + 1 for h, p in zip(hyps[g0:g0 + 32], prefixes[g0:g0 + 32])]
                self.n += 1  # upload
                if len(steps) >= 2:  # the engine's mt_batch_min_rows: smaller groups decode on the single-token kernel
                    self.n += -(-max(steps) // 16)  # one read-back per burst of the group
                else:
                    self.n += sum(-(-s // 16) for s in steps)  # per stream
            return hyps
        eng.pool_mt_greedy_incremental = mt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 8, 16, 32])
    ap.add_argument("--seconds", type=float, default=6.4, help="length of every utterance")
    ap.add_argument("--max-mt-positions", type=int, default=1024, help="the engine's MT cache entries (2048 for utterances above about 8 s)")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    single = StreamSpeechS2TTAgent(args_for(320, a.max_mt_positions))
    eng = single.engine
    n_max = max(max(a.streams), 16)
    pool = StreamPool(eng, n_slots=n_max, max_seconds=math.ceil(a.seconds) + 1, ctc_heads=2)
    syncs = SyncCounter(eng)
    workloads = [(f"{n}x320ms", [320] * n) for n in a.streams] + [("16x_mixed_320_640ms", [320 if j % 2 == 0 else 640 for j in range(16)])]
    result = {"gpu": gpu_info(), "utterance_seconds": a.seconds, "max_mt_positions": a.max_mt_positions, "rows": []}
    dictionary = single.dict["target_unigram"]
    for name, segs in workloads:
        wavs = [synth.make_audio(a.seconds, seed=9000 + j) for j in range(len(segs))]
        agents = [PooledS2TTAgent(pool, dictionary, args_for(s)) for s in segs]
        ref = run_single(single, wavs, segs)
        got = run_pooled(pool, agents, wavs, segs)
        for j in range(len(segs)):
            assert got[j] == ref[j], f"{name}: stream {j} differs from the single agent"
        times = {"pooled": [], "single": []}
        stage_ms, launches, flushes, n_sync = {}, 0, 0, 0
        for r in range(a.reps):
            t0 = time.perf_counter()
            run_single(single, wavs, segs)
            times["single"].append(time.perf_counter() - t0)
            if r == 0:
                pool.stage_ms = stage_ms
            steps0, l0, s0 = pool.steps, eng.launch_count(), syncs.n
            t0 = time.perf_counter()
            run_pooled(pool, agents, wavs, segs)
            times["pooled"].append(time.perf_counter() - t0)
            if r == 0:
                pool.stage_ms = None
                flushes, launches, n_sync = pool.steps - steps0, eng.launch_count() - l0, syncs.n - s0
        audio = a.seconds * len(segs)
        best = {k: min(v) for k, v in times.items()}
        row = {"workload": name, "streams": len(segs), "audio_s_per_s": {k: audio / v for k, v in best.items()},
               "speedup_pooled_vs_single": best["single"] / best["pooled"], "seconds_all": times, "flushes": flushes,
               "stage_ms_per_flush": {k: v / max(flushes, 1) for k, v in stage_ms.items()},
               "launches_per_flush": launches / max(flushes, 1), "host_syncs_per_flush": n_sync / max(flushes, 1),
               "identical_actions_text_tokens": True}
        print(json.dumps(row), flush=True)
        result["rows"].append(row)
        for ag in agents:
            pool.release(ag.slot)
    print(json.dumps({k: result[k] for k in ("gpu", "utterance_seconds", "max_mt_positions")}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
