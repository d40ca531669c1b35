#!/usr/bin/env python
"""MT decoder timing split: forced-prefix pass vs greedy single-token steps (CUDA events, warm)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from streamspeech_b200 import synth
from streamspeech_b200.agent import StreamSpeechS2STAgent

torch.set_grad_enabled(False)
agent = StreamSpeechS2STAgent(bench.agent_args(0, "cached"))
eng = agent.engine
enc = torch.randn(1024, 256, device="cuda") * 0.5
res = {}
toks, _ = eng.mt_greedy(enc[:160], None, 40)
toks = (toks + [17] * 40)[:40]
for T in (160,):
    for npre in (10, 30, 40):
        for new in (0, 3, 12):
            for stable in (T - 16,):
                def fn():
                    eng.encoder_stream_reset()
                    if stable:
                        eng.mt_greedy(enc[:T], toks[:npre], new, stable_rows=stable)  # primes the cross K/V of the final rows
                    return eng.mt_greedy(enc[:T], toks[:npre], new, stable_rows=stable)
                for _ in range(2): fn()
                ts = []
                for _ in range(5):
                    eng.encoder_stream_reset()
                    if stable:
                        eng.mt_greedy(enc[:T], toks[:npre], new, stable_rows=stable)
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize(); l0 = eng.launch_count(); s.record()
                    eng.mt_greedy(enc[:T], toks[:npre], new, stable_rows=stable)
                    e.record(); torch.cuda.synchronize()
                    ts.append(s.elapsed_time(e))
                ts.sort()
                res[f"T{T}_prefix{npre}_new{new}_stable{stable}"] = {"ms": ts[2], "launches": eng.launch_count() - l0}
                print(T, npre, new, stable, round(ts[2] * 1e3, 1), "us", eng.launch_count() - l0, "launches", flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "gpurun_out", "mt_profile.json"), "w"), indent=1)
