#!/usr/bin/env python
"""Large-M launches inside a cudaProfilerStart/Stop window (BASELINE configs[2] / configs[3] shapes) for
  ncu --profile-from-start off [--set full -k regex:umma2_kernel | --metrics gpu__time_duration.sum] python tools/ncu_large.py
1. FFN GEMMs of the offline batch (M = 32 x 375 = 12,000 rows) on the wgmma kernel, bf16x6
2. the vocoder generator on 750 frames
3. one batched multi-stream ASR step (32 streams x 8 rows)"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from streamspeech_b200 import synth
from streamspeech_b200.agent import StreamSpeechS2STAgent
from streamspeech_b200.scheduler import StreamPool

torch.set_grad_enabled(False)
agent = StreamSpeechS2STAgent(bench.agent_args(0, "cached"))
eng = agent.engine
rows = 12000
x = torch.randn(rows, 256, device="cuda")
hbuf = torch.randn(rows, 2048, device="cuda")
w1 = torch.randn(2048, 256, device="cuda") / 16
w2 = torch.randn(256, 2048, device="cuda") / 45
b1, b2 = torch.zeros(2048, device="cuda"), torch.zeros(256, device="cuda")
codes = torch.randint(0, 1000, (750,), device="cuda")
eng.vocoder_durations(codes, False)
eng.set_chunk(4, 4)
pool = StreamPool(eng, n_slots=32, max_seconds=11, ctc_heads=1)
slots = [pool.acquire() for _ in range(32)]
wavs = [synth.make_audio(10.0, seed=5000 + j) for j in range(32)]
for i in range(0, 2560 * 20, 2560):
    for j, sl in enumerate(slots):
        pool.push(sl, wavs[j][i:i + 2560])
    pool.flush()
for _ in range(2):  # warm: weight packing, workspaces
    eng.op_linear_umma(x, w1, b1, 2, 3)
    eng.op_linear_umma(hbuf, w2, b2, 0, 3)
    eng.vocoder_generate(750, 0, 750, 0)
torch.cuda.synchronize()
torch.cuda.profiler.start()
eng.op_linear_umma(x, w1, b1, 2, 3)      # FFN W1 + SiLU, M = 12,000, K = 256, N = 2048, bf16x6
eng.op_linear_umma(hbuf, w2, b2, 0, 3)   # FFN W2, K = 2048, N = 256
eng.vocoder_generate(750, 0, 750, 0)
i = 2560 * 20
for j, sl in enumerate(slots):
    pool.push(sl, wavs[j][i:i + 2560])
pool.flush()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("done")
