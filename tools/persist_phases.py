#!/usr/bin/env python
"""Per-phase time of the persistent encoder kernel (kernels_persist.cu), from the %globaltimer stamps it records when
option persistent_profile is set.  Prints the mean duration of each of the 11 phases of a layer (work + barrier) over
all layers and steps, the pure barrier cost, and the per-step GPU time with / without the persistent kernel."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from streamspeech_b200 import synth
from streamspeech_b200.agent import StreamSpeechS2STAgent

PHASES = ["ffn1_w1", "ffn1_w2", "qkv", "attention", "attn_out", "pw1_glu_dw", "pw2", "ffn2_w1", "ffn2_w2"]

torch.set_grad_enabled(False)
agent = StreamSpeechS2STAgent(bench.agent_args(0, "cached"))
eng = agent.engine
u = synth.make_audio(10.0, seed=1234).cuda()
feats = eng.fbank(u)
buf = torch.zeros(1024, 256, device="cuda")
L = agent.cfg.enc_layers
out = {}
for mode in (1, 0):
    eng.set_option("persistent_encoder", mode)
    eng.set_option("persistent_profile", mode)
    acc = [0.0] * len(PHASES)
    barrier, n, gpu = 0.0, 0, []
    for rep in range(2):
        eng.encoder_stream_reset()
        for k in range(1, 32):
            F = 32 * k - 2
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            eng.encoder_stream_step(feats[:F], buf)
            e.record()
            torch.cuda.synchronize()
            if rep == 1 and k > 4:
                gpu.append(s.elapsed_time(e))
                if mode:
                    ts = eng.persistent_phase_stamps(3 + L * len(PHASES))
                    barrier += (ts[2] - ts[0]) / 2
                    for li in range(L):
                        for p in range(len(PHASES)):
                            i = 3 + li * len(PHASES) + p
                            acc[p] += ts[i] - ts[i - 1]
                    n += 1
    key = "persistent" if mode else "per_kernel"
    out[key] = {"gpu_ms_per_step": sum(gpu) / len(gpu)}
    if mode:
        out[key]["barrier_us"] = barrier / n / 1e3
        out[key]["phase_us"] = {PHASES[p]: acc[p] / (n * L) / 1e3 for p in range(len(PHASES))}
        out[key]["layer_us"] = sum(acc) / (n * L) / 1e3
print(json.dumps(out, indent=1))
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "persist_phases.json"), "w"), indent=1)
# fine clock64 stamps of CTA 0 inside layer 1 of the last persistent step (see fine_stamp in kernels_persist.cu)
eng.set_option("persistent_encoder", 1)
eng.set_option("persistent_profile", 1)
eng.encoder_stream_reset()
for k in range(1, 20):
    eng.encoder_stream_step(feats[:32 * k - 2], buf)
torch.cuda.synchronize()
ts = eng.persistent_phase_stamps(256 + 240)[256:]
pairs = [(int(ts[2 * i]), int(ts[2 * i + 1])) for i in range(60) if ts[2 * i + 1]]
print("fine (tag: cycles since previous stamp), CTA 0, layer 1; tags: x0 gemm entry, x1 staged, x2 main loop done, x3 reduced, x4 epilogue done, x5 barrier arrive")
print(" ".join(f"{t}:{c - pairs[i - 1][1] if i else 0}" for i, (t, c) in enumerate(pairs)))
# arrival of every CTA at each barrier of layer 1, relative to the start of that phase (= end of the previous barrier)
all_ts = eng.persistent_phase_stamps(4096)
L1 = 3 + len(PHASES)  # index of the stamp taken after the last barrier of layer 0
import statistics
for p, name in enumerate(PHASES):
    start = all_ts[L1 + p - 1]
    n_ctas = torch.cuda.get_device_properties(0).multi_processor_count  # one CTA per SM
    arr = [all_ts[512 + c * 16 + p] - start for c in range(n_ctas)]
    order = sorted(range(n_ctas), key=lambda c: arr[c])
    print(f"{name:12s} arrive ns: min {min(arr)} med {int(statistics.median(arr))} max {max(arr)}  slowest CTAs {order[-4:]}  fastest {order[:3]}  barrier done {all_ts[L1 + p] - start}")
