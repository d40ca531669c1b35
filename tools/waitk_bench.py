"""The wait-k-stride-n S2ST agent (UnitY) on the synthetic UnitY checkpoint: N utterances of S seconds streamed at 320 ms with the
reference's defaults (k1 3, k2 1, n 1, n2 1, 15 units per subword, --segment-size 320).  Prints one JSON line with

  * audio_s_per_s: source seconds over the wall time of the whole stream loop (every call ends in a host read);
  * device time per stage per WRITE call (encoder, MT search, T2U encoder, unit search, vocoder), from CUDA events around each engine
    call; the MT features are rows of the MT search's own pass, so "mt_features + t2u" is the T2U encoder call;
  * launches per call (the engine's launch counter) and host synchronisations per call, counted from the burst rules of the calls
    (MT search: one read per burst of max(1, new tokens) steps or 16 for an ended source; unit search: one per 16 steps; vocoder: the
    duration read; the waveform's device-to-host copy), not traced;
  * unit_search_growth: units searched and unit-search time per WRITE call of the first utterance.  The unit search restarts from BOS
    on every call, as the reference's does (its tgt_units_indices is never assigned), so its cost grows with the output so far.

The card's name and power limit are read in the same run.

    python tools/waitk_bench.py [--utterances 4] [--seconds 10]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

STAGES = {"encoder": "encoder", "encoder_stream_step": "encoder", "mt_greedy": "mt_search", "t2u_encode_batch": "mt_features_t2u", "unit_search_batch": "unit_search",
          "vocoder_durations": "vocoder", "vocoder_generate": "vocoder"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def instrument(eng, log):
    """wrap the engine calls of a policy() call with CUDA events; log[stage] collects (start, end) event pairs"""
    for name, stage in STAGES.items():
        fn = getattr(eng, name)

        def wrapped(*a, _fn=fn, _stage=stage, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = _fn(*a, **k)
            e1.record()
            log.setdefault(_stage, []).append((e0, e1))
            return out

        setattr(eng, name, wrapped)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=4)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--variant", choices=("unity", "uni_unity", "chunk_unity"), default="unity",
                    help="the synthetic UnitY-family checkpoint (Uni-UnitY re-encodes the prefix, Chunk-UnitY encodes incrementally)")
    a = ap.parse_args()
    from streamspeech_b200 import synth
    from streamspeech_b200.simuleval_compat import SpeechSegment
    from streamspeech_b200.waitk import WaitkS2STAgent, add_waitk_args

    if not torch.cuda.is_available():
        raise SystemExit("waitk_bench needs a CUDA device")
    p = argparse.ArgumentParser()
    add_waitk_args(p)
    agent = WaitkS2STAgent(p.parse_args(["--model-path", "synthetic", "--user-dir", f"researches/{a.variant}", "--data-bin", ".",
                                         "--vocoder", "synthetic", "--vocoder-cfg", "none", "--dur-prediction"]))
    eng = agent.engine
    wavs = [synth.make_audio(a.seconds, seed=900 + i).tolist() for i in range(a.utterances)]
    step = 16 * 320

    def stream(wav, on_call=None):
        agent.reset()
        for i in range(0, len(wav), step):
            agent.push(SpeechSegment(content=wav[i:i + step], sample_rate=16000, finished=i + step >= len(wav)))
            act = agent.policy()
            if on_call is not None:
                on_call(act)

    stream(wavs[0])  # warm-up of every shape the timed loop uses
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for w in wavs:
        stream(w)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0

    # a second pass, instrumented, for the per-stage device times, launches and the unit-search growth
    log, calls, growth = {}, [], []
    instrument(eng, log)
    for ui, w in enumerate(wavs):
        state = {"l0": eng.launch_count()}

        def on_call(act, ui=ui, state=state):
            torch.cuda.synchronize()
            tr = agent.trace
            rec = {"launches": eng.launch_count() - state["l0"], "write": not act.is_read()}
            state["l0"] = eng.launch_count()
            for stage, evs in log.items():
                rec[stage] = sum(e0.elapsed_time(e1) for e0, e1 in evs)
            log.clear()
            if "mt_tokens" in tr:
                new = tr["new_subword_tokens"]
                produced = len(tr["mt_tokens"]) + 1
                rec["syncs"] = math.ceil(produced / (16 if new == -1 else max(1, new)))
                if "units" in tr:
                    rec["syncs"] += math.ceil((len(tr["units"]) + 1) / 16)
                if "dur" in tr:
                    rec["syncs"] += 2  # the duration read and the waveform's copy to the host
                if ui == 0 and "units" in tr:
                    growth.append({"units": len(tr["units"]), "unit_search_ms": round(rec.get("unit_search", 0.0), 3)})
            calls.append(rec)

        stream(w, on_call)
    full = [c for c in calls if "syncs" in c]  # calls that passed the gate
    stages = sorted({s for c in full for s in STAGES.values() if s in c})
    res = {"card": card(), "variant": a.variant, "utterances": a.utterances, "seconds": a.seconds, "segment_ms": 320,
           "audio_s_per_s": round(a.utterances * a.seconds / wall, 3), "policy_calls": len(calls), "calls_past_gate": len(full),
           "stage_ms_per_call": {s: round(float(np.mean([c.get(s, 0.0) for c in full])), 3) for s in stages},
           "stage_ms_max": {s: round(float(np.max([c.get(s, 0.0) for c in full])), 3) for s in stages},
           "launches_per_call": round(float(np.mean([c["launches"] for c in full])), 1),
           "host_syncs_per_call": round(float(np.mean([c["syncs"] for c in full])), 2),
           "unit_search_growth": growth}
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
