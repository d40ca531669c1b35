"""GPU: the ASR-BLEU transcriber (ss_asr_*) on the seeded Large-shape wav2vec 2.0 CTC checkpoint against the float64 oracle
(oracle/asr_oracle.py, run on the same device): every stage, conv-stride edges, a long input, ragged batches over several launch groups,
batch-of-one identity, letters against the fp64 arg-max, and refusals; the fixture's two small configurations (extractor width 64) against
fairseq's modules and the oracle, and wav2vec 2.0 Base's width (D = 768)."""
import os

import pytest
import torch

from oracle import asr_oracle as ao
from streamspeech_b200 import synth

pytestmark = pytest.mark.gpu

STRIDES = [s for (_, _, s) in synth.W2V_CONV_LAYERS]
KERNELS = [k for (_, k, _) in synth.W2V_CONV_LAYERS]
# relative bars (max |engine - fp64| / max |fp64|) per stage, about ten times the maxima measured on an H100 80GB HBM3 (test_stages prints
# them): extractor 2.3e-6, proj 4.3e-6, pos conv 4.3e-6, layer 0 1.0e-5, layer 11 2.2e-5, layer 23 2.2e-5, final LN 2.1e-5, emissions 1.5e-5
BARS = {"extractor": 2e-5, "proj": 5e-5, "pos": 5e-5, "layer0": 1e-4, "layer11": 2e-4, "layer23": 2e-4, "final_ln": 2e-4, "emissions": 2e-4}
TIE_MARGIN = 1e-2  # frames whose fp64 top-two emissions are closer than this may take either letter


def n_for_frames(T: int) -> int:
    return 400 + 320 * (T - 1)


@pytest.fixture(scope="module")
def model():
    from streamspeech_b200.engine import ASREngine

    sd = synth.make_w2v_ctc_state_dict()
    eng = ASREngine(sd, STRIDES, 0)
    sd64 = {k: v.to("cuda", torch.float64) for k, v in sd.items()}
    yield eng, sd64
    eng.close()


def ref(sd64, wav):
    return ao.forward(sd64, wav, STRIDES, normalize=True, dtype=torch.float64, device="cuda")


def stage_index(name: str) -> int:
    if name == "extractor":
        return 0
    if name == "proj":
        return 1
    if name == "pos":
        return 2
    if name.startswith("layer"):
        return 3 + int(name[5:])
    return {"final_ln": 27, "emissions": 28}[name]


def check_letters(am, tokens, emissions64):
    """the engine's per-frame arg-max equals the fp64 one except at near-ties; with no disagreement the tokens equal the fp64 path's"""
    bp = ao.best_path(emissions64)
    e = emissions64.clone()
    e[:, ao.UNK] = float("-inf")
    top2 = e.topk(2, dim=1).values
    margin = (top2[:, 0] - top2[:, 1]).cpu()
    diff = [t for t in range(len(bp)) if bp[t] != am[t]]
    assert all(float(margin[t]) < TIE_MARGIN for t in diff), [(t, float(margin[t])) for t in diff]
    if not diff:
        assert tokens == ao.get_tokens(bp)
    return len(diff)


def test_stages(model):
    eng, sd64 = model
    worst = {}
    for seconds, seed in ((1.0, 1), (2.3, 2)):
        wav = synth.make_audio(seconds, seed=seed)
        r = ref(sd64, wav)
        for name, bar in BARS.items():
            width = r[name].shape[1]
            got = eng.stage([wav], stage_index(name), width).double()
            assert got.shape == r[name].shape, name
            rel = float((got - r[name]).abs().max() / r[name].abs().max())
            worst[name] = max(worst.get(name, 0.0), rel)
            assert rel < bar, (name, rel)
    print("ASR stage max rel err:", {k: f"{v:.2e}" for k, v in worst.items()})


def test_conv_stride_edges_and_batch_of_one(model):
    eng, sd64 = model
    lengths = [400, 401, 404, 405, 409, 410, 559, 560, 719, 720] + [n_for_frames(T) for T in (1, 63, 64, 65, 1024, 1025)]
    lengths += [n_for_frames(64) - 1, n_for_frames(1025) + 319]
    waves = [synth.make_audio(n / 16000, seed=100 + i)[:n] for i, n in enumerate(lengths)]
    for n, w in zip(lengths, waves):
        assert w.numel() == n
        assert eng.num_frames(n) == ao.num_frames(n, KERNELS, STRIDES)
    toks, am, em = eng.transcribe(waves, emissions=True)
    r0, ties = 0, 0
    for i, w in enumerate(waves):
        T = eng.num_frames(w.numel())
        t1, a1, e1 = eng.transcribe([w], emissions=True)
        assert torch.equal(e1, em[r0:r0 + T]), i  # bit-identical to the batch of one
        assert t1[0] == toks[i] and a1 == am[r0:r0 + T]
        r = ref(sd64, w)
        rel = float((em[r0:r0 + T].double() - r["emissions"]).abs().max() / r["emissions"].abs().max())
        assert rel < BARS["emissions"], (i, rel)
        ties += check_letters(am[r0:r0 + T], toks[i], r["emissions"])
        r0 += T
    print(f"conv-stride edges: {len(waves)} utterances, {r0} frames, {ties} near-tie frames")


def test_long_input(model):
    eng, sd64 = model
    wav = synth.make_audio(41.0, seed=9)
    toks, am, em = eng.transcribe([wav], emissions=True)
    r = ref(sd64, wav)
    assert em.shape[0] == r["emissions"].shape[0] >= 2000
    rel = float((em.double() - r["emissions"]).abs().max() / r["emissions"].abs().max())
    assert rel < BARS["emissions"], rel
    ties = check_letters(am, toks[0], r["emissions"])
    print(f"41 s: {em.shape[0]} frames, emissions rel err {rel:.2e}, {ties} near-tie frames")


def test_ragged_batch_over_launch_groups(model):
    eng, _ = model
    secs = [30.0, 2.0, 29.0, 0.5, 31.0, 12.0, 28.0, 7.5, 30.5]  # ~8.6k frames: several launch groups of SS_ASR_BATCH_ROWS
    waves = [synth.make_audio(s, seed=200 + i) for i, s in enumerate(secs)]
    T = [eng.num_frames(w.numel()) for w in waves]
    assert sum(T) > 8192
    toks, am, em = eng.transcribe(waves, emissions=True)
    r0 = 0
    for i, w in enumerate(waves):
        t1, a1, e1 = eng.transcribe([w], emissions=True)
        assert torch.equal(e1, em[r0:r0 + T[i]]) and t1[0] == toks[i], i
        r0 += T[i]


def test_transcriber_letters(model):
    from streamspeech_b200.asr import ASRTranscriber

    _, sd64 = model
    tr = ASRTranscriber("synthetic", None, 0, max_batch_samples=3 * 16000)
    waves = [synth.make_audio(s, seed=300 + i).numpy() for i, s in enumerate((1.0, 2.5, 0.7, 3.1, 1.9))]
    out = tr.transcribe_tokens(waves)
    for w, (toks, am) in zip(waves, out):
        r = ref(sd64, torch.from_numpy(w))
        if check_letters(am, toks, r["emissions"]) == 0:
            assert tr.letters(toks) == ao.letters(ao.get_tokens(ao.best_path(r["emissions"])), tr.vocab)
    assert any(tr.letters(t) for t, _ in out)
    with pytest.raises(ValueError, match="fewer than one encoder frame"):
        tr.transcribe([waves[0][:399]])


def test_refusals_return_errors():
    from streamspeech_b200.engine import ASREngine, EngineError, SS_ERR_CAPACITY

    sd = synth.make_w2v_ctc_state_dict(dim=128, ffn=256, layers=2, pos_k=16, pos_groups=4)
    for setting, msg in (({"extractor_layer_norm": 0}, "group norm"), ({"layer_norm_first": 0}, "post-LN"), ({"pos_conv_depth": 2}, "pos_conv_depth"),
                         ({"conformer": 1}, "conformer"), ({"heads": 4}, "head dim")):
        with pytest.raises(EngineError, match=msg):
            ASREngine(sd, STRIDES, 0, **setting)
    eng = ASREngine(sd, STRIDES, 0, max_frames=10)
    with pytest.raises(EngineError, match="fewer than one encoder frame") as e:
        eng.transcribe([torch.zeros(399)])
    assert e.value.code == -1
    with pytest.raises(EngineError, match="max_frames") as e:
        eng.transcribe([torch.zeros(400), synth.make_audio(0.3)])
    assert e.value.code == SS_ERR_CAPACITY
    toks, am, _ = eng.transcribe([synth.make_audio(0.2)])  # the handle stays usable
    assert len(am) == eng.num_frames(3200) == 9
    missing = dict(sd)
    del missing["w2v_encoder.proj.bias"]
    with pytest.raises(EngineError, match="w2v_encoder.proj.bias"):
        ASREngine(missing, STRIDES, 0)


def small_stage_index(name: str, layers: int) -> int:
    if name.startswith("layer"):
        return 3 + int(name[5:])
    return {"extractor": 0, "proj": 1, "pos": 2, "final_ln": 3 + layers, "emissions": 4 + layers}[name]


def small_bar(name: str) -> float:
    return BARS[name] if name in BARS else BARS["layer11"]  # layers past the first take the deep-layer bar


@pytest.mark.parametrize("name", ["a", "b"])
def test_fixture_configurations(name):
    """Both configurations of tests/golden/asr_w2v.npz (extractor width 64, D = 128, conv_bias on / off, even / odd positional kernel):
    every stage against fairseq's own modules (the fixture) and against the float64 oracle.  Width 64 is outside the LayerNorm widths
    the encoder uses, so this also pins the feature LayerNorm at that width."""
    import numpy as np

    from oracle.gen_golden_asr import CONV, LAYERS, LENGTHS, config_state_dict
    from streamspeech_b200.engine import ASREngine

    golden = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "asr_w2v.npz"))
    sd = config_state_dict(name)
    strides = [s for (_, _, s) in CONV]
    layers = LAYERS
    eng = ASREngine(sd, strides, 0)
    sd64 = {k: v.to("cuda", torch.float64) for k, v in sd.items()}
    worst = {}
    try:
        for j, n in enumerate(LENGTHS):
            wav = torch.from_numpy(golden[f"{name}_{j}_wav"])
            r = ao.forward(sd64, wav, strides, normalize=True, dtype=torch.float64, device="cuda")
            for st in ["extractor", "proj", "pos"] + [f"layer{i}" for i in range(layers)] + ["final_ln", "emissions"]:
                fx = torch.from_numpy(golden[f"{name}_{j}_{st}"]).to("cuda", torch.float64)
                got = eng.stage([wav], small_stage_index(st, layers), fx.shape[1]).double()
                assert got.shape == fx.shape == r[st].shape, st
                for against, ref_ in (("fairseq", fx), ("fp64", r[st])):
                    rel = float((got - ref_).abs().max() / ref_.abs().max())
                    worst[(st, against)] = max(worst.get((st, against), 0.0), rel)
                    assert rel < small_bar(st), (name, j, st, against, rel)
    finally:
        eng.close()
    print(f"ASR fixture config {name} max rel err:", {f"{k[0]}/{k[1]}": f"{v:.1e}" for k, v in worst.items()})


def test_base_width_against_fp64():
    """wav2vec 2.0 Base's model width (D = 768, 12 heads; 3 layers, extractor width 512) against the float64 oracle at every stage"""
    from streamspeech_b200.engine import ASREngine

    layers = 3
    sd = synth.make_w2v_ctc_state_dict(seed=21, dim=768, ffn=3072, layers=layers, pos_k=128, pos_groups=16)
    eng = ASREngine(sd, STRIDES, 0)
    sd64 = {k: v.to("cuda", torch.float64) for k, v in sd.items()}
    worst = {}
    try:
        for seconds, seed in ((1.0, 31), (2.3, 32)):
            wav = synth.make_audio(seconds, seed=seed)
            r = ref(sd64, wav)
            for st in ["extractor", "proj", "pos"] + [f"layer{i}" for i in range(layers)] + ["final_ln", "emissions"]:
                got = eng.stage([wav], small_stage_index(st, layers), r[st].shape[1]).double()
                assert got.shape == r[st].shape, st
                rel = float((got - r[st]).abs().max() / r[st].abs().max())
                worst[st] = max(worst.get(st, 0.0), rel)
                assert rel < small_bar(st), (st, rel)
    finally:
        eng.close()
    print("ASR D = 768 max rel err:", {k: f"{v:.1e}" for k, v in worst.items()})
