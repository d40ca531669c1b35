"""CPU: oracle/asr_oracle.py against tests/golden/asr_w2v.npz, which oracle/gen_golden_asr.py made by running fairseq's own Wav2Vec2Model
(ConvFeatureExtractionModel, make_conv_pos, TransformerEncoder, TransformerSentenceEncoderLayer), the reference's own load_audiofile and
torchaudio's own CTCDecoder._get_tokens, in fp32 at small dims: conv_bias on with an even pos_conv kernel, and conv_bias off with an odd one.

Bounds, relative to the stage's max |value|: the fp32 oracle and fairseq's fp32 modules sum in different orders, measured at most 6.0e-7
(the extractor and projection bit-equal); the float64 oracle against the fp32 fixture is bounded by the fixture's own rounding, measured
at most 1.0e-6.  Bar 5e-6 for both; the per-frame arg-max must be equal."""
import os

import numpy as np
import pytest
import torch

from oracle import asr_oracle as ao
from oracle.gen_golden_asr import CONFIGS, CONV, LAYERS, LENGTHS, config_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "asr_w2v.npz")
STAGES = ["extractor", "proj", "pos"] + [f"layer{i}" for i in range(LAYERS)] + ["final_ln", "emissions"]
BAR = 5e-6


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", sorted(CONFIGS))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_forward_equals_fairseq_modules(golden, name, dtype):
    sd = config_state_dict(name)
    assert float(sum(v.double().sum() for v in sd.values())) == pytest.approx(float(golden[f"{name}_checksum"][0]), rel=1e-12)
    strides = [s for (_, _, s) in CONV]
    worst = {}
    for j, n in enumerate(LENGTHS):
        wav = torch.from_numpy(golden[f"{name}_{j}_wav"])
        assert wav.numel() == n
        x = wav.to(dtype).reshape(1, -1)
        norm = torch.nn.functional.layer_norm(x, x.shape)[0]
        ref_norm = torch.from_numpy(golden[f"{name}_{j}_normalized"]).to(dtype)
        assert float((norm - ref_norm).abs().max()) < 1e-5  # task.normalize: the reference's load_audiofile LayerNorm
        out = ao.forward(sd, wav, strides, normalize=True, dtype=dtype)
        for st in STAGES:
            ref = torch.from_numpy(golden[f"{name}_{j}_{st}"]).to(torch.float64)
            got = out[st].to(torch.float64)
            assert got.shape == ref.shape, (st, got.shape, ref.shape)
            rel = float((got - ref).abs().max() / ref.abs().max())
            worst[st] = max(worst.get(st, 0.0), rel)
            assert rel < BAR, (name, j, st, rel)
        am = ao.best_path(out["emissions"])
        assert am == ao.best_path(torch.from_numpy(golden[f"{name}_{j}_emissions"]).double())
    print(name, dtype, {k: f"{v:.1e}" for k, v in worst.items()})


def test_get_tokens_equals_torchaudio(golden):
    for i in range(len(golden["gt_in_off"]) - 1):
        path = golden["gt_in"][golden["gt_in_off"][i]:golden["gt_in_off"][i + 1]].tolist()
        assert ao.get_tokens(path) == golden["gt_out"][golden["gt_out_off"][i]:golden["gt_out_off"][i + 1]].tolist(), i


def test_fixture_configurations_need_no_reference_tree():
    """oracle/gen_golden_asr.config_state_dict, which the GPU tests import, opens nothing under the reference tree"""
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys, os\n"
            "ref = os.environ['STREAMSPEECH_REFERENCE']\n"
            "opened = []\n"
            "sys.addaudithook(lambda ev, a: opened.append(str(a[0])) if ev == 'open' and str(a[0]).startswith(ref) else None)\n"
            "from oracle.gen_golden_asr import config_state_dict\n"
            "sds = [config_state_dict(n) for n in ('a', 'b')]\n"
            "assert all(len(sd) > 10 for sd in sds)\n"
            "assert not opened, opened\n")
    env = dict(os.environ, STREAMSPEECH_REFERENCE=os.path.join(root, "no-such-reference-tree"), PYTHONPATH=root)
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
