"""The vocoder generator as one persistent kernel (option vocoder_fused) against the multi-launch path on the same frames."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig  # noqa: E402

torch.set_grad_enabled(False)


@pytest.fixture(scope="module")
def eng():
    from streamspeech_b200.engine import Engine

    cfg = ModelConfig()
    cfg.enc_layers = 3
    e = Engine(cfg, synth.make_model_state_dict(cfg, 0), synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=True), None)
    yield e
    e.close()


# (generator input frames N, new frames, explicit left context or -1): N = new frames + context.  N = 7 starts at frame 3, inside
# the receptive field; 750 is the offline leg's frame count.
CASES = [(1, 1, -1), (7, 4, -1), (45, 21, 24), (52, 28, 24), (180, 156, 24), (750, 726, 24)]


def test_fused_vocoder_matches_multi_launch(eng):
    g = torch.Generator().manual_seed(7)
    codes = torch.randint(0, eng.cfg.vocoder.num_embeddings, (800,), generator=g).cuda()
    _, cum = eng.vocoder_durations(codes, False)  # one frame per code
    assert int(cum[-1].item()) == 800
    diffs = {}
    try:
        for N, new, ctx in CASES:
            total = N + 10 if ctx >= 0 else N
            frame0 = total - new
            outs = {}
            for mode in (0, 1):
                eng.set_option("vocoder_fused", mode)
                eng.vocoder_generate(total, frame0, new, ctx)  # first use of this frame count: tables and packed weights
                l0 = eng.launch_count()
                outs[mode] = eng.vocoder_generate(total, frame0, new, ctx).clone()
                launches = eng.launch_count() - l0
                if mode == 1:
                    assert launches == 2, launches  # frame expansion + the generator kernel
                    again = eng.vocoder_generate(total, frame0, new, ctx)
                    assert torch.equal(again, outs[1])  # deterministic: the schedule does not change a sum
            eng.check_async_error()
            assert outs[1].numel() == new * eng.hop
            diffs[N] = float((outs[1] - outs[0]).abs().max())
            assert diffs[N] <= 1e-4, diffs
    finally:
        eng.set_option("vocoder_fused", -1)
    print("fused vs multi-launch max-abs by frame count:", diffs)
