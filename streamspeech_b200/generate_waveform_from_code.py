"""`generate_waveform_from_code.py` on the H100 engine (SURVEY.md §8 f4).

Front door of the reference's offline pipeline after `fairseq-generate`
(fairseq/examples/speech_to_speech/generate_waveform_from_code.py:40-111, used by
researches/ctc_unity/test_scripts/pred.offline-s2st.sh): one unit sequence per line in, `<i>_pred.wav` (16 kHz) per line out.  Lines are synthesised
32 at a time, each group in one vocoder call.
Same flags; `--cpu` is refused (there is no CPU path), multi-speaker vocoders are not part of StreamSpeech's unit vocoder.

    python -m streamspeech_b200.generate_waveform_from_code --in-code-file unit.txt --vocoder g_00500000 \\
        --vocoder-cfg config.json --results-path out/ --dur-prediction
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import wave
from pathlib import Path
from typing import List, Sequence

import numpy as np
import torch

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _REPO not in sys.path:
    sys.path.insert(0, _REPO)

from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig, VocoderConfig  # noqa: E402
from streamspeech_b200.engine import Engine  # noqa: E402
from streamspeech_b200.offline import vocode_whole  # noqa: E402

LINES_PER_CALL = 32  # code lines synthesised by one vocoder call (one generator kernel per group of the engine's ragged call)


def load_code(in_file: str) -> List[List[int]]:
    with open(in_file) as f:
        return [list(map(int, line.strip().split())) for line in f]


def write_wav(path: str, wav: np.ndarray, rate: int = 16000):
    """16-bit PCM like soundfile's default subtype for .wav (the reference uses sf.write, :26-31)"""
    pcm = np.clip(np.round(wav * 32768.0), -32768, 32767).astype("<i2")
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.writeframes(pcm.tobytes())


class VocoderOnly:
    """CodeHiFiGANVocoder(checkpoint, cfg) (fairseq/models/text_to_speech/vocoder.py) on the engine: only vocoder weights loaded."""

    def __init__(self, vocoder_path: str, vocoder_cfg: dict, device: int = 0):
        vc = VocoderConfig.from_json_dict(vocoder_cfg)
        if str(vocoder_path).startswith("synthetic"):
            sd = synth.make_vocoder_state_dict(vc, seed=1)
        else:
            sd = torch.load(vocoder_path, map_location="cpu", weights_only=False)["generator"]
        cfg = ModelConfig().tiny()      # the smallest model the engine accepts next to the vocoder (never run)
        cfg.vocoder = vc
        self.engine = Engine(cfg, synth.make_model_state_dict(cfg, 0), sd, None, device=device)

    def __call__(self, code: List[int], dur_prediction: bool = False) -> torch.Tensor:
        return self.batch([code], dur_prediction)[0]

    @torch.inference_mode()
    def batch(self, codes: Sequence[List[int]], dur_prediction: bool = False) -> List[torch.Tensor]:
        """__call__ of every code line in one vocoder call; each waveform equals __call__'s bit for bit"""
        return vocode_whole(self.engine, [[c for c in code if c >= 0] for code in codes], dur_prediction)  # "remove invalid code" (vocoder.py:52-54)


def main(args):
    if args.cpu:
        raise SystemExit("--cpu: the H100 engine has no CPU path")
    with open(args.vocoder_cfg) as f:
        vocoder_cfg = json.load(f)
    vocoder = VocoderOnly(args.vocoder, vocoder_cfg)
    data = load_code(args.in_code_file)
    Path(args.results_path).mkdir(exist_ok=True, parents=True)
    for g in range(0, len(data), LINES_PER_CALL):
        for i, wav in enumerate(vocoder.batch(data[g:g + LINES_PER_CALL], args.dur_prediction), start=g):
            write_wav(f"{args.results_path}/{i}_pred.wav", wav.detach().cpu().numpy())
    return len(data)


def cli_main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--in-code-file", type=str, required=True, help="one unit sequence per line")
    parser.add_argument("--vocoder", type=str, required=True, help="path to the CodeHiFiGAN vocoder")
    parser.add_argument("--vocoder-cfg", type=str, required=True, help="path to the CodeHiFiGAN vocoder config")
    parser.add_argument("--results-path", type=str, required=True)
    parser.add_argument("--dur-prediction", action="store_true", help="enable duration prediction (for reduced/unique code sequences)")
    parser.add_argument("--speaker-id", type=int, default=-1, help="(multi-speaker vocoders: not supported)")
    parser.add_argument("--cpu", action="store_true", help="refused: no CPU path")
    return main(parser.parse_args(argv))


if __name__ == "__main__":
    cli_main()
