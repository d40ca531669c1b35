"""The ASR-BLEU transcriber: asr_bleu/utils.py's ASRGenerator for the `en` model (fairseq Wav2VecCtc, wav2vec 2.0 Large LV-60 + self
training) on the engine's own kernels (ss_asr_*, ASREngine).  Reads the fairseq checkpoint and dict.ltr.txt from local paths; nothing is
downloaded.
"""
from __future__ import annotations

import ast
import pickle
import sys
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

SPECIALS = ["<s>", "<pad>", "</s>", "<unk>"]  # fairseq's special tokens, prepended to dict.ltr.txt (utils.py:199-202)
DEFAULT_CONV_LAYERS = "[(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512,2,2)] + [(512,2,2)]"  # Wav2Vec2Config.conv_feature_layers
MODEL_RATE = 16000
PRE = "w2v_encoder.w2v_model."


def _get(obj, key, default=None):
    if obj is None:
        return default
    if isinstance(obj, dict):
        return obj.get(key, default)
    return getattr(obj, key, default)


def checkpoint_settings(ckpt: dict) -> Dict[str, object]:
    """The settings the state dict's shapes do not carry, from a checkpoint's stored cfg (fairseq >= 0.10) or args; fairseq's defaults
    where neither has them"""
    cfg = ckpt.get("cfg")
    args = ckpt.get("args")
    model = _get(cfg, "model") or args
    w2v = _get(model, "w2v_args")
    w2v_model = _get(w2v, "model") or w2v
    task = _get(cfg, "task") or args
    pick = lambda k, d: _get(w2v_model, k, _get(model, k, d))  # noqa: E731
    return {
        "conv_feature_layers": pick("conv_feature_layers", DEFAULT_CONV_LAYERS),
        "extractor_mode": pick("extractor_mode", "default"),
        "layer_norm_first": bool(pick("layer_norm_first", False)),
        "pos_conv_depth": int(pick("pos_conv_depth", 1)),
        "layer_type": pick("layer_type", "transformer"),
        "encoder_attention_heads": int(pick("encoder_attention_heads", 12)),
        "normalize": bool(_get(task, "normalize", False)),
        "sample_rate": int(_get(task, "sample_rate", MODEL_RATE)),
    }


# the `en` model's published configuration (wav2vec_vox_960h_pl.pt): what a checkpoint that a plain torch.load cannot read is taken as
EN_SETTINGS = {"conv_feature_layers": DEFAULT_CONV_LAYERS, "extractor_mode": "layer_norm", "layer_norm_first": True, "pos_conv_depth": 1,
               "layer_type": "transformer", "encoder_attention_heads": 16, "normalize": True, "sample_rate": MODEL_RATE}


def conv_strides(conv_feature_layers: str) -> List[int]:
    layers = ast.literal_eval(conv_feature_layers) if "*" not in conv_feature_layers else eval(conv_feature_layers, {"__builtins__": {}})  # noqa: S307
    return [int(s) for (_, _, s) in layers]


class _Opaque:
    """stands in for a pickled class that is not installed (omegaconf's DictConfig in fairseq >= 0.10 checkpoints)"""

    def __init__(self, *a, **k):
        pass

    def __setstate__(self, state):
        self.__dict__["_state"] = state


class _LenientUnpickler(pickle.Unpickler):
    missing = False

    def find_class(self, module, name):
        try:
            return super().find_class(module, name)
        except (ModuleNotFoundError, AttributeError):
            _LenientUnpickler.missing = True  # (torch.load subclasses this Unpickler)
            return _Opaque


_lenient_pickle = type(sys)("lenient_pickle")
_lenient_pickle.Unpickler = _LenientUnpickler
_lenient_pickle.load = lambda f, **kw: _LenientUnpickler(f, **kw).load()
_lenient_pickle.__name__ = "lenient_pickle"


def load_checkpoint(path: str):
    """-> (checkpoint dict, whether every pickled class resolved).  Classes that are not installed become opaque placeholders, so the
    weights still load; the settings are then not read from them."""
    _LenientUnpickler.missing = False
    ckpt = torch.load(path, map_location="cpu", weights_only=False, pickle_module=_lenient_pickle)
    return ckpt, not _LenientUnpickler.missing


def parse_settings(items: Sequence[str]) -> Dict[str, object]:
    """--asr-setting KEY=VALUE overrides (VALUE a Python literal, or a bare string)"""
    out: Dict[str, object] = {}
    for it in items or []:
        k, _, v = it.partition("=")
        if k not in EN_SETTINGS:
            raise ValueError(f"--asr-setting {it}: unknown setting {k!r}; one of {sorted(EN_SETTINGS)}")
        try:
            out[k] = ast.literal_eval(v)
        except (ValueError, SyntaxError):
            out[k] = v
    return out


def read_letter_dict(path: str) -> List[str]:
    with open(path, encoding="utf-8") as f:
        return SPECIALS + [ln.split()[0] for ln in f if ln.strip()]


class ASRTranscriber:
    """transcribe(waveforms) -> lower-cased letters per waveform, as ASRGenerator.transcribe_audiofile returns them.
    model_path "synthetic": the seeded Large-shape checkpoint of synth.make_w2v_ctc_state_dict (dict_path is then ignored)."""

    def __init__(self, model_path: str, dict_path: Optional[str], device_index: int = 0, max_batch_samples: int = 160 * 16000,
                 settings: Optional[Dict[str, object]] = None, state_dict: Optional[Dict[str, torch.Tensor]] = None, time_stages: bool = False):
        from . import synth
        from .engine import ASREngine

        if state_dict is not None:
            sd, st = state_dict, dict(EN_SETTINGS)
            self.vocab = SPECIALS + [ln.split()[0] for ln in synth.w2v_letter_dict(int(sd["w2v_encoder.proj.weight"].shape[0])).splitlines()]
        elif model_path == "synthetic":
            sd, st = synth.make_w2v_ctc_state_dict(), dict(EN_SETTINGS)
            self.vocab = SPECIALS + [ln.split()[0] for ln in synth.w2v_letter_dict().splitlines()]
        else:
            ckpt, complete = load_checkpoint(model_path)
            st = checkpoint_settings(ckpt) if complete else dict(EN_SETTINGS)
            if not complete:
                print(f"{model_path}: the stored cfg needs classes that are not installed; taking the en model's settings {EN_SETTINGS} "
                      "(override with --asr-setting KEY=VALUE)", file=sys.stderr)
            sd = ckpt["model"] if "model" in ckpt else ckpt
            self.vocab = read_letter_dict(dict_path)
        st.update(settings or {})
        self.settings = st
        self.sample_rate = int(st["sample_rate"])
        self.max_batch_samples = max_batch_samples
        self.strides = conv_strides(str(st["conv_feature_layers"]))
        if "|" not in self.vocab:
            raise ValueError("the letter dictionary has no '|': only the en model's family (silence token '|') is supported")
        if "w2v_encoder.proj.weight" in sd and int(sd["w2v_encoder.proj.weight"].shape[0]) != len(self.vocab):
            raise ValueError(f"the dictionary has {len(self.vocab)} tokens with the specials, the checkpoint's proj {sd['w2v_encoder.proj.weight'].shape[0]}")
        heads = int(st.get("encoder_attention_heads", 0))
        self.engine = ASREngine(sd, self.strides, device_index, extractor_layer_norm=int(st["extractor_mode"] == "layer_norm"),
                                layer_norm_first=int(bool(st["layer_norm_first"])), pos_conv_depth=int(st["pos_conv_depth"]),
                                conformer=int(st["layer_type"] == "conformer"), heads=heads, normalize=int(bool(st["normalize"])),
                                time_stages=int(time_stages))

    def letters(self, tokens: Sequence[int]) -> str:
        """post_process "collapse" (utils.py:79-82) + strip().lower() (utils.py:306, compute_asr_bleu.py:145)"""
        return "".join(self.vocab[t] for t in tokens).replace("|", " ").strip().lower()

    def num_frames(self, n_samples: int) -> int:
        return self.engine.num_frames(n_samples)

    def batches(self, lengths: Sequence[int]) -> List[List[int]]:
        """indices in batches of at most max_batch_samples samples (a longer utterance alone), longest first so padding stays small"""
        order = sorted(range(len(lengths)), key=lambda i: -lengths[i])
        out: List[List[int]] = []
        cur, tot = [], 0
        for i in order:
            if cur and tot + lengths[i] > self.max_batch_samples:
                out.append(cur)
                cur, tot = [], 0
            cur.append(i)
            tot += lengths[i]
        if cur:
            out.append(cur)
        return out

    def transcribe_tokens(self, waves: Sequence) -> List[Tuple[List[int], List[int]]]:
        """(tokens, per-frame arg-max) per waveform; a waveform shorter than one encoder frame raises ValueError naming its index"""
        ts = [torch.as_tensor(np.asarray(w, dtype=np.float32)).reshape(-1) for w in waves]
        for i, t in enumerate(ts):
            if self.num_frames(t.numel()) <= 0:
                raise ValueError(f"waveform {i}: {t.numel()} samples are fewer than one encoder frame needs")
        res: List[Tuple[List[int], List[int]]] = [([], [])] * len(ts)
        for idx in self.batches([t.numel() for t in ts]):
            toks, am, _ = self.engine.transcribe([ts[i] for i in idx])
            r0 = 0
            for j, i in enumerate(idx):
                T = self.num_frames(ts[i].numel())
                res[i] = (toks[j], am[r0:r0 + T])
                r0 += T
        return res

    def transcribe(self, waves: Sequence) -> List[str]:
        return [self.letters(t) for t, _ in self.transcribe_tokens(waves)]

    def load_audio(self, path: str, rm_silence: bool = False) -> np.ndarray:
        """ASRGenerator.load_audiofile: 16-bit PCM scaled by 1 / 32768 or float32, mono only (the reference never averages channels:
        `audio_waveform.dim == 2` compares a method with 2).  Files the reference would read but this transcriber does not take (a rate
        other than the model's, more than one channel, another sample format, mp3) raise AudioRefused naming the file; a file that is
        not a readable WAV raises ValueError, as torchaudio.load would fail on it too."""
        from .evaluate import read_wav

        try:
            x, info = read_wav(path)
        except ValueError as e:
            if any(k in str(e) for k in _REFUSED_FORMATS):
                raise AudioRefused(f"{e} (the ASR-BLEU transcriber takes mono 16-bit PCM or float32 WAV)") from e
            raise
        if info.samplerate != self.sample_rate:
            raise AudioRefused(f"{path}: {info.samplerate} Hz; the transcriber takes {self.sample_rate} Hz WAV files (resampling is not supported)")
        if rm_silence:
            x = remove_silence(x)
        return x


class AudioRefused(ValueError):
    """a WAV file the reference transcribes but this transcriber refuses (rate, channels, sample format): never scored as an empty
    transcript"""


# read_wav's messages for files it parses but does not take (evaluate.read_wav)
_REFUSED_FORMATS = (" channels;", "WAV format ", "mp3 sources")


def remove_silence(x: np.ndarray) -> np.ndarray:
    """asr_bleu_rm_silence/utils.py:231-241: a zero is dropped when the 10 samples starting at it or the 10 ending at it are all zero,
    cyclically (torch.roll wraps around at both ends): a run of 10 zeros loses its two ends, a run of 19 or more goes whole"""
    x = np.asarray(x, dtype=np.float32)
    z = x == 0
    left = z.copy()
    right = z.copy()
    for i in range(10):
        left &= np.roll(z, -i)
        right &= np.roll(z, i)
    return x[~(z & (left | right))]
