"""`fairseq-generate --task speech_to_speech_ctc` for a data split on one engine: the offline S2ST evaluation of
researches/ctc_unity/test_scripts/pred.offline-s2st.sh with `fairseq-generate` replaced by this module:

    python -m streamspeech_b200.generate DATA --user-dir researches/ctc_unity \\
        --config-yaml config_gcmvn.yaml --multitask-config-yaml config_mtl_asr_st_ctcst.yaml \\
        --task speech_to_speech_ctc --target-is-code --target-code-size 1000 --vocoder code_hifigan \\
        --path CKPT --gen-subset test --beam-mt 1 --beam 1 --max-len-a 1 \\
        --max-tokens 10000 --required-batch-size-multiple 1 --results-path OUT > OUT/generate-test.log

The split is read, ordered and batched as fairseq does it (SpeechToTextDataset.ordered_indices, the task's max_positions filter,
data_utils.batch_by_size -> batch_by_size_vec, the collater's descending sort by n_frames inside each batch), because the unit
decoder's positional row is the sample's index in its batch (quirk N1, streamspeech_b200/offline.py): another batching would change
the units.  Each batch is one OfflineS2STGenerator.generate(..., scores=True) call.  Written:

  stdout                         per batch, in the collater's order: every `A-{id}\\t{ASR CTC text}`, then every `S-` (ST CTC text),
                                 then every `D-` (MT text) -- sequence_generator_multi_decoder_ctc.py:206-289's prints
  RESULTS/generate-{subset}.txt  per sample in batch order the unit hypothesis' `T-`, `H-`, `D-`, `P-` lines (fairseq_cli/generate.py:
                                 255-299: scores in base 2), then `Generate {subset} with beam={beam}: BLEU4 = ...` (fairseq's bleu
                                 scorer over unit ids)

Logger lines are not written.  With `--target-is-code` the reference's dataset creator replaces every target by the empty string
(speech_to_speech_dataset_modified.py:301-308), so, as there, every `T-` text is empty and BLEU is scored against a lone eos.
The vocoder is not loaded (fairseq-generate does not load it either); run streamspeech_b200.generate_waveform_from_code on the units.

`--task speech_to_speech_modified` with a UnitY checkpoint (unity.{fr,es,de}-en.pt) is researches/unitY/test_scripts/pred.sh's
`fairseq-generate --user-dir researches/translatotron ... --beam-mt 10 --beam 1 --max-len-a 1`: each batch is one
UnitYGenerator.generate call (MT search, T2U encoder, autoregressive unit search with max_len = min(int(max_len_a * F + max_len_b),
max_target_positions - 1), F the batch's padded fbank length).  stdout then carries only the `D-{id}\t{MT text}` prints
(sequence_generator_multi_decoder.py:217); the results file is written as above.  A Uni-UnitY checkpoint (arch uni_unity_conformer
or uni_unity_conformer_waitk) is researches/uni_unity/test_scripts/pred.sh (`--user-dir researches/uni_unity`): the same batching
and files, its encoder with a future mask and its T2U encoder causal, and the MT prints of fairseq's own generator, which that task
builds: `{MT text} (None-{id})`.  Chunk-UnitY is a simultaneous model and is refused here (offline_settings).
"""
from __future__ import annotations

import argparse
import csv
import io
import math
import os
import sys
import time
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _REPO not in sys.path:
    sys.path.insert(0, _REPO)

from streamspeech_b200 import workers  # noqa: E402

TASKS = ("speech_to_speech_ctc", "speech_to_speech_modified")  # StreamSpeech, UnitY
MAX_SOURCE_POSITIONS = 6000  # fairseq/tasks/speech_to_speech.py: --max-source-positions default
MAX_TARGET_POSITIONS = 1024  # --max-target-positions default
ENCODER_SUBSAMPLING = 4      # two stride-2 convolutions: ceil(ceil(F / 2) / 2) encoder frames (ss_encoder_out_frames)


# ------------------------------------------------------------------------------------------------------------------------ arguments

def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    p = argparse.ArgumentParser(prog="python -m streamspeech_b200.generate", description=__doc__,
                                formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("data", help="directory of the split manifests ({gen_subset}.tsv) and the configs")
    p.add_argument("--user-dir", default=None, help="the task is built in; with --path synthetic it names the UnitY-family model")
    p.add_argument("--config-yaml", default="config.yaml")
    p.add_argument("--multitask-config-yaml", default=None)
    p.add_argument("--task", default="speech_to_speech_ctc")
    p.add_argument("--target-is-code", action="store_true")
    p.add_argument("--target-code-size", type=int, default=None)
    p.add_argument("--vocoder", default="griffin_lim", help="accepted and ignored: fairseq-generate does not load it here")
    p.add_argument("--path", required=True, help="checkpoint (.pt), or synthetic[:seed] for the seeded synthetic checkpoint")
    p.add_argument("--gen-subset", default="test")
    p.add_argument("--beam-mt", type=int, default=1)
    p.add_argument("--beam", type=int, default=5)
    p.add_argument("--nbest", type=int, default=1)
    p.add_argument("--max-len-a", type=float, default=0, help="UnitY's unit search; ignored by the CTC unit decoder, which does not search")
    p.add_argument("--max-len-b", type=int, default=200, help="UnitY's unit search; ignored by the CTC unit decoder, which does not search")
    p.add_argument("--max-len-a-mt", type=float, default=0)
    p.add_argument("--max-len-b-mt", type=int, default=200)
    p.add_argument("--lenpen", type=float, default=1.0)
    p.add_argument("--max-tokens", type=int, default=None)
    p.add_argument("--batch-size", "--max-sentences", dest="batch_size", type=int, default=None)
    p.add_argument("--required-batch-size-multiple", type=int, default=8)
    p.add_argument("--max-source-positions", type=int, default=MAX_SOURCE_POSITIONS)
    p.add_argument("--max-target-positions", type=int, default=MAX_TARGET_POSITIONS)
    p.add_argument("--skip-invalid-size-inputs-valid-test", action="store_true")
    p.add_argument("--results-path", default=None, help="directory of generate-{gen_subset}.txt (default: the file goes to stdout)")
    p.add_argument("--device-index", type=int, default=0)
    workers.add_devices_arg(p)
    p.add_argument("--cpu", action="store_true", help="refused: the engine runs on the GPU")
    args = workers.parse_with_devices(p, argv, "--device-index")
    if args.cpu:
        p.error("--cpu is not offered: every stage runs on the H100 engine")
    if args.task not in TASKS:
        p.error(f"--task {args.task}: only speech_to_speech_ctc (StreamSpeech) and speech_to_speech_modified (UnitY) are offered")
    unity = args.task == "speech_to_speech_modified"
    if args.beam != 1:
        p.error(f"--beam {args.beam}: " + ("the UnitY unit search runs at beam 1 only" if unity else "the CTC unit decoder does not search")
                + "; pass --beam 1 (--beam-mt sets the MT beam)")
    if args.nbest != 1:
        p.error(f"--nbest {args.nbest}: the unit decoder gives one hypothesis here; pass --nbest 1")
    if unity and not math.isfinite(args.max_len_a):
        p.error(f"--max-len-a {args.max_len_a}: must be finite")
    if args.max_len_a_mt != 0:
        p.error(f"--max-len-a-mt {args.max_len_a_mt}: only 0 (the reference default) is supported")
    if not 1 <= args.beam_mt <= 32:
        p.error(f"--beam-mt {args.beam_mt}: must be in [1, 32]")
    if args.max_tokens is None and args.batch_size is None:
        p.error("--max-tokens or --batch-size is required")
    return args


# ----------------------------------------------------------------------------------------------------------------------------- data

def read_manifest(path: str) -> List[Dict[str, str]]:
    """SpeechToTextDatasetCreator._load_samples_from_tsv: a tab-separated file with a header row, no quoting"""
    if not os.path.isfile(path):
        raise FileNotFoundError(f"Dataset not found: {path}")
    with open(path, encoding="utf-8", newline="") as f:
        rows = list(csv.DictReader(f, delimiter="\t", quotechar=None, doublequote=False, lineterminator="\n", quoting=csv.QUOTE_NONE))
    for k in ("id", "src_audio", "src_n_frames"):
        if rows and k not in rows[0]:
            raise ValueError(f"{path}: no `{k}` column")
    return rows


def read_features(path: str) -> np.ndarray:
    """get_features_or_waveform for feature sources: `x.npy`, or `archive.zip:offset:length` (a .npy stored uncompressed in a zip).
    Waveform sources are refused."""
    parts = path.split(":")
    if len(parts) == 3:
        zpath, offset, length = parts[0], int(parts[1]), int(parts[2])
        if not zpath.endswith(".zip"):
            raise ValueError(f"{path}: a sliced source must point into a .zip")
        with open(zpath, "rb") as f:
            f.seek(offset)
            data = f.read(length)
        if len(data) != length:
            raise ValueError(f"{path}: the zip entry is truncated")
        if data[:6] != b"\x93NUMPY":
            raise ValueError(f"{path}: only .npy features are read (waveform sources are not supported; extract fbank features)")
        return np.load(io.BytesIO(data))
    if len(parts) != 1:
        raise ValueError(f"Invalid path: {path}")
    if not path.endswith(".npy"):
        raise ValueError(f"{path}: only .npy features are read (waveform sources such as .wav / .flac are not supported; "
                         "extract fbank features)")
    return np.load(path)


def feature_transforms(config: dict, split: str) -> List[str]:
    """S2TDataConfig.get_feature_transforms for an evaluation split: `transforms` (then `feature_transforms`) for the split, else
    `_eval`, else `*`"""
    out: Optional[List[str]] = None
    for key in ("transforms", "feature_transforms"):
        d = config.get(key) or {}
        cur = d.get(split)
        cur = d.get("_eval") if cur is None else cur
        cur = d.get("*") if cur is None else cur
        if cur is not None:
            out = list(cur) if out is None else out + list(cur)
    return out or []


def load_cmvn(config: dict, split: str) -> Optional[Tuple[np.ndarray, np.ndarray]]:
    """(mean, std) of GlobalCMVN when the split's transforms list global_cmvn; any other transform is refused"""
    names = feature_transforms(config, split)
    for n in names:
        if n != "global_cmvn":
            raise ValueError(f"feature transform `{n}` is not supported at evaluation (only global_cmvn)")
    if not names:
        return None
    stats = np.load(config["global_cmvn"]["stats_npz_path"])
    return stats["mean"], stats["std"]


def apply_cmvn(x: np.ndarray, cmvn) -> np.ndarray:
    """GlobalCMVN.__call__: np.subtract then np.divide, numpy's dtype promotion included"""
    if cmvn is None:
        return x
    return np.divide(np.subtract(x, cmvn[0]), cmvn[1])


# ------------------------------------------------------------------------------------------------------------------------- batching

def ordered_indices(n_frames: Sequence[int]) -> np.ndarray:
    """SpeechToTextDataset.ordered_indices without shuffling: descending n_frames, then manifest order"""
    return np.lexsort([np.arange(len(n_frames)), [-int(n) for n in n_frames]])


def filter_indices_by_size(indices: np.ndarray, src_n_frames: Sequence[int], tgt_n_frames: Sequence[int], max_positions: Tuple[int, int],
                           ignore_invalid: bool) -> np.ndarray:
    """FairseqTask.filter_indices_by_size with the dataset's size(i) = (src_n_frames, tgt_n_frames) against the task's
    (max_source_positions, max_target_positions)"""
    keep, ignored = [], []
    for i in indices.tolist():
        (keep if src_n_frames[i] <= max_positions[0] and tgt_n_frames[i] <= max_positions[1] else ignored).append(i)
    if ignored and not ignore_invalid:
        i = ignored[0]
        raise ValueError(f"Size of sample #{i} is invalid (={(src_n_frames[i], tgt_n_frames[i])}) since max_positions={max_positions}, "
                         "skip this example with --skip-invalid-size-inputs-valid-test")
    return np.array(keep, dtype=np.int64)


def batch_by_size_vec(indices: np.ndarray, num_tokens_vec: np.ndarray, max_tokens: int, max_sentences: int, bsz_mult: int) -> List[np.ndarray]:
    """fairseq/data/data_utils_fast.pyx batch_by_size_vec, line for line"""
    n = len(indices)
    if n == 0:
        return []
    if max_tokens > 0 and int(np.max(num_tokens_vec)) > max_tokens:
        raise ValueError(f"Sentences lengths should not exceed max_tokens={max_tokens}")
    ends = [0] * n
    batch_start = batches_count = 0
    tail_max_tokens = batch_max_tokens = 0
    for pos in range(n):
        tok = int(num_tokens_vec[pos])
        tail_max_tokens = max(tail_max_tokens, tok)
        new_batch_end = pos + 1
        new_batch_max_tokens = max(batch_max_tokens, tail_max_tokens)
        new_batch_sentences = new_batch_end - batch_start
        new_batch_num_tokens = new_batch_sentences * new_batch_max_tokens
        overflow = (max_sentences > 0 and new_batch_sentences > max_sentences) or (max_tokens > 0 and new_batch_num_tokens > max_tokens)
        size_matches_with_bsz_mult = new_batch_sentences < bsz_mult or new_batch_sentences % bsz_mult == 0
        if overflow:
            tail_num_tokens = tail_max_tokens * (new_batch_end - ends[batches_count])
            if max_tokens > 0 and tail_num_tokens > max_tokens:
                batches_count += 1
                ends[batches_count] = pos
                tail_max_tokens = tok
            batch_start = ends[batches_count]
            batches_count += 1
            new_batch_max_tokens = tail_max_tokens
        if overflow or size_matches_with_bsz_mult:
            ends[batches_count] = new_batch_end
            batch_max_tokens = new_batch_max_tokens
            tail_max_tokens = 0
    if ends[batches_count] != n:
        batches_count += 1
    return np.split(indices, ends[:batches_count])


def make_batches(src_n_frames: Sequence[int], tgt_n_frames: Sequence[int], max_tokens: Optional[int], batch_size: Optional[int],
                 required_batch_size_multiple: int, max_positions: Tuple[int, int], ignore_invalid: bool) -> List[List[int]]:
    """The dataset indices of every batch of get_batch_iterator, each in the collater's order"""
    indices = filter_indices_by_size(ordered_indices(src_n_frames), src_n_frames, tgt_n_frames, max_positions, ignore_invalid)
    nt = np.array([src_n_frames[i] for i in indices.tolist()], dtype=np.int64)
    b = batch_by_size_vec(indices, nt, int(max_tokens) if max_tokens is not None else -1,
                          int(batch_size) if batch_size is not None else -1, required_batch_size_multiple)
    if required_batch_size_multiple > 1 and b and len(b[-1]) % required_batch_size_multiple != 0:  # data_utils.batch_by_size
        b = b[:-1]
    return [collate_order(batch.tolist(), src_n_frames) for batch in b]


def collate_order(batch: Sequence[int], n_frames: Sequence[int]) -> List[int]:
    """the collater's `n_frames.sort(descending=True)`, which keeps the batch order among equal n_frames"""
    return [batch[j] for j in sorted(range(len(batch)), key=lambda j: -int(n_frames[batch[j]]))]


# -------------------------------------------------------------------------------------------------------------------------- output

def ctc_text(d, tokens: Sequence[int]) -> str:
    """the text rule of the generator's A- / S- / D- prints (sequence_generator_multi_decoder_ctc.py:216-225)"""
    text = "".join(d[int(c)] for c in tokens)
    text = text.replace("_", " ").replace("▁", " ").replace("<unk>", " ").replace("<s>", "").replace("</s>", "")
    if len(text) > 0 and text[0] == " ":
        text = text[1:]
    return text


def unit_string(d, tokens: Sequence[int], escape_unk: bool = False) -> str:
    """fairseq Dictionary.string with the generator's stripped symbols: bos and eos dropped, unk as <unk> (<<unk>> escaped)"""
    skip = {d.bos(), d.eos()}
    return " ".join(("<<unk>>" if escape_unk else "<unk>") if int(t) == d.unk() else d[int(t)] for t in tokens if int(t) not in skip)


def encode_line(d, line: str) -> List[int]:
    """Dictionary.encode_line(add_if_not_exist=False, append_eos=True) with fairseq's whitespace tokenizer"""
    return [d.index(w) for w in line.split()] + [d.eos()]


def hypothesis_lines(sample_id: str, target_str: str, hypo_str: str, score: float, positional: np.ndarray) -> List[str]:
    """generate.py:255-299 for one sample and its one hypothesis; score and positional scores in nats (converted to base 2)"""
    s = score / math.log(2)
    pos = (np.asarray(positional, dtype=np.float32) / np.float32(math.log(2))).tolist()
    return [f"T-{sample_id}\t{target_str}", f"H-{sample_id}\t{s}\t{hypo_str}", f"D-{sample_id}\t{s}\t{hypo_str}",
            "P-{}\t{}".format(sample_id, " ".join("{:.4f}".format(x) for x in pos))]


class BleuScorer:
    """fairseq/scoring/bleu.py Scorer over token ids with clib/libbleu's counting: refs and predictions are trimmed of leading pads
    and trailing pads / eos (the first token always stays), the ref's unks never match, n-grams up to 4 are clipped counts"""

    def __init__(self, pad: int, eos: int, unk: int):
        self.pad, self.eos, self.unk = pad, eos, unk
        self.reflen = self.predlen = 0
        self.match = [0] * 4
        self.count = [0] * 4

    def _trim(self, s: List[int]) -> List[int]:
        start = 0
        while start < len(s) and s[start] == self.pad:
            start += 1
        s = s[start:]
        if not s:
            return s
        end = len(s) - 1
        while end > 0 and (s[end] == self.eos or s[end] == self.pad):
            end -= 1
        return s[:end + 1]

    def add(self, ref: Sequence[int], pred: Sequence[int]):
        ref = self._trim([-999 if int(t) == self.unk else int(t) for t in ref])
        pred = self._trim([int(t) for t in pred])
        self.reflen += len(ref)
        self.predlen += len(pred)
        for n in range(1, 5):
            if len(pred) < n:
                continue
            grams: Dict[tuple, int] = {}
            for i in range(len(pred) - n + 1):
                g = tuple(pred[i:i + n])
                grams[g] = grams.get(g, 0) + 1
            self.count[n - 1] += len(pred) - n + 1
            for i in range(len(ref) - n + 1):
                g = tuple(ref[i:i + n])
                if grams.get(g, 0) > 0:
                    self.match[n - 1] += 1
                    grams[g] -= 1

    def precision(self) -> List[float]:
        return [m / c if c > 0 else 0 for m, c in zip(self.match, self.count)]

    def brevity(self) -> float:
        return min(1, math.exp(1 - self.reflen / self.predlen))

    def score(self, order: int = 4) -> float:
        psum = sum(math.log(p) if p > 0 else float("-Inf") for p in self.precision()[:order])
        return self.brevity() * math.exp(psum / order) * 100

    def result_string(self, order: int = 4) -> str:
        fmt = "BLEU{} = {:2.2f}, {:2.1f}" + "/{:2.1f}" * (order - 1) + " (BP={:.3f}, ratio={:.3f}, syslen={}, reflen={})"
        bleup = [p * 100 for p in self.precision()[:order]]
        return fmt.format(order, self.score(order=order), *bleup, self.brevity(), self.predlen / self.reflen, self.predlen, self.reflen)


# ------------------------------------------------------------------------------------------------------------------------- checkpoint

def _get(obj, key, default=None):
    if obj is None:
        return default
    if isinstance(obj, dict):
        return obj.get(key, default)
    return getattr(obj, key, default)


def offline_settings(state: dict, capacity: int) -> Tuple[bool, Optional[int]]:
    """(uni_encoder, chunk) of a checkpoint, from state["cfg"]["model"] or, in older checkpoints, state["args"].  A chunk size of at
    least the engine's encoder frame capacity (or none) is the offline model: chunk None, the engine's set_chunk(None, None).  A
    smaller chunk size is a simultaneous model, which this front door does not decode offline."""
    model_cfg = _get(_get(state, "cfg"), "model") or _get(state, "args")
    uni = bool(_get(model_cfg, "uni_encoder", False) or False)
    chunk = _get(model_cfg, "chunk_size", None)
    if chunk is not None and int(chunk) < capacity:
        raise ValueError(f"checkpoint trained with --chunk-size {int(chunk)}: a simultaneous model; offline decoding needs the offline "
                         f"model (chunk size at least {capacity} encoder frames, e.g. --chunk-size 999999)")
    return uni, None


def mt_print_line(cfg, sample_id: int, text: str) -> str:
    """the MT hypothesis line the UnitY generators print to stdout: researches/translatotron's MultiDecoderSequenceGenerator (UnitY)
    prints "D-{id}\\t{text}"; fairseq's own (examples/speech_to_speech/unity), which researches/uni_unity's task builds, prints
    "{text} (None-{id})"."""
    if cfg.unity_variant == "uni_unity":
        return "{} (None-{})".format(text, sample_id)
    return "D-{}\t{}".format(sample_id, text)


def load_offline_checkpoint(args: argparse.Namespace, capacity: int):
    """(cfg, model state dict, dictionaries) of --path; `synthetic[:seed]` is the seeded synthetic offline checkpoint"""
    import torch

    from streamspeech_b200 import synth
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.dictionary import Dictionary

    unity = args.task == "speech_to_speech_modified"
    if str(args.path).startswith("synthetic"):
        seed = int(args.path.split(":")[1]) if ":" in args.path else 0
        if unity:  # the seeded synthetic UnitY checkpoint at the released dimensions; --user-dir researches/uni_unity: Uni-UnitY's
            state = synth.make_unity_checkpoint(synth.synthetic_unity_variant(args.user_dir), seed=seed)
            offline_settings(state, capacity)
            cfg = ModelConfig.from_checkpoint(state)
            return cfg, state["model"], {"target_unigram": Dictionary.synthetic(cfg.tgt_vocab),
                                         "tgt": Dictionary.units(cfg.unit_vocab - 4, blank=False)}
        cfg = ModelConfig()
        cfg.uni_encoder = False
        dicts = {k: Dictionary.synthetic(n) for k, n in (("source_unigram", cfg.src_vocab), ("ctc_target_unigram", cfg.tgt_vocab),
                                                         ("target_unigram", cfg.tgt_vocab))}
        dicts["tgt"] = Dictionary.units(cfg.unit_vocab - 5)
        return cfg, synth.make_model_state_dict(cfg, seed=seed), dicts
    if not os.path.exists(args.path):
        raise IOError(f"Model file not found: {args.path}")
    state = torch.load(args.path, map_location="cpu", weights_only=False)
    uni, _ = offline_settings(state, capacity)
    cfg = ModelConfig.from_checkpoint(state)
    if cfg.unity != unity:
        raise ValueError(f"--task {args.task} does not match the checkpoint {args.path}: it is a "
                         f"{'UnitY' if cfg.unity else 'StreamSpeech'} model (pass --task "
                         f"{'speech_to_speech_modified' if cfg.unity else 'speech_to_speech_ctc'})")
    if not cfg.unity:
        cfg.uni_encoder = uni
    if args.multitask_config_yaml is None:
        raise ValueError("--multitask-config-yaml is required: it names the MT dictionary (and StreamSpeech's ASR and ST ones)")
    dicts = Dictionary.load_multitask(argparse.Namespace(data_bin=args.data, multitask_config_yaml=args.multitask_config_yaml), cfg)
    return cfg, state["model"], dicts


def load_config_yaml(args: argparse.Namespace) -> dict:
    path = os.path.join(args.data, args.config_yaml)
    if not os.path.isfile(path):
        if str(args.path).startswith("synthetic"):
            return {}
        raise FileNotFoundError(f"config not found: {path}")
    import yaml

    with open(path) as f:
        return yaml.safe_load(f) or {}


# --------------------------------------------------------------------------------------------------------------------------- runner

class Split:
    """The manifest of one split, its features as fairseq's dataset returns them, and fairseq's batches"""

    def __init__(self, args: argparse.Namespace, config: dict, max_encoder_frames: int):
        self.rows = read_manifest(os.path.join(args.data, f"{args.gen_subset}.tsv"))
        self.cmvn = load_cmvn(config, args.gen_subset)
        self.src_n_frames = [int(r["src_n_frames"]) for r in self.rows]
        self.tgt_n_frames = [int(r.get("tgt_n_frames") or 0) for r in self.rows]
        limit = max_encoder_frames * ENCODER_SUBSAMPLING
        for r, n in zip(self.rows, self.src_n_frames):
            if n > limit:
                raise ValueError(f"sample {r['id']}: {n} source frames; the engine's encoder takes at most {limit} "
                                 f"({max_encoder_frames} encoder frames)")
            if not (r["src_audio"].endswith(".npy") or r["src_audio"].count(":") == 2):
                raise ValueError(f"sample {r['id']}: source {r['src_audio']}: only .npy features (or .npy entries of a zip) are read; "
                                 "waveform sources are not supported")
        self.batches = make_batches(self.src_n_frames, self.tgt_n_frames, args.max_tokens, args.batch_size, args.required_batch_size_multiple,
                                    (args.max_source_positions, args.max_target_positions), args.skip_invalid_size_inputs_valid_test)
        self.target_is_code = args.target_is_code

    def features(self, i: int) -> np.ndarray:
        x = apply_cmvn(read_features(self.rows[i]["src_audio"]), self.cmvn)
        return np.asarray(x, dtype=np.float32)

    def target(self, i: int) -> str:
        """the target text of sample i as the reference's dataset holds it: "" for code targets (see the module docstring)"""
        return "" if self.target_is_code else self.rows[i].get("tgt_audio", "")


def run_batch(gen, split: Split, batch: Sequence[int]):
    """one generate(scores=True) call on the zero-padded features of the batch: its results in batch order"""
    import torch

    feats = [split.features(i) for i in batch]
    F = max(f.shape[0] for f in feats)
    x = torch.zeros(len(feats), F, feats[0].shape[1], dtype=torch.float32)
    for b, f in enumerate(feats):
        x[b, :f.shape[0]] = torch.from_numpy(f)
    return gen.generate(x.to(gen.engine.device), [f.shape[0] for f in feats], scores=True)


# (key, dictionary, result field) of the stdout prints per batch: StreamSpeech's A- / S- / D- CTC and MT texts, UnitY's MT text
STREAMSPEECH_PRINTS = (("A", "source_unigram", "asr_tokens"), ("S", "ctc_target_unigram", "st_tokens"), ("D", "target_unigram", "mt_tokens"))
UNITY_PRINTS = (("D", "target_unigram", "mt_tokens"),)


def make_generator(args: argparse.Namespace, cfg, engine):
    from streamspeech_b200.offline import OfflineS2STGenerator, UnitYGenerator

    if cfg.unity:
        return UnitYGenerator(engine, beam_size_mt=args.beam_mt, max_len_b_mt=args.max_len_b_mt, max_len_a=args.max_len_a,
                              max_len_b=args.max_len_b, len_penalty=args.lenpen)
    return OfflineS2STGenerator(engine, beam_size_mt=args.beam_mt, max_len_b_mt=args.max_len_b_mt, len_penalty=args.lenpen)


def batch_outputs(res, prints) -> List[Dict[str, object]]:
    """what the print loop reads from a batch's results, on the host: the printed tokens, units, unit score and positional scores"""
    return [{**{tok: [int(t) for t in r[tok]] for _, _, tok in prints}, "units": [int(t) for t in r["units"]],
             "unit_score": r["unit_score"], "unit_positional_scores": r["unit_positional_scores"].numpy()} for r in res]


def _generate_job(device: int, payload, next_item, emit):
    """one --devices worker: its own engine and generator on `device`, running whole batches of the split"""
    from streamspeech_b200.engine import Engine

    args, split, max_enc_frames = payload
    cfg, sd, _ = load_offline_checkpoint(args, max_enc_frames)
    engine = Engine(cfg, sd, None, None, device=device, max_enc_frames=max_enc_frames)
    try:
        gen = make_generator(args, cfg, engine)
        prints = UNITY_PRINTS if cfg.unity else STREAMSPEECH_PRINTS
        for key, batch in iter(next_item, None):
            emit(key, batch_outputs(run_batch(gen, split, batch), prints))
    finally:
        engine.close()


def main(argv: Optional[Sequence[str]] = None, stdout=None):
    args = parse_args(argv)
    stdout = stdout or sys.stdout
    from streamspeech_b200.engine import Engine

    max_enc_frames = 1024
    config = load_config_yaml(args)
    split = Split(args, config, max_enc_frames)  # the split is checked before the model is loaded
    cfg, sd, dicts = load_offline_checkpoint(args, max_enc_frames)
    prints = UNITY_PRINTS if cfg.unity else STREAMSPEECH_PRINTS
    engine = results = out_file = None
    try:
        if args.devices is None:
            engine = Engine(cfg, sd, None, None, device=args.device_index, max_enc_frames=max_enc_frames)
            gen = make_generator(args, cfg, engine)
            results = ((k, batch_outputs(run_batch(gen, split, batch), prints)) for k, batch in enumerate(split.batches))
        else:  # whole batches to the workers, each with its own engine, and their results back in batch order
            del sd  # every worker loads the checkpoint itself; this process keeps only cfg and the dictionaries
            results = workers.run(args.devices, _generate_job, (args, split, max_enc_frames), list(enumerate(split.batches)))
        if args.results_path is not None:
            os.makedirs(args.results_path, exist_ok=True)
            out_file = open(os.path.join(args.results_path, f"generate-{args.gen_subset}.txt"), "w", buffering=1, encoding="utf-8")
        out = out_file or stdout
        tgt = dicts["tgt"]
        scorer = BleuScorer(tgt.pad(), tgt.eos(), tgt.unk())
        t0 = time.perf_counter()
        seconds = 0.0
        for k, res in results:
            batch = split.batches[k]
            ids = list(batch)  # fairseq's sample["id"]: the dataset index
            for key, dname, tok in prints:
                for sid, r in zip(ids, res):
                    text = ctc_text(dicts[dname], r[tok])
                    print(mt_print_line(cfg, sid, text) if cfg.unity else f"{key}-{sid}\t{text}", file=stdout)
            for i, sid, r in zip(batch, ids, res):
                target_tokens = encode_line(tgt, split.target(i))
                target_str = unit_string(tgt, target_tokens, escape_unk=True)
                for line in hypothesis_lines(sid, target_str, unit_string(tgt, r["units"]), r["unit_score"], r["unit_positional_scores"]):
                    print(line, file=out)
                scorer.add(target_tokens, r["units"])
            seconds += sum(split.src_n_frames[i] for i in batch) / 100.0
        print("Generate {} with beam={}: {}".format(args.gen_subset, args.beam, scorer.result_string()), file=out)
        wall = time.perf_counter() - t0
        on = "" if args.devices is None else f" on devices {','.join(map(str, args.devices))}"
        print(f"| {len(split.rows)} samples in {len(split.batches)} batches, {seconds:.1f} s of source in {wall:.2f} s "
              f"({seconds / max(wall, 1e-9):.1f} audio-s/s){on}", file=sys.stderr)
    finally:
        if results is not None:
            results.close()  # stops the workers of --devices
        if out_file is not None:
            out_file.close()
        if engine is not None:
            engine.close()
    return split


if __name__ == "__main__":
    main()
