"""`python -m streamspeech_b200.asr_bleu`: asr_bleu/compute_asr_bleu.py (and, with --rm-silence, asr_bleu_rm_silence/compute_asr_bleu.py)
on the engine's transcriber.  Same flags, files and printed score line; the transcriber runs batched on the GPU (asr.ASRTranscriber) and
BLEU is sacrebleu 2.2.0's corpus_bleu restated (sacrebleu_compat).  Only the `en` model is offered, from local files: nothing is
downloaded.  `--devices LIST` transcribes groups of files on one worker process per entry (streamspeech_b200/workers.py) and writes the
same files and score line.
"""
from __future__ import annotations

import argparse
import glob
import os
import re
import sys
from contextlib import closing
from functools import partial
from pathlib import Path
from typing import Dict, List, Optional, Sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from streamspeech_b200 import workers  # noqa: E402
from streamspeech_b200.asr import AudioRefused  # noqa: E402
from streamspeech_b200.sacrebleu_compat import corpus_bleu  # noqa: E402

# asr_bleu/asr_model_cfgs.json, en / oct22: the files a user fetches once and passes as --asr-model / --asr-dict
EN_MODEL_URLS = {"oct22": ("https://dl.fbaipublicfiles.com/fairseq/wav2vec/wav2vec_vox_960h_pl.pt",
                           "https://dl.fbaipublicfiles.com/fairseq/wav2vec/dict.ltr.txt")}


def extract_audio_for_eval(audio_dirpath: str, audio_format: str, sort_numeric: bool = False) -> List[str]:
    """compute_asr_bleu.py:36-62: for i < the number of *_pred.wav files, {i}_pred.wav or else the one {i}_spk*_pred.wav"""
    if audio_format != "n_pred.wav":
        raise NotImplementedError(audio_format)
    audio_fp_list = glob.glob((Path(audio_dirpath) / "*_pred.wav").as_posix())
    if sort_numeric:  # the rm_silence variant sorts first (and fails on a name without a numeric prefix)
        audio_fp_list = sorted(audio_fp_list, key=lambda x: int(os.path.basename(x).split("_")[0]))
    out = []
    for i in range(len(audio_fp_list)):
        fp = (Path(audio_dirpath) / f"{i}_pred.wav").as_posix()
        if fp not in audio_fp_list:
            cands = glob.glob((Path(audio_dirpath) / f"{i}_spk*_pred.wav").as_posix())
            if len(cands) != 1:
                raise AssertionError(f"{i}_pred.wav does not exist in {audio_dirpath} and {len(cands)} files match {i}_spk*_pred.wav")
            fp = cands[0]
        out.append(fp)
    return out


_PANDAS_NA = {"", "#N/A", "#N/A N/A", "#NA", "-1.#IND", "-1.#QNAN", "-NaN", "-nan", "1.#IND", "1.#QNAN", "<NA>", "N/A", "NA", "NULL", "NaN",
              "None", "n/a", "nan", "null"}  # pd.read_csv's default na_values


def _is_number(c: str) -> bool:
    try:
        float(c)
        return True
    except ValueError:
        return False


def read_tsv_column(path: str, column: str) -> List[str]:
    """pd.read_csv(path, sep="\\t", quoting=3)[column]: no quote processing, blank lines skipped, the first line is the header"""
    with open(path, encoding="utf-8") as f:
        rows = [ln.rstrip("\r\n") for ln in f]
    rows = [r for r in rows if r.strip() != ""]
    header = rows[0].split("\t")
    if column not in header:
        raise KeyError(column)
    j = header.index(column)
    cells = [r.split("\t")[j] for r in rows[1:]]
    # pandas turns these into NaN, and a column of numbers into numbers; the reference's .strip() then fails on them
    for i, c in enumerate(cells):
        if c in _PANDAS_NA:
            raise ValueError(f"{path}: row {i + 1} of column {column!r} is {c!r}, which pd.read_csv reads as NaN; the reference fails on it")
    if cells and all(_is_number(c) for c in cells):
        raise ValueError(f"{path}: column {column!r} holds only numbers, which pd.read_csv reads as numbers; the reference fails on it")
    return cells


def extract_text_for_eval(references_filepath: str, reference_format: str, reference_tsv_column: Optional[str] = None) -> List[str]:
    """compute_asr_bleu.py:65-78"""
    if reference_format == "txt":
        with open(references_filepath, "r") as f:
            return [ln.strip() for ln in f.readlines()]
    if reference_format == "tsv":
        return [s.strip() for s in read_tsv_column(references_filepath, reference_tsv_column)]
    raise NotImplementedError(reference_format)


def _parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="ASR-BLEU between generated audio and text references, on the engine's GPU transcriber.")
    p.add_argument("--lang", type=str)
    p.add_argument("--asr_version", type=str, default="oct22")
    p.add_argument("--audio_dirpath", type=str)
    p.add_argument("--reference_path", type=str)
    p.add_argument("--reference_format", choices=["txt", "tsv"])
    p.add_argument("--reference_tsv_column", default=None, type=str)
    p.add_argument("--audio_format", default="n_pred.wav", choices=["n_pred.wav"])
    p.add_argument("--results_dirpath", default=None, type=str)
    p.add_argument("--transcripts_path", default=None, type=str, help="write the transcripts here, one per line (the rm_silence variant)")
    p.add_argument("--rm-silence", action="store_true", help="asr_bleu_rm_silence/: drop runs of >= 10 zero samples; a failed "
                                                             "transcription raises instead of scoring as an empty string; no pred.txt")
    p.add_argument("--asr-model", default=None, help="local path of the fairseq checkpoint (or 'synthetic': the seeded test model)")
    p.add_argument("--asr-dict", default=None, help="local path of dict.ltr.txt")
    p.add_argument("--asr-setting", action="append", default=[], metavar="KEY=VALUE",
                   help="override a setting read from the checkpoint's cfg (or the en model's published ones when the cfg cannot be "
                        "read): conv_feature_layers, extractor_mode, layer_norm_first, pos_conv_depth, layer_type, "
                        "encoder_attention_heads, normalize, sample_rate")
    p.add_argument("--device", type=int, default=0)
    workers.add_devices_arg(p)
    return p


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    return workers.parse_with_devices(_parser(), argv, "--device")


def check_model_args(args: argparse.Namespace):
    if args.lang != "en":
        raise SystemExit(f"--lang {args.lang}: only the `en` transcriber (fairseq wav2vec 2.0) is offered; the Hugging Face models of other "
                         "languages and the Hokkien model are not")
    if args.asr_version not in EN_MODEL_URLS:
        raise SystemExit(f"--asr_version {args.asr_version}: only {sorted(EN_MODEL_URLS)} exists for en")
    ckpt_url, dict_url = EN_MODEL_URLS[args.asr_version]
    for flag, val, url in (("--asr-model", args.asr_model, ckpt_url), ("--asr-dict", args.asr_dict, dict_url)):
        if val is None and not (flag == "--asr-dict" and args.asr_model == "synthetic"):
            raise SystemExit(f"{flag} is required: nothing is downloaded; fetch {url} and pass its local path")
        if val is not None and re.search("^https?://", val):
            raise SystemExit(f"{flag} {val}: nothing is downloaded; fetch {os.path.basename(val)} and pass its local path")


# ------------------------------------------------------------------------------------------------------------------- transcription

def asr_bleu_wave(tr, fp: str, rm_silence: bool):
    """compute_asr_bleu.py's reading of one file: its waveform, or None where the script's transcription fails and scores as ""
    (compute_asr_bleu.py:141-147).  A file the reference would transcribe but this transcriber refuses raises AudioRefused; with
    rm_silence every failure raises."""
    try:
        w = tr.load_audio(fp, rm_silence=rm_silence)
        if tr.num_frames(len(w)) <= 0:
            raise ValueError(f"{fp}: {len(w)} samples are fewer than one encoder frame needs")
        return w
    except AudioRefused:
        raise  # never scored as ""
    except Exception:
        if rm_silence:
            raise
        return None


def simuleval_wave(tr, fp: str):
    """the waveform of one file as SimulEval's compute_asr_bleu.py run reads it; too short for one encoder frame: SimulEvalASRFailed"""
    w = tr.load_audio(fp)
    if tr.num_frames(len(w)) <= 0:
        raise SimulEvalASRFailed(f"{fp}: {len(w)} samples are fewer than one encoder frame needs")
    return w


def transcribe_group(tr, files: Sequence[str], read) -> List[object]:
    """Per file its transcript, or the exception read(tr, file) raised (then nothing is transcribed).  read returns the waveform, or
    None for a file that transcribes as ""; the readable files are transcribed in one batched call."""
    waves: List[object] = []
    for fp in files:
        try:
            waves.append(read(tr, fp))
        except Exception as e:  # noqa: BLE001 (raised by transcribe_files in file order)
            waves.append(e)
    if any(isinstance(w, Exception) for w in waves):
        return waves
    ok = [i for i, w in enumerate(waves) if w is not None]
    out: List[object] = [""] * len(files)
    for i, t in zip(ok, tr.transcribe([waves[i] for i in ok])):
        out[i] = t
    return out


class DeviceTranscribers:
    """The transcription of `--devices`: one ASRTranscriber per entry of devices, each in its own worker process, over groups of
    files pulled from a shared queue (streamspeech_b200/workers.py); transcripts come back in file order.  A transcript does not
    depend on the batch it ran in (the transcriber's batch-of-one identity), so it equals the single-device one.  An error that is not
    scored (a refused or unreadable file) raises in its worker and stops every worker (workers.WorkerFailed names the device and the
    error); SimulEval's failure (a file too short for one frame) comes back and is raised in file order, to be scored as 0."""

    def __init__(self, devices: Sequence[int], model_path: str, dict_path: Optional[str], settings: Dict[str, object]):
        self.devices, self.model_path, self.dict_path, self.settings = list(devices), model_path, dict_path, settings

    def transcribe_files(self, files: Sequence[str], read) -> List[object]:
        size = max(1, min(64, -(-len(files) // (4 * len(self.devices)))))  # about four groups per worker, for balance
        groups = [(k, list(files[i:i + size])) for k, i in enumerate(range(0, len(files), size))]
        out: List[object] = []
        with closing(workers.run(self.devices, _transcribe_job, (self.model_path, self.dict_path, self.settings, read), groups)) as results:
            for _, outcomes in results:
                out += outcomes
        return out


def _transcribe_job(device: int, payload, next_item, emit):
    from streamspeech_b200.asr import ASRTranscriber

    model_path, dict_path, settings, read = payload
    tr = ASRTranscriber(model_path, dict_path, device, settings=settings)
    try:
        for key, files in iter(next_item, None):
            outcomes = transcribe_group(tr, files, read)
            for o in outcomes:  # an error the run cannot score stops every worker now (SimulEval's failure is scored, as 0)
                if isinstance(o, Exception) and not isinstance(o, SimulEvalASRFailed):
                    raise o
            emit(key, outcomes)
    finally:
        tr.engine.close()


def transcribe_files(tr, files: Sequence[str], read) -> List[str]:
    """the transcripts of files on tr (an ASRTranscriber, or DeviceTranscribers); read(tr, file) as in transcribe_group.  Where a
    read raised, the first such error in file order is raised, a SimulEvalASRFailed only when no other error was: as a single pass
    that reads every file before it checks any length raises."""
    outcomes = tr.transcribe_files(files, read) if isinstance(tr, DeviceTranscribers) else transcribe_group(tr, files, read)
    errors = [o for o in outcomes if isinstance(o, Exception)]
    for e in [e for e in errors if not isinstance(e, SimulEvalASRFailed)] + errors:
        raise e
    return outcomes


def run_asr_bleu(args: argparse.Namespace, transcriber=None):
    """-> (transcripts, BLEUScore); writes pred.txt (default variant)"""
    from streamspeech_b200.asr import ASRTranscriber, parse_settings

    references = extract_text_for_eval(args.reference_path, args.reference_format, args.reference_tsv_column)
    files = extract_audio_for_eval(args.audio_dirpath, args.audio_format, sort_numeric=args.rm_silence)
    assert len(files) == len(references)
    if transcriber is not None:
        tr = transcriber
    elif args.devices is not None:
        tr = DeviceTranscribers(args.devices, args.asr_model, args.asr_dict, parse_settings(args.asr_setting))
    else:
        tr = ASRTranscriber(args.asr_model, args.asr_dict, args.device, settings=parse_settings(args.asr_setting))
    transcripts = transcribe_files(tr, files, partial(asr_bleu_wave, rm_silence=args.rm_silence))
    if not args.rm_silence:
        with open(Path(args.audio_dirpath) / "pred.txt", "w") as f:
            f.write("\n".join(transcripts))
    bleu = corpus_bleu(transcripts, [references])
    print(bleu)
    return transcripts, bleu


class SimulEvalASRFailed(Exception):
    """where the compute_asr_bleu.py run that SimulEval makes fails on the run's files: a missing wav, a file too short to transcribe"""


def transcribe_simuleval(audio_dirpath: str, reference_path: str, make_transcriber) -> List[str]:
    """The run of fairseq's examples/speech_to_speech/asr_bleu/compute_asr_bleu.py that SimulEval's ASR_BLEU scorer makes
    (`--reference_path instances.log --reference_format txt`): the *_pred.wav files in numeric order, one per line of the reference
    file, each transcribed as written (no silence removal) in one batched pass -> the lower-cased transcripts, transcript i of
    {i}_pred.wav.  Where the script fails on the files, this raises SimulEvalASRFailed naming the cause: a wav {i}_pred.wav missing for
    some i below the number of lines, or a file too short for one encoder frame.  Anything else (an unreadable file, a transcriber
    error) propagates as it is.  make_transcriber() builds the transcriber, once the files are known to be there.  The script's own
    BLEU against the log's lines is not computed: SimulEval ignores it."""
    references = extract_text_for_eval(reference_path, "txt")
    try:
        files = extract_audio_for_eval(audio_dirpath, "n_pred.wav", sort_numeric=True)
    except AssertionError as e:
        raise SimulEvalASRFailed(str(e)) from e
    if len(files) != len(references):
        missing = [f"{i}_pred.wav" for i in range(len(references)) if not (Path(audio_dirpath) / f"{i}_pred.wav").exists()]
        raise SimulEvalASRFailed(f"{len(files)} *_pred.wav files in {audio_dirpath} for {len(references)} lines of {reference_path}; "
                                 f"missing: {', '.join(missing) or 'none'}")
    return transcribe_files(make_transcriber(), files, simuleval_wave)


def main(argv: Optional[Sequence[str]] = None, transcriber=None):
    args = parse_args(argv)
    if transcriber is None:
        check_model_args(args)
    transcripts, bleu = run_asr_bleu(args, transcriber)
    if args.results_dirpath is not None:
        Path(args.results_dirpath).mkdir(parents=True, exist_ok=True)
        with open(Path(args.results_dirpath) / f"{args.reference_format}_{args.lang}_bleu.txt", "w") as f:
            f.write(bleu.format(width=2))
    if args.transcripts_path is not None:
        with open(args.transcripts_path, "w") as f:
            for t in transcripts:
                f.write(t + "\n")
    return transcripts, bleu


if __name__ == "__main__":
    main()
