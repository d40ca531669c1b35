"""SimulEval's scorers, restated: the quality and latency metrics of a simultaneous run, and the files and table SimulEval writes.

Restated from the reference's SimulEval/simuleval/evaluator/: scorers/latency_scorer.py (AL, LAAL, AP, DAL, ATD, StartOffset,
EndOffset, NumChunks, DiscontinuitySum / Ave / Num, RTF, on the `delays` timestamps), scorers/quality_scorer.py (`BLEU`, `ASR_BLEU`
with the 13a tokenizer), evaluator.py (`quality`, `latency`, `results`, `dump_results`, `dump_metrics`, `from_args`) and
instance.py (`LogInstance`, what `--score-only` builds from instances.log).  SimulEval, sacrebleu, pandas and fairseq are not
imported: BLEU is sacrebleu_compat, the files and the table are written as pandas writes them, and ASR_BLEU transcribes on the
engine's batched wav2vec 2.0 transcriber (asr_bleu.transcribe_simuleval).  tests/golden/simuleval_scores.json pins all of it to
SimulEval's own code (oracle/gen_golden_scores.py).

SimulEval's quirks are kept, not fixed:
- a LogInstance's reference length always counts space-separated words, whatever --eval-latency-unit says (the live instances honour
  the unit);
- under --score-only ATD takes every instance as text output (target token length 0), even for a speech run;
- EndOffset and RTF end at the last interval (start + duration) for live speech output; from a log, EndOffset does when the line
  has intervals and RTF never does;
- `BLEU` on a live speech run scores the waveform paths: sacrebleu refuses a `Path`, and the scorer reports 0; from a log it scores
  the path strings;
- ASR_BLEU compares the lower-cased transcripts with the references as given.
"""
from __future__ import annotations

import csv
import io
import json
import logging
import math
import statistics
from pathlib import Path
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

from streamspeech_b200.sacrebleu_compat import corpus_bleu

logger = logging.getLogger("streamspeech_b200.scoring")

QUALITY_METRICS = ("BLEU", "ASR_BLEU")
LATENCY_METRICS = ("AL", "LAAL", "AP", "DAL", "ATD", "NumChunks", "DiscontinuitySum", "DiscontinuityAve", "DiscontinuityNum",
                   "StartOffset", "EndOffset", "RTF")
DISCONTINUITY = ("DiscontinuitySum", "DiscontinuityAve", "DiscontinuityNum")
# SimulEval's defaults (options.py): what a run scores when only the other metric flag is given
DEFAULT_QUALITY = ["BLEU"]
DEFAULT_LATENCY = ["LAAL", "AL", "AP", "DAL", "ATD"]


# ------------------------------------------------------------------------------------------------------------------------ instances

class ScoredInstance:
    """What the scorers read from one instance.  kind: "text" (a live SpeechToTextInstance), "speech" (a live
    SpeechToSpeechInstance) or "log" (a LogInstance, one line of instances.log).  metrics: what the latency scorers record."""

    def __init__(self, kind: str, index: int, delays, reference, source_length, prediction, reference_length: int,
                 durations=None, intervals=None, silences=None):
        self.kind, self.index, self.delays, self.reference = kind, index, delays, reference
        self.source_length, self.prediction, self.reference_length = source_length, prediction, reference_length
        self.durations = durations if durations is not None else []
        self.intervals = intervals if intervals is not None else []
        self.silences = silences
        self.metrics: dict = {}


def live_reference_length(reference: str, latency_unit: str) -> int:
    """Instance.reference_length (instance.py:114-121)"""
    if latency_unit == "word":
        return len(reference.split(" "))
    if latency_unit == "char":
        return len(reference.strip())
    raise NotImplementedError(latency_unit)


def live_instance(summary: dict, latency_unit: str, silences: Optional[List[float]] = None) -> ScoredInstance:
    """a live instance from its summarize() dict; speech output (a "durations" key) also needs the silences of its waveform"""
    ref_len = live_reference_length(summary["reference"], latency_unit)
    if "durations" in summary:
        return ScoredInstance("speech", summary["index"], summary["delays"], summary["reference"], summary["source_length"],
                              Path(summary["prediction"]), ref_len, summary["durations"], summary["intervals"], list(silences or []))
    return ScoredInstance("text", summary["index"], summary["delays"], summary["reference"], summary["source_length"],
                          summary["prediction"], ref_len)


def log_instance(line: str) -> ScoredInstance:
    """LogInstance (instance.py:443-457): its fields are the line's keys; no silences"""
    info = json.loads(line.strip())
    reference = info.get("reference", "")
    return ScoredInstance("log", info["index"], info.get("delays"), reference, info.get("source_length"), info.get("prediction"),
                          len(reference.split(" ")), info.get("durations"), info.get("intervals", []))


def read_log(output: Path) -> Dict[int, ScoredInstance]:
    """build_instances_from_log (evaluator.py:146-152)"""
    instances: Dict[int, ScoredInstance] = {}
    with open(Path(output) / "instances.log") as f:
        for line in f:
            ins = log_instance(line)
            instances[ins.index] = ins
    return instances


# ------------------------------------------------------------------------------------------------------------------ latency scorers

def _delays_lengths(ins: ScoredInstance, use_ref_len: bool):
    """LatencyScorer.get_delays_lengths"""
    delays = ins.delays
    assert delays
    tgt_len = len(delays) if not use_ref_len or ins.reference is None else ins.reference_length
    return delays, ins.source_length, tgt_len


def _al(ins, use_ref_len, laal=False):
    delays, source_length, target_length = _delays_lengths(ins, use_ref_len)
    if delays[0] > source_length:
        return delays[0]
    lagging = 0
    gamma = (max(len(delays), target_length) if laal else target_length) / source_length
    tau = 0
    for t_minus_1, d in enumerate(delays):
        lagging += d - t_minus_1 / gamma
        tau = t_minus_1 + 1
        if d >= source_length:
            break
    lagging /= tau
    return lagging


def _ap(ins, use_ref_len):
    delays, source_length, target_length = _delays_lengths(ins, use_ref_len)
    return sum(delays) / (source_length * target_length)


def _dal(ins, use_ref_len):
    delays, source_length, _ = _delays_lengths(ins, use_ref_len)
    dal = 0
    target_length = len(delays)
    gamma = target_length / source_length
    g_prime_last = 0
    for i_minus_1, g in enumerate(delays):
        g_prime = g if i_minus_1 == 0 else max([g, g_prime_last + 1 / gamma])
        dal += g_prime - i_minus_1 / gamma
        g_prime_last = g_prime
    dal /= target_length
    return dal


def _speech_output(ins):
    if ins.kind != "speech":  # SimulEval: assert isinstance(ins, SpeechOutputInstance)
        raise AssertionError(f"instance {ins.index}: the Discontinuity metrics need live speech output")
    return ins.silences


def _end_offset(ins, use_ref_len):
    delays, source_length, _ = _delays_lengths(ins, use_ref_len)
    if ins.kind == "speech" or (ins.kind == "log" and len(ins.intervals) > 0):
        delays = [start + duration for start, duration in ins.intervals]
    return delays[-1] - source_length


def _rtf(ins, use_ref_len):
    delays, source_length, _ = _delays_lengths(ins, use_ref_len)
    if ins.kind == "speech":
        delays = [start + duration for start, duration in ins.intervals]
    return delays[-1] / source_length


def _disc_ave(ins, use_ref_len):
    s = _speech_output(ins)
    return 0 if len(s) == 0 else sum(s) / len(s)


_COMPUTE: Dict[str, Callable] = {
    "AL": _al,
    "LAAL": lambda ins, u: _al(ins, u, laal=True),
    "AP": _ap,
    "DAL": _dal,
    "NumChunks": lambda ins, u: len(_delays_lengths(ins, u)[0]),
    "DiscontinuitySum": lambda ins, u: sum(_speech_output(ins)),
    "DiscontinuityAve": _disc_ave,
    "DiscontinuityNum": lambda ins, u: len(_speech_output(ins)),
    "StartOffset": lambda ins, u: _delays_lengths(ins, u)[0][0],
    "EndOffset": _end_offset,
    "RTF": _rtf,
}


def _skip(index) -> None:
    logger.warning(f"Instance {index} has no delay information. Skipped")


def latency_score(name: str, instances: Dict[int, ScoredInstance], use_ref_len: bool = True):
    """LatencyScorer.__call__ (ATDScorer.__call__ for ATD): the mean over the instances that have delays; each of them records its
    score in ins.metrics[name], except under ATD"""
    if name == "ATD":
        return _atd(instances)
    compute = _COMPUTE[name]
    scores = []
    for index, ins in instances.items():
        if ins.delays is None or len(ins.delays) == 0:
            _skip(index)
            continue
        score = compute(ins, use_ref_len)
        ins.metrics[name] = score
        scores.append(score)
    return statistics.mean(scores)


def _subtract(a, b):
    return [x - y for x, y in zip(a, b)]


def _atd(instances: Dict[int, ScoredInstance]):
    """ATDScorer.__call__, not computation-aware, speech input.  SimulEval reads the output type from instances[0]; here from the first
    instance, so a run that starts past index 0 is scored instead of raising KeyError."""
    first = next(iter(instances.values()), None)
    speech_out = first is not None and first.kind == "speech"
    src_token_len, tgt_token_len = 300, (300 if speech_out else 0)
    scores = []
    for index, ins in instances.items():
        delays = ins.delays
        if delays is None or len(delays) == 0:
            _skip(index)
            continue
        compute_times = [0] * len(delays)
        chunk_sizes = {"src": [0], "tgt": [0]}
        token_to_chunk = {"src": [0], "tgt": [0]}
        token_to_time = {"src": [0], "tgt": [0]}
        tgt_token_lens = []
        delays_no_duplicate = sorted(set(delays), key=delays.index)
        if not speech_out:
            prev_delay = None
            for delay in delays:
                if delay != prev_delay:
                    chunk_sizes["tgt"].append(1)
                else:
                    chunk_sizes["tgt"][-1] += 1
                prev_delay = delay
            for i, chunk_size in enumerate(chunk_sizes["tgt"][1:], 1):
                token_to_chunk["tgt"] += [i] * chunk_size
            tgt_token_lens = [tgt_token_len] * len(delays)
        else:
            s2s_delays, s2s_compute_times, chunk_durations, chunk_compute_times = [], [], [], []
            prev_delay = None
            for delay, compute_time, duration in zip(delays, compute_times, ins.durations):
                if delay != prev_delay:
                    chunk_durations.append(duration)
                    chunk_compute_times.append(compute_time)
                else:
                    chunk_durations[-1] += duration
                    chunk_compute_times[-1] += compute_time
                prev_delay = delay
            for i, chunk_duration in enumerate(chunk_durations, 1):
                num_tokens, rest = divmod(chunk_duration, tgt_token_len)
                token_lens = int(num_tokens) * [tgt_token_len] + ([rest] if rest != 0 else [])
                tgt_token_lens += token_lens
                chunk_sizes["tgt"] += [len(token_lens)]
                token_to_chunk["tgt"] += [i] * len(token_lens)
                s2s_delays += [delays_no_duplicate[i - 1]] * len(token_lens)
                s2s_compute_times += [chunk_compute_times[i - 1] / len(token_lens)] * len(token_lens)
            delays = s2s_delays
            compute_times = s2s_compute_times
        chunk_durations = _subtract(delays_no_duplicate, [0] + delays_no_duplicate[:-1])
        for i, chunk_duration in enumerate(chunk_durations, 1):
            num_tokens, rest = divmod(chunk_duration, src_token_len)
            token_lens = int(num_tokens) * [src_token_len] + ([rest] if rest != 0 else [])
            chunk_sizes["src"] += [len(token_lens)]
            for token_len in token_lens:
                token_to_time["src"].append(token_to_time["src"][-1] + token_len)
                token_to_chunk["src"].append(i)
        for delay, compute_time, token_len in zip(delays, compute_times, tgt_token_lens):
            tgt_start_time = max(delay, token_to_time["tgt"][-1])
            token_to_time["tgt"].append(tgt_start_time + token_len + compute_time)
        scores.append(_atd_compute(chunk_sizes, token_to_chunk, token_to_time))
    return statistics.mean(scores)


def _atd_compute(chunk_sizes, token_to_chunk, token_to_time) -> float:
    tgt_to_src = []
    for t in range(1, len(token_to_chunk["tgt"])):
        chunk_id = token_to_chunk["tgt"][t]
        acc_x = sum(chunk_sizes["src"][:chunk_id])
        acc_y = sum(chunk_sizes["tgt"][:chunk_id])
        s = t - max(0, acc_y - acc_x)
        current_src_size = sum(chunk_sizes["src"][:chunk_id + 1])
        tgt_to_src.append((t, s) if s < current_src_size else (t, current_src_size))
    return float(statistics.mean([token_to_time["tgt"][t] - token_to_time["src"][s] for t, s in tgt_to_src]))


# ------------------------------------------------------------------------------------------------------------------ quality scorers

def sacrebleu_corpus_score(hyps: Sequence, refs: Sequence[Sequence]):
    """sacrebleu 2.x BLEU(tokenize="13a").corpus_score(hyps, [refs]), with its argument check: a hypothesis that is not a string
    raises TypeError"""
    if not isinstance(hyps[0], str) or any(not isinstance(h, str) for h in hyps):
        raise TypeError("BLEU: Each element of `hyps` should be a string.")
    if not isinstance(refs[0][0], str) or any(not isinstance(r, str) for r in refs[0]):
        raise TypeError("BLEU: `refs` should be a sequence of sequence of strings.")
    return corpus_bleu(list(hyps), [list(refs[0])])


def bleu_score(instances: Dict[int, ScoredInstance]):
    """SacreBLEUScorer.__call__: a failure is logged and scores 0"""
    try:
        return sacrebleu_corpus_score([ins.prediction for ins in instances.values()],
                                      [[ins.reference for ins in instances.values()]]).score
    except Exception as e:  # noqa: BLE001 (SimulEval catches every exception here)
        logger.error(str(e))
        return 0


def asr_bleu_score(instances: Dict[int, ScoredInstance], make_transcriber: Callable):
    """ASRSacreBLEUScorer.__call__: transcribe the run's wavs/ as fairseq's compute_asr_bleu.py does (asr_bleu.transcribe_simuleval),
    write asr_transcripts.txt and wavs/{k}_pred.txt, and score BLEU of the transcripts against the references.  Where the script
    fails, every transcript is "" and nothing is written."""
    from streamspeech_b200.asr_bleu import SimulEvalASRFailed, transcribe_simuleval

    first = next(iter(instances.values()))
    wav_dir = Path(first.prediction).absolute().parent
    root_dir = wav_dir.parent
    try:
        transcripts = transcribe_simuleval(wav_dir.as_posix(), (root_dir / "instances.log").as_posix(), make_transcriber)
    except SimulEvalASRFailed as e:  # only where the script fails; any other error (a refused file, the transcriber) propagates
        logger.error(f"ASR on target speech failed: {e}")
        transcripts = ["" for _ in instances.keys()]
    else:
        with open(root_dir / "asr_transcripts.txt", "w") as f:
            for t in transcripts:
                f.write(t + "\n")
        transcripts = [t.strip() for t in transcripts]  # as SimulEval reads the file back
        for idx, item in enumerate(transcripts):
            with open(wav_dir / f"{idx}_pred.txt", "w") as f:
                f.write(item.lower() + "\n")
    return sacrebleu_corpus_score(transcripts, [[ins.reference for ins in instances.values()]]).score


# ------------------------------------------------------------------------------------------------------------------------- requests

def check_request(quality: Sequence[str], latency: Sequence[str], *, tokenizer: str = "13a", target_speech_lang: str = "en",
                  speech_output: Optional[bool] = None, score_only: bool = False, asr_model: Optional[str] = None,
                  n_instances: Optional[int] = None) -> None:
    """Refuse, with a message that names the metric or flag, what SimulEval cannot score or this module does not offer.
    speech_output None: unknown (--score-only).  n_instances None: unknown until instances.log is read."""
    for name in quality:
        if name == "WHISPER_ASR_BLEU":
            raise SystemExit("--quality-metrics WHISPER_ASR_BLEU is not offered: it needs OpenAI's whisper; ASR_BLEU scores speech "
                             "output on the engine's wav2vec 2.0 transcriber")
        if name not in QUALITY_METRICS:
            raise SystemExit(f"--quality-metrics {name}: no quality metric called {name}; one of {list(QUALITY_METRICS)}")
    for name in latency:
        if "_SpeechAlign_" in name:
            raise SystemExit(f"--latency-metrics {name} is not offered: the SpeechAlign metrics align the output speech with the "
                             "Montreal Forced Aligner (mfa)")
        if name not in LATENCY_METRICS:
            raise SystemExit(f"--latency-metrics {name}: no latency metric called {name}; one of {list(LATENCY_METRICS)}")
        if name in DISCONTINUITY and score_only:
            raise SystemExit(f"--latency-metrics {name} cannot be scored with --score-only: SimulEval computes it from the live "
                             "speech-output instances only (the lines of instances.log have no silences)")
        if name in DISCONTINUITY and speech_output is False:
            raise SystemExit(f"--latency-metrics {name} needs speech output; this agent writes text")
    if tokenizer != "13a":
        raise SystemExit(f"--sacrebleu-tokenizer {tokenizer}: only the 13a tokenizer is offered")
    if target_speech_lang != "en":
        raise SystemExit(f"--target-speech-lang {target_speech_lang}: only the `en` transcriber (fairseq wav2vec 2.0) is offered")
    if "ASR_BLEU" in quality:
        if speech_output is False:
            raise SystemExit("--quality-metrics ASR_BLEU needs speech output; this agent writes text (score it with BLEU)")
        if asr_model is None:
            raise SystemExit("--quality-metrics ASR_BLEU needs --asr-model (and --asr-dict): the local fairseq wav2vec 2.0 CTC "
                             "checkpoint and its dict.ltr.txt, or 'synthetic' for the seeded test model; nothing is downloaded")
    if n_instances == 0:
        raise SystemExit(f"{'--latency-metrics ' + latency[0] if latency else '--quality-metrics ' + quality[0]}: there are no "
                         "instances to score")


def metric_lists(quality: Optional[Sequence[str]], latency: Optional[Sequence[str]]):
    """(quality, latency) with SimulEval's defaults where one is not given; None when neither is"""
    if quality is None and latency is None:
        return None
    return (list(quality) if quality is not None else list(DEFAULT_QUALITY),
            list(latency) if latency is not None else list(DEFAULT_LATENCY))


# -------------------------------------------------------------------------------------------------------------------------- results

def score(instances: Dict[int, ScoredInstance], quality: Sequence[str], latency: Sequence[str], use_ref_len: bool = True,
          make_transcriber: Optional[Callable] = None) -> Dict[str, object]:
    """Evaluator.results before the frame: {name: round(value, 3)}, quality metrics first.  A latency metric with no instance to
    score raises SystemExit naming it (SimulEval raises statistics.StatisticsError)."""
    scores: Dict[str, object] = {}
    for name in quality:
        scores[name] = bleu_score(instances) if name == "BLEU" else asr_bleu_score(instances, make_transcriber)
    for name in latency:
        try:
            scores[name] = latency_score(name, instances, use_ref_len)
        except statistics.StatisticsError:
            raise SystemExit(f"--latency-metrics {name}: no instance has delays to score (every prediction was empty)") from None
    return {name: round(v, 3) if isinstance(v, (int, float)) else v for name, v in scores.items()}


def _is_int(v) -> bool:
    return isinstance(v, (int, np.integer)) and not isinstance(v, bool)


def _tsv(header: List[str], rows: List[List[str]]) -> str:
    """pandas to_csv(sep="\\t", index=False): the csv module's minimal quoting, "\\n" line ends"""
    buf = io.StringIO()
    w = csv.writer(buf, delimiter="\t", lineterminator="\n", quoting=csv.QUOTE_MINIMAL)
    w.writerow(header)
    w.writerows(rows)
    return buf.getvalue()


def _column(values: List) -> List[str]:
    """one frame column as to_csv writes it: int64 when every value is an int, else float64 (repr, NaN as "")"""
    if all(_is_int(v) for v in values):
        return [str(int(v)) for v in values]
    return ["" if v is None or (isinstance(v, float) and math.isnan(v)) else repr(float(v)) for v in values]


def scores_tsv(scores: Dict[str, object]) -> str:
    """dump_results' scores.tsv"""
    names = list(scores)
    return _tsv(names, [[_column([scores[n]])[0] for n in names]])


def metrics_tsv(instances: Dict[int, ScoredInstance]) -> str:
    """dump_metrics' metrics.tsv: pandas.DataFrame([ins.metrics ...]).round(3), one row per instance, columns in order of first
    appearance, a missing metric as an empty field"""
    rows = [ins.metrics for ins in instances.values()]
    names: List[str] = []
    for m in rows:
        names += [k for k in m if k not in names]
    cols = []
    for n in names:
        vals = [m.get(n) for m in rows]
        if all(_is_int(v) for v in vals):
            cols.append(_column(vals))
        else:  # DataFrame.round: numpy's rint(x * 1000) / 1000
            cols.append(_column([None if v is None else float(np.round(np.float64(v), 3)) for v in vals]))
    return _tsv(names, [[c[i] for c in cols] for i in range(len(rows))])


def _table_value(v) -> str:
    """one value of a one-row frame as to_string(index=False) formats it (display.precision 6)"""
    if _is_int(v):
        return str(int(v))
    v = float(v)
    if math.isnan(v):
        return "NaN"
    s = f"{v:.6f}"
    if "." in s:
        s = s.rstrip("0")
        s = s + "0" if s.endswith(".") else s
    if (abs(v) < 1e-6 and v != 0) or (len(s) > 12 and abs(v) > 1e6):
        s = f"{v:.6e}"
    return s


def results_table(scores: Dict[str, object]) -> str:
    """dump_results' printed table: DataFrame(scores).to_string(index=False), without the final newline print() adds.  A numeric
    column's header gets a leading space; each column is right-justified to its widest cell; columns are joined by one space."""
    heads, cells = [], []
    for name, v in scores.items():
        h, c = " " + name, _table_value(v)
        w = max(len(h), len(c))
        heads.append(h.rjust(w))
        cells.append(c.rjust(w))
    return " ".join(heads) + "\n" + " ".join(cells)


def dump(output: Optional[Path], instances: Dict[int, ScoredInstance], scores: Dict[str, object]) -> str:
    """dump_results + dump_metrics: write scores.tsv and metrics.tsv into output and print the table; -> the table"""
    table = results_table(scores)
    if output is not None:
        with open(Path(output) / "scores.tsv", "w") as f:
            f.write(scores_tsv(scores))
    print(table)
    if output is not None:
        with open(Path(output) / "metrics.tsv", "w") as f:
            f.write(metrics_tsv(instances))
    return table
