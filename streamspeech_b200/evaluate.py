"""`simuleval` for a whole source list on one engine: the agents of streamspeech_b200/agents/ evaluated with many instances in flight.

    python -m streamspeech_b200.evaluate --agent streamspeech_b200/agents/speech_to_speech.streamspeech.agent.py \\
        --source wav_list.txt --target target.txt --output DIR --source-segment-size 320 --streams 32 \\
        --model-path CKPT --data-bin DATA --vocoder VOCODER --vocoder-cfg VOCODER_CFG --dur-prediction

SimulEval's `SentenceLevelEvaluator.__call__` (SimulEval/simuleval/evaluator/evaluator.py:216-235) plays one instance at a time
through one agent.  Here every stream of a `StreamPool` plays its own instance: each round sends every active instance its next
segment and pops every agent (one batched flush), and an instance that has read its whole source frees its stream for the next
index of the list.  Each stream follows SimulEval's reset rule on its own: its agent is reset once before the first instance and
whenever an instance's prediction finishes, and never between instances otherwise.  With `--streams 1` (the default) the single
agent runs the list in order, without the pool.  The wait-k agents (UnitY checkpoints) have no pooled form and run `--streams 1`
only.

What SimulEval writes is written the same way: `instances.log` (one `summarize()` dict per line, in index order), `config.yaml`,
and for speech output `wavs/{index}_pred.wav`.  The instance classes below restate SimulEval's (evaluator/instance.py); `simuleval`
itself is not imported (its package import needs optional dependencies).  `--computation-aware` is refused: the pooled streams
share each flush, so one stream's compute time is undefined.

Scoring (streamspeech_b200/simuleval_scoring.py): with `--quality-metrics` or `--latency-metrics` the run is scored as SimulEval
scores it (the other flag then takes SimulEval's defaults), writing `scores.tsv` and `metrics.tsv` and printing the results table;
`ASR_BLEU` transcribes `wavs/` on the GPU transcriber (`--asr-model`, `--asr-dict`) after the agents' engine is closed.  A run with
neither flag is not scored (SimulEval would score it with its defaults).  `--score-only --output DIR` scores a finished run from its
`instances.log`, as `simuleval --score-only` does.

`--devices LIST` (streamspeech_b200/workers.py) runs the list on one worker process per entry, each with `--streams` agents on its own
engine on that device; the workers write the waveforms, and this process writes `config.yaml` and `instances.log` in index order and
scores the run (ASR_BLEU transcribed on the same devices).  Every file is the one the single-process run writes.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import struct
import sys
import time
from pathlib import Path
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _REPO not in sys.path:
    sys.path.insert(0, _REPO)

from streamspeech_b200 import simuleval_scoring as scoring  # noqa: E402
from streamspeech_b200 import workers  # noqa: E402
from streamspeech_b200.simuleval_compat import EmptySegment, SpeechSegment  # noqa: E402

# --agent file name -> (target type, single agent class name, pooled agent class name)
AGENTS = {
    "speech_to_speech.streamspeech.agent.py": ("speech", "StreamSpeechS2STAgent", "PooledS2STAgent"),
    "speech_to_text.s2tt.streamspeech.agent.py": ("text", "StreamSpeechS2TTAgent", "PooledS2TTAgent"),
    "speech_to_text.asr.streamspeech.agent.py": ("text", "StreamSpeechASRAgent", "PooledASRAgent"),
    # the wait-k-stride-n baselines on UnitY checkpoints (streamspeech_b200/waitk.py): one stream, no pooled class
    "speech_to_speech.wait-k-stride-n.agent.py": ("speech", "WaitkS2STAgent", None),
    "speech_to_text.wait-k-stride-n.agent.py": ("text", "WaitkS2TTAgent", None),
}


# ----------------------------------------------------------------------------------------------------------------------- WAV input

_WAVE_FORMAT_PCM, _WAVE_FORMAT_FLOAT, _WAVE_FORMAT_EXTENSIBLE = 1, 3, 0xFFFE


class AudioInfo:
    """What SimulEval reads from `soundfile.info(path)`: the sample rate, and the text of its repr (soundfile's _SoundFileInfo, not
    verbose), which a text-output instance logs as its "source"."""

    def __init__(self, path: str, samplerate: int, frames: int, subtype: str):
        self.name, self.samplerate, self.frames, self.subtype = path, samplerate, frames, subtype

    def _duration_str(self) -> str:
        hours, rest = divmod(self.frames, self.samplerate * 3600)
        minutes, rest = divmod(rest, self.samplerate * 60)
        seconds = rest / self.samplerate
        if hours:
            return "{0:.0g}:{1:02.0g}:{2:05.3f} h".format(hours, minutes, seconds)
        if minutes:
            return "{0:02.0g}:{1:05.3f} min".format(minutes, seconds)
        if seconds:
            return "{0:.3f} s".format(seconds)
        return "{0} samples".format(self.frames)

    def __str__(self) -> str:
        subtype_info = {"PCM_16": "Signed 16 bit PCM", "FLOAT": "32 bit float"}[self.subtype]
        return "\n".join([self.name, f"samplerate: {self.samplerate} Hz", "channels: 1", f"duration: {self._duration_str()}",
                          "format: WAV (Microsoft) [WAV]", f"subtype: {subtype_info} [{self.subtype}]"])


def read_wav(path: str, header_only: bool = False):
    """A mono PCM16 or float32 WAV file -> (samples as float32 in [-1, 1), AudioInfo); PCM16 is scaled by 1 / 32768, as
    soundfile.read(dtype="float32") does.  header_only: samples is None.  Anything else is refused with a ValueError that names the
    file."""
    with open(path, "rb") as f:
        head = f.read(12)
        if head[:3] == b"ID3" or (len(head) >= 2 and head[0] == 0xFF and head[1] & 0xE0 == 0xE0) or path.lower().endswith(".mp3"):
            raise ValueError(f"{path}: mp3 sources are not supported; convert them to 16-bit PCM or float32 WAV")
        if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
            raise ValueError(f"{path}: not a RIFF/WAVE file")
        fmt = None
        while True:
            ch = f.read(8)
            if len(ch) < 8:
                raise ValueError(f"{path}: no data chunk")
            cid, size = ch[:4], struct.unpack("<I", ch[4:])[0]
            if cid == b"fmt ":
                body = f.read(size + (size & 1))
                tag, channels, rate, _, _, bits = struct.unpack("<HHIIHH", body[:16])
                if tag == _WAVE_FORMAT_EXTENSIBLE and size >= 26:
                    tag = struct.unpack("<H", body[24:26])[0]  # first two bytes of the sub-format GUID
                fmt = (tag, channels, rate, bits)
            elif cid == b"data":
                if fmt is None:
                    raise ValueError(f"{path}: data chunk before the fmt chunk")
                tag, channels, rate, bits = fmt
                if channels != 1:
                    raise ValueError(f"{path}: {channels} channels; the agents take mono sources")
                if (tag, bits) == (_WAVE_FORMAT_PCM, 16):
                    dtype, subtype = "<i2", "PCM_16"
                elif (tag, bits) == (_WAVE_FORMAT_FLOAT, 32):
                    dtype, subtype = "<f4", "FLOAT"
                else:
                    raise ValueError(f"{path}: WAV format {tag} with {bits}-bit samples; only 16-bit PCM and 32-bit float are read")
                frames = size // np.dtype(dtype).itemsize
                info = AudioInfo(path, rate, frames, subtype)
                if header_only:
                    return None, info
                x = np.frombuffer(f.read(size), dtype=dtype)[:frames]
                if len(x) < frames:
                    raise ValueError(f"{path}: data chunk is truncated")
                x = x.astype(np.float32) / np.float32(32768.0) if subtype == "PCM_16" else x.astype(np.float32)
                return x, info
            else:
                f.seek(size + (size & 1), 1)


def read_lines(path: str) -> List[str]:
    """SimulEval's dataloader: one stripped line per instance"""
    with open(path) as f:
        return [line.strip() for line in f]


# ------------------------------------------------------------------------------------------------------------- instance bookkeeping

class SpeechInstance:
    """SimulEval's Instance + SpeechInputInstance (evaluator/instance.py:26-151, 231-320): the source segments and the delay of
    each prediction.  `clock` is time.time (a test can replace it)."""

    def __init__(self, index: int, samples: Sequence[float], info: AudioInfo, source_path: str, reference: str,
                 latency_unit: str = "word", clock: Callable[[], float] = time.time):
        self.index = index
        self.finish_prediction = False
        self.samples = samples
        self.info = info
        self.sample_rate = info.samplerate
        self.source_path = source_path
        self.reference = reference
        self.latency_unit = latency_unit
        self.clock = clock
        self.step = 0
        self.elapsed: List[float] = []
        self.prediction_list: list = []
        self.delays: List[float] = []
        self.start_time = None
        self.metrics: dict = {}
        self.source_finished_reading = False

    def send_source(self, segment_size: int):
        if self.step == 0:
            self.start_time = self.clock()
        assert segment_size >= 1, "instance size has to larger than 1 ms"
        num_samples = math.ceil(segment_size / 1000 * self.sample_rate)
        if self.step < len(self.samples):
            if self.step + num_samples >= len(self.samples):
                samples = self.samples[self.step:]
                is_finished = True
                self.source_finished_reading = True
            else:
                samples = self.samples[self.step:self.step + num_samples]
                is_finished = False
            self.step = min(self.step + num_samples, len(self.samples))
            return SpeechSegment(index=self.len_sample_to_ms(self.step), content=list(samples), sample_rate=self.sample_rate,
                                 finished=is_finished)
        self.source_finished_reading = True
        return EmptySegment(index=self.len_sample_to_ms(self.step), finished=True)

    @property
    def source_length(self) -> float:
        return self.len_sample_to_ms(len(self.samples))

    def len_sample_to_ms(self, length: int) -> float:
        return length * 1000 / self.sample_rate

    def step_to_delay(self, step) -> float:
        return self.len_sample_to_ms(self.step)

    def step_to_elapsed(self, step, current_time) -> float:
        return self.len_sample_to_ms(step) + (current_time - self.start_time) * 1000


class SpeechToTextInstance(SpeechInstance):
    """+ TextOutputInstance (instance.py:178-230)"""

    def receive_prediction(self, prediction):
        if self.finish_prediction or prediction.is_empty:
            self.finish_prediction = prediction.finished
            return
        if self.start_time is None:
            self.start_time = self.clock()
        self.finish_prediction = prediction.finished
        if len(prediction.content) == 0:
            return
        current_time = self.clock()
        if self.latency_unit == "word":
            prediction_list = prediction.content.strip().split()
        elif self.latency_unit == "char":
            prediction_list = list(prediction.content.replace(" ", ""))
        else:
            raise NotImplementedError(self.latency_unit)
        self.prediction_list += prediction_list
        self.elapsed += [self.step_to_elapsed(self.step, current_time)] * len(prediction_list)
        self.delays += [self.step_to_delay(self.step)] * len(prediction_list)

    @property
    def prediction(self) -> str:
        if self.latency_unit == "word":
            return "".join(self.prediction_list).replace("▁", " ")
        return "".join(self.prediction_list).replace("▁", "")

    def summarize(self) -> dict:
        return {"index": self.index, "prediction": self.prediction, "delays": self.delays, "elapsed": self.elapsed,
                "prediction_length": len(self.prediction_list), "reference": self.reference, "source": str(self.info).split("\n"),
                "source_length": self.source_length, "metric": self.metrics}


class SpeechToSpeechInstance(SpeechInstance):
    """+ SpeechOutputInstance (instance.py:322-420).  wav_path: where summarize() writes the waveform."""

    def __init__(self, *a, wav_path: Path, **kw):
        super().__init__(*a, **kw)
        self.wav_path = wav_path
        self.durations: List[float] = []
        self.intervals: list = []
        self.target_sample_rate = -1

    def receive_prediction(self, segment):
        if self.start_time is None:
            self.start_time = self.clock()
        if self.finish_prediction and self.source_finished_reading:
            return
        self.finish_prediction = segment.finished
        if segment.is_empty or len(segment.content) == 0:
            return
        current_time = self.clock()
        pred_duration = 1000 * len(segment.content) / segment.sample_rate
        if self.target_sample_rate < 0:
            self.target_sample_rate = segment.sample_rate
        self.durations.append(pred_duration)
        self.prediction_list.append(segment.content)
        self.elapsed.append(self.step_to_elapsed(self.step, current_time))
        self.delays.append(self.step_to_delay(self.step))

    def waveform(self):
        """(the written samples: each prediction at its delay, silence where it waits for the source; prediction_offset).  Sets
        intervals ([start, duration] per prediction) and silences (the length of each wait), as SimulEval's summarize() does."""
        samples: List[float] = []
        self.intervals = []
        self.silences: List[float] = []
        if not self.prediction_list:
            return samples, self.source_length
        start = prev_end = prediction_offset = self.delays[0]
        for i, delay in enumerate(self.delays):
            start = max(prev_end, delay)
            if start > prev_end:
                samples += [0.0] * int(self.target_sample_rate * (start - prev_end) / 1000)
                self.silences.append(start - prev_end)
            samples += self.prediction_list[i]
            prev_end = start + self.durations[i]
            self.intervals.append([start, self.durations[i]])
        return samples, prediction_offset

    def summarize(self) -> dict:
        from streamspeech_b200.generate_waveform_from_code import write_wav

        samples, prediction_offset = self.waveform()
        if self.prediction_list:
            write_wav(str(self.wav_path), np.asarray(samples, dtype=np.float32), self.target_sample_rate)
        return {"index": self.index, "prediction": Path(self.wav_path).as_posix(),
                "delays": self.delays, "durations": self.durations, "prediction_offset": prediction_offset, "elapsed": [],
                "intervals": self.intervals, "prediction_length": len(samples) / self.target_sample_rate,
                "source_length": self.source_length, "reference": self.reference, "source": self.source_path}


# ------------------------------------------------------------------------------------------------------------------------ arguments

def _add_evaluator_args(parser: argparse.ArgumentParser):
    """SimulEval's flags (options.py, dataloader.py) that a run of a speech source list needs, and its scoring flags"""
    parser.add_argument("--agent", required=True, help="one of the agent files under streamspeech_b200/agents/ (matched by file name)")
    parser.add_argument("--source", required=True, help="list of source WAV files, one per line")
    parser.add_argument("--target", required=True, help="list of references, one per line")
    parser.add_argument("--output", required=True, help="output directory")
    parser.add_argument("--source-segment-size", type=int, default=1, help="source segment size in ms")
    parser.add_argument("--start-index", type=int, default=0)
    parser.add_argument("--end-index", type=int, default=-1)
    parser.add_argument("--eval-latency-unit", type=str, default="word", choices=["word", "char"])
    parser.add_argument("--streams", type=int, default=1,
                        help="instances in flight; above 1 they share one stream pool, 1 runs the single agent")
    parser.add_argument("--computation-aware", action="store_true", default=False, help="refused (see --help of this module)")
    workers.add_devices_arg(parser)
    _add_scoring_args(parser)
    parser.add_argument("--device", type=str, default="gpu", help="accepted and ignored: the engine runs on --device-index")


def _add_scoring_args(parser: argparse.ArgumentParser):
    """SimulEval's scoring flags, and the ASR_BLEU transcriber's (those of the asr_bleu front door)"""
    parser.add_argument("--quality-metrics", nargs="+", default=None,
                        help=f"any of {list(scoring.QUALITY_METRICS)}; given alone, the latency metrics default to SimulEval's "
                             f"{scoring.DEFAULT_LATENCY}; neither flag: the run is not scored")
    parser.add_argument("--latency-metrics", nargs="+", default=None,
                        help=f"any of {list(scoring.LATENCY_METRICS)}; given alone, the quality metrics default to "
                             f"{scoring.DEFAULT_QUALITY}")
    parser.add_argument("--sacrebleu-tokenizer", type=str, default="13a", help="only 13a is offered")
    parser.add_argument("--no-use-ref-len", action="store_true", default=False,
                        help="latency metrics take the prediction's length, not the reference's, as the target length")
    parser.add_argument("--target-speech-lang", type=str, default="en", help="the language of the target speech (ASR_BLEU); only en")
    parser.add_argument("--asr-model", default=None, help="ASR_BLEU: local path of the fairseq wav2vec 2.0 CTC checkpoint (or "
                                                          "'synthetic': the seeded test model)")
    parser.add_argument("--asr-dict", default=None, help="ASR_BLEU: local path of dict.ltr.txt")
    parser.add_argument("--asr-setting", action="append", default=[], metavar="KEY=VALUE",
                        help="ASR_BLEU: override a transcriber setting read from the checkpoint (see python -m streamspeech_b200.asr_bleu)")


def agent_kind(agent_path: str):
    name = os.path.basename(agent_path)
    if name not in AGENTS:
        raise SystemExit(f"--agent {agent_path}: not one of the agent files {sorted(AGENTS)}")
    return AGENTS[name]


def single_agent_class(name: str):
    """the single-stream agent class of that name: streamspeech_b200.agent's, or the wait-k agents of streamspeech_b200.waitk"""
    from streamspeech_b200 import agent as _agents
    from streamspeech_b200 import waitk as _waitk

    return getattr(_agents, name) if hasattr(_agents, name) else getattr(_waitk, name)


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    pre = argparse.ArgumentParser(add_help=False)
    pre.add_argument("--agent")
    known, _ = pre.parse_known_args(argv)
    parser = argparse.ArgumentParser(prog="python -m streamspeech_b200.evaluate", description=__doc__,
                                     formatter_class=argparse.RawDescriptionHelpFormatter)
    _add_evaluator_args(parser)
    if known.agent is not None:
        target_type, single_name, _ = agent_kind(known.agent)
        single_agent_class(single_name).add_args(parser)
        if target_type == "text":  # the text agents share the S2ST agent's flags; the reference's text agents take no vocoder
            for action in parser._actions:
                if action.dest in ("vocoder", "vocoder_cfg"):
                    action.required = False
    args = workers.parse_with_devices(parser, argv, "--device-index")
    if args.computation_aware:
        parser.error("--computation-aware is not offered: pooled streams share every batched step, so a per-stream compute time "
                     "is undefined; the non-computation-aware latency metrics are scored from instances.log")
    if args.streams < 1:
        parser.error("--streams must be at least 1")
    if args.streams > 1 and agent_kind(args.agent)[2] is None:
        parser.error(f"--streams {args.streams}: the wait-k agent {os.path.basename(args.agent)} runs one stream (pass --streams 1)")
    return args


def get_indices(start_index: int, end_index: int, n_instances: int) -> range:
    """SentenceLevelEvaluator.get_indices (evaluator.py:181-189) with end_index < 0 read as the list's length (:113-115)"""
    if end_index < 0:
        end_index = n_instances
    return range(start_index, end_index)


# --------------------------------------------------------------------------------------------------------------------------- runner

class Evaluation:
    """One run: the agents (one per stream), the instances in flight, and the log written in index order."""

    def __init__(self, args: argparse.Namespace, agents: Sequence, target_type: str):
        self.args = args
        self.agents = list(agents)
        self.target_type = target_type
        self.output = Path(args.output)
        self.sources = read_lines(args.source)
        self.targets = read_lines(args.target)
        self.indices = get_indices(args.start_index, args.end_index, len(self.sources))
        self.infos: Dict[int, AudioInfo] = {}
        for i in self.indices:
            if i >= len(self.sources) or i >= len(self.targets):
                raise SystemExit(f"index {i} is past the end of --source ({len(self.sources)} lines) or --target ({len(self.targets)} lines)")
            self.infos[i] = check_source(self.sources[i], args.sample_rate)
        self.source_seconds = sum(info.frames / info.samplerate for info in self.infos.values())
        self.max_in_flight = 0
        # index -> what the scorers read from the finished instance (not its samples), in index order whatever order the streams
        # finish in; None: the run is not scored
        self.kept: Optional[Dict[int, scoring.ScoredInstance]] = None
        self.scores: Optional[Dict[str, object]] = None

    def _instance(self, index: int):
        samples, info = read_wav(self.sources[index])
        common = dict(info=info, source_path=self.sources[index], reference=self.targets[index], latency_unit=self.args.eval_latency_unit)
        if self.target_type == "speech":
            return SpeechToSpeechInstance(index, samples.tolist(), wav_path=(self.output / "wavs" / f"{index}_pred.wav").absolute(), **common)
        return SpeechToTextInstance(index, samples.tolist(), **common)

    def _open_output(self):
        self.output.mkdir(parents=True, exist_ok=True)
        if self.target_type == "speech":
            (self.output / "wavs").mkdir(exist_ok=True)
        with open(self.output / "config.yaml", "w") as f:  # evaluator.py:86-93, target_type written as the source type as there
            f.write("source_type: speech\ntarget_type: speech\n")
        return open(self.output / "instances.log", "w")

    def _write(self, log, index: int, line: str, kept: Optional["scoring.ScoredInstance"]):
        log.write(line + "\n")
        if self.kept is not None:  # in index order, as SimulEval scores and as the log lists them
            self.kept[index] = kept

    def play(self, next_index: Callable[[], Optional[int]], finished: Callable[[int, str, Optional["scoring.ScoredInstance"]], None]):
        """Play the instances next_index() returns (None: no more) on the agents, and call finished(index, log line, what the
        scorers read or None) for each as it finishes, in the order the streams finish them"""
        from streamspeech_b200.scheduler import pushpop_many

        active: Dict[int, object] = {}  # stream -> its instance
        for a in self.agents:
            a.reset()

        def admit(stream):
            i = next_index()
            if i is not None:
                active[stream] = self._instance(i)

        for j in range(len(self.agents)):
            admit(j)
        seg_ms = self.args.source_segment_size
        while active:
            self.max_in_flight = max(self.max_in_flight, len(active))
            streams = sorted(active)
            segments = [active[j].send_source(seg_ms) for j in streams]
            outputs = pushpop_many([self.agents[j] for j in streams], segments)
            for j, out in zip(streams, outputs):
                inst = active[j]
                inst.receive_prediction(out)
                if inst.finish_prediction:  # evaluator.py:224-229
                    self.agents[j].reset()
                if inst.source_finished_reading:
                    summary = inst.summarize()
                    kept = None
                    if self.kept is not None:
                        kept = scoring.live_instance(summary, self.args.eval_latency_unit, getattr(inst, "silences", None))
                    finished(inst.index, json.dumps(summary), kept)
                    del active[j]
                    admit(j)

    def run(self):
        log = self._open_output()
        queue = iter(self.indices)
        done: Dict[int, tuple] = {}  # index -> (its log line, what the scorers read), until every smaller index has been written
        next_to_write = [self.indices.start]

        def finished(index, line, kept):
            done[index] = (line, kept)
            while next_to_write[0] in done:
                self._write(log, next_to_write[0], *done.pop(next_to_write[0]))
                next_to_write[0] += 1

        try:
            self.play(lambda: next(queue, None), finished)
        finally:
            log.close()

    def run_devices(self, devices: Sequence[int], max_seconds: int):
        """run() with the instances spread over one worker process per entry of devices, each with --streams agents of its own on
        its own engine; the workers write the waveforms, the log is written here in index order"""
        from contextlib import closing

        from streamspeech_b200 import workers

        log = self._open_output()
        try:
            with closing(workers.run(devices, _evaluate_job, (self.args, self.target_type, self.kept is not None, max_seconds),
                                     [(i, None) for i in self.indices])) as results:
                for index, (line, kept) in results:
                    self._write(log, index, line, kept)
        finally:
            log.close()


def _evaluate_job(device: int, payload, next_item, emit):
    """one --devices worker: the agents of build_agents on `device`, playing the indices of the shared queue"""
    import copy

    args, target_type, scored, max_seconds = payload
    args = copy.copy(args)
    args.device_index = device
    agents, pool, _ = build_agents(args, max_seconds=max_seconds)
    ev = Evaluation(args, agents, target_type)
    ev.kept = {} if scored else None

    def next_index():
        item = next_item()
        return None if item is None else item[0]

    try:
        ev.play(next_index, lambda index, line, kept: emit(index, (line, kept)))
    finally:
        (pool.engine if pool is not None else agents[0].engine).close()


def check_source(path: str, sample_rate: int) -> AudioInfo:
    _, info = read_wav(path, header_only=True)
    if info.samplerate != sample_rate:
        raise ValueError(f"{path}: {info.samplerate} Hz source, but the agent runs at --sample-rate {sample_rate}")
    return info


def build_agents(args: argparse.Namespace, max_seconds: int = 60):
    """(agents, pool, target type): `args.streams` pooled agents on one StreamPool of the engine the single agent loads, or the
    single agent alone for one stream (the pool step is slower for one stream: it does not use the single-stream encoder kernels)"""
    from streamspeech_b200 import scheduler

    target_type, single_name, pooled_name = agent_kind(args.agent)
    single = single_agent_class(single_name)(args)
    if args.streams == 1:
        return [single], None, target_type
    ctc_heads = 1 if pooled_name == "PooledASRAgent" else 2
    pool = scheduler.StreamPool(single.engine, args.streams, max_seconds=max_seconds, ctc_heads=ctc_heads, sample_rate=args.sample_rate)
    cls = getattr(scheduler, pooled_name)
    if pooled_name == "PooledASRAgent":
        agents = [cls(pool, single.dict["source_unigram"], args) for _ in range(args.streams)]
    elif pooled_name == "PooledS2TTAgent":
        agents = [cls(pool, single.dict["target_unigram"], args) for _ in range(args.streams)]
    else:
        agents = [cls(pool, single.dict, args) for _ in range(args.streams)]
    return agents, pool, target_type


def parse_score_only_args(argv: Sequence[str]) -> argparse.Namespace:
    """`--score-only --output DIR` and the scoring flags; --agent, --source and --target are not required (and are ignored)"""
    parser = argparse.ArgumentParser(prog="python -m streamspeech_b200.evaluate --score-only",
                                     description="score the run in --output from its instances.log, as `simuleval --score-only` does")
    parser.add_argument("--score-only", action="store_true", required=True)
    parser.add_argument("--output", required=True, help="the output directory of a run")
    for flag in ("--agent", "--source", "--target"):
        parser.add_argument(flag, default=None, help="accepted and ignored")
    parser.add_argument("--eval-latency-unit", type=str, default="word", choices=["word", "char"],
                        help="accepted and ignored: SimulEval's LogInstance counts reference words whatever the unit")
    parser.add_argument("--computation-aware", action="store_true", default=False, help="refused")
    parser.add_argument("--device-index", type=int, default=0, help="CUDA device of the ASR_BLEU transcriber")
    workers.add_devices_arg(parser)
    _add_scoring_args(parser)
    parser.add_argument("--device", type=str, default="gpu", help="accepted and ignored")
    args = workers.parse_with_devices(parser, argv, "--device-index")
    if args.computation_aware:
        parser.error("--computation-aware is not offered: the computation-aware metrics are not scored")
    return args


def _transcriber_factory(args: argparse.Namespace):
    def make():
        from streamspeech_b200.asr import ASRTranscriber, parse_settings

        if getattr(args, "devices", None) is not None:
            from streamspeech_b200.asr_bleu import DeviceTranscribers

            return DeviceTranscribers(args.devices, args.asr_model, args.asr_dict, parse_settings(args.asr_setting))
        return ASRTranscriber(args.asr_model, args.asr_dict, getattr(args, "device_index", 0), settings=parse_settings(args.asr_setting))

    return make


def _check_scoring(args: argparse.Namespace, metrics, speech_output: Optional[bool], score_only: bool, n_instances: Optional[int]):
    quality, latency = metrics
    scoring.check_request(quality, latency, tokenizer=args.sacrebleu_tokenizer, target_speech_lang=args.target_speech_lang,
                          speech_output=speech_output, score_only=score_only, asr_model=args.asr_model, n_instances=n_instances)
    if args.asr_model is not None and "ASR_BLEU" in quality:
        from streamspeech_b200.asr import parse_settings

        try:
            parse_settings(args.asr_setting)
        except ValueError as e:
            raise SystemExit(str(e)) from None


def score_run(args: argparse.Namespace, instances: Dict[int, "scoring.ScoredInstance"], metrics) -> Dict[str, object]:
    """score the instances, write scores.tsv and metrics.tsv into --output and print the results table"""
    quality, latency = metrics
    scores = scoring.score(instances, quality, latency, use_ref_len=not args.no_use_ref_len, make_transcriber=_transcriber_factory(args))
    scoring.dump(Path(args.output), instances, scores)
    return scores


def score_only(argv: Sequence[str]) -> Dict[str, object]:
    args = parse_score_only_args(argv)
    metrics = scoring.metric_lists(args.quality_metrics, args.latency_metrics) or (scoring.DEFAULT_QUALITY, scoring.DEFAULT_LATENCY)
    _check_scoring(args, metrics, None, True, None)
    instances = scoring.read_log(Path(args.output))
    _check_scoring(args, metrics, None, True, len(instances))
    if "ASR_BLEU" in metrics[0] and instances and not str(next(iter(instances.values())).prediction).endswith("_pred.wav"):
        raise SystemExit("--quality-metrics ASR_BLEU needs speech output; the run in --output wrote text")
    return score_run(args, instances, metrics)


def main(argv: Optional[Sequence[str]] = None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if "--score-only" in argv:
        return score_only(argv)
    args = parse_args(argv)
    target_type = agent_kind(args.agent)[0]
    metrics = scoring.metric_lists(args.quality_metrics, args.latency_metrics)
    if metrics is not None:  # refused before the model is loaded, so a long run does not fail at its end
        _check_scoring(args, metrics, target_type == "speech", False, None)
    ev = Evaluation(args, [], target_type)  # sources checked before the model is loaded
    if metrics is not None:
        _check_scoring(args, metrics, target_type == "speech", False, len(ev.indices))
        ev.kept = {}
    longest = max((info.frames / info.samplerate for info in ev.infos.values()), default=1.0)
    if args.devices is not None:  # the workers build the agents, each on its own device
        t0 = time.perf_counter()
        ev.run_devices(args.devices, max_seconds=math.ceil(longest) + 1)
    else:
        agents, pool, _ = build_agents(args, max_seconds=math.ceil(longest) + 1)
        ev.agents = agents
        t0 = time.perf_counter()
        ev.run()
    seconds = time.perf_counter() - t0
    line = {"instances": len(ev.indices), "streams": args.streams}
    if args.devices is not None:  # streams is per worker; wall_seconds includes the workers' start-up and engine builds
        line["devices"] = ",".join(map(str, args.devices))
    line.update(source_seconds=round(ev.source_seconds, 3), wall_seconds=round(seconds, 3),
                audio_s_per_s=round(ev.source_seconds / max(seconds, 1e-9), 2), output=str(ev.output))
    if metrics is None:
        print(json.dumps(line))
    if args.devices is None:
        engine = pool.engine if pool is not None else agents[0].engine
        engine.close()
    if metrics is not None:  # after the engine is closed: the transcriber never shares the device with it
        t1 = time.perf_counter()
        ev.scores = score_run(args, ev.kept, metrics)
        line["scoring_seconds"] = round(time.perf_counter() - t1, 3)
        print(json.dumps(line))
    return ev


if __name__ == "__main__":
    main()
