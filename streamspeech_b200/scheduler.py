"""Multi-stream scheduler behind push() / pop(): many SimulEval agents, one engine, one batched streaming step.

The reference runs one agent (= one utterance) per process (agent/speech_to_text.asr.streamspeech.agent.py:385-433); BASELINE
configs[3] is 256 concurrent ASR streams, 32 per GPU.  `StreamPool` owns the engine's stream pool (ss_pool_*): every agent is bound
to a slot, `push()` only registers the new samples, and the first `pop()` after a round of pushes runs ONE ss_pool_step() for all
streams that have pending input (fbank -> chunk-Conformer encoder -> CTC heads over the concatenated rows), after which every agent
of the round finds its result ready.  A harness that feeds the agents round-robin (push all, pop all) -- or calls
`pushpop_many()` -- therefore gets cross-utterance batching without any change to the agent API.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from streamspeech_b200.engine import Engine
from streamspeech_b200.simuleval_compat import ReadAction, SpeechToTextAgent, WriteAction


class StreamPool:
    """sample_rate: the rate of the pushed samples, 16000 or 48000 (the reference agent's default input; decimated to 16 kHz per slot
    inside the batched step, with the single-stream agents' rule and arithmetic)"""

    def __init__(self, engine: Engine, n_slots: int, max_seconds: int = 60, ctc_heads: int = 1, sample_rate: int = 16000):
        self.engine = engine
        self.n_slots = n_slots
        self.ctc_heads = ctc_heads
        self.sample_rate = sample_rate
        engine.pool_create(n_slots, max_seconds, sample_rate)
        self.free: List[int] = list(range(n_slots))[::-1]
        self.pending: Dict[int, bool] = {}       # slot -> has pushed samples since its last step
        self.results: Dict[int, dict] = {}       # slot -> result of the last step that included it
        self.steps = 0                           # batched steps run (for tests / bench)
        self.rows_per_step: List[int] = []

    def acquire(self) -> int:
        if not self.free:
            raise RuntimeError("no free stream slot")
        slot = self.free.pop()
        self.reset(slot)
        return slot

    def release(self, slot: int):
        """give the slot back; it follows the handle's chunk setting again, so whoever acquires it next starts at the default
        latency"""
        self.engine.pool_reset(slot)
        self.engine.pool_set_chunk(slot, 0, 0)
        self.pending.pop(slot, None)
        self.results.pop(slot, None)
        self.free.append(slot)

    def set_chunk(self, slot: int, attn_chunk: int, conv_chunk: int):
        """the slot's own latency (encoder attention chunk, even conv chunk; (0, 0) = follow the engine's set_chunk).  Streams of
        different latencies share every batched step.  Only between utterances (the slot holds no samples); it survives reset()."""
        self.engine.pool_set_chunk(slot, attn_chunk, conv_chunk)

    def reset(self, slot: int):
        self.engine.pool_reset(slot)
        self.pending.pop(slot, None)
        self.results.pop(slot, None)

    def push(self, slot: int, samples: Sequence[float], finished: bool = False):
        """register new source samples of one stream (host -> device copy enqueued, nothing computed yet); finished: the
        stream's source ends with these samples (a 48 kHz stream's last 16 kHz samples are produced by the next step)"""
        if len(samples):
            t = samples if isinstance(samples, torch.Tensor) else torch.tensor(samples, dtype=torch.float32)
            self.engine.pool_push_audio(slot, t.contiguous())
        if finished:
            self.engine.pool_finish(slot)
        self.pending[slot] = True
        self.results.pop(slot, None)

    def flush(self):
        """one batched step for every stream with pending input"""
        slots = sorted(self.pending)
        if not slots:
            return
        res = self.engine.pool_step(slots, self.ctc_heads)
        for s, r in zip(slots, res):
            self.results[s] = r
        self.pending.clear()
        self.steps += 1
        self.rows_per_step.append(len(slots))

    def result(self, slot: int) -> dict:
        if slot not in self.results:
            self.flush()
        return self.results[slot]


class PooledASRAgent(SpeechToTextAgent):
    """StreamSpeechASRAgent (agent/speech_to_text.asr.streamspeech.agent.py:100-433) bound to a slot of a shared StreamPool:
    same push() / pop() / policy() contract and text output; the tensor work of all agents of a round is one batched step.
    Segments must come at the pool's sample rate (ValueError otherwise).  With args, the slot runs at args.source_segment_size
    like the single agent (chunk c = seg // 40, conv chunk min(c, 16), agent:361-375), whatever latency the other slots of the pool
    use; without args it follows the engine's set_chunk."""

    def __init__(self, pool: StreamPool, dictionary, args=None):
        self.pool = pool
        self.dictionary = dictionary
        self.slot = pool.acquire()
        if args is not None and getattr(args, "source_segment_size", None):
            chunk_size = args.source_segment_size // 40
            pool.set_chunk(self.slot, chunk_size, min(chunk_size, 16))  # once: it survives the reset between utterances
        super().__init__(args)
        self.trace = {}

    def reset(self):
        self.asr_text = ""
        self.states.reset()
        if hasattr(self, "slot"):
            self.pool.reset(self.slot)

    def push(self, source_segment, states=None):  # GenericAgent.push (SimulEval agents/agent.py:71-83) + device mirror of the new samples
        if states is None:
            states = self.states
        rate = getattr(source_segment, "sample_rate", -1)  # SpeechSegment's default -1 = not stated: taken as the pool's rate
        if rate > 0 and rate != self.pool.sample_rate:
            raise ValueError(f"a {rate} Hz segment was pushed to a {self.pool.sample_rate} Hz stream pool")
        before = len(states.source)
        states.update_source(source_segment)
        self.pool.push(self.slot, states.source[before:], finished=states.source_finished)

    def policy(self):
        r = self.pool.result(self.slot)
        if r["T"] == 0 and not self.states.source_finished:
            return ReadAction()
        toks = r["ctc"][0][0] if r["T"] > 0 else []
        self.trace = {"asr_tokens": toks}
        text = " ".join(self.dictionary[t] for t in toks)  # :419-425
        new_text = text[len(self.asr_text):]
        self.asr_text = text
        if self.states.source_finished:
            self.states.target_finished = True
            self.reset()
        return WriteAction(new_text, finished=self.states.target_finished)


def pushpop_many(agents: Sequence[PooledASRAgent], segments: Sequence) -> list:
    """the batched front door: push one segment to every agent, then pop all (one batched engine step)"""
    for a, s in zip(agents, segments):
        a.push(s)
    return [a.pop() for a in agents]
