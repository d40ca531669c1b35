"""Multi-stream scheduler behind push() / pop(): many SimulEval agents, one engine, one batched streaming step.

The reference runs one agent (= one utterance) per process (agent/speech_to_text.asr.streamspeech.agent.py:385-433); BASELINE
configs[3] is 256 concurrent ASR streams, 32 per GPU.  `StreamPool` owns the engine's stream pool (ss_pool_*): every agent is bound
to a slot, `push()` only registers the new samples, and the first `pop()` after a round of pushes runs ONE ss_pool_step() for all
streams that have pending input (fbank -> chunk-Conformer encoder -> CTC heads over the concatenated rows), after which every agent
of the round finds its result ready.  A harness that feeds the agents round-robin (push all, pop all) -- or calls
`pushpop_many()` -- therefore gets cross-utterance batching without any change to the agent API.

`PooledS2STAgent` extends this to simultaneous speech-to-speech translation: the flush that serves its streams also runs ONE batched
MT search (ss_pool_mt_greedy) for every stream whose policy gate says WRITE and ONE T2U + unit-decoder call
(ss_t2u_unit_decode_ragged) for every stream that still has something to say, then ONE vocoder durations call and ONE generate call
(ss_vocoder_durations_ragged / ss_vocoder_generate_ragged) for every stream that has new units.  The host stages around those calls
are the single agent's own methods (StreamSpeechS2STAgent._gate / _after_mt / _before_vocoder / _after_vocoder).

`PooledS2TTAgent` does the same for simultaneous speech-to-text translation: ONE incremental MT search
(ss_pool_mt_greedy_incremental) for every writing stream, each on its slot's own incremental decoder state, between the single
agent's host stages (StreamSpeechS2TTAgent._gate / _after_mt).  S2ST and S2TT agents can share one pool: a flush runs the decode
round of each kind for its own streams.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from streamspeech_b200.agent import READ, SAMPLE_RATE, StreamSpeechS2STAgent, StreamSpeechS2TTAgent
from streamspeech_b200.engine import Engine
from streamspeech_b200.simuleval_compat import ReadAction, SpeechToSpeechAgent, SpeechToTextAgent, WriteAction


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
        self.decoders: Dict[int, "_PooledDecoder"] = {}  # slot -> its S2ST / S2TT agent: a flush also runs the decoders of these slots
        self.stage_ms: Optional[Dict[str, float]] = None  # a dict: device time per stage of every flush is added to it (CUDA events)

    @property
    def s2st(self) -> Dict[int, "PooledS2STAgent"]:
        """the S2ST agents among the decoding agents, by slot"""
        return {s: a for s, a in self.decoders.items() if isinstance(a, PooledS2STAgent)}

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
        self.decoders.pop(slot, None)
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
        """one batched step for every stream with pending input, then the decode round of its S2ST streams and that of its S2TT
        streams"""
        slots = sorted(self.pending)
        if not slots:
            return
        clock = _StageClock(self.stage_ms)
        clock.mark("pool_step")
        res = self.engine.pool_step(slots, self.ctc_heads)
        for s, r in zip(slots, res):
            self.results[s] = r
        self.pending.clear()
        self.steps += 1
        self.rows_per_step.append(len(slots))
        rounds: Dict[type, list] = {}  # agent class -> its agents of this flush, in slot order
        for s in slots:
            if s in self.decoders:
                rounds.setdefault(type(self.decoders[s]), []).append(self.decoders[s])
        for kind, agents in rounds.items():
            kind.decode_round(self, agents, clock)
        clock.close()

    def result(self, slot: int) -> dict:
        if slot not in self.results:
            self.flush()
        return self.results[slot]


class _StageClock:
    """CUDA events on the current stream at stage boundaries; close() adds each stage's time to `into` (nothing without a dict)"""

    def __init__(self, into: Optional[Dict[str, float]]):
        self.into = into
        self.events = []

    def mark(self, name: str):
        if self.into is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.events.append((name, ev))

    def close(self):
        if self.into is None or not self.events:
            return
        self.mark("")
        self.events[-1][1].synchronize()
        for (name, e0), (_, e1) in zip(self.events, self.events[1:]):
            self.into[name] = self.into.get(name, 0.0) + e0.elapsed_time(e1)
        self.events = []


class _PooledSource:
    """push() of a pooled agent: the segment's samples go to the agent's slot (they must come at the pool's sample rate)"""

    def push(self, source_segment, states=None):  # GenericAgent.push (SimulEval agents/agent.py:71-83) + device mirror of the new samples
        if states is None:
            states = self.states
        rate = getattr(source_segment, "sample_rate", -1)  # SpeechSegment's default -1 = not stated: taken as the pool's rate
        if rate > 0 and rate != self.pool.sample_rate:
            raise ValueError(f"a {rate} Hz segment was pushed to a {self.pool.sample_rate} Hz stream pool")
        before = len(states.source)
        states.update_source(source_segment)
        self.pool.push(self.slot, states.source[before:], finished=states.source_finished)


class PooledASRAgent(_PooledSource, SpeechToTextAgent):
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


class _PooledDecoder(_PooledSource):
    """an agent whose policy() result is computed by its pool's flush (decode_round of its class) and kept until it is asked for"""

    def _policy_impl(self):
        if self._action is None:
            self.pool.flush()  # this agent's segment is pending: the round computes the action of every pending agent
        action, self._action = self._action, None
        if action is None:
            raise RuntimeError("policy() of a pooled agent needs a pushed segment first")
        return action


class PooledS2STAgent(_PooledDecoder, StreamSpeechS2STAgent):
    """StreamSpeechS2STAgent (agent/speech_to_speech.streamspeech.agent.py:101-770) bound to a slot of a shared StreamPool: same
    push() / pop() / policy() contract and WriteAction(SpeechSegment) output, the same policy code (the single agent's host stages),
    but the tensor work of all agents of a round runs as one pool step, one batched MT search and one T2U + unit-decoder call.
    The pool needs both CTC heads (StreamPool(..., ctc_heads=2)).  The slot takes the S2ST agent's latency rule: chunk c =
    source_segment_size // 40, conv chunk 16 if c >= 16 else 8 (agent:406-413); whole-word output at >= 640 ms (agent:207-210).
    args: the single agent's flags (lagging_k1, stride_n, dur_prediction, vocoder_context, ...); the model comes from the pool's
    engine and `dicts` (the single agent's `dict`: "target_unigram" and "tgt" are read)."""

    def __init__(self, pool: StreamPool, dicts, args):
        if pool.ctc_heads != 2:
            raise ValueError("a pooled S2ST agent needs a stream pool with both CTC heads (ctc_heads=2)")
        self.pool = pool
        self.engine = pool.engine
        self.cfg = pool.engine.cfg
        self.torch_device = pool.engine.device
        self.dict = dicts
        self.eos = self.cfg.eos
        self.max_len = args.max_len
        self.force_finish = args.force_finish
        self.dur_prediction = args.dur_prediction
        self.lagging_k1 = args.lagging_k1
        self.lagging_k2 = args.lagging_k2
        self.segment_size = args.segment_size
        self.stride_n = args.stride_n
        self.unit_per_subword = args.unit_per_subword
        self.stride_n2 = args.stride_n2
        self.whole_word = args.source_segment_size >= 640  # agent:207-210
        self.vocoder_context = getattr(args, "vocoder_context", "receptive-field")
        self.trace = {}
        self._action = None
        self.slot = pool.acquire()
        chunk_size = args.source_segment_size // 40  # agent:395-413
        pool.set_chunk(self.slot, chunk_size, 16 if chunk_size >= 16 else 8)  # once: it survives the reset between utterances
        pool.decoders[self.slot] = self
        SpeechToSpeechAgent.__init__(self, args)  # states + reset()

    def _reset_caches(self):
        """new utterance: the slot starts over (audio, encoder state, cross K / V cache)"""
        if hasattr(self, "slot"):
            self.pool.reset(self.slot)
        self._action = None

    @staticmethod
    @torch.inference_mode()
    def decode_round(pool: StreamPool, agents: Sequence["PooledS2STAgent"], clock: _StageClock):
        """Stages 2-7 of a flush for the agents whose slots the pool step just ran: the gate per stream, one batched MT search for
        the writing streams, the post-MT checks per stream, teacher-forced features for finishing whole-word streams (once per
        utterance, N2 pad tail), one T2U + unit-decoder call for every stream that goes on, then one vocoder call (durations, one host
        read of the cumsums, generate) for every stream with new units."""
        eng = pool.engine
        writing = []
        for a in agents:
            a.trace = {}
            r = pool.results[a.slot]
            if r["T"] == 0:  # no encoder row yet (fewer samples than one fbank frame)
                a._action = READ
                continue
            (src, _), (tgt, _) = r["ctc"]  # agent:437, 461
            a.trace["asr_tokens"], a.trace["st_tokens"] = src, tgt
            new = a._gate(src, tgt)
            if new is None:
                a._action = READ
            else:
                writing.append((a, new, r["T"]))
        if not writing:
            return
        clock.mark("mt")
        hyps, feats = eng.pool_mt_greedy([a.slot for a, _, _ in writing], [a.tgt_subwords_indices for a, _, _ in writing],
                                         [new for _, new, _ in writing], max_len_b=100)
        going = []  # (agent, new_subword_tokens, T, row of feats, prev_output_tokens_mt, n_pad_tail)
        for k, (a, new, T) in enumerate(writing):
            action, t2u_input = a._after_mt(hyps[k])
            if action is not None:
                a._action = action
            else:
                going.append((a, new, T, k) + t2u_input)
        if not going:
            return
        lengths = [len(g[4]) for g in going]
        S = max(lengths)
        rows = feats[torch.tensor([g[3] for g in going], device=feats.device), :S]  # [B, S, mt_dim] (rows >= S_b unused)
        x = torch.nn.functional.pad(rows, (0, 0, 0, S - rows.shape[1])).contiguous()  # (a pad position can lie past the search's rows)
        padded = [j for j, g in enumerate(going) if g[5]]
        if padded:  # whole-word streams at their end: mt_decoder(prev_output_tokens_mt) with the pad position (agent:576-642)
            clock.mark("features")
            Tp = max(going[j][2] for j in padded)
            enc = torch.zeros(len(padded), Tp, eng.cfg.enc_dim, dtype=torch.float32, device=eng.device)
            for m, j in enumerate(padded):
                enc[m, :going[j][2]] = eng.pool_encoder_rows(going[j][0].slot, going[j][2])
            Sp = max(lengths[j] for j in padded)
            toks = [going[j][4] + [eng.cfg.pad] * (Sp - lengths[j]) for j in padded]
            pf = eng.mt_features_batch(enc, [going[j][2] for j in padded], toks)
            for m, j in enumerate(padded):
                x[j, :lengths[j]] = pf[m, :lengths[j]]
        clock.mark("t2u")
        units, _, _ = eng.t2u_unit_decode_ragged(x, lengths, [g[5] for g in going])
        clock.mark("vocoder")  # (unit mapping included, as in the single agent's post-T2U stage)
        voc = []  # (agent, new_subword_tokens, unit)
        for (a, new, _, _, _, _), u in zip(going, units):
            action, unit = a._before_vocoder(u)
            if action is not None:
                a._action = action
            else:
                voc.append((a, new, unit))
        if not voc:
            return
        wavs = StreamSpeechS2STAgent._vocode(eng, [a for a, _, _ in voc], [unit for _, _, unit in voc])
        for (a, new, unit), w in zip(voc, wavs):
            a._action = a._after_vocoder(unit, w, new)


class PooledS2TTAgent(_PooledDecoder, StreamSpeechS2TTAgent):
    """StreamSpeechS2TTAgent (agent/speech_to_text.s2tt.streamspeech.agent.py:101-545) bound to a slot of a shared StreamPool: same
    push() / pop() / policy() contract and text output, the same policy code (the single agent's host stages), but the tensor work of
    all agents of a round runs as one pool step and one incremental MT search.  The reference's incremental MT decoder state (N12) lives
    in the slot (ss_pool_mt_greedy_incremental) and is cleared with it by reset(), as the single agent clears the handle's.  The pool
    needs both CTC heads (StreamPool(..., ctc_heads=2)).  The slot takes the S2TT agent's latency rule: chunk c = source_segment_size //
    40, conv chunk min(c, 16) (:359-366).  dictionary: the target subword dictionary (the single agent's dict["target_unigram"]);
    args: the single agent's flags (lagging_k1, stride_n, ...); the model comes from the pool's engine."""

    def __init__(self, pool: StreamPool, dictionary, args):
        if pool.ctc_heads != 2:
            raise ValueError("a pooled S2TT agent needs a stream pool with both CTC heads (ctc_heads=2)")
        self.pool = pool
        self.engine = pool.engine
        self.cfg = pool.engine.cfg
        self.torch_device = pool.engine.device
        self.dict = {"target_unigram": dictionary}
        self.lagging_k1 = args.lagging_k1
        self.lagging_k2 = args.lagging_k2
        self.segment_size = args.segment_size
        self.stride_n = args.stride_n
        self.unit_per_subword = args.unit_per_subword
        self.stride_n2 = args.stride_n2
        self.max_decoder_positions = getattr(args, "max_decoder_positions", 1200)
        self.trace = {}
        self._action = None
        self.slot = pool.acquire()
        chunk_size = args.source_segment_size // 40  # :359-366
        pool.set_chunk(self.slot, chunk_size, min(chunk_size, 16))  # once: it survives the reset between utterances
        pool.decoders[self.slot] = self
        SpeechToTextAgent.__init__(self, args)  # states + reset()

    def _reset_caches(self):
        """new utterance: the slot starts over (audio, encoder state, incremental MT state)"""
        if hasattr(self, "slot"):
            self.pool.reset(self.slot)
        self._action = None

    def policy(self):
        return self._policy_impl()

    @staticmethod
    @torch.inference_mode()
    def decode_round(pool: StreamPool, agents: Sequence["PooledS2TTAgent"], clock: _StageClock):
        """The S2TT stages of a flush for the agents whose slots the pool step just ran: the gate per stream, one incremental MT
        search for the writing streams, then the text delta per stream."""
        eng = pool.engine
        writing = []
        for a in agents:
            a.trace = {}
            r = pool.results[a.slot]
            if r["T"] == 0 and not a.states.source_finished:  # no fbank frame yet
                a._action = ReadAction()
                continue
            (src, _), (tgt, _) = r["ctc"]
            a.trace["asr_tokens"], a.trace["st_tokens"] = src, tgt
            new = a._gate(src, tgt)
            if new is None:
                a._action = ReadAction()
            else:
                writing.append((a, new))
        if not writing:
            return
        clock.mark("mt_incremental")
        hyps = writing[0][0]._mt_capacity_named(lambda: eng.pool_mt_greedy_incremental(
            [a.slot for a, _ in writing], [a.tgt_subwords_indices for a, _ in writing], [new for _, new in writing],
            [a._max_len(eng.pool_info(a.slot)["n_feat"]) for a, _ in writing]))
        for (a, new), tokens in zip(writing, hyps):
            a._action = a._after_mt(tokens, new)


def pushpop_many(agents: Sequence, segments: Sequence) -> list:
    """the batched front door: push one segment to every agent, then pop all (one batched engine step)"""
    for a, s in zip(agents, segments):
        a.push(s)
    return [a.pop() for a in agents]
