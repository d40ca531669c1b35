"""SimulEval agents backed by the H100 engine: same classes, flags, policy()/push()/pop() behaviour as

  agent/speech_to_speech.streamspeech.agent.py   (StreamSpeechS2STAgent, :101-770)
  agent/speech_to_text.asr.streamspeech.agent.py (StreamSpeechASRAgent,  :100-433)

but every tensor op of policy() runs in libstreamspeech_b200.so.  The classes here carry no @entrypoint: SimulEval
accepts exactly one registered system per `--agent` file (utils/agent.py:51-56), so each agent has its own thin file under
streamspeech_b200/agents/ named like the reference's (`speech_to_speech.streamspeech.agent.py`, ...).  Host code keeps exactly the
reference's control flow (READ/WRITE gate, prefix bookkeeping, wav tail slicing, the reset quirk).
What differs on purpose, without changing results:
  * new source samples are appended to a device buffer instead of re-converting the whole python list;
  * fbank frames are cached (each frame depends only on its own 400 samples);
  * the vocoder is run on the new units plus the generator's receptive field of left context
    (`--vocoder-context full` restores the reference's whole-sequence pass).
"""
from __future__ import annotations

import array
import json
import os
import sys
from typing import List, Optional, Sequence

import numpy as np
import torch

# Absolute imports with a path bootstrap: SimulEval loads `--agent FILE` as a top-level module named "agents"
# (SimulEval/simuleval/utils/agent.py:25-28), where relative imports do not resolve.
_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _REPO not in sys.path:
    sys.path.insert(0, _REPO)

from streamspeech_b200.config import ModelConfig, VocoderConfig  # noqa: E402
from streamspeech_b200.dictionary import Dictionary  # noqa: E402
from streamspeech_b200.engine import SS_ERR_CAPACITY, Engine, EngineError  # noqa: E402
from streamspeech_b200.simuleval_compat import (ReadAction, SpeechSegment, SpeechToSpeechAgent, SpeechToTextAgent, WriteAction)  # noqa: E402
from streamspeech_b200 import synth  # noqa: E402

SHIFT_SIZE = 10
WINDOW_SIZE = 25
ORG_SAMPLE_RATE = 48000
SAMPLE_RATE = 16000
FEATURE_DIM = 80
BOW_PREFIX = "▁"
DEFAULT_EOS = 2
READ = ("read", None, False, False)  # the policy's READ action as (kind, wav, SpeechSegment.finished, WriteAction.finished)


def load_streamspeech_checkpoint(args):
    """What `load_model_vocab` (agent:355-420) needs from disk: model cfg + state dict, gcmvn, dictionaries.

    `--model-path synthetic[:seed]` builds the seeded synthetic checkpoint (no real checkpoint exists in
    the build/GPU containers); anything else is a fairseq `.pt` whose "model" entry is the state dict.
    """
    if str(args.model_path).startswith("synthetic"):
        seed = int(args.model_path.split(":")[1]) if ":" in args.model_path else 0
        cfg = ModelConfig()
        sd = synth.make_model_state_dict(cfg, seed=seed)
        gcmvn = synth.make_gcmvn(cfg)
        dicts = {k: Dictionary.synthetic(n) for k, n in (("source_unigram", cfg.src_vocab), ("ctc_target_unigram", cfg.tgt_vocab),
                                                         ("target_unigram", cfg.tgt_vocab))}
        dicts["tgt"] = Dictionary.units(cfg.unit_vocab - 5)
        return cfg, sd, gcmvn, dicts
    if not os.path.exists(args.model_path):
        raise IOError("Model file not found: {}".format(args.model_path))
    state = torch.load(args.model_path, map_location="cpu", weights_only=False)
    sd = state["model"]
    cfg = ModelConfig.from_state_dict(sd)
    gcmvn = None
    if getattr(args, "config_yaml", None) is not None:
        import yaml

        with open(os.path.join(args.data_bin, args.config_yaml)) as f:
            config = yaml.load(f, Loader=yaml.BaseLoader)
        if "global_cmvn" in config:
            gcmvn = np.load(config["global_cmvn"]["stats_npz_path"])
    dicts = Dictionary.load_multitask(args, cfg)
    return cfg, sd, gcmvn, dicts


def load_vocoder(args, cfg: ModelConfig):
    """CodeHiFiGANVocoderWithDur.__init__ (agent/tts/vocoder.py:31-45): JSON config + torch.load(ckpt)["generator"]."""
    if str(args.vocoder).startswith("synthetic"):
        seed = int(args.vocoder.split(":")[1]) if ":" in args.vocoder else 1
        return cfg.vocoder, synth.make_vocoder_state_dict(cfg.vocoder, seed=seed)
    with open(args.vocoder_cfg) as f:
        vc = VocoderConfig.from_json_dict(json.load(f))
    sd = torch.load(args.vocoder, map_location="cpu", weights_only=False)["generator"]
    return vc, sd


class _DeviceAudio:
    """states.source mirrored on the device; only new samples cross PCIe.  With a 48 kHz source (the reference's default,
    agent:32-35: OnlineFeatureExtractor resamples states.source to 16 kHz on every call) the raw samples are kept at 48 kHz and
    the 16 kHz signal the fbank reads is extended on the device (ss_resample_48k_to_16k): only samples whose filter support is
    complete are produced while the source is open, the rest when it finishes."""

    def __init__(self, device, capacity=16000 * 60, engine=None, sample_rate=SAMPLE_RATE):
        self.rate = sample_rate
        self.engine = engine
        self.buf = torch.zeros(capacity * (sample_rate // SAMPLE_RATE), dtype=torch.float32, device=device)
        self.n = 0
        if sample_rate != SAMPLE_RATE:
            self.buf16 = torch.zeros(capacity, dtype=torch.float32, device=device)
            self.n16 = 0

    def reset(self):
        self.n = 0
        if self.rate != SAMPLE_RATE:
            self.n16 = 0

    def sync(self, source: List[float], finished: bool = False):
        n = len(source)
        if n < self.n:
            self.reset()
        if n > self.buf.numel():
            nb = torch.zeros(max(n * 2, self.buf.numel() * 2), dtype=torch.float32, device=self.buf.device)
            nb[: self.n] = self.buf[: self.n]
            self.buf = nb
        if n > self.n:
            # python list -> fp32 through array('f') (3x faster than torch.tensor(list)) into a persistent pinned staging buffer
            # (the previous chunk's copy has completed: policy() read results back since)
            m = n - self.n
            if getattr(self, "_stage", None) is None or self._stage.numel() < m:
                self._stage = torch.empty(max(m, 16384), dtype=torch.float32).pin_memory()
            if getattr(self, "_stage_ev", None) is not None:
                self._stage_ev.synchronize()  # (normally long complete)
            self._stage[:m].copy_(torch.frombuffer(array.array("f", source[self.n:]), dtype=torch.float32))
            self.buf[self.n:n].copy_(self._stage[:m], non_blocking=True)
            self._stage_ev = torch.cuda.Event()
            self._stage_ev.record()
            self.n = n
        if self.rate == SAMPLE_RATE:
            return self.buf[:n]
        n16 = self.engine.resample_out_len(n, finished)
        if n16 > self.buf16.numel():
            nb = torch.zeros(max(n16 * 2, self.buf16.numel() * 2), dtype=torch.float32, device=self.buf16.device)
            nb[: self.n16] = self.buf16[: self.n16]
            self.buf16 = nb
        if n16 > self.n16:
            self.engine.resample_48k_to_16k(self.buf[:n], self.buf16, self.n16, n16 - self.n16)
            self.n16 = n16
        return self.buf16[: self.n16]


class _EngineAgentMixin:
    def _init_engine(self, args, need_vocoder: bool):
        if args.sample_rate not in (SAMPLE_RATE, ORG_SAMPLE_RATE):
            raise NotImplementedError("the H100 front-end takes 16 kHz or 48 kHz input (the reference's two cases: agent:32-35)")
        override = getattr(args, "checkpoint_override", None)  # (cfg, model state dict, vocoder state dict, gcmvn) already in memory
        if override is not None:                                # (bench.py: the NCCL-broadcast copy of rank 0's checkpoint)
            cfg, sd, vsd_o, gcmvn = override
            dicts = {k: Dictionary.synthetic(n) for k, n in (("source_unigram", cfg.src_vocab), ("ctc_target_unigram", cfg.tgt_vocab),
                                                             ("target_unigram", cfg.tgt_vocab))}
            dicts["tgt"] = Dictionary.units(cfg.unit_vocab - 5)
        else:
            cfg, sd, gcmvn, dicts = load_streamspeech_checkpoint(args)
        vsd = None
        if need_vocoder:
            if override is not None:
                vsd = vsd_o
            else:
                cfg.vocoder, vsd = load_vocoder(args, cfg)
        self.cfg = cfg
        self.dict = dicts
        dev = getattr(args, "device_index", 0)
        self.engine = Engine(cfg, sd, vsd, gcmvn, device=dev, max_enc_frames=getattr(args, "max_enc_frames", 1024),
                             max_mt_positions=getattr(args, "max_mt_positions", 1024))
        self.torch_device = self.engine.device
        self.audio = _DeviceAudio(self.torch_device, engine=self.engine, sample_rate=args.sample_rate)
        self.feat_cache = torch.zeros(6000, cfg.feat_dim, dtype=torch.float32, device=self.torch_device)
        self.n_feat = 0
        self._resident = None
        self.encoder_mode = getattr(args, "encoder_mode", "cached")
        self.enc_buf = torch.zeros(getattr(args, "max_enc_frames", 1024), cfg.enc_dim, dtype=torch.float32, device=self.torch_device)
        self._enc_final = 0
        self._ctc_valid = [0, 0]

    def _encode(self, feature: torch.Tensor) -> torch.Tensor:
        """forward_encoder (agent:433).  "cached": only the rows of the not yet final chunk group are recomputed
        (ss_encoder_stream_step); "recompute": the whole prefix every call, like the reference."""
        if self.encoder_mode == "recompute":
            return self.engine.encoder(feature.unsqueeze(0))[0]
        T, t_final = self.engine.encoder_stream_step(feature, self.enc_buf)
        self._enc_final = t_final  # rows below it never change again (their CTC arg-max can be cached, see _ctc)
        return self.enc_buf[:T]

    def step_resident(self, audio_dev: torch.Tensor, n_valid: int, finished: bool):
        """Device-resident variant of pushpop(): the first `n_valid` samples of `audio_dev` (fp32, on the engine's
        device) are the source so far; returns (is_write, wav tensor on the device or None).  Same policy code,
        no python-list conversions."""
        self._resident = (audio_dev, n_valid)
        self.states.source_finished = finished
        try:
            kind, wav, _, _ = self._policy_impl()
        finally:
            self._resident = None
        return kind == "write", wav

    def _reset_caches(self):
        """new utterance: drop the device audio mirror and the fbank frame cache"""
        if hasattr(self, "audio"):
            self.audio.reset()
            self.n_feat = 0
            self.engine.encoder_stream_reset()
        self._enc_final = 0
        self._ctc_valid = [0, 0]

    def _features(self):
        """OnlineFeatureExtractor.__call__ (agent:66-87) with a per-frame cache."""
        if self._resident is not None:  # bench "value" leg: the utterance already lives in HBM
            samples = self._resident[0][: self._resident[1]]
        else:
            samples = self.audio.sync(self.states.source, self.states.source_finished)
        F = self.engine.num_fbank_frames(samples.numel())
        if F < self.n_feat:
            self.n_feat = 0
        if F > self.feat_cache.shape[0]:
            raise EngineError("utterance longer than the feature cache")
        if F > self.n_feat:
            self.feat_cache[self.n_feat:F] = self.engine.fbank(samples, self.n_feat, F - self.n_feat)
            self.n_feat = F
        return self.feat_cache[:F]

    def _ctc(self, head: int, enc: torch.Tensor):
        """CTC greedy over the encoder rows so far.  Encoder rows below the previous step's T_final are final, so their
        arg-max is cached on the device and only the newer rows are projected (ss_ctc_greedy_rows)."""
        if not hasattr(self, "_ctc_am") or self._ctc_am.shape[1] < self.enc_buf.shape[0]:
            self._ctc_am = torch.zeros(2, self.enc_buf.shape[0], dtype=torch.int64, device=self.enc_buf.device)
        row0 = min(self._ctc_valid[head], enc.shape[0]) if self.encoder_mode == "cached" else 0
        out = self.engine.ctc_greedy_rows(head, enc, row0, self._ctc_am[head])
        self._ctc_valid[head] = min(self._enc_final, enc.shape[0])  # arg-max of rows that are final now is reusable
        return out

    def _ctc_pair(self, enc: torch.Tensor):
        """ASR and ST CTC heads of one policy() call with a single device->host read (see _ctc)."""
        if not hasattr(self, "_ctc_am") or self._ctc_am.shape[1] < self.enc_buf.shape[0]:
            self._ctc_am = torch.zeros(2, self.enc_buf.shape[0], dtype=torch.int64, device=self.enc_buf.device)
        cached = self.encoder_mode == "cached"
        row0s = [min(self._ctc_valid[h], enc.shape[0]) if cached else 0 for h in (0, 1)]
        a, b = self.engine.ctc_greedy_rows_pair(enc, row0s, [self._ctc_am[0], self._ctc_am[1]])
        self._ctc_valid = [min(self._enc_final, enc.shape[0])] * 2
        return a, b


class StreamSpeechS2STAgent(_EngineAgentMixin, SpeechToSpeechAgent):
    """Drop-in for the reference class of the same name (agent:101-770)."""

    def __init__(self, args):
        super().__init__(args)
        self.eos = DEFAULT_EOS
        self.args = args
        self._init_engine(args, need_vocoder=True)
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
        chunk_size = args.source_segment_size // 40  # agent:395-413
        self.engine.set_chunk(chunk_size, 16 if chunk_size >= 16 else 8)
        self.vocoder_context = getattr(args, "vocoder_context", "receptive-field")
        self.trace = {}
        self.reset()

    @staticmethod
    def add_args(parser):
        """Same flags as the reference (agent:214-326) plus two engine knobs."""
        parser.add_argument("--model-path", type=str, required=True, help="path to your pretrained model.")
        parser.add_argument("--data-bin", type=str, required=True, help="Path of data binary")
        parser.add_argument("--config-yaml", type=str, default=None, help="Path to config yaml file")
        parser.add_argument("--multitask-config-yaml", type=str, default=None, help="Path to config yaml file")
        parser.add_argument("--global-stats", type=str, default=None, help="Path to json file containing cmvn stats")
        parser.add_argument("--tgt-splitter-type", type=str, default="SentencePiece")
        parser.add_argument("--tgt-splitter-path", type=str, default=None)
        parser.add_argument("--user-dir", type=str, default="researches/ctc_unity")
        parser.add_argument("--agent-dir", type=str, default="agent")
        parser.add_argument("--max-len", type=int, default=200, help="Max length of translation")
        parser.add_argument("--force-finish", default=False, action="store_true")
        parser.add_argument("--shift-size", type=int, default=SHIFT_SIZE)
        parser.add_argument("--window-size", type=int, default=WINDOW_SIZE)
        parser.add_argument("--sample-rate", type=int, default=ORG_SAMPLE_RATE, help="Sample rate")
        parser.add_argument("--feature-dim", type=int, default=FEATURE_DIM)
        parser.add_argument("--vocoder", type=str, required=True, help="path to the CodeHiFiGAN vocoder")
        parser.add_argument("--vocoder-cfg", type=str, required=True, help="path to the CodeHiFiGAN vocoder config")
        parser.add_argument("--dur-prediction", action="store_true")
        parser.add_argument("--lagging-k1", type=int, default=0)
        parser.add_argument("--lagging-k2", type=int, default=0)
        parser.add_argument("--segment-size", type=int, default=320)
        parser.add_argument("--stride-n", type=int, default=1)
        parser.add_argument("--stride-n2", type=int, default=1)
        parser.add_argument("--unit-per-subword", type=int, default=15)
        parser.add_argument("--extra-output-dir", type=str, default=None)
        parser.add_argument("--output-asr-translation", type=bool, default=False)
        parser.add_argument("--vocoder-context", type=str, default="receptive-field", choices=["receptive-field", "full"])
        parser.add_argument("--device-index", type=int, default=0)
        parser.add_argument("--encoder-mode", type=str, default="cached", choices=["cached", "recompute"])

    def reset(self):  # agent:328-347
        self.src_seg_num = 0
        self.tgt_subwords_indices = None
        self.src_ctc_indices = None
        self.src_ctc_prefix_length = 0
        self.tgt_ctc_prefix_length = 0
        self.tgt_units_indices = None
        self.prev_output_tokens_mt = None
        self.tgt_text = []
        self.mt_decoder_out = None
        self.unit = None
        self.wav = []
        self.post_transcription = ""
        self.unfinished_wav = None
        self.states.reset()
        self._reset_caches()

    def _finished_write_tuple(self):  # agent:615-626: WriteAction(SpeechSegment(unfinished_wav or [], finished=True), finished=True)
        return ("write", self.unfinished_wav, True, True)

    def policy(self):
        kind, wav, seg_finished, finished = self._policy_impl()
        if kind == "read":
            return ReadAction()
        content = wav.cpu().numpy().tolist() if wav is not None else []  # agent:765 (device -> host -> python list)
        return WriteAction(SpeechSegment(content=content, sample_rate=SAMPLE_RATE, finished=seg_finished), finished=finished)

    @torch.inference_mode()
    def _policy_impl(self):
        """The body of the reference policy(); returns (kind, wav on the device, SpeechSegment.finished, WriteAction.finished).
        The host stages between the engine calls are methods of their own (_gate, _after_mt, _before_vocoder, _after_vocoder), which the pooled agent
        (scheduler.PooledS2STAgent) calls between its batched engine calls."""
        eng = self.engine
        tr = self.trace = {}
        feature = self._features()
        if feature.size(0) == 0 and not self.states.source_finished:
            return READ
        enc = self._encode(feature)  # [T, 256]
        self.encoder_out = enc
        (src_ctc_indices, _), (tgt_ctc_indices, _) = self._ctc_pair(enc)  # agent:437, 461
        tr["asr_tokens"], tr["st_tokens"] = src_ctc_indices, tgt_ctc_indices
        new_subword_tokens = self._gate(src_ctc_indices, tgt_ctc_indices)
        if new_subword_tokens is None:
            return READ

        # 1. MT decoder (agent:520-538); the hypothesis comes back without its trailing eos
        # encoder rows below T_final are final in cached mode: their cross-attention K / V are projected once (ss_mt_stable_rows)
        stable = self._enc_final if self.encoder_mode == "cached" else 0
        tokens, feats = eng.mt_greedy(enc, self.tgt_subwords_indices, new_subword_tokens, max_len_b=100, stable_rows=stable)
        action, t2u_input = self._after_mt(tokens)
        if action is not None:
            return action
        prev_output_tokens_mt, n_pad_tail = t2u_input
        # mt_decoder(prev_output_tokens_mt, features_only=True) (agent:638-642): already produced by the greedy pass
        # unless whole-word trimming changed the sequence
        if n_pad_tail:
            feats = eng.mt_features(enc, prev_output_tokens_mt, stable_rows=stable)
        else:  # causal decoder: the features of [eos, t1..tj] are the first j + 1 rows of the greedy pass
            feats = feats[: len(prev_output_tokens_mt)]
        # 2./3. T2U encoder + CTC unit decoder (agent:662-689)
        r = eng.t2u_unit_decode(feats.contiguous(), n_pad_tail=n_pad_tail)
        return self._after_t2u(eng.units_to_host(r), new_subword_tokens)

    def _gate(self, src_ctc_indices, tgt_ctc_indices) -> Optional[int]:
        """READ / WRITE gate on the CTC prefixes (agent:480-509): None = READ, else the MT call's new_subword_tokens (-1 once the
        source is finished)."""
        if not self.states.source_finished:  # agent:480-509
            src_ctc_prefix_length = len(src_ctc_indices)
            tgt_ctc_prefix_length = len(tgt_ctc_indices)
            self.src_ctc_indices = src_ctc_indices
            if (src_ctc_prefix_length < self.src_ctc_prefix_length + self.stride_n
                    or tgt_ctc_prefix_length < self.tgt_ctc_prefix_length + self.stride_n):
                return None
            self.src_ctc_prefix_length = max(src_ctc_prefix_length, self.src_ctc_prefix_length)
            self.tgt_ctc_prefix_length = max(tgt_ctc_prefix_length, self.tgt_ctc_prefix_length)
            subword_tokens = ((tgt_ctc_prefix_length - self.lagging_k1) // self.stride_n) * self.stride_n
            if self.whole_word:
                subword_tokens += 1
            new_subword_tokens = (subword_tokens - len(self.tgt_subwords_indices)) if self.tgt_subwords_indices is not None else subword_tokens
            if new_subword_tokens < 1:
                return None
        else:
            self.src_ctc_indices = src_ctc_indices
            new_subword_tokens = -1
        new_subword_tokens = int(new_subword_tokens)
        self.trace["new_subword_tokens"] = new_subword_tokens
        return new_subword_tokens

    def _after_mt(self, tokens: List[int]):
        """Whole-word trimming and the "same hypothesis" / "not longer" checks on the MT hypothesis (agent:540-636).  Returns
        (action, None) when the call ends here, else (None, (prev_output_tokens_mt, n_pad_tail)): the T2U input."""
        c = self.cfg
        tgt_subwords_indices = list(tokens)
        n_pad_tail = 0
        if self.whole_word:  # agent:540-574
            if not self.states.source_finished:
                j = 999999
                for j in range(len(tgt_subwords_indices) - 1, -1, -1):
                    if self.dict["target_unigram"][tgt_subwords_indices[j]].startswith(BOW_PREFIX):
                        break
                tgt_subwords_indices = tgt_subwords_indices[:j]
                tokens = tokens[:j]
                if j == 0:
                    return READ, None
            else:
                # source finished: the hypothesis keeps its eos, max_tgt_len = len + 1 -> ONE trailing <pad> (agent:576-591).
                # While reading, the hypothesis was cut to [:j] (no eos) and max_tgt_len = j + 1: no pad position.
                n_pad_tail = 1
        prev_output_tokens_mt = [c.eos] + list(tokens) + [c.pad] * n_pad_tail  # agent:576-591
        self.trace["mt_tokens"] = list(tokens)

        if self.tgt_subwords_indices is not None and self.tgt_subwords_indices == tgt_subwords_indices:  # agent:609-626
            if not self.states.source_finished:
                return READ, None
            return self._finished_write_tuple(), None
        self.tgt_subwords_indices = tgt_subwords_indices
        if not self.states.source_finished and self.prev_output_tokens_mt is not None:  # agent:629-636
            if self.prev_output_tokens_mt == prev_output_tokens_mt or len(prev_output_tokens_mt) <= len(self.prev_output_tokens_mt):
                return READ, None
        self.prev_output_tokens_mt = prev_output_tokens_mt
        return None, (prev_output_tokens_mt, n_pad_tail)

    def _after_t2u(self, tmp: List[int], new_subword_tokens: int):
        """From the collapsed unit indices of the T2U + unit-decoder call to the action (agent:690-770), as a batch of one of the
        three stages the pooled agent runs for all of its streams: _before_vocoder, _vocode, _after_vocoder."""
        action, unit = self._before_vocoder(tmp)
        if action is not None:
            return action
        new_wav = self._vocode(self.engine, [self], [unit])[0]
        return self._after_vocoder(unit, new_wav, new_subword_tokens)

    def _before_vocoder(self, tmp: List[int]):
        """Unit dictionary mapping and the new units (cur_unit) (agent:690-742).  Returns (action, None) when the call ends here,
        else (None, unit): the vocoder's input, the whole unit sequence so far."""
        if len(tmp) == 0:
            if not self.states.source_finished:
                return READ, None
            return self._finished_write_tuple(), None
        if tmp[-1] == self.eos:
            tmp = tmp[:-1]
        unit = []
        for t in tmp:  # agent:713-717
            u = self.dict["tgt"][t].replace("<s>", "").replace("</s>", "")
            if u != "":
                unit.append(int(u))
        self.trace["units"] = list(unit)
        cur_unit = unit if self.unit is None else unit[len(self.unit):]
        if len(unit) < 1 or len(cur_unit) < 1:
            if not self.states.source_finished:
                return READ, None
            return self._finished_write_tuple(), None
        return None, unit

    @staticmethod
    def _vocode(eng, agents: Sequence["StreamSpeechS2STAgent"], units: Sequence[List[int]]) -> List[torch.Tensor]:
        """4. vocoder (agent:743-753): the wav of each agent's new units, for all agents in one durations call, one host read of the
        cumsums and one generate call per dur_prediction setting.  Each agent's wav equals that of a call of its own, bit for bit."""
        if len(agents) == 1:  # a batch of one: the single-sequence calls (the n = 1 case of the same entry points), one cumsum read
            a, unit = agents[0], units[0]
            _, cum = eng.vocoder_durations(torch.tensor(unit, dtype=torch.long, device=eng.device), a.dur_prediction)
            cum_h = cum.tolist()
            total = cum_h[-1]
            new = total - cum_h[0 if a.unit is None else len(a.unit)]
            a.trace["dur"] = [cum_h[j + 1] - cum_h[j] for j in range(len(unit))]
            if a.vocoder_context == "full":
                return [eng.vocoder_generate(total, 0, total, 0)[-new * eng.hop:]]
            return [eng.vocoder_generate(total, total - new, new, -1)]
        out: List[Optional[torch.Tensor]] = [None] * len(agents)
        for dp in sorted({bool(a.dur_prediction) for a in agents}):
            idx = [i for i, a in enumerate(agents) if bool(a.dur_prediction) == dp]
            _, cums, _ = eng.vocoder_durations_ragged([units[i] for i in idx], dp)
            args, new_frames = [], []  # (total_frames, frame0, n_frames, left_context) per stream; its new frames
            for i, cum_h in zip(idx, cums):
                a, unit = agents[i], units[i]
                total = cum_h[-1]
                a.trace["dur"] = [cum_h[j + 1] - cum_h[j] for j in range(len(unit))]
                new = total - cum_h[0 if a.unit is None else len(a.unit)]
                new_frames.append(new)
                args.append((total, 0, total, 0) if a.vocoder_context == "full" else (total, total - new, new, -1))
            wavs = eng.vocoder_generate_ragged(*zip(*args))
            for i, w, new in zip(idx, wavs, new_frames):
                out[i] = w[-new * eng.hop:]  # ("full": the tail of the whole-sequence pass)
        return out

    def _after_vocoder(self, unit: List[int], new_wav: torch.Tensor, new_subword_tokens: int):
        """The wav tail, unfinished_wav and the reset quirk (agent:754-770)."""
        if self.unfinished_wav is not None and len(self.unfinished_wav) > 0:
            new_wav = torch.cat((self.unfinished_wav, new_wav), dim=0)
        self.unit = unit
        if self.states.source_finished and new_subword_tokens == -1:
            self.states.target_finished = True
            self.reset()  # NB: resets the states as well, so both flags below read False (agent:759-770)
        return ("write", new_wav, self.states.source_finished, self.states.target_finished)


class StreamSpeechASRAgent(_EngineAgentMixin, SpeechToTextAgent):
    """Drop-in for agent/speech_to_text.asr.streamspeech.agent.py: fbank -> encoder -> ASR CTC -> text delta."""

    def __init__(self, args):
        super().__init__(args)
        self.args = args
        self._init_engine(args, need_vocoder=False)
        chunk_size = args.source_segment_size // 40
        self.engine.set_chunk(chunk_size, min(chunk_size, 16))  # :361-375 (N8)
        self.trace = {}
        self.reset()

    add_args = StreamSpeechS2STAgent.add_args

    def reset(self):
        self.asr_text = ""
        self.states.reset()
        self._reset_caches()

    @torch.inference_mode()
    def policy(self):
        feature = self._features()
        if feature.size(0) == 0 and not self.states.source_finished:
            return ReadAction()
        enc = self._encode(feature)
        toks, _ = self._ctc(0, enc)
        self.trace = {"asr_tokens": toks}
        text = " ".join(self.dict["source_unigram"][t] for t in toks)  # :419-425
        new_text = text[len(self.asr_text):]
        self.asr_text = text
        if self.states.source_finished:
            self.states.target_finished = True
            self.reset()
        return WriteAction(new_text, finished=self.states.target_finished)


class StreamSpeechS2TTAgent(_EngineAgentMixin, SpeechToTextAgent):
    """Drop-in for agent/speech_to_text.s2tt.streamspeech.agent.py (StreamSpeechS2TTAgent, :101-545): fbank -> encoder ->
    ASR / ST CTC -> policy gate -> MT decoder -> text delta.  The reference runs this agent's MT generator with incremental
    states that live across policy() calls (:161-179, SURVEY.md N12); the engine keeps the same state in the handle
    (ss_mt_greedy_incremental) and reproduces its two quirks (duplicate self-attention entry per call, cross-attention K / V of
    early encoder rows never refreshed)."""

    def __init__(self, args):
        super().__init__(args)
        self.args = args
        self._init_engine(args, need_vocoder=False)
        self.lagging_k1 = args.lagging_k1
        self.lagging_k2 = args.lagging_k2
        self.segment_size = args.segment_size
        self.stride_n = args.stride_n
        self.unit_per_subword = args.unit_per_subword
        self.stride_n2 = args.stride_n2
        chunk_size = args.source_segment_size // 40
        self.engine.set_chunk(chunk_size, min(chunk_size, 16))  # :359-366
        self.max_decoder_positions = getattr(args, "max_decoder_positions", 1200)  # model.max_decoder_positions() (unit decoder)
        self.trace = {}
        self.reset()

    add_args = StreamSpeechS2STAgent.add_args

    def reset(self):  # :300-309
        self.src_seg_num = 0
        self.tgt_subwords_indices = None
        self.src_ctc_indices = None
        self.src_ctc_prefix_length = 0
        self.tgt_ctc_prefix_length = 0
        self.tgt_text = ""
        self.states.reset()
        self._reset_caches()

    def _reset_caches(self):
        """new utterance: the mixin's caches and the handle's incremental MT state"""
        super()._reset_caches()
        if hasattr(self, "engine"):
            self.engine.mt_incremental_reset()

    @torch.inference_mode()
    def policy(self):
        """The body of the reference policy().  The host stages around the MT call are methods of their own (_gate, _after_mt), which
        the pooled agent (scheduler.PooledS2TTAgent) calls around its batched MT call."""
        tr = self.trace = {}
        feature = self._features()
        if feature.size(0) == 0 and not self.states.source_finished:
            return ReadAction()
        enc = self._encode(feature)
        (src_ctc_indices, _), (tgt_ctc_indices, _) = self._ctc_pair(enc)
        tr["asr_tokens"], tr["st_tokens"] = src_ctc_indices, tgt_ctc_indices
        new_subword_tokens = self._gate(src_ctc_indices, tgt_ctc_indices)
        if new_subword_tokens is None:
            return ReadAction()
        tokens = self._mt_capacity_named(lambda: self.engine.mt_greedy_incremental(enc, self.tgt_subwords_indices, new_subword_tokens,
                                                                                     self._max_len(feature.size(0))))
        return self._after_mt(tokens, new_subword_tokens)

    def _mt_capacity_named(self, search):
        """Runs the incremental MT search; its SS_ERR_CAPACITY (refused before any launch: the cache must hold max_len + 2 entries plus
        one per earlier call of the utterance, wherever eos would fall) comes back as an error that says what to change."""
        try:
            return search()
        except EngineError as e:
            if e.code != SS_ERR_CAPACITY:
                raise
            raise EngineError(f"utterance too long for this agent's MT decoder cache (max_mt_positions = {self.engine.max_mt_positions}): "
                              f"{e.detail}.  Build the agent with a larger args.max_mt_positions; 2048 covers every utterance the encoder "
                              f"admits") from e

    def _max_len(self, n_frames: int) -> int:
        """generator_mt: max_len_a = 1, max_len_b = 200 (:161-179); src_len = src_tokens.size(1) = fbank frames"""
        return min(int(n_frames + 200), self.max_decoder_positions - 1)

    def _gate(self, src_ctc_indices, tgt_ctc_indices) -> Optional[int]:
        """READ / WRITE gate on the CTC prefixes (:437-465): None = READ, else the MT call's new_subword_tokens (-1 once the source is
        finished)."""
        if not self.states.source_finished:  # :437-465
            src_ctc_prefix_length, tgt_ctc_prefix_length = len(src_ctc_indices), len(tgt_ctc_indices)
            self.src_ctc_indices = src_ctc_indices
            if (src_ctc_prefix_length < self.src_ctc_prefix_length + self.stride_n
                    or tgt_ctc_prefix_length < self.tgt_ctc_prefix_length + self.stride_n):
                return None
            self.src_ctc_prefix_length = max(src_ctc_prefix_length, self.src_ctc_prefix_length)
            self.tgt_ctc_prefix_length = max(tgt_ctc_prefix_length, self.tgt_ctc_prefix_length)
            subword_tokens = ((tgt_ctc_prefix_length - self.lagging_k1) // self.stride_n) * self.stride_n
            new_subword_tokens = (subword_tokens - len(self.tgt_subwords_indices)) if self.tgt_subwords_indices is not None else subword_tokens
            if new_subword_tokens < 1:
                return None
        else:
            self.src_ctc_indices = src_ctc_indices
            new_subword_tokens = -1
        new_subword_tokens = int(new_subword_tokens)
        self.trace["new_subword_tokens"] = new_subword_tokens
        return new_subword_tokens

    def _after_mt(self, tokens: List[int], new_subword_tokens: int):
        """From the MT hypothesis (without eos) to the action (:519-545): the "same hypothesis" check, the text delta and the reset
        quirk at the end of the utterance."""
        self.trace["mt_tokens"] = list(tokens)
        if self.tgt_subwords_indices is not None and self.tgt_subwords_indices == tokens:  # :519-529
            if not self.states.source_finished:
                return ReadAction()
            return WriteAction("", finished=True)
        self.tgt_subwords_indices = tokens
        text = " ".join(self.dict["target_unigram"][t] for t in tokens)  # :532-535
        new_text = text[len(self.tgt_text):]
        self.tgt_text = text
        if self.states.source_finished and new_subword_tokens == -1:
            self.states.target_finished = True
            self.reset()
        return WriteAction(new_text, finished=self.states.target_finished)
