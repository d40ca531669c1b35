"""The reference's wait-k-stride-n baselines on UnitY, Uni-UnitY and Chunk-UnitY checkpoints, backed by the H100 engine: same classes, flags and policy() behaviour as

  agent/speech_to_speech.wait-k-stride-n.agent.py   (WaitkS2STAgent, :101-581)
  agent/speech_to_text.wait-k-stride-n.agent.py     (EnglishSpeechCounter, :100-477; WaitkS2TTAgent here)

The policy counts source segments instead of reading CTC prefixes: after `lagging_k1` segments of `--segment-size` ms it lets the MT
search emit one subword per `stride_n` segments, and the unit search `unit_per_subword` units per `stride_n2` subwords after the first
`lagging_k2`.  Every policy() call that passes the gate runs, like the reference (whose generators keep no incremental state):

  fbank + gcmvn of the whole source                       ss_fbank (frames cached: each depends only on its own samples)
  forward_encoder on the whole prefix                     UnitY (bidirectional) and Uni-UnitY (future mask, symmetric convs):
                                                            ss_encoder_forward, B = 1, every row recomputed;
                                                          Chunk-UnitY (chunk mask and chunk-causal convs at the training
                                                            --chunk-size): ss_encoder_stream_step, the rows of the open chunk
                                                            group only (earlier rows are final)
  MT search with the previous hypothesis as prefix        ss_mt_greedy (cross K / V of every encoder row re-projected; Chunk-UnitY:
                                                            of the rows that are not final, ss_mt_stable_rows)
  S2ST: MT decoder features of [eos, tokens...]           the rows of the same ss_mt_greedy pass (causal decoder)
  S2ST: synthesizer_encoder                               ss_t2u_encode_batch, B = 1 (causal with --uni-encoder: Uni-UnitY, Chunk-UnitY)
  S2ST: unit search from BOS (tgt_units_indices is        ss_unit_search_batch, B = 1, max_len = the absolute unit count
        never assigned in the reference)                    or min(F + 200, max_decoder_positions - 1) once the source ended
  S2ST: vocoder on all units, the new units' samples      the S2ST agent's receptive-field tail window (_vocode)

Quirks kept as the reference has them: the S2TT agent gates on the unit count too; the text is " ".join of the raw subword symbols;
`self.reset()` inside policy() also resets `states`, so both finished flags of the last WRITE read False.

One rule differs on purpose: the reference counts segments as len(source) // (segment_size * 48000 / 1000) while its feature
extractor's --sample-rate defaults to 16000.  Here a segment is `segment_size` ms of source samples at --sample-rate (16 or 48 kHz).
"""
from __future__ import annotations

import os
from typing import List, Optional

import numpy as np
import torch

from streamspeech_b200 import synth
from streamspeech_b200.agent import (READ, SAMPLE_RATE, StreamSpeechS2STAgent, _DeviceAudio, _EngineAgentMixin, load_vocoder)
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.dictionary import Dictionary
from streamspeech_b200.engine import Engine
from streamspeech_b200.simuleval_compat import (ReadAction, SpeechSegment, SpeechToSpeechAgent, SpeechToTextAgent, WriteAction)

DEFAULT_EOS = 2


def load_unity_checkpoint(args):
    """(cfg, model state dict, gcmvn, dictionaries) of --model-path: `synthetic[:seed]` is the seeded synthetic checkpoint of the
    UnitY-family model --user-dir names (synth.make_unity_checkpoint: researches/uni_unity, researches/chunk_unity, else UnitY);
    anything else is a fairseq `.pt`, which must hold a UnitY, Uni-UnitY or Chunk-UnitY model (ModelConfig.from_checkpoint)."""
    if str(args.model_path).startswith("synthetic"):
        seed = int(args.model_path.split(":")[1]) if ":" in args.model_path else 0
        state = synth.make_unity_checkpoint(synth.synthetic_unity_variant(getattr(args, "user_dir", None)), seed=seed)
        cfg = ModelConfig.from_checkpoint(state)
        dicts = {"target_unigram": Dictionary.synthetic(cfg.tgt_vocab), "tgt": Dictionary.units(cfg.unit_vocab - 4, blank=False)}
        return cfg, state["model"], synth.make_gcmvn(cfg), dicts
    if not os.path.exists(args.model_path):
        raise IOError("Model file not found: {}".format(args.model_path))
    state = torch.load(args.model_path, map_location="cpu", weights_only=False)
    cfg = ModelConfig.from_checkpoint(state)
    if not cfg.unity:
        raise ValueError(f"{args.model_path} is a StreamSpeech (CTC) checkpoint; the wait-k agents run UnitY checkpoints "
                         f"(unity.{{fr,es,de}}-en.pt).  Evaluate StreamSpeech with the streamspeech agents")
    gcmvn = None
    if getattr(args, "config_yaml", None) is not None:
        import yaml

        with open(os.path.join(args.data_bin, args.config_yaml)) as f:
            config = yaml.load(f, Loader=yaml.BaseLoader)
        if "global_cmvn" in config:
            gcmvn = np.load(config["global_cmvn"]["stats_npz_path"])
    return cfg, state["model"], gcmvn, Dictionary.load_multitask(args, cfg)


def waitk_counts(n_samples: int, segment_size: int, sample_rate: int, lagging_k1: int, stride_n: int, lagging_k2: int, stride_n2: int,
                 unit_per_subword: int):
    """(src_seg_num, subword_tokens, unit_tokens) of the gate (agent:359-384) for a source of n_samples samples"""
    src_seg_num = int(n_samples // (segment_size * sample_rate / 1000))
    subword_tokens = ((src_seg_num - lagging_k1) // stride_n) * stride_n
    return src_seg_num, subword_tokens, unit_tokens_of(subword_tokens, lagging_k2, stride_n2, unit_per_subword)


def unit_tokens_of(subword_tokens: int, lagging_k2: int, stride_n2: int, unit_per_subword: int) -> int:
    return ((subword_tokens - lagging_k2) // stride_n2) * stride_n2 * unit_per_subword


class _WaitkMixin(_EngineAgentMixin):
    def _init_waitk(self, args, need_vocoder: bool):
        if args.sample_rate not in (SAMPLE_RATE, 48000):
            raise NotImplementedError("the H100 front-end takes 16 kHz or 48 kHz input")
        cfg, sd, gcmvn, dicts = load_unity_checkpoint(args)
        vsd = None
        if need_vocoder:
            cfg.vocoder, vsd = load_vocoder(args, cfg)
        self.cfg, self.dict, self.args = cfg, dicts, args
        # model.max_decoder_positions() (the unit decoder's): both generators' max_len for max_new_tokens == -1
        self.max_decoder_positions = cfg.max_target_positions
        # the MT search of an ended source runs to at most max_decoder_positions - 1 tokens and needs two more positions
        self.engine = Engine(cfg, sd, vsd, gcmvn, device=getattr(args, "device_index", 0), max_enc_frames=getattr(args, "max_enc_frames", 1024),
                             max_mt_positions=max(getattr(args, "max_mt_positions", 1024), cfg.max_target_positions + 1))
        # UnitY: the offline (bidirectional) encoder; Uni-UnitY: a future mask with symmetric convolutions, whose rows still change as
        # the source grows (re-encoded whole on every call, as the reference does); Chunk-UnitY: the chunk encoder, whose rows of
        # complete chunk groups are final (encoded incrementally, their MT cross K / V projected once)
        self.engine.set_chunk(*cfg.encoder_chunk())
        self.incremental = cfg.unity_variant == "chunk_unity"
        self.torch_device = self.engine.device
        if self.incremental:
            self.enc_buf = torch.zeros(getattr(args, "max_enc_frames", 1024), cfg.enc_dim, dtype=torch.float32, device=self.torch_device)
        self.sample_rate = args.sample_rate
        self.audio = _DeviceAudio(self.torch_device, engine=self.engine, sample_rate=args.sample_rate)
        self.feat_cache = torch.zeros(6000, cfg.feat_dim, dtype=torch.float32, device=self.torch_device)
        self.n_feat = 0
        self._resident = None
        self._enc_final = 0
        self._ctc_valid = [0, 0]
        self.lagging_k1, self.lagging_k2 = args.lagging_k1, args.lagging_k2
        self.segment_size = args.segment_size
        self.stride_n, self.stride_n2 = args.stride_n, args.stride_n2
        self.unit_per_subword = args.unit_per_subword
        self.trace = {}

    def _n_source(self) -> int:
        return self._resident[1] if self._resident is not None else len(self.states.source)

    def _gate(self):
        """agent:359-405: None = READ, else (new_subword_tokens, new_unit_tokens), both -1 once the source has ended"""
        fin = self.states.source_finished
        src_seg_num, subword_tokens, unit_tokens = waitk_counts(self._n_source(), self.segment_size, self.sample_rate, self.lagging_k1,
                                                                self.stride_n, self.lagging_k2, self.stride_n2, self.unit_per_subword)
        if (src_seg_num <= self.src_seg_num or src_seg_num < self.lagging_k1) and not fin:
            return None
        self.src_seg_num = src_seg_num
        new_subword_tokens = subword_tokens - len(self.tgt_subwords_indices) if self.tgt_subwords_indices is not None else subword_tokens
        new_unit_tokens = unit_tokens  # tgt_units_indices is never assigned after reset()
        if (new_subword_tokens < 1 or new_unit_tokens < 1) and not fin:
            return None
        if fin:
            new_subword_tokens = new_unit_tokens = -1
        self.trace["new_subword_tokens"], self.trace["new_unit_tokens"] = int(new_subword_tokens), int(new_unit_tokens)
        return int(new_subword_tokens), int(new_unit_tokens)

    def _full_max_len(self, n_frames: int) -> int:
        """generate_decoder's max_len for max_new_tokens == -1 (sequence_generator.py:205-213): max_len_a = 1, max_len_b = 200,
        src_len = the number of fbank frames"""
        return min(int(1 * n_frames + 200), self.max_decoder_positions - 1)

    def _encode_and_translate(self, new_subword_tokens: int):
        """features, encoder and MT search (agent:407-436).  None = READ (no fbank frame yet), else (tokens, MT features of
        [eos] + tokens, number of fbank frames)"""
        feature = self._features()
        F = int(feature.size(0))
        if F == 0 and not self.states.source_finished:
            return None
        if self.incremental:  # only the rows of the open chunk group are computed; rows below t_final are final
            T, t_final = self.engine.encoder_stream_step(feature, self.enc_buf)
            enc, stable = self.enc_buf[:T], t_final
        else:
            enc, stable = self.engine.encoder(feature.unsqueeze(0))[0], 0  # the whole prefix; no stable-rows hint: every row changes
        self._enc_final = stable
        tokens, feats = self.engine.mt_greedy(enc, self.tgt_subwords_indices, new_subword_tokens, max_len_b=self._full_max_len(F),
                                              stable_rows=stable)
        self.trace["mt_tokens"] = list(tokens)
        self.tgt_subwords_indices = list(tokens)
        return tokens, feats, F


def add_waitk_args(parser):
    """The reference's flags (agent:186-288) plus the engine's device index"""
    parser.add_argument("--model-path", type=str, required=True, help="path to your pretrained model.")
    parser.add_argument("--data-bin", type=str, required=True, help="Path of data binary")
    parser.add_argument("--config-yaml", type=str, default=None, help="Path to config yaml file")
    parser.add_argument("--multitask-config-yaml", type=str, default=None, help="Path to config yaml file")
    parser.add_argument("--global-stats", type=str, default=None, help="Path to json file containing cmvn stats")
    parser.add_argument("--tgt-splitter-type", type=str, default="SentencePiece", help="Subword splitter type for target text")
    parser.add_argument("--tgt-splitter-path", type=str, default=None, help="Subword splitter model path for target text")
    parser.add_argument("--user-dir", type=str, default="researches/ctc_unity", help="User directory for model")
    parser.add_argument("--agent-dir", type=str, default="agent", help="User directory for agents")
    parser.add_argument("--max-len", type=int, default=200, help="Max length of translation")
    parser.add_argument("--force-finish", default=False, action="store_true",
                        help="Force the model to finish the hypothsis if the source is not finished")
    parser.add_argument("--shift-size", type=int, default=10, help="Shift size of feature extraction window.")
    parser.add_argument("--window-size", type=int, default=25, help="Window size of feature extraction window.")
    parser.add_argument("--sample-rate", type=int, default=SAMPLE_RATE, help="Sample rate")
    parser.add_argument("--feature-dim", type=int, default=80, help="Acoustic feature dimension.")
    parser.add_argument("--vocoder", type=str, required=True, help="path to the CodeHiFiGAN vocoder")
    parser.add_argument("--vocoder-cfg", type=str, required=True, help="path to the CodeHiFiGAN vocoder config")
    parser.add_argument("--dur-prediction", action="store_true", help="enable duration prediction (for reduced/unique code sequences)")
    parser.add_argument("--lagging-k1", type=int, default=3, help="lagging number")
    parser.add_argument("--lagging-k2", type=int, default=1, help="lagging number")
    parser.add_argument("--segment-size", type=int, default=320, help="segment-size")
    parser.add_argument("--stride-n", type=int, default=1, help="lagging number")
    parser.add_argument("--stride-n2", type=int, default=1, help="lagging number")
    parser.add_argument("--unit-per-subword", type=int, default=15, help="lagging number")
    parser.add_argument("--device-index", type=int, default=0)


class WaitkS2STAgent(_WaitkMixin, SpeechToSpeechAgent):
    """Drop-in for the reference class of the same name (agent/speech_to_speech.wait-k-stride-n.agent.py:101-581)."""

    def __init__(self, args):
        super().__init__(args)
        self.eos = DEFAULT_EOS
        self._init_waitk(args, need_vocoder=True)
        self.max_len = args.max_len
        self.force_finish = args.force_finish
        self.dur_prediction = args.dur_prediction
        self.vocoder_context = "receptive-field"  # what StreamSpeechS2STAgent._vocode reads
        self.reset()

    add_args = staticmethod(add_waitk_args)

    def reset(self):  # agent:290-296
        self.src_seg_num = 0
        self.tgt_subwords_indices = None
        self.tgt_units_indices = None
        self.unit = None
        self.wav = []
        self.states.reset()
        self._reset_caches()

    def policy(self):
        kind, wav, seg_finished, finished = self._policy_impl()
        if kind == "read":
            return ReadAction()
        content = wav.cpu().numpy().tolist() if wav is not None else []
        return WriteAction(SpeechSegment(content=content, sample_rate=SAMPLE_RATE, finished=seg_finished), finished=finished)

    @torch.inference_mode()
    def _policy_impl(self):
        """The body of the reference policy() (agent:358-581); returns (kind, wav on the device or None, SpeechSegment.finished,
        WriteAction.finished) like StreamSpeechS2STAgent._policy_impl, which step_resident() calls."""
        eng, c = self.engine, self.cfg
        self.trace = {}
        fin = self.states.source_finished
        gate = self._gate()
        if gate is None:
            return READ
        new_subword_tokens, new_unit_tokens = gate
        r = self._encode_and_translate(new_subword_tokens)
        if r is None:
            return READ
        tokens, feats, F = r
        new_unit_tokens = unit_tokens_of(len(tokens), self.lagging_k2, self.stride_n2, self.unit_per_subword)  # agent:438-453
        if new_unit_tokens < 1 and not fin:
            return READ
        if fin:
            new_unit_tokens = -1
        # prev_output_tokens_mt = [eos, tokens...] (the hypothesis always ends in eos: no pad position); its features are the
        # first len(tokens) + 1 rows of the greedy pass
        S = len(tokens) + 1
        t2u = eng.t2u_encode_batch(feats[:S].unsqueeze(0).contiguous(), [S])
        max_len = new_unit_tokens if new_unit_tokens != -1 else self._full_max_len(F)
        hyp = eng.unit_search_batch(t2u, [S], max_len)[0]["tokens"]  # from BOS on every call (agent:520-533)
        tmp = hyp[:-1] if hyp[-1] == c.eos else hyp
        unit = [int(self.dict["tgt"][t]) for t in tmp]  # agent:541
        self.trace["units"] = list(unit)
        cur_unit = unit if self.unit is None else unit[len(self.unit):]
        if len(unit) < 1 or len(cur_unit) < 1:  # agent:545-556
            if not fin:
                return READ
            return ("write", None, True, True)
        new_wav = StreamSpeechS2STAgent._vocode(eng, [self], [unit])[0]  # agent:558-566: the samples of cur_unit
        self.unit = unit
        if new_subword_tokens == -1 and new_unit_tokens == -1:
            self.states.target_finished = True
            self.reset()  # resets the states as well: both flags below read False (agent:570-581)
        return ("write", new_wav, self.states.source_finished, self.states.target_finished)


class WaitkS2TTAgent(_WaitkMixin, SpeechToTextAgent):
    """Drop-in for agent/speech_to_text.wait-k-stride-n.agent.py (class EnglishSpeechCounter there, :100-477).  It takes
    --vocoder / --vocoder-cfg like the reference and does not load them."""

    def __init__(self, args):
        super().__init__(args)
        self.eos = DEFAULT_EOS
        self._init_waitk(args, need_vocoder=False)
        self.max_len = args.max_len
        self.force_finish = args.force_finish
        self.reset()

    add_args = staticmethod(add_waitk_args)

    def reset(self):  # :290-297
        self.src_seg_num = 0
        self.tgt_subwords_indices = None
        self.tgt_units_indices = None
        self.unit = None
        self.wav = []
        self.tgt_text = ""
        self.states.reset()
        self._reset_caches()

    @torch.inference_mode()
    def policy(self):
        """The body of the reference policy() (:358-477)"""
        self.trace = {}
        gate = self._gate()  # the unit count gates this agent too (:370-400)
        if gate is None:
            return ReadAction()
        new_subword_tokens, _ = gate
        r = self._encode_and_translate(new_subword_tokens)
        if r is None:
            return ReadAction()
        tokens = r[0]
        text = " ".join(self.dict["target_unigram"][t] for t in tokens)  # :451-463; the replace chain's text is discarded
        new_text = text[len(self.tgt_text):]
        self.tgt_text = text
        if self.states.source_finished and new_subword_tokens == -1:
            self.states.target_finished = True
            self.reset()
        return WriteAction(new_text, finished=self.states.target_finished)
