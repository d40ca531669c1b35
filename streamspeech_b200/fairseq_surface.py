"""The fairseq model surface of StreamSpeech on top of the H100 engine (SURVEY.md §8b(ii)).

The reference agents never call kernels directly: they poke attributes of a fairseq model object and call its sub-modules
(agent/speech_to_speech.streamspeech.agent.py:395-413,433,520-538,638-689).  `StreamSpeechB200Model` offers exactly those
attributes as thin `nn.Module` shims whose `forward()` runs the engine:

  model.encoder.chunk_size = c                                         (agent:404)            -> ss_set_chunk
  model.encoder.subsample.conv_layers[i].chunk_size = cc               (agent:410-411)        -> ss_set_chunk
  model.encoder.conformer_layers[i].conv_module.depthwise_conv.chunk_size = cc  (agent:412-413)
  model.encoder(src_tokens [B,F,80], src_lengths [B]) -> {"encoder_out": [T x B x C], "encoder_padding_mask": [B x T] or [], ...}
                                                                        (chunk_unity/models/s2t_conformer.py:154-163)
  model.mt_task_name, getattr(model, f"{task}_decoder"), model.synthesizer_encoder, model.decoder,
  model.get_normalized_probs, model.max_decoder_positions()             (streamspeech_model.py:182-258)

so a maintainer can hand this object to the reference's own agent / generators (INTEGRATION.md path B) without editing them.
`register_with_fairseq()` registers the class as model "streamspeech_b200" (+ arch of the same name) when fairseq is importable,
mirroring `@register_model("streamspeech")` / `@register_model_architecture` (streamspeech_model.py:57,418).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F


class _ChunkHolder(nn.Module):
    """a module whose only job is the `chunk_size` attribute the agents assign (ChunkCausalConv1d.chunk_size)"""

    def __init__(self, owner: "B200Encoder", role: str):
        super().__init__()
        object.__setattr__(self, "_owner", owner)
        object.__setattr__(self, "_role", role)
        object.__setattr__(self, "_chunk", None)

    @property
    def chunk_size(self):
        return self._chunk

    @chunk_size.setter
    def chunk_size(self, v):
        object.__setattr__(self, "_chunk", None if v is None else int(v))
        self._owner._conv_chunk_changed(v)


class _ConvModule(nn.Module):
    def __init__(self, owner):
        super().__init__()
        self.depthwise_conv = _ChunkHolder(owner, "depthwise")


class _LayerShim(nn.Module):
    def __init__(self, owner):
        super().__init__()
        self.conv_module = _ConvModule(owner)


class _Subsample(nn.Module):
    def __init__(self, owner, n_layers=2):
        super().__init__()
        self.conv_layers = nn.ModuleList([_ChunkHolder(owner, "subsample") for _ in range(n_layers)])


class B200Encoder(nn.Module):
    """ChunkS2SConformerEncoder (chunk_unity/models/s2s_conformer.py:37-62) surface over ss_encoder_forward."""

    def __init__(self, engine, cfg):
        super().__init__()
        object.__setattr__(self, "_engine", engine)
        self.cfg = cfg
        object.__setattr__(self, "_attn_chunk", None)
        object.__setattr__(self, "_conv_chunk", None)
        self.subsample = _Subsample(self)
        self.conformer_layers = nn.ModuleList([_LayerShim(self) for _ in range(cfg.enc_layers)])

    # encoder.chunk_size (agent:404); None / >= 999 = offline model (N10)
    @property
    def chunk_size(self):
        return self._attn_chunk

    @chunk_size.setter
    def chunk_size(self, v):
        object.__setattr__(self, "_attn_chunk", None if v is None else int(v))
        self._push()

    def _conv_chunk_changed(self, v):
        object.__setattr__(self, "_conv_chunk", None if v is None else int(v))
        self._push()

    def _push(self):
        a, c = self._attn_chunk, self._conv_chunk
        offline = a is None or a >= 999
        if offline:
            self._engine.set_chunk(None)
        else:
            self._engine.set_chunk(a, c if c is not None else (16 if a >= 16 else 8))

    def forward(self, src_tokens: torch.Tensor, src_lengths: Optional[torch.Tensor] = None, **kw) -> Dict[str, List[torch.Tensor]]:
        eng = self._engine
        x = src_tokens.to(device=eng.device, dtype=torch.float32).contiguous()
        B, Fr, _ = x.shape
        lens = None if src_lengths is None else [int(v) for v in src_lengths.tolist()]
        out = eng.encoder(x, lens)  # [B, T, C]
        T = out.shape[1]
        masks: List[torch.Tensor] = []
        if lens is not None:
            tl = torch.tensor([eng.encoder_out_frames(v) for v in lens], device=out.device)
            m = torch.arange(T, device=out.device)[None, :] >= tl[:, None]
            if bool(m.any()):
                masks = [m]
        return {"encoder_out": [out.transpose(0, 1)], "encoder_padding_mask": masks, "encoder_embedding": [], "encoder_states": [],
                "src_tokens": [], "src_lengths": []}

    def forward_torchscript(self, net_input: Dict[str, torch.Tensor]):  # fairseq/models/fairseq_encoder.py
        return self.forward(net_input["src_tokens"], net_input.get("src_lengths"))

    def reorder_encoder_out(self, encoder_out, new_order):
        return {"encoder_out": [x.index_select(1, new_order) for x in encoder_out["encoder_out"]],
                "encoder_padding_mask": [x.index_select(0, new_order) for x in encoder_out["encoder_padding_mask"]],
                "encoder_embedding": [], "encoder_states": [], "src_tokens": [], "src_lengths": []}


class B200CTCDecoder(nn.Module):
    """CTCDecoder (fairseq/models/speech_to_speech/modules/ctc_decoder.py:11-18): Linear enc_dim -> vocab over [T,B,C]."""

    def __init__(self, engine, weight: torch.Tensor, bias: torch.Tensor):
        super().__init__()
        object.__setattr__(self, "_engine", engine)
        self.register_buffer("weight", weight.to(engine.device).float().contiguous(), persistent=False)
        self.register_buffer("bias", bias.to(engine.device).float().contiguous(), persistent=False)

    def forward(self, src_tokens, src_lengths=None, **kw):
        x = src_tokens  # the reference passes encoder_out["encoder_out"][0]: [T, B, C]
        T, B, C = x.shape
        y = self._engine.op_linear(x.reshape(T * B, C).contiguous().float(), self.weight, self.bias)
        return {"encoder_out": y.view(T, B, -1)}


class B200MTDecoder(nn.Module):
    """first-pass TransformerDecoder (ctc_unity/modules/transformer_decoder.py:39-523) surface: forward(prev_output_tokens,
    encoder_out, features_only) -> (x [B,L,C or V], {"attn": [None], "inner_states": []}); batch 1 (the streaming agents)."""

    padding_idx = 1

    def __init__(self, engine, cfg):
        super().__init__()
        object.__setattr__(self, "_engine", engine)
        self.cfg = cfg
        self.padding_idx = cfg.pad

    def forward(self, prev_output_tokens, encoder_out=None, features_only=False, **kw):
        if prev_output_tokens.shape[0] != 1:
            raise NotImplementedError("B200MTDecoder.forward is the batch-1 surface of the streaming agents")
        enc = encoder_out["encoder_out"][0][:, 0].contiguous()  # [T, C]
        toks = [int(t) for t in prev_output_tokens[0].tolist()]
        feats = self._engine.mt_features(enc, toks)
        if features_only:
            return feats.unsqueeze(0), {"attn": [None], "inner_states": []}
        raise NotImplementedError("logits of every position are not part of the agents' path (they call generate_decoder -> ss_mt_greedy)")


class StreamSpeechB200Model(nn.Module):
    """The attribute surface of StreamSpeechModel (researches/ctc_unity/models/streamspeech_model.py:57-258)."""

    mt_task_name = "target_unigram"

    def __init__(self, engine, cfg, model_sd: Dict[str, torch.Tensor]):
        super().__init__()
        object.__setattr__(self, "engine", engine)
        self.cfg = cfg
        self.encoder = B200Encoder(engine, cfg)
        self.source_unigram_decoder = B200CTCDecoder(engine, model_sd["source_unigram_decoder.proj.weight"], model_sd["source_unigram_decoder.proj.bias"])
        self.ctc_target_unigram_decoder = B200CTCDecoder(engine, model_sd["ctc_target_unigram_decoder.proj.weight"],
                                                         model_sd["ctc_target_unigram_decoder.proj.bias"])
        self.target_unigram_decoder = B200MTDecoder(engine, cfg)

    @classmethod
    def from_checkpoint(cls, model_sd, vocoder_sd=None, gcmvn=None, device: int = 0, **kw):
        from streamspeech_b200.config import ModelConfig
        from streamspeech_b200.engine import Engine

        cfg = ModelConfig.from_state_dict(model_sd)
        return cls(Engine(cfg, model_sd, vocoder_sd, gcmvn, device=device, **kw), cfg, model_sd)

    def max_decoder_positions(self):
        return 1200

    def get_normalized_probs(self, net_output, log_probs, sample=None):
        logits = net_output[0].float()
        return F.log_softmax(logits, dim=-1) if log_probs else F.softmax(logits, dim=-1)

    def forward_encoder(self, net_input):  # EnsembleModel.forward_encoder's per-model call
        return self.encoder.forward_torchscript(net_input)


def register_with_fairseq() -> bool:
    """@register_model("streamspeech_b200") + architecture, when fairseq is importable (streamspeech_model.py:57,418-430)."""
    try:
        from fairseq.models import register_model, register_model_architecture  # type: ignore
    except Exception:  # noqa: BLE001 -- fairseq is not installable in the build image (DESIGN.md)
        return False
    register_model("streamspeech_b200")(StreamSpeechB200Model)

    def _arch(args):
        return None

    register_model_architecture("streamspeech_b200", "streamspeech_b200")(_arch)
    return True
