"""TEST INFRASTRUCTURE (CPU oracle) -- not part of the product path.

The CPU restatements of UnitY (oracle.unity_oracle, oracle.waitk_oracle) for the two other models of the family, which share its
state-dict keys and differ only in masks (ModelConfig.unity_variant):

  Uni-UnitY    researches/uni_unity: the Conformer encoder with a future mask on self-attention when --uni-encoder is set
               (uni_unity/models/s2t_conformer.py:97,132-133,170-182; espnet_multihead_attention.py:197-205), i.e. the chunk mask of
               chunk size 1, with the subsampler and depthwise convolutions left symmetric (CausalConv1d is commented out,
               conformer_layer.py:71-82); a causal T2U encoder (uni_unity/modules/transformer_encoder.py:29,36-37)
  Chunk-UnitY  researches/chunk_unity: StreamSpeech's ChunkS2TConformerEncoder at the training --chunk-size, for the attention mask
               and the chunk-causal convolutions alike (chunk_unity/models/s2t_conformer.py:52-100,195-213); its future mask is
               commented out (:144), so --uni-encoder makes only the T2U encoder causal (s2s_conformer_chunk_unity.py:249)

The decoders and searches are UnitY's.  Every class takes `dtype` (float32 restates the reference, float64 gives margins).
"""
from __future__ import annotations

from dataclasses import replace

import torch

from .unity_oracle import UnitYOracle
from .waitk_oracle import OracleWaitkS2STAgent, OracleWaitkS2TTAgent


def oracle_geometry(cfg):
    """(chunk_size, conv_chunk_size) of StreamSpeechOracle for the model's encoder: None = no attention mask / plain convolutions"""
    if cfg.unity_variant == "uni_unity" and cfg.uni_encoder:
        return 1, None
    if cfg.unity_variant == "chunk_unity":
        return cfg.chunk_size, cfg.chunk_size
    return None, None


def configure(o, cfg):
    """point a StreamSpeechOracle at the variant: its encoder masks and the T2U encoder's causality (cfg.uni_encoder)"""
    o.cfg = cfg
    o.chunk_size, o.conv_chunk_size = oracle_geometry(cfg)


def _unity_base(cfg):
    return replace(cfg, uni_encoder=False)  # what UnitYOracle's constructor accepts; configure() restores the variant


class VariantUnitYOracle(UnitYOracle):
    def __init__(self, cfg, model_sd, dtype: torch.dtype = torch.float32, device="cpu"):
        super().__init__(_unity_base(cfg), model_sd, dtype, device)
        self.cfg = cfg
        configure(self.o, cfg)


class VariantWaitkS2STAgent(OracleWaitkS2STAgent):
    def __init__(self, cfg, sd, gcmvn, vsd, **kw):
        super().__init__(_unity_base(cfg), sd, gcmvn, vsd, **kw)
        self.cfg = cfg
        configure(self.o, cfg)
        self.u = VariantUnitYOracle(cfg, sd, self.o.dtype)


class VariantWaitkS2TTAgent(OracleWaitkS2TTAgent):
    def __init__(self, cfg, sd, gcmvn, vsd=None, **kw):
        super().__init__(_unity_base(cfg), sd, gcmvn, vsd, **kw)
        self.cfg = cfg
        configure(self.o, cfg)
