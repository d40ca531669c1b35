"""Model dimensions of the StreamSpeech simultaneous S2ST checkpoint family.

Every number here is a *default* taken from the reference's training recipe and arch
functions; a real checkpoint's `cfg` / vocoder `config.json` overrides them:

* encoder / decoder sizes: researches/ctc_unity/train_scripts/train.simul-s2st.sh:11-31,
  researches/ctc_unity/models/streamspeech_model.py:418-430,
  fairseq/fairseq/models/speech_to_speech/s2s_transformer.py:619-669
* multitask heads: configs/fr-en/config_mtl_asr_st_ctcst.yaml:1-36
* unit dictionary = 4 specials + 1000 units + <blank> (researches/ctc_unity/tasks/speech_to_speech_ctc.py:15-17)
* vocoder: public unit-HiFiGAN config (not in the reference tree; read from JSON at run time)
"""
from __future__ import annotations

import ctypes
import json
from dataclasses import dataclass, field, asdict
from typing import List


@dataclass
class VocoderConfig:
    upsample_rates: List[int] = field(default_factory=lambda: [5, 4, 4, 2, 2])
    upsample_kernel_sizes: List[int] = field(default_factory=lambda: [11, 8, 8, 4, 4])
    upsample_initial_channel: int = 512
    resblock_kernel_sizes: List[int] = field(default_factory=lambda: [3, 7, 11])
    resblock_dilation_sizes: List[List[int]] = field(
        default_factory=lambda: [[1, 3, 5], [1, 3, 5], [1, 3, 5]]
    )
    num_embeddings: int = 1000
    embedding_dim: int = 128
    model_in_dim: int = 128
    dur_hidden: int = 128  # dur_predictor_params.var_pred_hidden_dim
    dur_kernel: int = 3  # dur_predictor_params.var_pred_kernel_size

    @property
    def hop(self) -> int:
        h = 1
        for u in self.upsample_rates:
            h *= u
        return h

    def to_json_dict(self) -> dict:
        """Same schema as the reference vocoder `config.json` (agent/tts/codehifigan.py:9-33)."""
        return {
            "resblock": "1",
            "upsample_rates": self.upsample_rates,
            "upsample_kernel_sizes": self.upsample_kernel_sizes,
            "upsample_initial_channel": self.upsample_initial_channel,
            "resblock_kernel_sizes": self.resblock_kernel_sizes,
            "resblock_dilation_sizes": self.resblock_dilation_sizes,
            "num_embeddings": self.num_embeddings,
            "embedding_dim": self.embedding_dim,
            "model_in_dim": self.model_in_dim,
            "dur_predictor_params": {
                "encoder_embed_dim": self.embedding_dim,
                "var_pred_hidden_dim": self.dur_hidden,
                "var_pred_kernel_size": self.dur_kernel,
                "var_pred_dropout": 0.5,
            },
        }

    @staticmethod
    def from_json_dict(d: dict) -> "VocoderConfig":
        dp = d.get("dur_predictor_params") or {}
        return VocoderConfig(
            upsample_rates=list(d["upsample_rates"]),
            upsample_kernel_sizes=list(d["upsample_kernel_sizes"]),
            upsample_initial_channel=int(d["upsample_initial_channel"]),
            resblock_kernel_sizes=list(d["resblock_kernel_sizes"]),
            resblock_dilation_sizes=[list(x) for x in d["resblock_dilation_sizes"]],
            num_embeddings=int(d["num_embeddings"]),
            embedding_dim=int(d["embedding_dim"]),
            model_in_dim=int(d.get("model_in_dim", 80)),
            dur_hidden=int(dp.get("var_pred_hidden_dim", 128)),
            dur_kernel=int(dp.get("var_pred_kernel_size", 3)),
        )

    @staticmethod
    def from_json_file(path: str) -> "VocoderConfig":
        with open(path) as f:
            return VocoderConfig.from_json_dict(json.load(f))


UNITY_VARIANTS = ("unity", "uni_unity", "chunk_unity")
# the registered arch names of the UnitY family (researches/translatotron, researches/uni_unity, researches/chunk_unity and fairseq's own)
UNITY_ARCHS = {
    "unity_conformer_modified": "unity",
    "unity_conformer": "unity",
    "uni_unity_conformer": "uni_unity",
    "uni_unity_conformer_waitk": "uni_unity",
    "chunk_unity_conformer": "chunk_unity",
}
# stored settings the engine's Conformer encoder assumes (every recipe of the family trains with them), and their values
UNITY_FIXED_SETTINGS = (("pos_enc_type", "rel_pos"), ("attn_type", "espnet"), ("conv_version", "s2t_transformer"))


def unity_variant_of(get):
    """(unity_variant, uni_encoder, chunk_size) of a UnitY-family checkpoint from its stored model cfg (`get(key)`, None when
    absent).  A checkpoint without an arch is UnitY, as are unity_conformer_modified ones: both take the bidirectional encoder and T2U
    encoder whatever else is stored (their models read neither --uni-encoder nor --chunk-size).  Raises ValueError, naming the
    setting, for any arch or stored setting the engine does not reproduce."""
    arch = get("arch")
    if arch is not None and arch not in UNITY_ARCHS:
        raise ValueError(f"arch {arch!r}: not a UnitY-family model the engine runs (one of {', '.join(sorted(UNITY_ARCHS))})")
    for key, want in UNITY_FIXED_SETTINGS:
        have = get(key)
        if have is not None and have != want:
            raise ValueError(f"{key} {have!r}: the engine's encoder implements {key} {want!r} only")
    variant = UNITY_ARCHS.get(arch, "unity")
    if variant == "unity":
        return variant, False, 0
    uni = bool(get("uni_encoder") or False)
    if variant == "uni_unity":
        return variant, uni, 0
    chunk = get("chunk_size")
    if chunk is None or not 0 < int(chunk) < 999 or int(chunk) % 2:
        raise ValueError(f"chunk_size {chunk!r}: a chunk_unity_conformer checkpoint runs on the engine with an even --chunk-size "
                         "between 2 and 998 (its attention and convolution chunk)")
    return variant, uni, int(chunk)


@dataclass
class ModelConfig:
    # front-end
    feat_dim: int = 80
    # chunk-Conformer encoder
    enc_dim: int = 256
    enc_ffn: int = 2048
    enc_heads: int = 4
    enc_layers: int = 12
    dw_kernel: int = 31
    conv_channels: int = 1024  # subsampler mid channels
    conv_kernel: int = 5
    max_source_positions: int = 6000
    # CTC heads (ASR: source_unigram, ST: ctc_target_unigram) and MT dictionary
    src_vocab: int = 6000
    tgt_vocab: int = 6000
    # first-pass MT decoder (target_unigram)
    mt_dim: int = 512
    mt_ffn: int = 2048
    mt_heads: int = 8
    mt_layers: int = 4
    # T2U ("synthesizer") encoder
    t2u_layers: int = 2
    # NAR CTC unit decoder
    unit_dim: int = 512
    unit_ffn: int = 2048
    unit_heads: int = 8
    unit_layers: int = 2
    unit_vocab: int = 1005  # 4 specials + 1000 units + <blank>
    ctc_upsample_rate: int = 25
    # dictionary conventions (fairseq Dictionary: <s>=0 <pad>=1 </s>=2 <unk>=3)
    bos: int = 0
    pad: int = 1
    eos: int = 2
    unk: int = 3
    uni_encoder: bool = True  # --uni-encoder: causal T2U encoder
    # UnitY (researches/translatotron: unity_conformer_modified): no CTC heads, an autoregressive unit decoder over 4 specials +
    # 1000 units (no blank) searched token by token, whose sinusoidal positions cover max_target_positions
    unity: bool = False
    max_target_positions: int = 1024
    # which UnitY-family model (unity only; see UNITY_ARCHS): "unity" (bidirectional encoder), "uni_unity" (the Conformer with a
    # future mask on self-attention when uni_encoder is set, symmetric convolutions) or "chunk_unity" (StreamSpeech's chunk encoder at
    # the training --chunk-size, attention mask and convolutions alike).  uni_encoder makes the T2U encoder causal in both variants.
    unity_variant: str = "unity"
    chunk_size: int = 0  # chunk_unity: the training --chunk-size (encoder frames)
    vocoder: VocoderConfig = field(default_factory=VocoderConfig)

    @property
    def unit_blank(self) -> int:
        return self.unit_vocab - 1

    def encoder_chunk(self):
        """(attention chunk, conv chunk) of Engine.set_chunk for a UnitY-family model's whole-prefix encoder: (None, None) is the
        bidirectional encoder, (1, 0) a future mask with symmetric convolutions, (c, c) the chunk encoder of chunk size c"""
        assert self.unity
        if self.unity_variant == "uni_unity" and self.uni_encoder:
            return 1, 0
        if self.unity_variant == "chunk_unity":
            return self.chunk_size, self.chunk_size
        return None, None

    @staticmethod
    def from_state_dict(sd) -> "ModelConfig":
        """Infer the dimensions from a fairseq StreamSpeech or UnitY state dict (checkpoint `cfg` is hydra-pickled and
        not loadable without fairseq; every size is recoverable from tensor shapes).  A UnitY unit decoder's
        max_target_positions is not a shape: it stays 1024 here, use from_checkpoint to read it."""
        c = ModelConfig()
        c.conv_channels, c.feat_dim, c.conv_kernel = (int(x) for x in sd["encoder.subsample.conv_layers.0.weight"].shape)
        c.enc_dim = int(sd["encoder.linear.weight"].shape[0])
        c.enc_ffn = int(sd["encoder.conformer_layers.0.ffn1.w_1.weight"].shape[0])
        c.enc_heads = int(sd["encoder.conformer_layers.0.self_attn.pos_bias_u"].shape[0])
        c.dw_kernel = int(sd["encoder.conformer_layers.0.conv_module.depthwise_conv.weight"].shape[-1])
        n = lambda prefix: 1 + max(int(k[len(prefix):].split(".")[0]) for k in sd if k.startswith(prefix))  # noqa: E731
        c.enc_layers = n("encoder.conformer_layers.")
        c.tgt_vocab, c.mt_dim = (int(x) for x in sd["target_unigram_decoder.embed_tokens.weight"].shape)
        heads = [k in sd for k in ("source_unigram_decoder.proj.weight", "ctc_target_unigram_decoder.proj.weight")]
        if any(heads) and not all(heads):
            raise KeyError("a StreamSpeech state dict needs both CTC heads (source_unigram_decoder.proj, ctc_target_unigram_decoder.proj); "
                           "a UnitY one has neither")
        c.unity = not any(heads)
        c.src_vocab = c.tgt_vocab if c.unity else int(sd["source_unigram_decoder.proj.weight"].shape[0])
        c.mt_ffn = int(sd["target_unigram_decoder.layers.0.fc1.weight"].shape[0])
        c.mt_heads = c.mt_dim // 64
        c.mt_layers = n("target_unigram_decoder.layers.")
        c.t2u_layers = n("synthesizer_encoder.layers.")
        c.unit_vocab, c.unit_dim = (int(x) for x in sd["decoder.embed_tokens.weight"].shape)
        c.unit_ffn = int(sd["decoder.layers.0.fc1.weight"].shape[0])
        c.unit_heads = c.unit_dim // 64
        c.unit_layers = n("decoder.layers.")
        if c.unity:
            c.uni_encoder = False  # TransformerEncoderNoEmb: bidirectional
        return c

    @staticmethod
    def from_checkpoint(state) -> "ModelConfig":
        """from_state_dict(state["model"]) plus what only the checkpoint's stored cfg carries: a UnitY unit decoder's
        max_target_positions (state["cfg"]["model"], or state["args"] in older checkpoints; fairseq's default 1024 when absent).
        The released UnitY checkpoints were trained with --max-target-positions 1200, which sets the unit search's length limit."""
        c = ModelConfig.from_state_dict(state["model"])
        if c.unity:
            def get(o, k):
                return None if o is None else (o.get(k) if isinstance(o, dict) else getattr(o, k, None))

            model_cfg = get(get(state, "cfg"), "model") or get(state, "args")
            c.max_target_positions = int(get(model_cfg, "max_target_positions") or 1024)
            c.unity_variant, c.uni_encoder, c.chunk_size = unity_variant_of(lambda k: get(model_cfg, k))
        return c

    @staticmethod
    def unity_default(variant: str = "unity") -> "ModelConfig":
        """The released UnitY checkpoints' dimensions (unity.{fr,es,de}-en.pt): StreamSpeech's encoder, MT decoder and T2U encoder,
        and a 2-layer autoregressive unit decoder over 1004 symbols with 1200 positions.  `variant` "uni_unity" / "chunk_unity" is the
        same model with the training recipes' --uni-encoder (and --chunk-size 8) of researches/{uni,chunk}_unity/train_scripts."""
        if variant not in UNITY_VARIANTS:
            raise ValueError(f"unknown UnitY variant {variant!r}; one of {', '.join(UNITY_VARIANTS)}")
        c = ModelConfig()
        c.unity, c.uni_encoder, c.unit_vocab, c.max_target_positions = True, False, 1004, 1200
        c.unity_variant = variant
        if variant != "unity":
            c.uni_encoder = True
        if variant == "chunk_unity":
            c.chunk_size = 8
        return c

    def tiny(self) -> "ModelConfig":
        """A shrunken variant with the same structure (used by fast CPU tests)."""
        c = ModelConfig(**{k: v for k, v in asdict(self).items() if k != "vocoder"})
        c.enc_layers = 2
        c.mt_layers = 1
        c.t2u_layers = 1
        c.unit_layers = 1
        c.vocoder = VocoderConfig()
        return c
