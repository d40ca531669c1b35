"""ctypes binding of libstreamspeech_b200.so (include/streamspeech_b200.h): PyTorch tensors in, PyTorch tensors out.

PyTorch is plumbing here (device memory, streams); every FLOP of the path runs in the library's own
sm_90a kernels.  There is NO CPU fallback: importing this module without the built library, or
constructing an Engine without a CUDA device, raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import constants
from .config import ModelConfig

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstreamspeech_b200.so")
SS_MAX_UPS, SS_MAX_RB, SS_MAX_DIL = 8, 4, 4


class SSConfig(ctypes.Structure):
    _fields_ = (
        [(n, ctypes.c_int32) for n in (
            "feat_dim", "enc_dim", "enc_ffn", "enc_heads", "enc_layers", "dw_kernel", "conv_channels", "conv_kernel",
            "src_vocab", "tgt_vocab", "mt_dim", "mt_ffn", "mt_heads", "mt_layers",
            "t2u_layers", "unit_dim", "unit_ffn", "unit_heads", "unit_layers", "unit_vocab", "ctc_upsample_rate",
            "bos", "pad", "eos", "unk", "uni_encoder", "max_enc_frames", "max_mt_positions", "voc_n_ups")]
        + [("voc_up_rates", ctypes.c_int32 * SS_MAX_UPS), ("voc_up_kernels", ctypes.c_int32 * SS_MAX_UPS),
           ("voc_init_channels", ctypes.c_int32), ("voc_n_rb", ctypes.c_int32),
           ("voc_rb_kernels", ctypes.c_int32 * SS_MAX_RB), ("voc_rb_ndil", ctypes.c_int32),
           ("voc_rb_dils", (ctypes.c_int32 * SS_MAX_DIL) * SS_MAX_RB)]
        + [(n, ctypes.c_int32) for n in ("voc_num_embeddings", "voc_embedding_dim", "voc_in_dim", "voc_dur_hidden", "voc_dur_kernel")]
    )


SS_ERR_CAPACITY = -5
SS_ASR_MAX_CONV = 8
SS_ASR_BATCH_ROWS = 8192


class ASRConfig(ctypes.Structure):
    _fields_ = [("n_conv", ctypes.c_int32), ("conv_stride", ctypes.c_int32 * SS_ASR_MAX_CONV)] + [
        (n, ctypes.c_int32) for n in ("extractor_layer_norm", "layer_norm_first", "pos_conv_depth", "conformer", "heads", "normalize",
                                      "max_frames", "time_stages")]


_P, _I, _F = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float


class GemmArgs(ctypes.Structure):
    """ctypes mirror of `struct ss_op_gemm_args` (the ss_op_gemm parity hook)"""
    _fields_ = (
        [("x", _P), ("lengths", _P)]
        + [(n, _I) for n in ("B", "L_in", "L_rows", "C_in", "ldx", "ksize", "stride", "dil", "pad_left", "chunk")]
        + [("pre_lrelu", _F)]
        + [(n, _I) for n in ("t_offset", "x_row0", "x_rows", "k_tiles_per_split")]
        + [("w", _P), ("N", _I), ("bias", _P), ("act", _I), ("glu", _I), ("alpha", _F), ("residual", _P), ("res_scale", _F),
           ("accumulate", _I), ("out", _P)]
        + [(n, _I) for n in ("ldo", "out_L", "out_row_stride", "out_row_offset")]
        + [("ln_gamma", _P), ("ln_beta", _P), ("split_n", _I), ("out2", _P), ("out3", _P), ("ldo2", _I), ("ldo3", _I),
           ("kernel", _I), ("splitk", _I)]
        + [(n, _I) for n in ("route_kernel", "route_bm", "route_bn", "route_splits", "route_mr", "route_ks", "route_cpt", "route_grid",
                             "route_u_bn", "route_u_ck", "route_u_upt", "route_u_sb")]
    )


class EngineError(RuntimeError):
    """code: the ss_status of a failed library call (None for errors raised on the host side); detail: the library's message"""

    def __init__(self, message: str, code: Optional[int] = None, detail: str = ""):
        super().__init__(message)
        self.code, self.detail = code, detail


_lib = None


def load_library() -> ctypes.CDLL:
    """Load the in-tree shared library; raise loudly if it has not been built (`python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EngineError(f"{LIB_PATH} is missing: build it with `make -C streamspeech_b200/csrc` "
                          "(or __graft_entry__.build()).  There is no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    lib.ss_create.argtypes = [ctypes.POINTER(vp), i32, ctypes.POINTER(SSConfig)]
    lib.ss_destroy.argtypes = [vp]
    lib.ss_last_error.argtypes = [vp]
    lib.ss_last_error.restype = ctypes.c_char_p
    lib.ss_version.restype = ctypes.c_char_p
    lib.ss_load_tensor.argtypes = [vp, ctypes.c_char_p, vp, i32, ctypes.POINTER(i64)]
    lib.ss_finalize.argtypes = [vp]
    lib.ss_set_chunk.argtypes = [vp, i32, i32]
    lib.ss_fbank_num_frames.argtypes = [i64]
    lib.ss_fbank_num_frames.restype = i64
    lib.ss_encoder_out_frames.argtypes = [i64]
    lib.ss_encoder_out_frames.restype = i64
    lib.ss_fbank.argtypes = [vp, vp, vp, i64, i64, i64, vp]
    lib.ss_encoder_forward.argtypes = [vp, vp, vp, vp, i32, i32, vp]
    lib.ss_encoder_stream_reset.argtypes = [vp]
    lib.ss_encoder_stream_step.argtypes = [vp, vp, vp, i32, vp, ctypes.POINTER(i32), ctypes.POINTER(i32)]
    lib.ss_ctc_greedy.argtypes = [vp, vp, i32, vp, i32, vp, vp, vp, vp]
    lib.ss_ctc_greedy_rows.argtypes = [vp, vp, i32, vp, i32, i32, vp, vp, vp, vp]
    lib.ss_ctc_greedy_pair.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp]
    lib.ss_mt_greedy.argtypes = [vp, vp, vp, i32, vp, i32, i32, i32, vp, i32, ctypes.POINTER(i32), vp]
    lib.ss_mt_greedy_batch.argtypes = [vp, vp, vp, i32, i32, vp, i32, vp, i32, vp]
    lib.ss_mt_beam_batch.argtypes = [vp, vp, vp, i32, i32, vp, i32, i32, ctypes.c_float, vp, i32, vp, vp, vp]
    lib.ss_mt_stable_rows.argtypes = [vp, i32]
    lib.ss_mt_incremental_reset.argtypes = [vp]
    lib.ss_mt_greedy_incremental.argtypes = [vp, vp, vp, i32, vp, i32, i32, i32, vp, i32, ctypes.POINTER(i32)]
    lib.ss_mt_features.argtypes = [vp, vp, vp, i32, vp, i32, vp, vp]
    lib.ss_t2u_unit_decode.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp]
    lib.ss_ctc_greedy_batch.argtypes = [vp, vp, vp, i32, i32, vp]
    lib.ss_mt_features_batch.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, vp]
    lib.ss_t2u_unit_decode_batch.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, vp, vp]
    lib.ss_t2u_unit_decode_batch_scored.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, vp, vp, vp]
    lib.ss_unit_position_row.argtypes = [vp, vp]
    lib.ss_vocoder_durations.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    lib.ss_vocoder_generate.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    lib.ss_vocoder_durations_ragged.argtypes = [vp, vp, i32, vp, vp, i32, vp, vp]
    lib.ss_vocoder_generate_ragged.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    lib.ss_vocoder_hop.argtypes = [vp]
    lib.ss_vocoder_receptive_field.argtypes = [vp]
    lib.ss_op_linear.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, i32, vp]
    lib.ss_op_linear_umma.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, i32, i32, vp]
    lib.ss_op_conv1d.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, i32, i32, i32, ctypes.c_float, i32, vp]
    lib.ss_set_option.argtypes = [vp, ctypes.c_char_p, i32]
    lib.ss_op_layer_norm.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp, i32]
    lib.ss_op_gemm.argtypes = [vp, vp, ctypes.POINTER(GemmArgs)]
    lib.ss_op_argmax_rows.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp, vp]
    lib.ss_debug_copy.argtypes = [vp, ctypes.c_char_p, vp, ctypes.c_size_t]
    lib.ss_launch_count.argtypes = [vp]
    lib.ss_launch_count.restype = i64
    lib.ss_async_error.argtypes = [vp]
    lib.ss_resample_out_len.argtypes = [i64, i32]
    lib.ss_resample_out_len.restype = i64
    lib.ss_resample_48k_to_16k.argtypes = [vp, vp, vp, i64, i64, i64, vp]
    lib.ss_pool_create.argtypes = [vp, i32, i32]
    lib.ss_pool_create_rate.argtypes = [vp, i32, i32, i32]
    lib.ss_pool_reset.argtypes = [vp, i32]
    lib.ss_pool_finish.argtypes = [vp, i32]
    lib.ss_pool_set_chunk.argtypes = [vp, i32, i32, i32]
    lib.ss_pool_push_audio.argtypes = [vp, vp, i32, vp, i32]
    lib.ss_pool_info.argtypes = [vp, i32, ctypes.POINTER(i64), ctypes.POINTER(i32), ctypes.POINTER(i32), ctypes.POINTER(vp), ctypes.POINTER(vp)]
    lib.ss_pool_step.argtypes = [vp, vp, i32, vp, i32, vp, i64, vp, vp, vp]
    lib.ss_pool_mt_greedy.argtypes = [vp, vp, i32, vp, vp, vp, vp, i32, vp, i32, vp, vp, i32]
    lib.ss_pool_mt_greedy_incremental.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp, vp, i32, vp]
    lib.ss_t2u_unit_decode_ragged.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, i32, vp, vp]
    lib.ss_t2u_encode_batch.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    lib.ss_unit_search_batch.argtypes = [vp, vp, vp, i32, i32, vp, i32, ctypes.c_float, vp, i32, vp, vp, vp]
    f32 = ctypes.c_float
    lib.ss_op_relpos_attention.argtypes = [vp, vp, vp, i32, vp, i32, vp, i32, vp, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, i32]
    lib.ss_op_mha_attention.argtypes = [vp, vp, vp, i32, vp, i32, vp, i32, vp, i32, i32, i32, i32, i32, f32, i32, i32, vp, i32]
    lib.ss_op_grouped_causal_attention.argtypes = [vp, vp, vp, i32, vp, i32, vp, i32, vp, i32, i32, i32, i32, f32, i32, vp]
    lib.ss_op_depthwise_bn_silu.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32]
    lib.ss_op_ms_relpos_attention.argtypes = [vp, vp, vp, i32, vp, vp, i64, i32, vp, i32, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.ss_op_ms_depthwise.argtypes = [vp, vp, vp, i64, i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.ss_asr_create.argtypes = [ctypes.POINTER(vp), i32, ctypes.POINTER(ASRConfig)]
    lib.ss_asr_destroy.argtypes = [vp]
    lib.ss_asr_last_error.argtypes = [vp]
    lib.ss_asr_last_error.restype = ctypes.c_char_p
    lib.ss_asr_load_tensor.argtypes = [vp, ctypes.c_char_p, vp, i32, ctypes.POINTER(i64)]
    lib.ss_asr_finalize.argtypes = [vp]
    lib.ss_asr_num_frames.argtypes = [vp, i64]
    lib.ss_asr_num_frames.restype = i64
    lib.ss_asr_transcribe.argtypes = [vp, vp, vp, vp, i32, vp, i64, vp, vp]
    lib.ss_asr_debug_stage.argtypes = [vp, vp, vp, vp, i32, i32, vp]
    lib.ss_asr_stage_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_double)]
    _lib = lib
    return lib


EXPORTED_SYMBOLS = [
    "ss_asr_create", "ss_asr_destroy", "ss_asr_last_error", "ss_asr_load_tensor", "ss_asr_finalize", "ss_asr_num_frames", "ss_asr_transcribe",
    "ss_asr_debug_stage", "ss_asr_stage_ms",
    "ss_create", "ss_destroy", "ss_last_error", "ss_version", "ss_load_tensor", "ss_finalize", "ss_set_chunk",
    "ss_fbank_num_frames", "ss_fbank", "ss_encoder_out_frames", "ss_encoder_forward", "ss_encoder_stream_reset", "ss_encoder_stream_step", "ss_ctc_greedy", "ss_ctc_greedy_rows", "ss_mt_greedy",
    "ss_mt_features", "ss_mt_stable_rows", "ss_t2u_unit_decode", "ss_unit_position_row", "ss_vocoder_durations", "ss_vocoder_generate", "ss_vocoder_durations_ragged", "ss_vocoder_generate_ragged", "ss_vocoder_hop",
    "ss_vocoder_receptive_field", "ss_op_linear", "ss_op_linear_umma", "ss_op_conv1d", "ss_set_option", "ss_debug_copy", "ss_op_layer_norm", "ss_launch_count", "ss_async_error", "ss_mt_incremental_reset", "ss_mt_greedy_incremental", "ss_ctc_greedy_pair", "ss_resample_out_len", "ss_resample_48k_to_16k", "ss_pool_create", "ss_pool_reset", "ss_pool_push_audio", "ss_pool_info", "ss_pool_step",
    "ss_pool_create_rate", "ss_pool_finish", "ss_pool_set_chunk", "ss_mt_greedy_batch", "ss_mt_beam_batch", "ss_ctc_greedy_batch", "ss_mt_features_batch",
    "ss_t2u_unit_decode_batch", "ss_pool_mt_greedy", "ss_pool_mt_greedy_incremental", "ss_t2u_unit_decode_ragged", "ss_op_relpos_attention", "ss_op_mha_attention",
    "ss_op_grouped_causal_attention", "ss_op_depthwise_bn_silu", "ss_op_ms_relpos_attention", "ss_op_ms_depthwise",
    "ss_t2u_unit_decode_batch_scored", "ss_op_argmax_rows", "ss_t2u_encode_batch", "ss_unit_search_batch",
    "ss_op_gemm",
]


def _i32_array(xs: Optional[Sequence[int]]):
    return None if xs is None else (ctypes.c_int32 * max(len(xs), 1))(*[int(x) for x in xs])


def make_ss_config(cfg: ModelConfig, max_enc_frames: int, max_mt_positions: int = 1024) -> SSConfig:
    c = SSConfig()
    for n in ("feat_dim", "enc_dim", "enc_ffn", "enc_heads", "enc_layers", "dw_kernel", "conv_channels", "conv_kernel",
              "src_vocab", "tgt_vocab", "mt_dim", "mt_ffn", "mt_heads", "mt_layers", "t2u_layers", "unit_dim", "unit_ffn",
              "unit_heads", "unit_layers", "unit_vocab", "ctc_upsample_rate", "bos", "pad", "eos", "unk"):
        setattr(c, n, int(getattr(cfg, n)))
    c.uni_encoder = int(cfg.uni_encoder)
    c.max_enc_frames = max_enc_frames
    c.max_mt_positions = max_mt_positions
    v = cfg.vocoder
    c.voc_n_ups = len(v.upsample_rates)
    for i, (u, k) in enumerate(zip(v.upsample_rates, v.upsample_kernel_sizes)):
        c.voc_up_rates[i], c.voc_up_kernels[i] = u, k
    c.voc_init_channels = v.upsample_initial_channel
    c.voc_n_rb = len(v.resblock_kernel_sizes)
    c.voc_rb_ndil = len(v.resblock_dilation_sizes[0])
    for j, (k, dils) in enumerate(zip(v.resblock_kernel_sizes, v.resblock_dilation_sizes)):
        c.voc_rb_kernels[j] = k
        assert len(dils) == c.voc_rb_ndil
        for m, d in enumerate(dils):
            c.voc_rb_dils[j][m] = d
    c.voc_num_embeddings, c.voc_embedding_dim, c.voc_in_dim = v.num_embeddings, v.embedding_dim, v.model_in_dim
    c.voc_dur_hidden, c.voc_dur_kernel = v.dur_hidden, v.dur_kernel
    return c


def remove_weight_norm(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """`model.remove_weight_norm()` at vocoder load (agent/tts/vocoder.py:45): w = v * (g / ||v||)."""
    out = dict(sd)
    for k in list(sd.keys()):
        if k.endswith(".weight_g"):
            base = k[: -len(".weight_g")]
            g, v = sd[k].float(), sd[base + ".weight_v"].float()
            norm = v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))
            out[base + ".weight"] = v * (g / norm)
            del out[k], out[base + ".weight_v"]
    return out


def ctc_record(host: torch.Tensor, off: int, T: int) -> Tuple[List[int], List[int]]:
    """(tokens, index) of the packed CTC record [count (int32 in the first int64) | tokens[T] | index[T] (int32)] at host[off:]"""
    row = host[off:off + 2 * T + 2]
    n = int(row[:1].view(torch.int32)[0])
    return row[1:1 + n].tolist(), row[1 + T:].view(torch.int32)[:n].tolist()


class Engine:
    """One model replica on one GPU.  Not thread-safe (one host thread per handle)."""

    def __init__(self, cfg: ModelConfig, model_sd: Dict[str, torch.Tensor], vocoder_sd: Optional[Dict[str, torch.Tensor]] = None,
                 gcmvn: Optional[dict] = None, device: int = 0, max_enc_frames: int = 1024, max_mt_positions: int = 1024):
        if not torch.cuda.is_available():
            raise EngineError("streamspeech_b200.Engine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = load_library()
        self.cfg = cfg
        self.device = torch.device("cuda", device)
        self.max_mt_positions = max_mt_positions
        self._h = ctypes.c_void_p()
        sc = make_ss_config(cfg, max_enc_frames, max_mt_positions)
        rc = self.lib.ss_create(ctypes.byref(self._h), device, ctypes.byref(sc))
        if rc != 0:
            raise EngineError(f"ss_create failed with {rc}: {self.lib.ss_last_error(None).decode()}")
        try:
            for k, v in model_sd.items():
                if v.is_floating_point():
                    self._load(k, v)
            if vocoder_sd is not None:
                for k, v in remove_weight_norm(vocoder_sd).items():
                    self._load("vocoder." + k, v)
            self._load("__const__.mel_bank", constants.mel_bank())
            self._load("__const__.window", constants.povey_window())
            self._load("__const__.resample_3to1", constants.resample_kernel_3to1()[0])
            self._load("__const__.enc_pe", constants.rel_pos_table(max_enc_frames, cfg.enc_dim))
            self._load("__const__.mt_pos_table", constants.sinusoidal_table(max_mt_positions + cfg.pad + 2, cfg.mt_dim, cfg.pad))
            self._load("__const__.unit_pos_row", constants.sinusoidal_table(cfg.pad + 4, cfg.unit_dim, cfg.pad)[cfg.pad + 1])
            if cfg.unity:  # the autoregressive unit decoder's positions (SinusoidalPositionalEmbedding of max_target_positions)
                self._load("__const__.unit_pos_table", constants.sinusoidal_table(cfg.max_target_positions + cfg.pad + 1, cfg.unit_dim, cfg.pad))
            if gcmvn is not None:
                self._load("__const__.gcmvn_mean", torch.as_tensor(gcmvn["mean"], dtype=torch.float32))
                self._load("__const__.gcmvn_std", torch.as_tensor(gcmvn["std"], dtype=torch.float32))
            self._check(self.lib.ss_finalize(self._h))
        except Exception:
            self.close()
            raise
        # tensor-core routing (kernels_umma2.cu): vocoder convs tolerate the 3-MMA split (1e-3 waveform bar, measured 7e-6);
        # linears that feed an arg-max stay on the exact fp32 kernels unless explicitly switched on
        self.set_option("umma_vocoder", int(os.environ.get("SS_UMMA_VOCODER", "12")))
        self.set_option("umma_linear", int(os.environ.get("SS_UMMA_LINEAR", "13")))
        self.set_option("umma_min_rows", int(os.environ.get("SS_UMMA_MIN_ROWS", "128")))
        self.set_option("umma_min_channels", int(os.environ.get("SS_UMMA_MIN_CHANNELS", "16")))
        self.set_option("persistent_encoder", int(os.environ.get("SS_PERSISTENT_ENCODER", "1")))
        self.set_option("persistent_mt", int(os.environ.get("SS_PERSISTENT_MT", "1")))
        self.set_option("fbank_tma", int(os.environ.get("SS_FBANK_TMA", "1")))
        self.set_option("persistent_ffn_fused", int(os.environ.get("SS_PERSISTENT_FFN_FUSED", "1")))
        # cluster kernel for encoder steps with <= 16 active rows (larger steps and refused launches take the one-CTA-per-SM kernel)
        self.set_option("persistent_encoder_cluster", int(os.environ.get("SS_PERSISTENT_ENCODER_CLUSTER", "1")))
        self.set_option("cluster_cooperative", int(os.environ.get("SS_CLUSTER_COOPERATIVE", "1")))
        self.set_option("persistent_mt_prefix", int(os.environ.get("SS_PERSISTENT_MT_PREFIX", "1")))
        self.set_option("vocoder_streams", int(os.environ.get("SS_VOCODER_STREAMS", "1")))
        self.set_option("unit_grouped", int(os.environ.get("SS_UNIT_GROUPED", "1")))
        # vocoder generator as one persistent kernel: -1 (default) for short frame windows, 0 never (multi-launch path), 1 always
        self.set_option("vocoder_fused", int(os.environ.get("SS_VOCODER_FUSED", "-1")))
        self.hop = self.lib.ss_vocoder_hop(self._h)
        self.vocoder_receptive_field = self.lib.ss_vocoder_receptive_field(self._h)

    # ------------------------------------------------------------------ plumbing
    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.ss_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            detail = self.lib.ss_last_error(self._h).decode()
            raise EngineError(f"libstreamspeech_b200 error {rc}: {detail}", rc, detail)

    def _load(self, key: str, t: torch.Tensor):
        t = t.detach().to(torch.float32).cpu().contiguous()
        shape = (ctypes.c_int64 * max(t.dim(), 1))(*t.shape)
        self._check(self.lib.ss_load_tensor(self._h, key.encode(), t.data_ptr(), t.dim(), shape))

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _f32(self, *shape) -> torch.Tensor:
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    @staticmethod
    def _ptr(t: Optional[torch.Tensor]):
        return None if t is None else t.data_ptr()

    def persistent_phase_stamps(self, n: int):
        """ns timestamps the persistent encoder kernel recorded on its last step (option persistent_profile)"""
        buf = (ctypes.c_uint64 * n)()
        self._check(self.lib.ss_debug_copy(self._h, b"persist_ts", ctypes.cast(buf, ctypes.c_void_p), n * 8))
        return list(buf)

    def launch_count(self) -> int:
        return int(self.lib.ss_launch_count(self._h))

    def check_async_error(self):
        """raise if a persistent kernel's grid barrier timed out since the last check (synchronises the device)"""
        self._check(self.lib.ss_async_error(self._h))

    def set_chunk(self, attn_chunk: Optional[int], conv_chunk: Optional[int] = None):
        """encoder.chunk_size and the conv chunk sizes the agents poke (agent:395-413).  None = offline model."""
        a = 0 if attn_chunk is None else int(attn_chunk)
        if conv_chunk is None:
            conv_chunk = 0 if attn_chunk is None else (16 if a >= 16 else 8)
        self._check(self.lib.ss_set_chunk(self._h, a, int(conv_chunk)))

    # ------------------------------------------------------------------ blocks
    def num_fbank_frames(self, n_samples: int) -> int:
        return int(self.lib.ss_fbank_num_frames(n_samples))

    def encoder_out_frames(self, F: int) -> int:
        return int(self.lib.ss_encoder_out_frames(F))

    def fbank(self, samples: torch.Tensor, frame0: int = 0, n_frames: Optional[int] = None) -> torch.Tensor:
        """samples: fp32 [n] on the engine's device (16 kHz, unscaled) -> [F, 80] features after global CMVN."""
        assert samples.is_cuda and samples.dtype == torch.float32 and samples.is_contiguous()
        F = self.num_fbank_frames(samples.numel())
        if n_frames is None:
            n_frames = F - frame0
        out = self._f32(max(n_frames, 0), self.cfg.feat_dim)
        if n_frames > 0:
            self._check(self.lib.ss_fbank(self._h, self._stream(), samples.data_ptr(), samples.numel(), frame0, n_frames, out.data_ptr()))
        return out

    def resample_out_len(self, n_in_48k: int, finished: bool) -> int:
        return int(self.lib.ss_resample_out_len(int(n_in_48k), int(finished)))

    def resample_48k_to_16k(self, x48: torch.Tensor, out16: torch.Tensor, out0: int, n_out: int):
        """x48: all 48 kHz samples so far (device fp32); writes out16[out0 : out0 + n_out]"""
        assert x48.is_cuda and out16.is_cuda and x48.is_contiguous() and out16.is_contiguous() and out16.numel() >= out0 + n_out
        self._check(self.lib.ss_resample_48k_to_16k(self._h, self._stream(), x48.data_ptr(), x48.numel(), int(out0), int(n_out), out16.data_ptr()))

    def encoder(self, feats: torch.Tensor, lengths: Optional[Sequence[int]] = None) -> torch.Tensor:
        """feats [B, F, 80] -> [B, T, enc_dim] (batch-major; the reference's encoder_out is the T x B x C transpose)."""
        assert feats.is_cuda and feats.dtype == torch.float32 and feats.is_contiguous() and feats.dim() == 3
        B, F, _ = feats.shape
        T = self.encoder_out_frames(F)
        out = self._f32(B, T, self.cfg.enc_dim)
        lens = None
        if lengths is not None:
            lens = (ctypes.c_int32 * B)(*[int(x) for x in lengths])
        self._check(self.lib.ss_encoder_forward(self._h, self._stream(), feats.data_ptr(), lens, B, F, out.data_ptr()))
        return out

    def encoder_stream_reset(self):
        self._check(self.lib.ss_encoder_stream_reset(self._h))

    def encoder_stream_step(self, feats: torch.Tensor, out_buf: torch.Tensor) -> Tuple[int, int]:
        """feats [F, 80] = all fbank frames of the utterance so far; out_buf [>= T, enc_dim] persistent.  Returns (T, T_final)."""
        assert feats.is_cuda and feats.is_contiguous() and out_buf.is_cuda and out_buf.is_contiguous()
        T, Tf = ctypes.c_int32(0), ctypes.c_int32(0)
        assert out_buf.shape[0] >= self.encoder_out_frames(feats.shape[0])
        self._check(self.lib.ss_encoder_stream_step(self._h, self._stream(), feats.data_ptr(), feats.shape[0], out_buf.data_ptr(),
                                                    ctypes.byref(T), ctypes.byref(Tf)))
        return T.value, Tf.value

    def ctc_greedy(self, head: int, enc: torch.Tensor):
        """enc [T, enc_dim] of one utterance -> dict of device tensors (argmax, tokens, index, count)."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 2
        T = enc.shape[0]
        am = torch.empty(T, dtype=torch.int64, device=self.device)
        toks = torch.empty(T, dtype=torch.int64, device=self.device)
        idx = torch.empty(T, dtype=torch.int32, device=self.device)
        cnt = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._check(self.lib.ss_ctc_greedy(self._h, self._stream(), head, enc.data_ptr(), T, am.data_ptr(), toks.data_ptr(), idx.data_ptr(), cnt.data_ptr()))
        return {"argmax": am, "tokens": toks, "index": idx, "count": cnt}

    def ctc_greedy_rows(self, head: int, enc: torch.Tensor, row0: int, argmax: torch.Tensor):
        """Incremental form for a growing sequence: `argmax` (int64, >= T entries, owned by the caller) already holds the
        arg-max of rows < row0 from earlier calls; rows [row0, T) are computed, then all T rows are collapsed.
        Returns (tokens, index) as python lists with ONE device->host copy."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 2 and argmax.dtype == torch.int64
        T = enc.shape[0]
        out = torch.empty(2 * T + 2, dtype=torch.int64, device=self.device)  # [count | tokens[T] | index (int32 pairs)]
        toks = out[1:1 + T]
        idx = out[1 + T:].view(torch.int32)[:T]
        cnt = out[:1].view(torch.int32)
        cnt.zero_()
        self._check(self.lib.ss_ctc_greedy_rows(self._h, self._stream(), head, enc.data_ptr(), T, int(row0), argmax.data_ptr(), toks.data_ptr(),
                                                idx.data_ptr(), cnt.data_ptr()))
        return ctc_record(out.cpu(), 0, T)

    def ctc_greedy_rows_pair(self, enc: torch.Tensor, row0s: Sequence[int], argmaxes: Sequence[torch.Tensor]):
        """Both CTC heads (0 = ASR, 1 = ST) of one policy() call: the two launches are enqueued back to back and read with
        ONE device->host copy.  Returns ((tokens0, index0), (tokens1, index1))."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 2
        T = enc.shape[0]
        W = 2 * T + 2
        if int(row0s[0]) == int(row0s[1]):  # one projection over both heads + one arg-max / collapse kernel
            out = torch.empty(2 * W, dtype=torch.int64, device=self.device)  # per head: [count | tokens[T] | index (int32 pairs)]
            self._check(self.lib.ss_ctc_greedy_pair(self._h, self._stream(), enc.data_ptr(), T, int(row0s[0]), argmaxes[0].data_ptr(),
                                                    argmaxes[1].data_ptr(), out.data_ptr()))
        else:
            out = torch.zeros(2 * W, dtype=torch.int64, device=self.device)
            for hd in (0, 1):
                o = out[hd * W:(hd + 1) * W]
                self._check(self.lib.ss_ctc_greedy_rows(self._h, self._stream(), hd, enc.data_ptr(), T, int(row0s[hd]), argmaxes[hd].data_ptr(),
                                                        o[1:1 + T].data_ptr(), o[1 + T:].view(torch.int32)[:T].data_ptr(), o[:1].view(torch.int32).data_ptr()))
        host = out.cpu()
        return ctc_record(host, 0, T), ctc_record(host, W, T)

    def mt_greedy(self, enc: torch.Tensor, prefix: Optional[Sequence[int]], max_new_tokens: int, max_len_b: int = 100,
                  stable_rows: int = 0) -> Tuple[List[int], torch.Tensor]:
        """Returns (tokens without the trailing eos, decoder features of [eos]+tokens as [n+1, mt_dim]).
        stable_rows: leading rows of `enc` that are final for this utterance (ss_mt_stable_rows); 0 = project every row."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 2
        if stable_rows > 0:
            self._check(self.lib.ss_mt_stable_rows(self._h, int(stable_rows)))
        prefix = list(prefix) if prefix is not None else []
        cap = self.max_mt_positions
        pfx = (ctypes.c_int64 * max(len(prefix), 1))(*prefix)
        out = (ctypes.c_int64 * cap)()
        n_out = ctypes.c_int32(0)
        feats = self._f32(cap, self.cfg.mt_dim)
        self._check(self.lib.ss_mt_greedy(self._h, self._stream(), enc.data_ptr(), enc.shape[0], pfx, len(prefix), int(max_new_tokens),
                                          int(max_len_b), out, cap, ctypes.byref(n_out), feats.data_ptr()))
        n = n_out.value
        return [int(out[i]) for i in range(n)], feats[: n + 1]

    def mt_greedy_batch(self, enc: torch.Tensor, enc_lengths: Sequence[int], max_len_b: int) -> List[List[int]]:
        """Greedy MT search of every sample of a padded encoder batch enc [B, T, C] (ss_mt_greedy_batch): sample b uses its
        first enc_lengths[b] rows.  Returns the hypotheses without eos; each equals mt_greedy(enc[b, :T_b], None, -1, max_len_b)."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 3
        B, T = int(enc.shape[0]), int(enc.shape[1])
        if len(enc_lengths) != B:
            raise EngineError(f"{len(enc_lengths)} lengths for a batch of {B}")
        lens = (ctypes.c_int32 * max(B, 1))(*[int(x) for x in enc_lengths])
        cap = self.max_mt_positions
        out = (ctypes.c_int64 * (max(B, 1) * cap))()
        n_out = (ctypes.c_int32 * max(B, 1))()
        self._check(self.lib.ss_mt_greedy_batch(self._h, self._stream(), enc.data_ptr(), B, T, lens, int(max_len_b), out, cap, n_out))
        return [[int(out[b * cap + i]) for i in range(n_out[b])] for b in range(B)]

    def mt_beam_batch(self, enc: torch.Tensor, enc_lengths: Sequence[int], beam: int, max_len_b: int,
                      len_penalty: float = 1.0) -> List[List[Dict[str, object]]]:
        """MT beam search of width `beam` (>= 2) over every sample of a padded encoder batch enc [B, T, C] (ss_mt_beam_batch):
        SequenceGenerator.generate_decoder with beam_size = beam, len_penalty and normalize_scores, max_len as mt_greedy_batch.
        Returns per sample the `beam` finalized hypotheses in the order of the reference's finalized[b] (score, highest first),
        each {"tokens": [...] without eos, "score": float, "positional_scores": [...] one per token, eos's last}."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 3
        B, T = int(enc.shape[0]), int(enc.shape[1])
        if len(enc_lengths) != B:
            raise EngineError(f"{len(enc_lengths)} lengths for a batch of {B}")
        K = int(beam)
        lens = (ctypes.c_int32 * max(B, 1))(*[int(x) for x in enc_lengths])
        cap = self.max_mt_positions
        n = max(B, 1) * max(K, 1)
        out = (ctypes.c_int64 * (n * cap))()
        n_out = (ctypes.c_int32 * n)()
        scores = (ctypes.c_float * n)()
        pos = (ctypes.c_float * (n * (cap + 1)))()
        self._check(self.lib.ss_mt_beam_batch(self._h, self._stream(), enc.data_ptr(), B, T, lens, K, int(max_len_b), float(len_penalty),
                                              out, cap, n_out, scores, pos))
        res = []
        for b in range(B):
            hyps = []
            for i in range(K):
                h = b * K + i
                hyps.append({"tokens": [int(out[h * cap + t]) for t in range(n_out[h])], "score": float(scores[h]),
                             "positional_scores": [float(pos[h * (cap + 1) + t]) for t in range(n_out[h] + 1)]})
            res.append(hyps)
        return res

    def mt_incremental_reset(self):
        self._check(self.lib.ss_mt_incremental_reset(self._h))

    def mt_greedy_incremental(self, enc: torch.Tensor, prefix: Optional[Sequence[int]], max_new_tokens: int, max_len: int) -> List[int]:
        """generate_decoder with use_incremental_states=True (S2TT agent): decoder state persists in the handle across calls
        (ss_mt_greedy_incremental).  `max_len` = the generator's max_len for max_new_tokens == -1.  Returns tokens without eos."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 2
        prefix = list(prefix) if prefix is not None else []
        cap = self.max_mt_positions
        pfx = (ctypes.c_int64 * max(len(prefix), 1))(*prefix)
        out = (ctypes.c_int64 * cap)()
        n_out = ctypes.c_int32(0)
        self._check(self.lib.ss_mt_greedy_incremental(self._h, self._stream(), enc.data_ptr(), enc.shape[0], pfx, len(prefix), int(max_new_tokens),
                                                      int(max_len), out, cap, ctypes.byref(n_out)))
        return [int(out[i]) for i in range(n_out.value)]

    def mt_features(self, enc: torch.Tensor, tokens: Sequence[int], want_logits: bool = False, stable_rows: int = 0):
        if stable_rows > 0:
            self._check(self.lib.ss_mt_stable_rows(self._h, int(stable_rows)))
        toks = (ctypes.c_int64 * len(tokens))(*[int(t) for t in tokens])
        feats = self._f32(len(tokens), self.cfg.mt_dim)
        logits = self._f32(self.cfg.tgt_vocab) if want_logits else None
        self._check(self.lib.ss_mt_features(self._h, self._stream(), enc.data_ptr(), enc.shape[0], toks, len(tokens), feats.data_ptr(), self._ptr(logits)))
        return (feats, logits) if want_logits else feats

    def t2u_unit_decode(self, mt_feats: torch.Tensor, n_pad_tail: int = 0, mask_eos: bool = False, debug: bool = False):
        assert mt_feats.is_cuda and mt_feats.is_contiguous() and mt_feats.dim() == 2
        S = mt_feats.shape[0]
        L = S * self.cfg.ctc_upsample_rate
        am = torch.empty(L, dtype=torch.int64, device=self.device)
        packed = torch.zeros(L + 1, dtype=torch.int64, device=self.device)  # [count | units]: one device->host copy reads both
        units = packed[1:]
        cnt = packed[:1].view(torch.int32)[:1]
        t2u = self._f32(S, self.cfg.unit_dim) if debug else None
        logits = self._f32(L, self.cfg.unit_vocab) if debug else None
        self._check(self.lib.ss_t2u_unit_decode(self._h, self._stream(), mt_feats.data_ptr(), S, n_pad_tail, int(mask_eos), am.data_ptr(),
                                                units.data_ptr(), cnt.data_ptr(), self._ptr(t2u), self._ptr(logits)))
        return {"argmax": am, "units": units, "count": cnt, "t2u_out": t2u, "logits": logits, "packed": packed}

    @staticmethod
    def units_to_host(r) -> List[int]:
        """the collapsed unit sequence of a t2u_unit_decode result as a python list (one device->host copy)"""
        host = r["packed"].cpu()
        n = int(host[:1].view(torch.int32)[0])
        return host[1:1 + n].tolist()

    def unit_position_row(self, b: int) -> torch.Tensor:
        """positional row of batch element b in the reference's unit decoder: pad + 1 + b at every time step (SURVEY.md N1)"""
        return constants.sinusoidal_table(self.cfg.pad + 4 + int(b), self.cfg.unit_dim, self.cfg.pad)[self.cfg.pad + 1 + int(b)].contiguous().float()

    def set_unit_batch_index(self, b: int):
        """Batch element b of the reference's unit decoder gets positional row pad + 1 + b at every time step (SURVEY.md N1).
        b = 0 is what the streaming agents use (and what the engine is created with)."""
        row = self.unit_position_row(b)
        self._check(self.lib.ss_unit_position_row(self._h, row.data_ptr()))

    # ------------------------------------------------------------------ offline batch (one call per stage for all samples)
    def ctc_greedy_batch(self, enc: torch.Tensor):
        """Both CTC heads over every row of a padded batch enc [B, T, C] (ss_ctc_greedy_batch, padded rows included).  Returns
        ([((tokens0, index0), (tokens1, index1)) per sample], packed device tensor) after ONE device->host copy."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 3
        B, T = int(enc.shape[0]), int(enc.shape[1])
        W = 2 * T + 2
        packed = torch.empty(B * 2 * W, dtype=torch.int64, device=self.device)
        self._check(self.lib.ss_ctc_greedy_batch(self._h, self._stream(), enc.data_ptr(), B, T, packed.data_ptr()))
        host = packed.cpu()
        return [(ctc_record(host, 2 * b * W, T), ctc_record(host, (2 * b + 1) * W, T)) for b in range(B)], packed

    def mt_features_batch(self, enc: torch.Tensor, enc_lengths: Sequence[int], tokens: Sequence[Sequence[int]]) -> torch.Tensor:
        """mt_features for every sample of a padded batch (ss_mt_features_batch): enc [B, T, C], sample b attends to its first
        enc_lengths[b] rows; tokens [B][S] = [eos, hyp..., pad...].  Returns the features [B, S, mt_dim] (device)."""
        assert enc.is_cuda and enc.is_contiguous() and enc.dim() == 3
        B, T = int(enc.shape[0]), int(enc.shape[1])
        if len(enc_lengths) != B or len(tokens) != B:
            raise EngineError(f"{len(enc_lengths)} lengths and {len(tokens)} token rows for a batch of {B}")
        S = len(tokens[0]) if B else 0
        if any(len(t) != S for t in tokens):
            raise EngineError("every token row of the batch must have the same length")
        lens = (ctypes.c_int32 * max(B, 1))(*[int(x) for x in enc_lengths])
        toks = (ctypes.c_int64 * max(B * S, 1))(*[int(t) for row in tokens for t in row])
        feats = self._f32(B, S, self.cfg.mt_dim)
        self._check(self.lib.ss_mt_features_batch(self._h, self._stream(), enc.data_ptr(), B, T, lens, toks, S, feats.data_ptr()))
        return feats

    def t2u_encode_batch(self, mt_feats: torch.Tensor, lengths: Sequence[int]) -> torch.Tensor:
        """UnitY's synthesizer_encoder on a padded batch (ss_t2u_encode_batch): mt_feats [B, S, dim], sample b's positions >=
        lengths[b] are masked keys.  Returns the T2U states [B, S, dim] (device)."""
        assert mt_feats.is_cuda and mt_feats.is_contiguous() and mt_feats.dim() == 3
        B, S = int(mt_feats.shape[0]), int(mt_feats.shape[1])
        if len(lengths) != B:
            raise EngineError(f"{len(lengths)} lengths for a batch of {B}")
        out = self._f32(B, S, self.cfg.unit_dim)
        self._check(self.lib.ss_t2u_encode_batch(self._h, self._stream(), mt_feats.data_ptr(), B, S, _i32_array(lengths), out.data_ptr()))
        return out

    def unit_search_batch(self, t2u: torch.Tensor, lengths: Sequence[int], max_len: int, len_penalty: float = 1.0) -> List[Dict[str, object]]:
        """UnitY's unit search at beam 1 (ss_unit_search_batch) over t2u [B, S, dim], sample b cross-attending to its first
        lengths[b] rows, with one max_len for the batch.  Returns per sample {"tokens": [...] eos last (finalized[b][0]["tokens"]),
        "score": float, "positional_scores": [...] one per token}."""
        assert t2u.is_cuda and t2u.is_contiguous() and t2u.dim() == 3
        B, S = int(t2u.shape[0]), int(t2u.shape[1])
        if len(lengths) != B:
            raise EngineError(f"{len(lengths)} lengths for a batch of {B}")
        cap = max(int(max_len), 1)
        out = torch.empty(max(B, 1) * cap, dtype=torch.int64)
        n_out = torch.empty(max(B, 1), dtype=torch.int32)
        scores = torch.empty(max(B, 1), dtype=torch.float32)
        pos = torch.empty(max(B, 1) * (cap + 1), dtype=torch.float32)
        self._check(self.lib.ss_unit_search_batch(self._h, self._stream(), t2u.data_ptr(), B, S, _i32_array(lengths), int(max_len),
                                                  float(len_penalty), out.data_ptr(), cap, n_out.data_ptr(), scores.data_ptr(), pos.data_ptr()))
        res = []
        for b in range(B):
            n = int(n_out[b])
            res.append({"tokens": out[b * cap:b * cap + n].tolist() + [self.cfg.eos], "score": float(scores[b]),
                        "positional_scores": pos[b * (cap + 1):b * (cap + 1) + n + 1].clone()})
        return res

    def t2u_unit_decode_batch(self, mt_feats: torch.Tensor, n_pad_tail: Sequence[int], mask_eos: bool = False):
        """t2u_unit_decode for every sample of a padded batch mt_feats [B, S, mt_dim] (ss_t2u_unit_decode_batch), sample b with
        positional row unit_position_row(b) (N1).  Returns (units per sample, arg-max per sample, {"argmax": [B, S*rate],
        "packed": [B, S*rate + 1]} device tensors); the python lists come from ONE device->host copy."""
        assert mt_feats.is_cuda and mt_feats.is_contiguous() and mt_feats.dim() == 3
        B, S = int(mt_feats.shape[0]), int(mt_feats.shape[1])
        if len(n_pad_tail) != B:
            raise EngineError(f"{len(n_pad_tail)} pad-tail lengths for a batch of {B}")
        L = S * self.cfg.ctc_upsample_rate
        rows = torch.stack([self.unit_position_row(b) for b in range(B)]).to(self.device) if B else self._f32(0, self.cfg.unit_dim)
        buf = torch.empty(B * (2 * L + 1), dtype=torch.int64, device=self.device)  # [argmax B*L | packed B*(L+1)]
        am, packed = buf[:B * L].view(B, L), buf[B * L:].view(B, L + 1)
        pads = (ctypes.c_int32 * max(B, 1))(*[int(x) for x in n_pad_tail])
        self._check(self.lib.ss_t2u_unit_decode_batch(self._h, self._stream(), mt_feats.data_ptr(), B, S, pads, rows.data_ptr(), int(mask_eos),
                                                      am.data_ptr(), packed.data_ptr()))
        host = buf.cpu()
        h_am, h_packed = host[:B * L].view(B, L), host[B * L:].view(B, L + 1)
        units = [h_packed[b, 1:1 + int(h_packed[b, :1].view(torch.int32)[0])].tolist() for b in range(B)]
        return units, [h_am[b].tolist() for b in range(B)], {"argmax": am, "packed": packed}

    def t2u_unit_decode_batch_scored(self, mt_feats: torch.Tensor, n_pad_tail: Sequence[int], mask_eos: bool = False):
        """t2u_unit_decode_batch plus every upsampled row's arg-max log-probability (ss_t2u_unit_decode_batch_scored: the reference's
        CTCSequenceGenerator positional scores, pad-tail rows included).  Returns (units per sample, arg-max per sample, lprob per
        sample as fp32 [S*rate] host tensors, {"argmax", "packed", "lprob": [B, S*rate] device}); units, arg-max and lprob come from
        ONE device->host copy."""
        assert mt_feats.is_cuda and mt_feats.is_contiguous() and mt_feats.dim() == 3
        B, S = int(mt_feats.shape[0]), int(mt_feats.shape[1])
        if len(n_pad_tail) != B:
            raise EngineError(f"{len(n_pad_tail)} pad-tail lengths for a batch of {B}")
        L = S * self.cfg.ctc_upsample_rate
        rows = torch.stack([self.unit_position_row(b) for b in range(B)]).to(self.device) if B else self._f32(0, self.cfg.unit_dim)
        n_lp = (B * L + 1) // 2  # int64 words holding the fp32 scores
        buf = torch.empty(B * (2 * L + 1) + n_lp, dtype=torch.int64, device=self.device)  # [argmax B*L | packed B*(L+1) | lprob]
        am, packed = buf[:B * L].view(B, L), buf[B * L:B * (2 * L + 1)].view(B, L + 1)
        lprob = buf[B * (2 * L + 1):].view(torch.float32)[:B * L].view(B, L)
        pads = (ctypes.c_int32 * max(B, 1))(*[int(x) for x in n_pad_tail])
        self._check(self.lib.ss_t2u_unit_decode_batch_scored(self._h, self._stream(), mt_feats.data_ptr(), B, S, pads, rows.data_ptr(),
                                                             int(mask_eos), am.data_ptr(), packed.data_ptr(), lprob.data_ptr()))
        host = buf.cpu()
        h_am, h_packed = host[:B * L].view(B, L), host[B * L:B * (2 * L + 1)].view(B, L + 1)
        h_lp = host[B * (2 * L + 1):].view(torch.float32)[:B * L].view(B, L)
        units = [h_packed[b, 1:1 + int(h_packed[b, :1].view(torch.int32)[0])].tolist() for b in range(B)]
        return units, [h_am[b].tolist() for b in range(B)], [h_lp[b] for b in range(B)], {"argmax": am, "packed": packed, "lprob": lprob}

    def t2u_unit_decode_ragged(self, mt_feats: torch.Tensor, lengths: Sequence[int], n_pad_tail: Sequence[int], pos_rows: Optional[torch.Tensor] = None,
                               mask_eos: bool = False):
        """t2u_unit_decode for every sample of mt_feats [B, S_stride, mt_dim] where sample b has only its first lengths[b] positions
        (ss_t2u_unit_decode_ragged), n_pad_tail[b] of them N2 pad positions.  pos_rows [B, unit_dim] (device): each sample's positional
        row, default unit_position_row(0) for every sample (what each streaming agent uses).  Returns (units per sample, arg-max per
        sample (its lengths[b] * rate rows), {"argmax": [B, S_stride*rate], "packed": [B, S_stride*rate + 1]} device tensors); the python
        lists come from ONE device->host copy."""
        assert mt_feats.is_cuda and mt_feats.is_contiguous() and mt_feats.dim() == 3
        B, S = int(mt_feats.shape[0]), int(mt_feats.shape[1])
        if len(lengths) != B or len(n_pad_tail) != B:
            raise EngineError(f"{len(lengths)} lengths and {len(n_pad_tail)} pad-tail lengths for a batch of {B}")
        R = self.cfg.ctc_upsample_rate
        L = S * R
        if pos_rows is None:
            pos_rows = self.unit_position_row(0).to(self.device).expand(max(B, 1), -1).contiguous()
        assert pos_rows.is_cuda and pos_rows.is_contiguous() and pos_rows.shape[0] >= B
        buf = torch.empty(B * (2 * L + 1), dtype=torch.int64, device=self.device)  # [argmax B*L | packed B*(L+1)]
        am, packed = buf[:B * L].view(B, L), buf[B * L:].view(B, L + 1)
        lens = (ctypes.c_int32 * max(B, 1))(*[int(x) for x in lengths])
        pads = (ctypes.c_int32 * max(B, 1))(*[int(x) for x in n_pad_tail])
        self._check(self.lib.ss_t2u_unit_decode_ragged(self._h, self._stream(), mt_feats.data_ptr(), B, S, lens, pads, pos_rows.data_ptr(),
                                                       int(mask_eos), am.data_ptr(), packed.data_ptr()))
        host = buf.cpu()
        h_am, h_packed = host[:B * L].view(B, L), host[B * L:].view(B, L + 1)
        units = [h_packed[b, 1:1 + int(h_packed[b, :1].view(torch.int32)[0])].tolist() for b in range(B)]
        return units, [h_am[b, :int(lengths[b]) * R].tolist() for b in range(B)], {"argmax": am, "packed": packed}

    def vocoder_durations(self, codes: torch.Tensor, dur_prediction: bool = True):
        assert codes.is_cuda and codes.dtype == torch.int64 and codes.is_contiguous()
        U = codes.numel()
        dur = torch.empty(U, dtype=torch.int64, device=self.device)
        cum = torch.empty(U + 1, dtype=torch.int32, device=self.device)
        self._check(self.lib.ss_vocoder_durations(self._h, self._stream(), codes.data_ptr(), U, int(dur_prediction), dur.data_ptr(), cum.data_ptr()))
        return dur, cum

    def vocoder_generate(self, total_frames: int, frame0: int, n_frames: int, left_context: int = -1) -> torch.Tensor:
        wav = self._f32(n_frames * self.hop)
        self._check(self.lib.ss_vocoder_generate(self._h, self._stream(), total_frames, frame0, n_frames, left_context, wav.data_ptr()))
        return wav

    def vocoder_durations_ragged(self, codes_list: Sequence, dur_prediction: bool = True):
        """vocoder_durations of every code sequence in codes_list (1-D int64 tensors or lists) in one call
        (ss_vocoder_durations_ragged).  Returns (durations per sequence, cumsum per sequence (U_s + 1 frame offsets), as host lists
        from ONE device->host copy, and {"dur": packed durations, "cumsum": packed cumsums} device tensors).  The sequences stay
        cached for vocoder_generate_ragged."""
        n = len(codes_list)
        if n == 0:
            raise EngineError("vocoder_durations_ragged needs at least one code sequence")
        if all(isinstance(c, torch.Tensor) for c in codes_list):
            U = [int(c.numel()) for c in codes_list]
            codes = torch.cat([c.reshape(-1).to(self.device, torch.int64) for c in codes_list])
        else:  # host lists: one host->device copy
            U = [len(c) for c in codes_list]
            codes = torch.tensor([int(u) for c in codes_list for u in c], dtype=torch.int64, device=self.device)
        n_dur, n_cum = sum(U), sum(U) + n
        buf = torch.empty(n_dur + (n_cum + 1) // 2, dtype=torch.int64, device=self.device)  # [durations | cumsums (int32)]
        dur, cum = buf[:n_dur], buf[n_dur:].view(torch.int32)[:n_cum]
        lens = (ctypes.c_int32 * n)(*U)
        self._check(self.lib.ss_vocoder_durations_ragged(self._h, self._stream(), n, codes.data_ptr(), lens, int(dur_prediction),
                                                         dur.data_ptr(), cum.data_ptr()))
        host = buf.cpu()
        h_dur, h_cum = host[:n_dur].tolist(), host[n_dur:].view(torch.int32)[:n_cum].tolist()
        durs, cums, o = [], [], 0
        for s, u in enumerate(U):
            durs.append(h_dur[o:o + u])
            cums.append(h_cum[o + s:o + s + u + 1])
            o += u
        return durs, cums, {"dur": dur, "cumsum": cum}

    def vocoder_generate_ragged(self, totals: Sequence[int], frame0s: Sequence[int], n_frames: Sequence[int],
                                left_contexts: Sequence[int]) -> List[torch.Tensor]:
        """vocoder_generate of every sequence of the last vocoder_durations_ragged call in one call (ss_vocoder_generate_ragged).
        Returns each sequence's n_frames[s] * hop samples as views of one device buffer."""
        n = len(totals)
        if not (len(frame0s) == len(n_frames) == len(left_contexts) == n) or n == 0:
            raise EngineError("vocoder_generate_ragged needs one total, frame0, n_frames and left context per sequence")
        arr = lambda v: (ctypes.c_int32 * n)(*[int(x) for x in v])
        wav = self._f32(sum(int(x) for x in n_frames) * self.hop)
        self._check(self.lib.ss_vocoder_generate_ragged(self._h, self._stream(), n, arr(totals), arr(frame0s), arr(n_frames),
                                                        arr(left_contexts), wav.data_ptr()))
        out, o = [], 0
        for nf in n_frames:
            out.append(wav[o:o + int(nf) * self.hop])
            o += int(nf) * self.hop
        return out

    # single ops (parity tests)
    def op_linear(self, x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], act: int = 0) -> torch.Tensor:
        M, K = x.shape
        N = w.shape[0]
        out = self._f32(M, N)
        self._check(self.lib.ss_op_linear(self._h, self._stream(), x.data_ptr(), M, K, w.data_ptr(), self._ptr(b), N, act, out.data_ptr()))
        return out

    def op_linear_umma(self, x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], act: int = 0, pieces: int = 3) -> torch.Tensor:
        M, K = x.shape
        N = w.shape[0]
        out = self._f32(M, N)
        self._check(self.lib.ss_op_linear_umma(self._h, self._stream(), x.data_ptr(), M, K, w.data_ptr(), self._ptr(b), N, act, pieces, out.data_ptr()))
        return out

    def op_conv1d(self, x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], ksize: int, dil: int = 1, pad_left: int = 0,
                  pre_lrelu: float = 1.0, mode: int = 0) -> torch.Tensor:
        """x [L][C_in] channels-last, w [N][ksize*C_in] tap-major; mode 0 = fp32 CUDA cores, 12/13 = wgmma (bf16x3 / bf16x6)"""
        L, C = x.shape
        N = w.shape[0]
        out = self._f32(L, N)
        self._check(self.lib.ss_op_conv1d(self._h, self._stream(), x.data_ptr(), L, C, w.data_ptr(), self._ptr(b), N, ksize, dil, pad_left,
                                          float(pre_lrelu), mode, out.data_ptr()))
        return out

    def persistent_time(self):
        """(summed ms, launches, summed algorithmic bytes) of the persistent encoder kernel since the last query
        (CUDA events on the launching stream; enable with set_option('persistent_time', 1))"""
        buf = (ctypes.c_double * 3)()
        self._check(self.lib.ss_debug_copy(self._h, b"persist_time", buf, ctypes.sizeof(buf)))
        return float(buf[0]), int(buf[1]), float(buf[2])

    def mt_time(self):
        """(summed ms, launches, summed greedy steps) of the single-token MT kernel since the last query (CUDA events on the launching
        stream; enable with set_option('persistent_time', 1))"""
        buf = (ctypes.c_double * 3)()
        self._check(self.lib.ss_debug_copy(self._h, b"mt_time", buf, ctypes.sizeof(buf)))
        return float(buf[0]), int(buf[1]), float(buf[2])

    def mt_incremental_state(self, slot: Optional[int] = None) -> Dict[str, object]:
        """the incremental MT state of the handle (slot None: mt_greedy_incremental's) or of one pool slot (ss_debug_copy "mt_inc_state" /
        "pool_mt_inc_state:<slot>") as CPU tensors: {"entries", "cross_rows", "self_k", "self_v" [mt_layers, entries, mt_dim],
        "cross_kv" [mt_layers, cross_rows, 2 * mt_dim]}"""
        name = b"mt_inc_state" if slot is None else b"pool_mt_inc_state:%d" % int(slot)
        counts = (ctypes.c_int32 * 2)()
        self._check(self.lib.ss_debug_copy(self._h, name, counts, ctypes.sizeof(counts)))
        E, R = int(counts[0]), int(counts[1])
        L, D = self.cfg.mt_layers, self.cfg.mt_dim
        buf = torch.empty(2 + 2 * L * E * D + 2 * L * R * D, dtype=torch.float32)
        self._check(self.lib.ss_debug_copy(self._h, name, buf.data_ptr(), buf.numel() * 4))
        assert buf[:2].view(torch.int32).tolist() == [E, R]
        kv = buf[2:2 + 2 * L * E * D].view(2, L, E, D)
        return {"entries": E, "cross_rows": R, "self_k": kv[0], "self_v": kv[1], "cross_kv": buf[2 + 2 * L * E * D:].view(L, R, 2 * D)}

    def cluster_steps(self) -> int:
        """encoder steps taken by the cluster kernel (option persistent_encoder_cluster) since the engine was created"""
        buf = ctypes.c_longlong(0)
        self._check(self.lib.ss_debug_copy(self._h, b"cluster_steps", ctypes.byref(buf), ctypes.sizeof(buf)))
        return int(buf.value)

    # ------------------------------------------------------------------ multi-stream pool (ss_pool_*)
    def pool_create(self, n_slots: int, max_seconds: int = 60, sample_rate: int = 16000):
        """sample_rate 16000 or 48000: the rate of the samples pool_push_audio takes (48 kHz is resampled per slot on the device)"""
        self._check(self.lib.ss_pool_create_rate(self._h, int(n_slots), int(max_seconds), int(sample_rate)))
        self._pool_slots = int(n_slots)
        self._pool_out = None

    def pool_reset(self, slot: int):
        self._check(self.lib.ss_pool_reset(self._h, int(slot)))

    def pool_set_chunk(self, slot: int, attn_chunk: int, conv_chunk: int):
        """the slot's own latency (attention chunk, even conv chunk, as set_chunk); (0, 0) = follow the handle's set_chunk.  Only
        while the slot holds no samples (after pool_reset); the setting survives pool_reset"""
        self._check(self.lib.ss_pool_set_chunk(self._h, int(slot), int(attn_chunk), int(conv_chunk)))

    def pool_finish(self, slot: int):
        """the slot's source is closed: the next step produces the rest of its 16 kHz signal; pushes fail until pool_reset"""
        self._check(self.lib.ss_pool_finish(self._h, int(slot)))

    def pool_resample_time(self):
        """(summed ms, launches, summed algorithmic bytes) of the pool's resample kernel since the last query (CUDA events on the
        launching stream; enable with set_option('persistent_time', 1))"""
        buf = (ctypes.c_double * 3)()
        self._check(self.lib.ss_debug_copy(self._h, b"pool_resample_time", buf, ctypes.sizeof(buf)))
        return float(buf[0]), int(buf[1]), float(buf[2])

    def pool_push_audio(self, slot: int, samples: torch.Tensor):
        """samples: fp32 CPU tensor (contiguous) at the pool's rate; appended to the slot's device audio"""
        assert samples.dtype == torch.float32 and not samples.is_cuda and samples.is_contiguous()
        self._check(self.lib.ss_pool_push_audio(self._h, self._stream(), int(slot), samples.data_ptr(), samples.numel()))

    def pool_info(self, slot: int):
        na, nf, tf = ctypes.c_int64(0), ctypes.c_int32(0), ctypes.c_int32(0)
        enc, feats = ctypes.c_void_p(), ctypes.c_void_p()
        self._check(self.lib.ss_pool_info(self._h, int(slot), ctypes.byref(na), ctypes.byref(nf), ctypes.byref(tf), ctypes.byref(enc), ctypes.byref(feats)))
        return {"n_audio": na.value, "n_feat": nf.value, "T_final": tf.value, "enc_out_ptr": enc.value, "feats_ptr": feats.value}

    def pool_step(self, slots: Sequence[int], ctc_heads: int = 1, max_rows: int = 1024):
        """One batched streaming step (fbank -> encoder -> CTC heads) of the listed slots.  Returns a list, per slot, of
        {"T", "T_final", "ctc": [(tokens, index) per head]} with ONE device->host copy for all streams."""
        n = len(slots)
        cap = n * max(ctc_heads, 1) * (2 * max_rows + 2)
        if self._pool_out is None or self._pool_out.numel() < cap:
            self._pool_out = torch.empty(cap, dtype=torch.int64, device=self.device)
        sl = (ctypes.c_int32 * n)(*[int(x) for x in slots])
        T, Tf, off = (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)(), (ctypes.c_int64 * n)()
        self._check(self.lib.ss_pool_step(self._h, self._stream(), n, sl, int(ctc_heads), self._pool_out.data_ptr(), self._pool_out.numel(), T, Tf, off))
        res = [{"T": int(T[i]), "T_final": int(Tf[i]), "ctc": []} for i in range(n)]
        if ctc_heads:
            used = int(off[n - 1]) + ctc_heads * (2 * int(T[n - 1]) + 2)
            host = self._pool_out[:used].cpu()
            for i in range(n):
                Ti = int(T[i])
                res[i]["ctc"] = [ctc_record(host, int(off[i]) + hd * (2 * Ti + 2), Ti) for hd in range(ctc_heads)]
        return res

    def pool_mt_greedy(self, slots: Sequence[int], prefixes: Sequence[Optional[Sequence[int]]], max_new_tokens: Sequence[int],
                       max_len_b: int = 100) -> Tuple[List[List[int]], torch.Tensor]:
        """Greedy MT search of several pool streams at once (ss_pool_mt_greedy) on each slot's encoder rows of its last pool_step:
        stream i continues prefixes[i] (None = empty) with max_new_tokens[i] (-1 = source finished).  Returns (hypotheses without eos,
        prefix included; decoder features [n, feats_ld, mt_dim] on the device, stream i's features of [eos] + hyp_i in its first
        len(hyp_i) + 1 rows).  Each stream equals mt_greedy(enc_slot, prefixes[i], max_new_tokens[i], max_len_b)."""
        n = len(slots)
        if len(prefixes) != n or len(max_new_tokens) != n:
            raise EngineError(f"{len(prefixes)} prefixes and {len(max_new_tokens)} token limits for {n} streams")
        pfx = [list(p) if p is not None else [] for p in prefixes]
        cap = self.max_mt_positions
        mlen = [min(int(max_len_b), cap - 1) if int(m) == -1 else len(p) + int(m) for p, m in zip(pfx, max_new_tokens)]
        feats_ld = max(max(mlen, default=0), 0) + 1
        flat = [int(t) for p in pfx for t in p]
        sl = (ctypes.c_int32 * max(n, 1))(*[int(x) for x in slots])
        cat = (ctypes.c_int64 * max(len(flat), 1))(*flat)
        npf = (ctypes.c_int32 * max(n, 1))(*[len(p) for p in pfx])
        mnt = (ctypes.c_int32 * max(n, 1))(*[int(m) for m in max_new_tokens])
        out = (ctypes.c_int64 * (max(n, 1) * cap))()
        n_out = (ctypes.c_int32 * max(n, 1))()
        feats = self._f32(max(n, 1), feats_ld, self.cfg.mt_dim)
        self._check(self.lib.ss_pool_mt_greedy(self._h, self._stream(), n, sl, cat, npf, mnt, int(max_len_b), out, cap, n_out, feats.data_ptr(),
                                               feats_ld))
        return [[int(out[i * cap + k]) for k in range(n_out[i])] for i in range(n)], feats[:n]

    def pool_mt_greedy_incremental(self, slots: Sequence[int], prefixes: Sequence[Optional[Sequence[int]]], max_new_tokens: Sequence[int],
                                   max_lens: Sequence[int]) -> List[List[int]]:
        """mt_greedy_incremental of several pool streams at once (ss_pool_mt_greedy_incremental), each on its slot's own incremental
        state (kept until pool_reset) and its encoder rows of the last pool_step: stream i continues prefixes[i] (None = empty) with
        max_new_tokens[i] (-1 = source finished, then max_lens[i] is the generator's max_len).  Returns hypotheses without eos."""
        n = len(slots)
        if len(prefixes) != n or len(max_new_tokens) != n or len(max_lens) != n:
            raise EngineError(f"{len(prefixes)} prefixes, {len(max_new_tokens)} token limits and {len(max_lens)} max_lens for {n} streams")
        pfx = [list(p) if p is not None else [] for p in prefixes]
        cap = self.max_mt_positions
        flat = [int(t) for p in pfx for t in p]
        sl = (ctypes.c_int32 * max(n, 1))(*[int(x) for x in slots])
        cat = (ctypes.c_int64 * max(len(flat), 1))(*flat)
        npf = (ctypes.c_int32 * max(n, 1))(*[len(p) for p in pfx])
        mnt = (ctypes.c_int32 * max(n, 1))(*[int(m) for m in max_new_tokens])
        mls = (ctypes.c_int32 * max(n, 1))(*[int(m) for m in max_lens])
        out = (ctypes.c_int64 * (max(n, 1) * cap))()
        n_out = (ctypes.c_int32 * max(n, 1))()
        self._check(self.lib.ss_pool_mt_greedy_incremental(self._h, self._stream(), n, sl, cat, npf, mnt, mls, out, cap, n_out))
        return [[int(out[i * cap + k]) for k in range(n_out[i])] for i in range(n)]

    def pool_encoder_rows(self, slot: int, T: int) -> torch.Tensor:
        """the slot's first T encoder rows [T, enc_dim] as a tensor over the pool's device memory (a view: valid until the next pool_step)"""
        ptr = self.pool_info(slot)["enc_out_ptr"]
        numel = int(T) * self.cfg.enc_dim

        class _Rows:
            __cuda_array_interface__ = {"shape": (numel,), "typestr": "<f4", "data": (ptr, False), "version": 3}
        return torch.as_tensor(_Rows(), device=self.device).view(int(T), self.cfg.enc_dim)

    def set_option(self, name: str, value: int):
        self._check(self.lib.ss_set_option(self._h, name.encode(), int(value)))

    def op_layer_norm(self, x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """LayerNorm over the C = g.numel() columns of the rows of x [rows, >= C] (row stride x.stride(0)) into out [rows, >= C] (default: a
        new [rows, C] tensor)"""
        C = g.numel()
        if out is None:
            out = self._f32(x.shape[0], C)
        self._check(self.lib.ss_op_layer_norm(self._h, self._stream(), x.data_ptr(), self._ld(x), x.shape[0], C, g.data_ptr(), b.data_ptr(),
                                              out.data_ptr(), self._ld(out)))
        return out

    def op_gemm(self, args: GemmArgs) -> GemmArgs:
        """ss_op_gemm: one GEMM with every field of the kernel layer's contract (pointers are device addresses); the route_* fields of
        `args` are filled in"""
        self._check(self.lib.ss_op_gemm(self._h, self._stream(), ctypes.byref(args)))
        return args

    def op_argmax_rows(self, logits: torch.Tensor, n_masked: int, scored: bool):
        """ss_op_argmax_rows on a 2-D fp32 device tensor: (indices, log-probabilities or None)"""
        assert logits.is_cuda and logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
        rows, V = logits.shape
        idx = torch.empty(rows, dtype=torch.int64, device=self.device)
        lp = torch.empty(rows, dtype=torch.float32, device=self.device) if scored else None
        self._check(self.lib.ss_op_argmax_rows(self._h, self._stream(), logits.data_ptr(), rows, V, logits.stride(0), n_masked, idx.data_ptr(),
                                               self._ptr(lp)))
        return idx, lp

    # Attention / depthwise-conv parity hooks (ss_op_*_attention, ss_op_*depthwise*).  Matrices are 2-D device fp32 tensors whose rows
    # may be strided (column slices of a fused buffer); kernel: 0 = the engine's choice, 1 = row kernel, 2 = tile kernel.
    @staticmethod
    def _ld(t: torch.Tensor) -> int:
        assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1, (t.shape, t.stride())
        return t.stride(0)

    def op_relpos_attention(self, q, k, v, pos, bias_u, bias_v, B: int, nQ: int, q_offset: int, T: int, H: int, chunk: int,
                            lengths: Optional[Sequence[int]] = None, kernel: int = 0) -> torch.Tensor:
        """q [B*nQ, >=D] (absolute positions q_offset ..), k / v [B*T, >=D], pos [2*Tpos-1, D] -> out [B*nQ, D]"""
        D = H * 64
        Tpos = (pos.shape[0] + 1) // 2
        out = self._f32(B * nQ, D)
        self._check(self.lib.ss_op_relpos_attention(self._h, self._stream(), q.data_ptr(), self._ld(q), k.data_ptr(), self._ld(k), v.data_ptr(),
                                                    self._ld(v), pos.data_ptr(), Tpos, bias_u.data_ptr(), bias_v.data_ptr(), out.data_ptr(), B,
                                                    nQ, q_offset, T, H, D, chunk, _i32_array(lengths), kernel))
        return out

    def op_mha_attention(self, q, k, v, B: int, Tq: int, Tk: int, H: int, scale: float, causal: bool = False, causal_offset: int = 0,
                         kv_len: Optional[Sequence[int]] = None, kernel: int = 0) -> torch.Tensor:
        """q [B*Tq, >=D], k / v [B*Tk, >=D] -> out [B*Tq, D]"""
        out = self._f32(B * Tq, H * 64)
        self._check(self.lib.ss_op_mha_attention(self._h, self._stream(), q.data_ptr(), self._ld(q), k.data_ptr(), self._ld(k), v.data_ptr(),
                                                 self._ld(v), out.data_ptr(), self._ld(out), B, Tq, Tk, H, float(scale), int(causal),
                                                 causal_offset, _i32_array(kv_len), kernel))
        return out

    def op_grouped_causal_attention(self, q, k, v, B: int, S: int, R: int, H: int, scale: float,
                                    kv_len: Optional[Sequence[int]] = None) -> torch.Tensor:
        """q / k / v [B*S, >=D] (one row per group) -> out [B*S*R, D]"""
        out = self._f32(B * S * R, H * 64)
        self._check(self.lib.ss_op_grouped_causal_attention(self._h, self._stream(), q.data_ptr(), self._ld(q), k.data_ptr(), self._ld(k),
                                                            v.data_ptr(), self._ld(v), out.data_ptr(), self._ld(out), S, R, H, float(scale), B,
                                                            _i32_array(kv_len)))
        return out

    def op_depthwise_bn_silu(self, x, w, scale, shift, B: int, T: int, t0: int, n: int, chunk: int) -> torch.Tensor:
        """x [B*T, >=C], w [k, C] -> y [B*n, C] for positions t0 .. t0+n-1"""
        k, C = w.shape
        y = self._f32(B * n, C)
        self._check(self.lib.ss_op_depthwise_bn_silu(self._h, self._stream(), x.data_ptr(), self._ld(x), w.data_ptr(), scale.data_ptr(),
                                                     shift.data_ptr(), y.data_ptr(), C, B, T, t0, n, C, k, chunk))
        return y

    @staticmethod
    def _ms_args(streams: Sequence[dict], chunk_key: str):
        return [_i32_array([s[f] for s in streams]) for f in ("slot", "a0", "nA", "T", chunk_key, "row0")]

    def op_ms_relpos_attention(self, q, kc, vc, pos, bias_u, bias_v, out, H: int, streams: Sequence[dict]):
        """kc / vc [n_slots, slot_rows, D] key / value caches; streams: dicts of slot, a0, nA, T, attn_chunk, row0; writes the rows of
        out [rows, >=D] the streams own (the others are left as they are)"""
        n_slots = kc.shape[0]
        self._check(self.lib.ss_op_ms_relpos_attention(self._h, self._stream(), q.data_ptr(), self._ld(q), kc.data_ptr(), vc.data_ptr(),
                                                       kc.stride(0), n_slots, pos.data_ptr(), (pos.shape[0] + 1) // 2, bias_u.data_ptr(),
                                                       bias_v.data_ptr(), out.data_ptr(), self._ld(out), out.shape[0], H, len(streams),
                                                       *self._ms_args(streams, "attn_chunk")))

    def op_ms_depthwise(self, x, w, scale, shift, y, streams: Sequence[dict]):
        """x [n_slots, slot_rows, C] conv-input caches; streams: dicts of slot, a0, nA, T, conv_chunk, row0; writes the rows of
        y [rows, >=C] the streams own"""
        k, C = w.shape
        self._check(self.lib.ss_op_ms_depthwise(self._h, self._stream(), x.data_ptr(), x.stride(0), x.shape[0], w.data_ptr(), scale.data_ptr(),
                                                shift.data_ptr(), y.data_ptr(), self._ld(y), y.shape[0], C, k, len(streams),
                                                *self._ms_args(streams, "conv_chunk")))


class ASREngine:
    """The ASR-BLEU transcriber's handle (ss_asr_*): wav2vec 2.0 CTC emissions, beam-1 arg-max and collapse on one GPU.  `settings`:
    the ASRConfig fields (n_conv is taken from `strides`)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], strides: Sequence[int], device: int = 0, **settings):
        if not torch.cuda.is_available():
            raise EngineError("streamspeech_b200.ASREngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = load_library()
        self.device = torch.device("cuda", device)
        self.vocab_size = int(state_dict["w2v_encoder.proj.weight"].shape[0]) if "w2v_encoder.proj.weight" in state_dict else 0
        c = ASRConfig()
        c.n_conv = len(strides)
        for i, s in enumerate(strides[:SS_ASR_MAX_CONV]):
            c.conv_stride[i] = s
        defaults = dict(extractor_layer_norm=1, layer_norm_first=1, pos_conv_depth=1, conformer=0, heads=0, normalize=1, max_frames=0,
                        time_stages=0)
        defaults.update(settings)
        for k, v in defaults.items():
            setattr(c, k, int(v))
        self._h = ctypes.c_void_p()
        rc = self.lib.ss_asr_create(ctypes.byref(self._h), device, ctypes.byref(c))
        if rc != 0:
            raise EngineError(f"ss_asr_create failed with {rc}: {self.lib.ss_asr_last_error(None).decode()}", rc,
                              self.lib.ss_asr_last_error(None).decode())
        try:
            for k, v in state_dict.items():
                if v.is_floating_point():
                    t = v.detach().to(torch.float32).cpu().contiguous()
                    shape = (ctypes.c_int64 * max(t.dim(), 1))(*t.shape)
                    self._check(self.lib.ss_asr_load_tensor(self._h, k.encode(), t.data_ptr(), t.dim(), shape))
            self._check(self.lib.ss_asr_finalize(self._h))
        except Exception:
            self.close()
            raise

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.ss_asr_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            detail = self.lib.ss_asr_last_error(self._h).decode()
            raise EngineError(f"libstreamspeech_b200 error {rc}: {detail}", rc, detail)

    def num_frames(self, n_samples: int) -> int:
        return int(self.lib.ss_asr_num_frames(self._h, n_samples))

    def _audio(self, waves: Sequence[torch.Tensor]):
        offs = [0]
        for w in waves:
            offs.append(offs[-1] + int(w.numel()))
        audio = torch.cat([w.reshape(-1).to(torch.float32) for w in waves]).to(self.device) if offs[-1] else torch.zeros(1, device=self.device)
        return audio, (ctypes.c_int64 * len(offs))(*offs)

    def transcribe(self, waves: Sequence[torch.Tensor], emissions: bool = False):
        """-> (token lists, per-frame arg-max list, emissions [sum T][V] or None).  Utterances shorter than one frame raise EngineError."""
        audio, offs = self._audio(waves)
        T = [self.num_frames(int(w.numel())) for w in waves]
        stride = max(T + [0]) + 1
        packed = torch.zeros(len(waves), stride, dtype=torch.int64, device=self.device)
        am = torch.empty(max(1, sum(T)), dtype=torch.int64, device=self.device)
        em = None
        if emissions:
            em = torch.empty(max(1, sum(T)), self.vocab_size, dtype=torch.float32, device=self.device)
        self._check(self.lib.ss_asr_transcribe(self._h, torch.cuda.current_stream(self.device).cuda_stream, audio.data_ptr(), offs, len(waves),
                                               packed.data_ptr(), stride, am.data_ptr(), None if em is None else em.data_ptr()))
        host = packed.cpu()
        toks = []
        for b in range(len(waves)):
            n = int(host[b, 0].item() & 0xFFFFFFFF)
            toks.append(host[b, 1:1 + n].tolist())
        return toks, am.cpu()[:sum(T)].tolist(), em

    def stage(self, waves: Sequence[torch.Tensor], stage: int, width: int) -> torch.Tensor:
        """ss_asr_debug_stage: activations after `stage`, rows of the utterances in order"""
        audio, offs = self._audio(waves)
        rows = sum(max(0, self.num_frames(int(w.numel()))) for w in waves)
        out = torch.empty(max(1, rows), width, dtype=torch.float32, device=self.device)
        self._check(self.lib.ss_asr_debug_stage(self._h, torch.cuda.current_stream(self.device).cuda_stream, audio.data_ptr(), offs, len(waves),
                                                stage, out.data_ptr()))
        return out[:rows]

    def stage_ms(self) -> List[float]:
        buf = (ctypes.c_double * 4)()
        self._check(self.lib.ss_asr_stage_ms(self._h, buf))
        return list(buf)
