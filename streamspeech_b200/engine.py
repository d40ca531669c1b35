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


class EngineError(RuntimeError):
    pass


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
    lib.ss_mt_stable_rows.argtypes = [vp, i32]
    lib.ss_mt_incremental_reset.argtypes = [vp]
    lib.ss_mt_greedy_incremental.argtypes = [vp, vp, vp, i32, vp, i32, i32, i32, vp, i32, ctypes.POINTER(i32)]
    lib.ss_mt_features.argtypes = [vp, vp, vp, i32, vp, i32, vp, vp]
    lib.ss_t2u_unit_decode.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp]
    lib.ss_unit_position_row.argtypes = [vp, vp]
    lib.ss_vocoder_durations.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    lib.ss_vocoder_generate.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    lib.ss_vocoder_hop.argtypes = [vp]
    lib.ss_vocoder_receptive_field.argtypes = [vp]
    lib.ss_op_linear.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, i32, vp]
    lib.ss_op_linear_umma.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, i32, i32, vp]
    lib.ss_op_conv1d.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, i32, i32, i32, ctypes.c_float, i32, vp]
    lib.ss_set_option.argtypes = [vp, ctypes.c_char_p, i32]
    lib.ss_op_layer_norm.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp]
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
    _lib = lib
    return lib


EXPORTED_SYMBOLS = [
    "ss_create", "ss_destroy", "ss_last_error", "ss_version", "ss_load_tensor", "ss_finalize", "ss_set_chunk",
    "ss_fbank_num_frames", "ss_fbank", "ss_encoder_out_frames", "ss_encoder_forward", "ss_encoder_stream_reset", "ss_encoder_stream_step", "ss_ctc_greedy", "ss_ctc_greedy_rows", "ss_mt_greedy",
    "ss_mt_features", "ss_mt_stable_rows", "ss_t2u_unit_decode", "ss_unit_position_row", "ss_vocoder_durations", "ss_vocoder_generate", "ss_vocoder_hop",
    "ss_vocoder_receptive_field", "ss_op_linear", "ss_op_linear_umma", "ss_op_conv1d", "ss_set_option", "ss_debug_copy", "ss_op_layer_norm", "ss_launch_count", "ss_async_error", "ss_mt_incremental_reset", "ss_mt_greedy_incremental", "ss_ctc_greedy_pair", "ss_resample_out_len", "ss_resample_48k_to_16k", "ss_pool_create", "ss_pool_reset", "ss_pool_push_audio", "ss_pool_info", "ss_pool_step",
    "ss_pool_create_rate", "ss_pool_finish", "ss_pool_set_chunk", "ss_mt_greedy_batch",
]


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
            raise EngineError(f"ss_create failed with {rc}")
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
            if gcmvn is not None:
                self._load("__const__.gcmvn_mean", torch.as_tensor(gcmvn["mean"], dtype=torch.float32))
                self._load("__const__.gcmvn_std", torch.as_tensor(gcmvn["std"], dtype=torch.float32))
            self._check(self.lib.ss_finalize(self._h))
        except Exception:
            self.close()
            raise
        # tensor-core routing (kernels_umma2.cu): vocoder convs tolerate the 3-MMA split (1e-3 waveform bar, measured 7e-6);
        # linears that feed an arg-max stay on the exact fp32 kernels unless explicitly switched on
        self.set_option("prefer_shared", int(os.environ.get("SS_PREFER_SHARED", "0")))
        self.set_option("umma_vocoder", int(os.environ.get("SS_UMMA_VOCODER", "12")))
        self.set_option("umma_linear", int(os.environ.get("SS_UMMA_LINEAR", "13")))
        self.set_option("umma_min_rows", int(os.environ.get("SS_UMMA_MIN_ROWS", "128")))
        self.set_option("umma_min_channels", int(os.environ.get("SS_UMMA_MIN_CHANNELS", "16")))
        self.set_option("persistent_encoder", int(os.environ.get("SS_PERSISTENT_ENCODER", "1")))
        self.set_option("persistent_mt", int(os.environ.get("SS_PERSISTENT_MT", "1")))
        self.set_option("umma2_fused_reduce", int(os.environ.get("SS_UMMA2_FUSED_REDUCE", "0")))
        self.set_option("fbank_tma", int(os.environ.get("SS_FBANK_TMA", "1")))
        self.set_option("persistent_ffn_fused", int(os.environ.get("SS_PERSISTENT_FFN_FUSED", "1")))
        # cluster kernel for encoder steps with <= 16 active rows (larger steps and refused launches take the one-CTA-per-SM kernel)
        self.set_option("persistent_encoder_cluster", int(os.environ.get("SS_PERSISTENT_ENCODER_CLUSTER", "1")))
        self.set_option("cluster_cooperative", int(os.environ.get("SS_CLUSTER_COOPERATIVE", "1")))
        self.set_option("persistent_mt_v2", int(os.environ.get("SS_PERSISTENT_MT_V2", "1")))
        self.set_option("persistent_mt_prefix", int(os.environ.get("SS_PERSISTENT_MT_PREFIX", "1")))
        self.set_option("vocoder_streams", int(os.environ.get("SS_VOCODER_STREAMS", "1")))
        self.set_option("unit_grouped", int(os.environ.get("SS_UNIT_GROUPED", "1")))
        self.set_option("vocoder_graph", int(os.environ.get("SS_VOCODER_GRAPH", "0")))
        # vocoder generator as one persistent kernel: -1 (default) for short frame windows, 0 never (multi-launch path), 1 always
        self.set_option("vocoder_fused", int(os.environ.get("SS_VOCODER_FUSED", "-1")))
        self.set_option("graph_pdl", int(os.environ.get("SS_GRAPH_PDL", "0")))
        self.set_option("persistent_prefetch", int(os.environ.get("SS_PERSISTENT_PREFETCH", "0")))
        self.set_option("umma2_split_below", int(os.environ.get("SS_UMMA2_SPLIT_BELOW", "60")))
        self.set_option("umma2_min_units", int(os.environ.get("SS_UMMA2_MIN_UNITS", "4")))
        self.set_option("persistent_barrier", int(os.environ.get("SS_PERSISTENT_BARRIER", "1")))
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
            raise EngineError(f"libstreamspeech_b200 error {rc}: {self.lib.ss_last_error(self._h).decode()}")

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
        host = out.cpu()
        n = int(host[:1].view(torch.int32)[0])
        return host[1:1 + n].tolist(), host[1 + T:].view(torch.int32)[:n].tolist()

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
        res = []
        for hd in (0, 1):
            hrow = host[hd * W:(hd + 1) * W]
            n = int(hrow[:1].view(torch.int32)[0])
            res.append((hrow[1:1 + n].tolist(), hrow[1 + T:].view(torch.int32)[:n].tolist()))
        return res[0], res[1]

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

    def set_unit_batch_index(self, b: int):
        """Batch element b of the reference's unit decoder gets positional row pad + 1 + b at every time step (SURVEY.md N1).
        b = 0 is what the streaming agents use (and what the engine is created with)."""
        row = constants.sinusoidal_table(self.cfg.pad + 4 + int(b), self.cfg.unit_dim, self.cfg.pad)[self.cfg.pad + 1 + int(b)].contiguous().float()
        self._check(self.lib.ss_unit_position_row(self._h, row.data_ptr()))

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
                for hd in range(ctc_heads):
                    o = int(off[i]) + hd * (2 * Ti + 2)
                    row = host[o:o + 2 * Ti + 2]
                    cnt = int(row[:1].view(torch.int32)[0])
                    res[i]["ctc"].append((row[1:1 + cnt].tolist(), row[1 + Ti:].view(torch.int32)[:cnt].tolist()))
        return res

    def set_option(self, name: str, value: int):
        self._check(self.lib.ss_set_option(self._h, name.encode(), int(value)))

    def op_layer_norm(self, x: torch.Tensor, g: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        out = torch.empty_like(x)
        self._check(self.lib.ss_op_layer_norm(self._h, self._stream(), x.data_ptr(), x.shape[0], x.shape[1], g.data_ptr(), b.data_ptr(), out.data_ptr()))
        return out
