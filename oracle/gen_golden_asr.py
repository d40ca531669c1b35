"""Generate tests/golden/asr_w2v.npz from the REAL reference code (build container only, CPU, seconds).

Run:  python -m oracle.gen_golden_asr      (needs /root/reference and torchaudio's installed source)

The fixture of the ASR-BLEU transcriber's restatement (oracle/asr_oracle.py) and of asr.remove_silence:

  forward     fairseq's own Wav2Vec2Model (fairseq/models/wav2vec/wav2vec2.py), exec'd from its class source together with
              ConvFeatureExtractionModel, make_conv_pos, TransformerEncoder and TransformerSentenceEncoderLayer, built at small dims
              from a seeded synth.make_w2v_ctc_state_dict and run as Wav2VecEncoder does (extract_features with an all-False padding
              mask, then proj).  The input goes through the reference's own ASRGenerator.load_audiofile (asr_bleu/utils.py, with
              torchaudio.load returning the waveform), so the task.normalize LayerNorm is the reference's too.  Two configurations:
              conv_bias on with an even pos_conv kernel (SamePad drops a frame), conv_bias off with an odd one.  Stages are caught
              with forward hooks: extractor output, post_extract_proj output, pos_conv output, every layer, the encoder output and
              the emissions, all fp32.
  rm_silence  asr_bleu_rm_silence/utils.py's load_audiofile from its own source on known patterns and random signals.
  get_tokens  torchaudio's CTCDecoder._get_tokens from its own source (the module itself needs flashlight) on random paths.
"""
from __future__ import annotations

import ast
import itertools
import os
import sys
import types
from types import SimpleNamespace as NS

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from streamspeech_b200 import synth  # noqa: E402

REF = ref_loader.REF
W2V = REF + "/fairseq/fairseq/models/wav2vec/wav2vec2.py"
OUT = os.path.join(ROOT, "tests", "golden", "asr_w2v.npz")
CONV = [(64, 10, 5), (64, 3, 2), (64, 3, 2), (64, 3, 2), (64, 2, 2)]
CONFIGS = {  # name: (seed, conv_bias, pos_k, pos_groups)
    "a": (11, True, 16, 4),
    "b": (12, False, 15, 2),
}
DIM, FFN, LAYERS, VOCAB = 128, 256, 2, 32
LENGTHS = (2000, 4321)
RM_PATTERNS = [[1] + [0] * 9 + [1], [1] + [0] * 10 + [1], [1] + [0] * 12 + [1], [1] + [0] * 19 + [1], [0] * 5 + [1, 1] + [0] * 5,
               [0] * 4 + [1, 1] + [0] * 5, [0] * 12, [1, 0, 1, 0] * 6]


def config_state_dict(name):
    seed, conv_bias, k, g = CONFIGS[name]
    sd = synth.make_w2v_ctc_state_dict(seed=seed, dim=DIM, ffn=FFN, layers=LAYERS, conv_layers=CONV, pos_k=k, pos_groups=g, vocab=VOCAB)
    if not conv_bias:
        sd = {key: v for key, v in sd.items() if not (".conv_layers." in key and key.endswith(".0.bias"))}
    return sd


def w2v_namespace():
    from oracle.gen_golden import extract_class

    ref_loader.load_full()
    import fairseq.utils as U
    from fairseq.modules.fp32_group_norm import Fp32GroupNorm
    from fairseq.modules.grad_multiply import GradMultiply
    from fairseq.modules.layer_norm import Fp32LayerNorm, LayerNorm
    from fairseq.modules.multihead_attention import MultiheadAttention
    from fairseq.modules.same_pad import SamePad
    from fairseq.modules.transpose_last import TransposeLast

    w = sys.modules.setdefault("fairseq.models.wav2vec", types.ModuleType("fairseq.models.wav2vec"))
    w.__path__ = [REF + "/fairseq/fairseq/models/wav2vec"]
    from fairseq.models.wav2vec.utils import pad_to_multiple

    class _Unused:
        def __init__(self, *a, **k):
            raise RuntimeError("not part of the en model's forward pass")

    ns = dict(torch=torch, nn=nn, F=F, np=np, math=__import__("math"), utils=U, LayerNorm=LayerNorm, Fp32LayerNorm=Fp32LayerNorm,
              Fp32GroupNorm=Fp32GroupNorm, TransposeLast=TransposeLast, SamePad=SamePad, GradMultiply=GradMultiply,
              MultiheadAttention=MultiheadAttention, index_put=U.index_put, is_xla_tensor=U.is_xla_tensor, buffered_arange=U.buffered_arange,
              get_activation_fn=U.get_activation_fn, pad_to_multiple=pad_to_multiple, fsdp_wrap=lambda m, **k: m,
              checkpoint_wrapper=lambda m, **k: m, init_bert_params=lambda m: None, FullyShardedDataParallel=_Unused,
              ConformerWav2Vec2EncoderLayer=_Unused, TransformerSentenceEncoderWithAdapterLayer=_Unused, GumbelVectorQuantizer=_Unused,
              ConformerEncoder=_Unused, compute_mask_indices=None, BaseFairseqModel=nn.Module, Wav2Vec2Config=object,
              register_model=lambda *a, **k: (lambda c: c), List=list, Tuple=tuple)
    tree = ast.parse(open(W2V).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "make_conv_pos"][0]
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "wav2vec2.py:make_conv_pos", "exec"), ns)
    for cls in ("TransformerSentenceEncoderLayer", "ConvFeatureExtractionModel", "TransformerEncoder", "Wav2Vec2Model"):
        ns[cls] = extract_class(W2V, cls, ns)
    return ns


def w2v_cfg(k, g, conv_bias):
    """the Wav2Vec2Config fields Wav2Vec2Model / TransformerEncoder read, at the en model's settings"""
    return NS(conv_feature_layers=repr(CONV), extractor_mode="layer_norm", conv_bias=conv_bias, encoder_embed_dim=DIM, quantize_input=False,
              crop_seq_to_multiple=1, mask_prob=0.0, mask_selection="static", mask_other=0, mask_length=10, no_mask_overlap=False,
              mask_min_space=1, mask_channel_prob=0.0, mask_channel_before=False, mask_channel_selection="static", mask_channel_other=0,
              mask_channel_length=10, no_mask_channel_overlap=False, mask_channel_min_space=1, dropout_input=0.0, dropout_features=0.0,
              feature_grad_mult=0.0, num_negatives=0, cross_sample_negatives=0, codebook_negatives=0, negatives_from_everywhere=False,
              logit_temp=0.1, final_dim=0, quantize_targets=False, layer_type="transformer", pos_enc_type="abs", target_glu=False,
              dropout=0.0, encoder_layers=LAYERS, encoder_ffn_embed_dim=FFN, encoder_attention_heads=DIM // 64, attention_dropout=0.0,
              activation_dropout=0.0, activation_fn="gelu", layer_norm_first=True, encoder_layerdrop=0.0, conv_pos=k, conv_pos_groups=g,
              pos_conv_depth=1, required_seq_len_multiple=2, checkpoint_activations=False, offload_activations=False,
              min_params_to_wrap=100000000, max_positions=100000, adp_num=-1, adp_dim=64, adp_act_fn="relu", adp_trf_idx="all")


def reference_load_audiofile(path_utils, wav, normalize):
    """the reference's ASRGenerator.load_audiofile from its own source; torchaudio.load returns `wav` at the model's rate"""
    from oracle.gen_golden import extract_functions

    ta = types.SimpleNamespace(load=lambda p: (wav.reshape(1, -1).clone(), 16000), functional=types.SimpleNamespace(resample=None))
    fns = extract_functions(path_utils, "ASRGenerator", ["load_audiofile"], {"torch": torch, "torchaudio": ta})
    return fns["load_audiofile"](NS(sampling_rate=16000, normalize_input=normalize), "unused.wav")


def run_forward(ns, name, wavs):
    from oracle.gen_golden import sub_state

    seed, conv_bias, k, g = CONFIGS[name]
    sd = config_state_dict(name)
    torch.manual_seed(0)
    model = ns["Wav2Vec2Model"](w2v_cfg(k, g, conv_bias)).eval()
    missing, unexpected = model.load_state_dict(sub_state(sd, "w2v_encoder.w2v_model."), strict=False)
    assert not unexpected, unexpected
    assert set(missing) <= {"mask_emb", "project_q.weight", "project_q.bias", "final_proj.weight", "final_proj.bias"}, missing
    out = {}
    caught = {}
    model.feature_extractor.register_forward_hook(lambda m, i, o: caught.__setitem__("extractor", o[0].t().clone()))
    model.post_extract_proj.register_forward_hook(lambda m, i, o: caught.__setitem__("proj", o[0].clone()))
    model.encoder.pos_conv.register_forward_hook(lambda m, i, o: caught.__setitem__("pos_conv", o[0].t().clone()))
    for li, layer in enumerate(model.encoder.layers):
        layer.register_forward_hook(lambda m, i, o, li=li: caught.__setitem__(f"layer{li}", o[0][:, 0].clone()))
    for j, wav in enumerate(wavs):
        src = reference_load_audiofile(REF + "/asr_bleu/utils.py", wav, True)
        caught.clear()
        with torch.no_grad():
            res = model.extract_features(src, torch.zeros(src.shape, dtype=torch.bool), mask=False)
            emis = F.linear(res["x"], sd["w2v_encoder.proj.weight"], sd["w2v_encoder.proj.bias"])
        T = emis.shape[1]
        out[f"{name}_{j}_wav"] = wav.numpy()
        out[f"{name}_{j}_normalized"] = src[0].numpy()
        out[f"{name}_{j}_extractor"] = caught["extractor"].numpy()
        out[f"{name}_{j}_proj"] = caught["proj"].numpy()
        out[f"{name}_{j}_pos"] = (caught["proj"] + caught["pos_conv"]).numpy()  # x + pos_conv(x) (extract_features, no padding)
        for li in range(LAYERS):
            out[f"{name}_{j}_layer{li}"] = caught[f"layer{li}"][:T].numpy()
        out[f"{name}_{j}_final_ln"] = res["x"][0].numpy()
        out[f"{name}_{j}_emissions"] = emis[0].numpy()
    out[f"{name}_checksum"] = np.array([float(sum(v.double().sum() for v in sd.values()))])
    return out


def reference_rm_silence(x):
    return reference_load_audiofile(REF + "/asr_bleu_rm_silence/utils.py", torch.from_numpy(x), False)[0]


def torchaudio_get_tokens():
    import importlib.util

    spec = importlib.util.find_spec("torchaudio")
    path = os.path.join(os.path.dirname(spec.origin), "models", "decoder", "_ctc_decoder.py")
    from oracle.gen_golden import extract_functions

    fns = extract_functions(path, "CTCDecoder", ["_get_tokens"], {"it": itertools, "torch": torch})
    return fns["_get_tokens"]


def main():
    ns = w2v_namespace()
    out = {}
    g = torch.Generator().manual_seed(5)
    wavs = [synth.make_audio(n / 16000, seed=40 + i)[:n] for i, n in enumerate(LENGTHS)]
    for name in CONFIGS:
        out.update(run_forward(ns, name, wavs))
    # rm_silence: known patterns (values 1..n where the pattern is 1) and random signals with zero runs
    rm_in, rm_out = [], []
    for p in RM_PATTERNS:
        x = np.where(np.array(p) == 0, 0.0, np.arange(1, len(p) + 1)).astype(np.float32)
        rm_in.append(x)
    rng = np.random.default_rng(3)
    for _ in range(40):
        x = rng.standard_normal(rng.integers(1, 200)).astype(np.float32)
        for _ in range(rng.integers(0, 5)):
            a = rng.integers(0, len(x))
            x[a:a + rng.integers(1, 25)] = 0.0
        rm_in.append(x)
    for x in rm_in:
        rm_out.append(reference_rm_silence(x).numpy())
    out["rm_in"] = np.concatenate(rm_in)
    out["rm_in_off"] = np.cumsum([0] + [len(x) for x in rm_in])
    out["rm_out"] = np.concatenate(rm_out)
    out["rm_out_off"] = np.cumsum([0] + [len(x) for x in rm_out])
    # _get_tokens on random arg-max paths over a small vocabulary (repeats and blanks frequent)
    get_tokens = torchaudio_get_tokens()
    paths = [torch.randint(0, 4, (int(torch.randint(0, 40, (1,), generator=g)),), generator=g, dtype=torch.int32) for _ in range(60)]
    toks = [get_tokens(NS(blank=0), p).numpy() for p in paths]
    out["gt_in"] = np.concatenate([p.numpy() for p in paths]).astype(np.int64)
    out["gt_in_off"] = np.cumsum([0] + [len(p) for p in paths])
    out["gt_out"] = np.concatenate(toks).astype(np.int64)
    out["gt_out_off"] = np.cumsum([0] + [len(t) for t in toks])
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(out)} arrays")


if __name__ == "__main__":
    main()
