"""CPU: the C-ABI library builds, loads and exports every symbol include/streamspeech_b200.h declares;
host-side logic (dictionary, constants, SimulEval API mirror, synthetic checkpoint keys)."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    from streamspeech_b200 import engine

    if not os.path.exists(engine.LIB_PATH):
        g.build()
    lib = engine.load_library()
    header = open(os.path.join(ROOT, "include", "streamspeech_b200.h")).read()
    declared = set(re.findall(r"\b(ss_[a-z0-9_]+)\s*\(", header))
    assert declared == set(engine.EXPORTED_SYMBOLS), declared ^ set(engine.EXPORTED_SYMBOLS)
    for s in declared:
        assert hasattr(lib, s), s
    assert b"sm_90a" in lib.ss_version()
    # pure host helpers need no GPU
    assert lib.ss_fbank_num_frames(160000) == 998 and lib.ss_fbank_num_frames(239) == 0
    assert lib.ss_encoder_out_frames(998) == 250 and lib.ss_encoder_out_frames(1498) == 375 and lib.ss_encoder_out_frames(1) == 1


def test_engine_refuses_to_run_without_cuda():
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.engine import Engine, EngineError

    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    with pytest.raises(EngineError, match="no CPU fallback"):
        Engine(ModelConfig(), {}, None, None)


def test_ss_config_struct_layout_matches_header():
    """ctypes mirror of `struct ss_config`: same field order and count as the header."""
    from streamspeech_b200.engine import SSConfig

    header = open(os.path.join(ROOT, "include", "streamspeech_b200.h")).read()
    body = header[header.index("typedef struct ss_config {"):header.index("} ss_config;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"\b([a-z_0-9]+)(?:\[[A-Z_]+\])*\s*[,;]", body)
    assert names == [n for n, _ in SSConfig._fields_], (names, [n for n, _ in SSConfig._fields_])


def test_ss_op_gemm_args_struct_layout_matches_header():
    """ctypes mirror of `struct ss_op_gemm_args`: same field order, names and C types as the header, so every offset agrees."""
    import ctypes

    from streamspeech_b200.engine import GemmArgs

    header = open(os.path.join(ROOT, "include", "streamspeech_b200.h")).read()
    body = header[header.index("typedef struct ss_op_gemm_args {") + len("typedef struct ss_op_gemm_args {"):header.index("} ss_op_gemm_args;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    ctype = {"float*": ctypes.c_void_p, "int32_t*": ctypes.c_void_p, "int32_t": ctypes.c_int32, "float": ctypes.c_float}
    fields = []
    for decl in body.split(";"):
        decl = " ".join(decl.split())
        if not decl:
            continue
        m = re.fullmatch(r"(?:const )?(float|int32_t)(\*?) ?(.*)", decl)
        assert m, decl
        for name in m.group(3).split(","):
            fields.append((name.strip(), ctype[m.group(1) + m.group(2)]))
    assert [(n, t) for n, t in GemmArgs._fields_] == fields, ([n for n, _ in GemmArgs._fields_], [n for n, _ in fields])
    assert "ss_op_gemm" in re.findall(r"\b(ss_[a-z0-9_]+)\s*\(", header)


def test_constants_match_oracle_tables():
    from oracle import streamspeech_oracle as so
    from streamspeech_b200 import constants

    assert torch.equal(constants.rel_pos_table(17, 256), so.rel_positional_encoding(17, 256))
    assert torch.equal(constants.sinusoidal_table(40, 512, 1), so.sinusoidal_table(40, 512, 1))
    assert torch.equal(constants.mel_bank()[:, :256], so._mel_banks())


def test_dictionary_and_simuleval_mirror():
    from streamspeech_b200.dictionary import Dictionary
    from streamspeech_b200.simuleval_compat import (AgentStates, EmptySegment, ReadAction, SpeechSegment, SpeechToSpeechAgent,
                                                    WriteAction)

    d = Dictionary.units(1000)
    assert len(d) == 1005 and d[4] == "0" and d[1003] == "999" and d.blank_index == 1004 and d[2] == "</s>"
    s = Dictionary.synthetic(6000)
    assert len(s) == 6000 and s[4].startswith("▁") and not s[5].startswith("▁")

    class Echo(SpeechToSpeechAgent):
        def policy(self):
            if len(self.states.source) < 4:
                return ReadAction()
            return WriteAction(SpeechSegment(content=list(self.states.source), sample_rate=16000, finished=self.states.source_finished),
                               finished=self.states.source_finished)

    a = Echo(None)
    assert a.pushpop(SpeechSegment(content=[0.1, 0.2], sample_rate=16000)).is_empty
    out = a.pushpop(SpeechSegment(content=[0.3, 0.4], sample_rate=16000, finished=True))
    assert out.content == [0.1, 0.2, 0.3, 0.4] and out.finished
    st = AgentStates()
    st.update_source(EmptySegment(finished=True))
    assert st.source_finished and st.source == []


def test_synthetic_checkpoint_keys_and_determinism():
    from streamspeech_b200 import synth
    from streamspeech_b200.config import ModelConfig

    cfg = ModelConfig()
    a, b = synth.make_model_state_dict(cfg, 0), synth.make_model_state_dict(cfg, 0)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert a["encoder.conformer_layers.11.conv_module.depthwise_conv.weight"].shape == (256, 1, 31)
    assert a["decoder.embed_tokens.weight"].shape == (1005, 512)
    assert ModelConfig.from_state_dict(a).enc_layers == 12 and ModelConfig.from_state_dict(a).unit_vocab == 1005
    n_enc = sum(v.numel() for k, v in a.items() if k.startswith("encoder.") and "num_batches" not in k)
    assert abs(n_enc - 33.45e6) < 0.1e6  # SURVEY.md §8: encoder ~33.45 M parameters


def test_utterances_shard_across_ranks_gloo():
    """N>1 path of bench.py: utterance ids are partitioned over ranks with no data-path collective."""
    import torch.distributed as dist
    import torch.multiprocessing as mp

    mp.spawn(_shard_worker, args=(2,), nprocs=2, join=True)


def _shard_worker(rank, world):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = "29533"
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import bench

    mine = bench.shard_utterances(7, rank, world)
    gathered = [None] * world
    dist.all_gather_object(gathered, mine)
    flat = sorted(x for g in gathered for x in g)
    assert flat == list(range(7))
    t = torch.tensor([float(len(mine))])
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    assert t.item() == 4.0
    dist.destroy_process_group()


def test_agent_files_load_the_way_simuleval_loads_them():
    """`simuleval --agent FILE` imports the file as a top-level module named "agents" and then requires exactly ONE class
    registered by @entrypoint (SimulEval/simuleval/utils/agent.py:25-28,46-56).  Each file under streamspeech_b200/agents/ must
    survive that (no relative imports) and register exactly its own agent, with the reference's class name and flags."""
    import argparse
    import importlib.util

    from streamspeech_b200 import simuleval_compat as sc

    expected = {"speech_to_speech.streamspeech.agent.py": ("StreamSpeechS2STAgent", "speech"),
                "speech_to_text.asr.streamspeech.agent.py": ("StreamSpeechASRAgent", "text"),
                "speech_to_text.s2tt.streamspeech.agent.py": ("StreamSpeechS2TTAgent", "text")}
    d = os.path.join(ROOT, "streamspeech_b200", "agents")
    assert sorted(os.listdir(d)) == sorted(expected) or sorted(f for f in os.listdir(d) if f.endswith(".py")) == sorted(expected)
    for fname, (cls_name, target) in expected.items():
        before = len(sc.EVALUATION_SYSTEM_LIST)
        spec = importlib.util.spec_from_file_location("agents", os.path.join(d, fname))  # import_file()
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        new = sc.EVALUATION_SYSTEM_LIST[before:]
        assert len(new) == 1 and new[0].__name__ == cls_name, (fname, new)
        klass = new[0]
        assert klass.source_type == "speech" and klass.target_type == target
        p = argparse.ArgumentParser()
        klass.add_args(p)
        a = p.parse_args(["--model-path", "m", "--data-bin", "d", "--vocoder", "v", "--vocoder-cfg", "c"])
        for flag in ("config_yaml", "multitask_config_yaml", "lagging_k1", "stride_n", "segment_size", "sample_rate", "dur_prediction",
                     "extra_output_dir", "max_len", "force_finish"):
            assert hasattr(a, flag), (fname, flag)
        assert a.sample_rate == 48000  # the reference's default (agent:32-35)


def test_resample_filter_matches_torchaudio():
    """constants.resample_kernel_3to1 restates torchaudio's windowed-sinc kernel (the oracle of the 48 kHz -> 16 kHz front end)."""
    import math

    import torch
    from torchaudio.functional.functional import _get_sinc_resample_kernel

    from streamspeech_b200.constants import resample_kernel_3to1

    k, w = _get_sinc_resample_kernel(48000, 16000, math.gcd(48000, 16000))
    k2, w2 = resample_kernel_3to1()
    assert w == w2 == 19 and k2.numel() == 41 and float((k.view(-1) - k2).abs().max()) == 0.0


class _FakeEngine:
    """records the calls the fairseq-surface shims make (CPU test double; no compute)"""

    def __init__(self):
        import torch

        self.device = torch.device("cpu")
        self.calls = []

    def set_chunk(self, attn, conv=None):
        self.calls.append(("set_chunk", attn, conv))


def test_fairseq_surface_attribute_pokes_reach_the_engine():
    """agent:395-413: the agent assigns encoder.chunk_size and the conv chunk sizes on the model object; the shims of
    streamspeech_b200/fairseq_surface.py must translate every assignment into ss_set_chunk with the agent's values."""
    import sys
    import types

    import torch

    from streamspeech_b200 import synth
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.fairseq_surface import B200Encoder, StreamSpeechB200Model, register_with_fairseq

    cfg = ModelConfig()
    eng = _FakeEngine()
    enc = B200Encoder(eng, cfg)
    assert len(enc.conformer_layers) == cfg.enc_layers and len(enc.subsample.conv_layers) == 2
    # the reference's own lines, verbatim in spirit (agent:404-413)
    chunk_size = 320 // 40
    enc.chunk_size = chunk_size
    chunk_size = 16 if chunk_size >= 16 else 8
    for conv in enc.subsample.conv_layers:
        conv.chunk_size = chunk_size
    for layer in enc.conformer_layers:
        layer.conv_module.depthwise_conv.chunk_size = chunk_size
    assert eng.calls[0] == ("set_chunk", 8, 8) and eng.calls[-1] == ("set_chunk", 8, 8)
    assert enc.chunk_size == 8 and enc.subsample.conv_layers[1].chunk_size == 8
    # ASR agent rule (speech_to_text.asr agent :361-375): 160 ms -> attention 4, conv min(4, 16) = 4
    enc.chunk_size = 4
    for conv in enc.subsample.conv_layers:
        conv.chunk_size = 4
    assert eng.calls[-1] == ("set_chunk", 4, 4)
    # offline model (--chunk-size 999999, N10)
    enc.chunk_size = 999999
    assert eng.calls[-1] == ("set_chunk", None, None)
    # registration with a fairseq that offers the two decorators
    reg = {}
    fm = types.ModuleType("fairseq.models")
    fm.register_model = lambda name: (lambda cls: reg.setdefault("model:" + name, cls))
    fm.register_model_architecture = lambda m, a: (lambda fn: reg.setdefault("arch:" + a, fn))
    saved = {k: sys.modules.get(k) for k in ("fairseq", "fairseq.models")}
    sys.modules["fairseq"] = types.ModuleType("fairseq")
    sys.modules["fairseq.models"] = fm
    try:
        assert register_with_fairseq() and reg["model:streamspeech_b200"] is StreamSpeechB200Model and "arch:streamspeech_b200" in reg
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_checkpoint_files_round_trip(tmp_path):
    """`--model-path file.pt --config-yaml ... --multitask-config-yaml ... --vocoder g.pt --vocoder-cfg config.json`
    (agent:355-393, agent/tts/vocoder.py:31-45): everything the agent reads from disk -- fairseq .pt with a "model" entry, gcmvn
    npz behind the yaml, SPM-style dictionary files behind the multitask yaml, weight-normed vocoder checkpoint + JSON -- comes
    back as the tensors / config / dictionaries of the synthetic checkpoint it was written from."""
    import argparse
    import json

    import numpy as np
    import torch
    import yaml

    from streamspeech_b200 import synth
    from streamspeech_b200.agent import load_streamspeech_checkpoint, load_vocoder
    from streamspeech_b200.config import ModelConfig
    from streamspeech_b200.dictionary import Dictionary
    from streamspeech_b200.engine import remove_weight_norm

    cfg = ModelConfig().tiny()
    cfg.src_vocab = cfg.tgt_vocab = 64
    sd = synth.make_model_state_dict(cfg, 0)
    vsd = synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=True)
    d = tmp_path
    torch.save({"model": sd, "cfg": None, "args": None}, d / "model.pt")
    torch.save({"generator": vsd}, d / "g_00500000")
    json.dump(cfg.vocoder.to_json_dict(), open(d / "config.json", "w"))
    g = synth.make_gcmvn(cfg)
    np.savez(d / "gcmvn.npz", mean=g["mean"], std=g["std"])
    yaml.safe_dump({"global_cmvn": {"stats_npz_path": str(d / "gcmvn.npz")}, "input_feat_per_channel": 80}, open(d / "config_gcmvn.yaml", "w"))
    mt = {}
    for name in ("source_unigram", "ctc_target_unigram", "target_unigram"):
        sub = d / name
        sub.mkdir()
        dic = Dictionary.synthetic(64)
        with open(sub / "spm_unigram.txt", "w", encoding="utf-8") as f:
            for sym in dic.symbols[4:]:
                f.write(f"{sym} 1\n")
        mt[name] = {"decoder_type": "transformer" if name == "target_unigram" else "ctc", "dict": str(sub / "spm_unigram.txt")}
    yaml.safe_dump(mt, open(d / "config_mtl.yaml", "w"))
    args = argparse.Namespace(model_path=str(d / "model.pt"), data_bin=str(d), config_yaml="config_gcmvn.yaml", multitask_config_yaml="config_mtl.yaml",
                              vocoder=str(d / "g_00500000"), vocoder_cfg=str(d / "config.json"))
    cfg2, sd2, gc2, dicts = load_streamspeech_checkpoint(args)
    for k in ("enc_dim", "enc_ffn", "enc_heads", "enc_layers", "dw_kernel", "conv_channels", "conv_kernel", "src_vocab", "tgt_vocab", "mt_dim", "mt_ffn",
              "mt_layers", "t2u_layers", "unit_dim", "unit_layers", "unit_vocab"):
        assert getattr(cfg2, k) == getattr(cfg, k), k
    assert set(sd2) == set(sd) and all(torch.equal(sd2[k], sd[k]) for k in sd)
    assert np.array_equal(gc2["mean"], g["mean"]) and np.array_equal(gc2["std"], g["std"])
    assert dicts["target_unigram"].symbols == Dictionary.synthetic(64).symbols and len(dicts["tgt"]) == cfg.unit_vocab
    vc, vsd2 = load_vocoder(args, cfg2)
    assert vc.upsample_rates == cfg.vocoder.upsample_rates and vc.dur_hidden == cfg.vocoder.dur_hidden
    plain = synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=False)
    folded = remove_weight_norm(vsd2)
    assert set(folded) == set(plain) and all(float((folded[k] - plain[k]).abs().max()) < 1e-5 for k in plain)
