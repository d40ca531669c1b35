"""Pin the wait-k-stride-n agents on UnitY to the reference's own policy() (build container only, CPU, a few minutes).

Run:  python -m oracle.gen_golden_waitk        (needs /root/reference)

`WaitkS2STAgent.policy` / `.reset` (agent/speech_to_speech.wait-k-stride-n.agent.py:290-296,358-581), the S2TT twin's
(agent/speech_to_text.wait-k-stride-n.agent.py) and `OnlineFeatureExtractor.__call__` / `.transform` are executed FROM THEIR OWN
SOURCE (ast) against a `self` built as the agents' __init__ builds it (beam 1, max_len_a 1, max_len_b 200, min_len 1, no incremental
state): the reference's own `agent/sequence_generator.py:SequenceGenerator` twice (MT and units), over the UnitY modules assembled as
oracle.gen_golden_unity assembles them (fairseq's S2TConformerEncoder, TransformerDecoderBase, TransformerEncoderNoEmb,
TransformerUnitDecoder) with the seeded synthetic UnitY checkpoint, the reference's CodeGenerator behind
CodeHiFiGANVocoderWithDur.forward with the synthetic vocoder, and SimulEval's action / segment / states classes from their files.

Substitutions: the sources are 16 kHz, so convert_waveform is the identity and ORG_SAMPLE_RATE (the gate's segment length in
samples per ms) is 16000; the reference's literal 48000 would count 48 kHz samples in a 16 kHz source.

Every setting is streamed in SimulEval's segments; oracle.waitk_oracle must reproduce every action (READ / WRITE, both finished
flags, MT tokens, text, units, durations, waveform within 1e-5) before tests/golden/waitk_policy.npz is written.
"""
from __future__ import annotations

import ast
import math
import os
import sys
import types
from copy import deepcopy

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import GOLD, REF, extract_functions  # noqa: E402
from oracle.gen_golden_agent import load_file_module  # noqa: E402
from oracle.gen_golden_unity import RefUnitY, load_reference_classes  # noqa: E402
from oracle.waitk_oracle import OracleWaitkS2STAgent, OracleWaitkS2TTAgent  # noqa: E402
from streamspeech_b200 import synth  # noqa: E402
from streamspeech_b200.config import ModelConfig, VocoderConfig  # noqa: E402
from streamspeech_b200.dictionary import Dictionary  # noqa: E402

# tag, agent, lagging_k1, lagging_k2, stride_n, stride_n2, unit_per_subword, --segment-size, SimulEval segment (ms), seconds, seed
SETTINGS = [
    ("s2st_default", "s2st", 3, 1, 1, 1, 15, 320, 320, 3.3, 41),    # the reference's defaults; the source ends mid-segment
    ("s2st_k5n2", "s2st", 5, 1, 2, 2, 15, 640, 320, 8.1, 42),       # k1 = 5, n = n2 = 2, --segment-size 640 fed in 320 ms pieces
    ("s2tt_default", "s2tt", 3, 1, 1, 1, 15, 320, 320, 3.3, 41),
    ("s2tt_k5n2", "s2tt", 5, 1, 2, 2, 15, 640, 320, 8.1, 42),
]
SAMPLE_RATE = 16000


def reference_globals(seg, act, gcmvn):
    glb = {"torch": torch, "np": np, "math": math, "deepcopy": deepcopy, "ReadAction": act.ReadAction, "WriteAction": act.WriteAction,
           "SpeechSegment": seg.SpeechSegment, "SAMPLE_RATE": SAMPLE_RATE, "ORG_SAMPLE_RATE": SAMPLE_RATE,
           "convert_waveform": lambda w, sr, to_mono=True, to_sample_rate=None: (w, SAMPLE_RATE)}
    # extract_fbank_features (fairseq/examples/speech_to_text/data_utils.py) + _get_torchaudio_fbank (audio_utils.py)
    tree = ast.parse(open(REF + "/fairseq/fairseq/data/audio/audio_utils.py").read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "_get_torchaudio_fbank"]
    ns = {"torch": torch, "np": np, "Optional": __import__("typing").Optional}
    exec(compile(ast.Module(body=fn, type_ignores=[]), "audio_utils.py", "exec"), ns)
    tree = ast.parse(open(REF + "/fairseq/examples/speech_to_text/data_utils.py").read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "extract_fbank_features"]
    ns2 = {"torch": torch, "np": np, "Optional": __import__("typing").Optional, "Path": __import__("pathlib").Path,
           "convert_waveform": glb["convert_waveform"], "_get_kaldi_fbank": lambda *a: None, "_get_torchaudio_fbank": ns["_get_torchaudio_fbank"]}
    exec(compile(ast.Module(body=fn, type_ignores=[]), "data_utils.py", "exec"), ns2)
    glb["extract_fbank_features"] = ns2["extract_fbank_features"]
    return glb


def load_simuleval():
    seg = load_file_module("_ref_simuleval_segments", REF + "/SimulEval/simuleval/data/segments.py")
    for name in ("simuleval", "simuleval.data", "simuleval.agents"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
    sys.modules["simuleval.data.segments"] = seg
    act = load_file_module("simuleval.agents.actions", REF + "/SimulEval/simuleval/agents/actions.py")
    sys.modules["simuleval.agents.actions"] = act
    sts = load_file_module("simuleval.agents.states", REF + "/SimulEval/simuleval/agents/states.py")
    return seg, act, sts


def build_reference_agent(kind, model, cfg, gcmvn, vsd_wn, k1, k2, n, n2, ups, segment_size, R):
    """A `self` for the reference policy(), constructed as the agents' __init__ (:107-183) constructs it"""
    from agent.sequence_generator import SequenceGenerator
    from agent.tts.codehifigan import CodeGenerator

    search = R["search"]
    seg, act, sts = load_simuleval()
    glb = reference_globals(seg, act, gcmvn)
    path = REF + ("/agent/speech_to_speech.wait-k-stride-n.agent.py" if kind == "s2st" else "/agent/speech_to_text.wait-k-stride-n.agent.py")
    cls = "WaitkS2STAgent" if kind == "s2st" else "EnglishSpeechCounter"
    fe = extract_functions(path, "OnlineFeatureExtractor", ["__call__", "transform"], glb)
    ag = extract_functions(path, cls, ["policy", "reset"], glb)

    class FeatureExtractor:  # OnlineFeatureExtractor.__init__ (:45-60) with the agent's default --sample-rate 16000
        shift_size, window_size, sample_rate, feature_dim = 10, 25, SAMPLE_RATE, 80
        num_samples_per_shift = 160
        num_samples_per_window = 400
        len_ms_to_samples = staticmethod(lambda x: x * SAMPLE_RATE / 1000)
        global_cmvn = gcmvn
        device = "cpu"
        __call__ = fe["__call__"]
        transform = fe["transform"]

    gen = CodeGenerator(VocoderConfig().to_json_dict())
    gen.load_state_dict(vsd_wn, strict=True)
    gen.eval()
    gen.remove_weight_norm()
    voc_forward = extract_functions(REF + "/agent/tts/vocoder.py", "CodeHiFiGANVocoderWithDur", ["forward"], {"torch": torch, "Dict": dict})["forward"]

    class Vocoder:
        model = gen

        def __call__(self, x, dur_prediction=False):
            return voc_forward(self, x, dur_prediction)

    tgt_dict_mt = Dictionary.synthetic(cfg.tgt_vocab)
    tgt_dict = Dictionary.units(cfg.unit_vocab - 4, blank=False)

    class RefAgent:
        policy = ag["policy"]
        reset = ag["reset"]

        def __init__(self):
            self.device = "cpu"
            self.eos = 2
            self.states = sts.AgentStates()
            self.feature_extractor = FeatureExtractor()
            self.models = [model]
            self.dict = {"tgt": tgt_dict, "target_unigram": tgt_dict_mt}
            common = dict(beam_size=1, max_len_a=1, max_len_b=200, max_len=0, min_len=1, normalize_scores=True, len_penalty=1.0,
                          unk_penalty=0.0, temperature=1.0, match_source_len=False, no_repeat_ngram_size=0, symbols_to_strip_from_output=None)
            self.generator = SequenceGenerator(self.models, tgt_dict, search_strategy=search.BeamSearch(tgt_dict), eos=tgt_dict.eos(), **common)
            self.generator_mt = SequenceGenerator(self.models, tgt_dict_mt, search_strategy=search.BeamSearch(tgt_dict_mt), eos=tgt_dict_mt.eos(),
                                                  **common)
            self.vocoder = Vocoder()
            self.dur_prediction = True
            self.lagging_k1, self.lagging_k2, self.segment_size = k1, k2, segment_size
            self.stride_n, self.unit_per_subword, self.stride_n2 = n, ups, n2
            self.reset()

        def push(self, samples, finished):  # SimulEval agents/agent.py -> states.update_source
            self.states.update_source(seg.SpeechSegment(content=samples, sample_rate=SAMPLE_RATE, finished=finished))

    return RefAgent(), tgt_dict_mt


def run_setting(setting, model, cfg, sd, gcmvn, vsd_wn, R, report):
    tag, kind, k1, k2, n, n2, ups, segment_size, chunk_ms, seconds, seed = setting
    ref, tdict = build_reference_agent(kind, model, cfg, gcmvn, vsd_wn, k1, k2, n, n2, ups, segment_size, R)
    kw = dict(lagging_k1=k1, lagging_k2=k2, stride_n=n, stride_n2=n2, unit_per_subword=ups, segment_size=segment_size, sample_rate=SAMPLE_RATE,
              symbols=lambda t: tdict[t])
    mine = OracleWaitkS2STAgent(cfg, sd, gcmvn, vsd_wn, **kw) if kind == "s2st" else OracleWaitkS2TTAgent(cfg, sd, gcmvn, **kw)
    wav = synth.make_audio(seconds, seed=seed)
    step = math.ceil(chunk_ms / 1000 * SAMPLE_RATE)  # SimulEval's segment (evaluator/instance.py send_source)
    out = {"setting": np.array([k1, k2, n, n2, ups, segment_size, chunk_ms, seed]), "kind": np.array(kind), "seconds": np.array(seconds)}
    kinds, flags, texts, worst, empty_finish = [], [], [], 0.0, False
    for ci, i in enumerate(range(0, len(wav), step)):
        fin = i + step >= len(wav)
        chunk = wav[i:i + step].tolist()
        ref.push(chunk, fin)
        mine.push(chunk, finished=fin)
        a_ref = ref.policy()
        a = mine.policy()
        for k in ("new_subword_tokens", "new_unit_tokens", "mt_tokens", "units", "dur"):
            if k in a.trace:
                out[f"call{ci}_{k}"] = np.array(a.trace[k], dtype=np.int64)
        if "unit_margin" in a.trace:
            out[f"call{ci}_unit_margin"] = np.array(a.trace["unit_margin"])
        if a_ref.is_read():
            assert a.kind == "read", (tag, ci)
            kinds.append(0)
            flags.append([False, False])
            texts.append("")
            continue
        assert a.kind == "write", (tag, ci)
        kinds.append(1)
        if kind == "s2st":
            content = a_ref.content.content
            assert a_ref.finished == a.finished and a_ref.content.finished == a.seg_finished, (tag, ci)
            assert len(content) == len(a.wav), (tag, ci, len(content), len(a.wav))
            if len(content):
                worst = max(worst, float(np.abs(np.array(content) - np.array(a.wav)).max()))
            else:
                empty_finish = True
            out[f"call{ci}_wav"] = np.array(content, dtype=np.float32)
            flags.append([a_ref.finished, a_ref.content.finished])
            texts.append("")
            if ref.unit is not None:  # (None after the finishing reset)
                assert ref.unit == a.trace["units"], (tag, ci)
        else:
            assert a_ref.content == a.wav and a_ref.finished == a.finished, (tag, ci, a_ref.content, a.wav)
            flags.append([a_ref.finished, False])
            texts.append(a_ref.content)
        if ref.tgt_subwords_indices is not None:
            assert ref.tgt_subwords_indices.view(-1).tolist() == a.trace["mt_tokens"], (tag, ci)
    assert worst < 1e-5, (tag, worst)
    assert sum(kinds) >= 2, (tag, kinds)
    out.update(kinds=np.array(kinds), flags=np.array(flags), texts=np.array(texts), empty_finish=np.array(empty_finish))
    last_mt = max((ci for ci in range(len(kinds)) if f"call{ci}_mt_tokens" in out), default=None)
    report[tag] = (f"{len(kinds)} calls, kinds {''.join(map(str, kinds))}, final MT {len(out[f'call{last_mt}_mt_tokens'])} tokens"
                   + (f", wav max-abs {worst:.2e}, empty finishing write: {empty_finish}" if kind == "s2st" else ""))
    return out


def main():
    assert ref_loader.available(), "reference tree missing"
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    R = load_reference_classes()
    cfg = ModelConfig.unity_default()
    sd = synth.make_unity_state_dict(cfg, seed=0)
    gcmvn = synth.make_gcmvn(cfg)
    vsd_wn = synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=True)
    model = RefUnitY(cfg, sd, R).eval()
    report, gold = {}, {"tags": np.array([s[0] for s in SETTINGS])}
    for s in SETTINGS:
        gold.update({f"{s[0]}_{k}": v for k, v in run_setting(s, model, cfg, sd, gcmvn, vsd_wn, R, report).items()})
    path = os.path.join(GOLD, "waitk_policy.npz")
    np.savez_compressed(path, **gold)
    for k, v in report.items():
        print(f"{k:14s} {v}")
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
