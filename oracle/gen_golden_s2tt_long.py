"""Pin the S2TT agent on the 10 s bench utterance, whose finishing MT call is allowed more than 1024 positions (build container only).

Run:  python -m oracle.gen_golden_s2tt_long        (needs the reference tree; CPU only, under a minute)

The reference's own `StreamSpeechS2TTAgent.policy()` (run from source on reference modules, exactly as gen_golden_agent.py's s2tt320
case: `SequenceGenerator` with use_incremental_states=True, max_len_a = 1, max_len_b = 200) streams the 10 s bench utterance
(synth.make_audio(10.0, seed=1234)) in 320 ms segments next to `OracleS2TTAgent`.  The finishing call runs with max_len = min(F + 200,
max_decoder_positions - 1) = 1198, and the incremental state keeps one duplicate entry per earlier MT call on top (SURVEY.md N12).
The reference neither asserts nor truncates; what ends the search is the model: the synthetic checkpoint's eos is a positional
feature (synth.py), and the hypothesis of this utterance stops at 91 tokens, far below max_len.  So the state of the reference holds
final_len + MT calls entries, not more than 1024: the fixture pins what the agent must output for an utterance whose max_len exceeds
1024, and the searches that really fill more than 1024 entries are tested against the float64 oracle on a checkpoint without eos
(tests/test_s2tt_long.py).  Recorded per call: the action, the text delta, the CTC tokens and the MT hypothesis; plus the final
hypothesis length, the finishing call's max_len and the self-attention entries the reference's state held when the utterance ended.

Writes tests/golden/agent_policy_s2tt_long.npz only; agent_policy.npz is gen_golden_agent.py's and is not touched.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle.agent_oracle import OracleS2TTAgent
from oracle.gen_golden_agent import GOLD, build_reference_agent
from oracle.streamspeech_oracle import StreamSpeechOracle
from streamspeech_b200 import synth
from streamspeech_b200.config import ModelConfig
from streamspeech_b200.dictionary import Dictionary

SEGMENT_MS, SECONDS, SEED = 320, 10.0, 1234


def self_attention_entries(model, generator) -> int:
    """entries of the reference's incremental self-attention state (prev_key [1, heads, entries, head_dim]), equal in every layer"""
    state = generator.incremental_states[0]
    n = {int(layer.self_attn._get_input_buffer(state)["prev_key"].size(2)) for layer in model.target_unigram_decoder.layers}
    assert len(n) == 1, n
    return n.pop()


def main():
    torch.set_grad_enabled(False)
    cfg = ModelConfig()
    sd = synth.make_model_state_dict(cfg, 0)
    gcmvn = synth.make_gcmvn(cfg)
    vsd_wn = synth.make_vocoder_state_dict(cfg.vocoder, 1, weight_norm=True)
    ref, model, _, _ = build_reference_agent(cfg, sd, vsd_wn, gcmvn, SEGMENT_MS, kind="s2tt")
    d = Dictionary.synthetic(cfg.tgt_vocab)
    mine = OracleS2TTAgent(StreamSpeechOracle(cfg, sd, None, gcmvn), SEGMENT_MS, symbols=lambda t: d[t])

    # the finishing call resets the agent, and with it the generator's state: note the entries it held just before
    entries = []
    reset_states = ref.generator_mt.reset_incremental_states

    def noting_reset():
        if ref.generator_mt.incremental_states is not None:
            entries.append(self_attention_entries(model, ref.generator_mt))
        reset_states()

    ref.generator_mt.reset_incremental_states = noting_reset

    wav = synth.make_audio(SECONDS, seed=SEED)
    n = 16 * SEGMENT_MS
    out = {"segment_ms": np.array(SEGMENT_MS), "seconds": np.array(SECONDS), "seed": np.array(SEED)}
    kinds, texts, mt_calls = [], [], 0
    for ci, i in enumerate(range(0, len(wav), n)):
        fin = i + n >= len(wav)
        chunk = wav[i:i + n].tolist()
        ref.push(chunk, fin)
        mine.push(chunk, finished=fin)
        a_ref, a = ref.policy(), mine.policy()
        for k in ("asr_tokens", "st_tokens"):
            out[f"call{ci}_{k}"] = np.array(a.trace.get(k, []), dtype=np.int64)
        mt_calls += "mt_tokens" in a.trace
        if a_ref.is_read():
            assert a.kind == "read", ci
            kinds.append(0)
            texts.append("")
            continue
        assert a.kind == "write" and a_ref.content == a.wav and a_ref.finished == a.finished, (ci, a_ref.content, a.wav)
        if not fin:  # (after the finishing WRITE the reference has reset itself)
            assert ref.tgt_subwords_indices.view(-1).tolist() == mine.tgt_subwords_indices, ci
        kinds.append(1)
        texts.append(a_ref.content)
        out[f"call{ci}_mt_tokens"] = np.array(a.trace["mt_tokens"], dtype=np.int64)
        out[f"call{ci}_finished"] = np.array(a_ref.finished)
    final_len = len(out[f"call{len(kinds) - 1}_mt_tokens"])
    frames = (len(wav) - 240) // 160
    max_len = min(frames + 200, 1199)
    assert kinds[-1] == 1 and max_len > 1024 and final_len <= max_len, (kinds, final_len, frames)
    assert len(entries) == 1 and entries[0] == final_len + mt_calls, (entries, final_len, mt_calls)
    out["kinds"] = np.array(kinds)
    out["texts"] = np.array(texts)
    out["final_len"] = np.array(final_len)
    out["final_max_len"] = np.array(max_len)
    out["self_attention_entries"] = np.array(entries[0])
    out["mt_calls"] = np.array(mt_calls)
    np.savez_compressed(os.path.join(GOLD, "agent_policy_s2tt_long.npz"), **out)
    print(f"{len(kinds)} calls, kinds {''.join(map(str, kinds))}, {mt_calls} MT calls, final hypothesis {final_len} tokens (max_len {max_len}), "
          f"{entries[0]} self-attention entries in the reference's incremental state")


if __name__ == "__main__":
    main()
