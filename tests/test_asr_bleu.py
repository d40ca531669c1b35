"""CPU: the ASR-BLEU front door's host side.  sacrebleu 2.2.0's corpus_bleu restatement against hand-computed answers, the beam-1 CTC
decoding rule and letter post-processing, the rm_silence rule, file discovery, references and the output files of both variants."""
import math
import os
import struct

import numpy as np
import pytest
import torch

from oracle import asr_oracle as ao
from streamspeech_b200 import asr_bleu
from streamspeech_b200.asr import ASRTranscriber, AudioRefused, load_checkpoint, parse_settings, remove_silence
from streamspeech_b200.sacrebleu_compat import corpus_bleu, ngram_counts, tokenize_13a

VOCAB = ao.SPECIALS + ["|", "e", "t", "a"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "asr_w2v.npz")


# ---- BLEU
def test_bleu_perfect_match():
    b = corpus_bleu(["the cat sat on the mat"], [["the cat sat on the mat"]])
    assert (b.counts, b.totals) == ([6, 5, 4, 3], [6, 5, 4, 3])
    assert b.score == pytest.approx(100.0)
    assert str(b) == "BLEU = 100.00 100.0/100.0/100.0/100.0 (BP = 1.000 ratio = 1.000 hyp_len = 6 ref_len = 6)"
    assert b.format(width=2) == str(b)


def test_bleu_empty_hypothesis():
    b = corpus_bleu([""], [["a b c"]])
    assert (b.counts, b.totals, b.sys_len, b.ref_len) == ([0, 0, 0, 0], [0, 0, 0, 0], 0, 3)
    assert str(b) == "BLEU = 0.00 0.0/0.0/0.0/0.0 (BP = 0.000 ratio = 0.000 hyp_len = 0 ref_len = 3)"


def test_bleu_brevity_penalty():
    b = corpus_bleu(["a b c d"], [["a b c d e f g h"]])
    assert (b.counts, b.totals) == ([4, 3, 2, 1], [4, 3, 2, 1])
    assert b.bp == pytest.approx(math.exp(1 - 8 / 4))
    assert b.score == pytest.approx(100 * math.exp(-1))
    assert str(b) == "BLEU = 36.79 100.0/100.0/100.0/100.0 (BP = 0.368 ratio = 0.500 hyp_len = 4 ref_len = 8)"


def test_bleu_exp_smoothing_of_zero_higher_orders():
    # unigrams 5/5; bigrams ab bc cd de vs ac ce eb bd: 0/4; trigrams 0/3; 4-grams 0/2
    b = corpus_bleu(["a b c d e"], [["a c e b d"]])
    assert (b.counts, b.totals) == ([5, 0, 0, 0], [5, 4, 3, 2])
    p = [100.0, 100 / (2 * 4), 100 / (4 * 3), 100 / (8 * 2)]
    assert b.precisions == pytest.approx(p)
    assert b.score == pytest.approx((p[0] * p[1] * p[2] * p[3]) ** 0.25)
    assert str(b) == f"BLEU = {b.score:.2f} 100.0/12.5/8.3/6.2 (BP = 1.000 ratio = 1.000 hyp_len = 5 ref_len = 5)"


def test_bleu_corpus_sums_statistics():
    b = corpus_bleu(["a b", "c d e"], [["a b", "c x e"]])
    # unigrams: 2 + 2 of 2 + 3; bigrams: 1 + 0 of 1 + 2; trigrams: 0 + 0 of 0 + 1; 4-grams: none
    assert (b.counts, b.totals, b.sys_len, b.ref_len) == ([4, 1, 0, 0], [5, 3, 1, 0], 5, 5)
    # the 4-gram total is 0: the loop stops and its precision stays 0, so the score is 0 (sacrebleu without effective order)
    assert b.precisions[:3] == pytest.approx([80.0, 100 / 3, 100 / 2]) and b.precisions[3] == 0.0
    assert b.score == pytest.approx(0.0, abs=1e-12)


def test_bleu_is_case_sensitive_and_counts_clip():
    b = corpus_bleu(["the the the the"], [["The cat the"]])
    assert b.counts[0] == 1  # "the" clipped to its one lower-case occurrence; "The" does not match
    assert ngram_counts(["a", "a", "a"])[("a", "a")] == 2


def test_13a_punctuation_and_numbers():
    assert tokenize_13a("Hello, world! It costs $3.50 (i.e. 1,000-2).") == "Hello , world ! It costs $ 3.50 ( i . e . 1,000 - 2 ) ."
    assert tokenize_13a("well-known a.b 3,b x&amp;y") == "well-known a . b 3 , b x & y"
    assert tokenize_13a("  many   spaces\n") == "many spaces"


# ---- decoding rule
def emissions(rows):
    e = torch.full((len(rows), len(VOCAB)), -1.0, dtype=torch.float64)
    for t, r in enumerate(rows):
        for idx, v in r.items():
            e[t, idx] = v
    return e


def test_unk_winning_the_raw_argmax_is_skipped():
    e = emissions([{3: 5.0, 5: 1.0}, {3: 5.0, 6: 2.0, 5: 2.0}])
    assert ao.best_path(e) == [5, 5]  # unk excluded; the lowest index wins the 6 / 5 tie


def test_repeats_split_by_blanks_and_silences():
    a, e_, bar = 7, 5, 4
    path = [a, a, 0, a, bar, bar, e_, 0, 0, e_]
    assert ao.get_tokens(path) == [a, a, bar, e_, e_]
    assert ao.letters(ao.get_tokens(path), VOCAB) == "aa ee"


def test_leading_trailing_silence_and_all_blank():
    assert ao.letters(ao.get_tokens([4, 4, 0, 7, 0, 4, 6, 4]), VOCAB) == "a t"
    assert ao.letters(ao.get_tokens([0] * 7), VOCAB) == ""
    assert ao.letters(ao.get_tokens([4, 0, 4]), VOCAB) == ""  # "||" -> two spaces -> stripped
    assert ao.letters(ao.get_tokens([7, 4, 0, 4, 6]), VOCAB) == "a  t"  # a blank between two silences keeps both


# ---- rm_silence
def zeros_case(pattern):
    x = np.ones(len(pattern), dtype=np.float32)
    x[np.array(pattern) == 0] = 0.0
    return x


# A zero goes when the 10 samples starting at it, or the 10 ending at it, are all zero (cyclically): in a run of L >= 10 zeros the
# ones at offsets p <= L - 10 or p >= 9 go, so a run of 10 loses its two ends and a run of 19 or more goes whole.
@pytest.mark.parametrize("pattern,kept", [
    ([1] + [0] * 9 + [1], 11),                       # a run of 9 stays
    ([1] + [0] * 10 + [1], 10),                      # a run of exactly 10 loses its first and last zero
    ([1] + [0] * 12 + [1], 8),                       # offsets 0-2 and 9-11 of a run of 12
    ([1] + [0] * 19 + [1], 2),                       # a run of 19 goes whole
    ([0] * 5 + [1, 1] + [0] * 5, 10),                # 5 + 5 wrap around the ends into one run of 10
    ([0] * 4 + [1, 1] + [0] * 5, 11),                # 4 + 5 = 9 wrapped: stays
    ([0] * 12, 0),
    ([1, 0, 1, 0] * 6, 24),
])
def test_rm_silence_rule(pattern, kept):
    x = zeros_case(pattern) * np.arange(1, len(pattern) + 1, dtype=np.float32)
    got = remove_silence(x)
    z = np.array(pattern) == 0
    n = len(z)
    want = [x[i] for i in range(n) if not (z[i] and (all(z[(i + j) % n] for j in range(10)) or all(z[(i - j) % n] for j in range(10))))]
    assert len(got) == kept and np.array_equal(got, np.array(want, dtype=np.float32))


def test_rm_silence_matches_the_reference_fixture():
    """asr_bleu_rm_silence/utils.py's own load_audiofile, run by oracle/gen_golden_asr.py on the patterns above and random signals"""
    g = np.load(GOLDEN)
    for i in range(len(g["rm_in_off"]) - 1):
        x = g["rm_in"][g["rm_in_off"][i]:g["rm_in_off"][i + 1]]
        assert np.array_equal(remove_silence(x), g["rm_out"][g["rm_out_off"][i]:g["rm_out_off"][i + 1]]), i


# ---- files
def write_wav(path, x, rate=16000, channels=1):
    pcm = (np.clip(x, -1, 1 - 1 / 32768) * 32768).astype("<i2").tobytes()
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(pcm)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<IHHIIHH", 16, 1, channels, rate, rate * 2 * channels, 2 * channels, 16))
        f.write(b"data" + struct.pack("<I", len(pcm)) + pcm)


def test_file_discovery(tmp_path):
    for name in ("0_pred.wav", "1_spk3_pred.wav", "2_pred.wav"):
        write_wav(tmp_path / name, np.zeros(10))
    got = asr_bleu.extract_audio_for_eval(str(tmp_path), "n_pred.wav")
    assert [os.path.basename(p) for p in got] == ["0_pred.wav", "1_spk3_pred.wav", "2_pred.wav"]
    assert asr_bleu.extract_audio_for_eval(str(tmp_path), "n_pred.wav", sort_numeric=True) == got
    os.remove(tmp_path / "1_spk3_pred.wav")
    write_wav(tmp_path / "3_pred.wav", np.zeros(10))
    with pytest.raises(AssertionError, match="1_pred.wav"):
        asr_bleu.extract_audio_for_eval(str(tmp_path), "n_pred.wav")


def test_references(tmp_path):
    (tmp_path / "ref.txt").write_text("  Hello world \nsecond\n")
    assert asr_bleu.extract_text_for_eval(str(tmp_path / "ref.txt"), "txt") == ["Hello world", "second"]
    (tmp_path / "ref.tsv").write_text('id\ttgt_text\n0\t "quoted" text \n\n1\tnext\n')
    assert asr_bleu.extract_text_for_eval(str(tmp_path / "ref.tsv"), "tsv", "tgt_text") == ['"quoted" text', "next"]


class FakeTranscriber:
    """the transcriber's host side (ASRTranscriber.load_audio, the real one) with a stand-in for the GPU: 'transcribes' a waveform as
    the letters of its length"""

    sample_rate = 16000
    load_audio = ASRTranscriber.load_audio

    def num_frames(self, n):
        return ao.num_frames(n, [10, 3, 3, 3, 3, 2, 2], [5, 2, 2, 2, 2, 2, 2])

    def transcribe(self, waves):
        return [f"len {len(w)}" for w in waves]


def test_output_files_of_both_variants(tmp_path, capsys):
    d = tmp_path / "wavs"
    d.mkdir()
    write_wav(d / "0_pred.wav", np.full(800, 0.5))
    write_wav(d / "1_pred.wav", np.zeros(300))               # too short for one frame
    write_wav(d / "2_pred.wav", np.concatenate([np.full(600, 0.25), np.zeros(40)]))
    (tmp_path / "ref.txt").write_text("len 800\nlen 300\nlen 640\n")
    argv = ["--lang", "en", "--audio_dirpath", str(d), "--reference_path", str(tmp_path / "ref.txt"), "--reference_format", "txt",
            "--results_dirpath", str(tmp_path / "res")]
    tr, bleu = asr_bleu.main(argv, transcriber=FakeTranscriber())
    assert tr == ["len 800", "", "len 640"]  # a failed transcription scores as "" in the default variant
    assert (d / "pred.txt").read_text() == "len 800\n\nlen 640"
    assert (tmp_path / "res" / "txt_en_bleu.txt").read_text() == bleu.format(width=2)
    assert capsys.readouterr().out == str(bleu) + "\n"
    # rm_silence variant: silence removed, transcripts file, no pred.txt, and a failure propagates
    os.remove(d / "pred.txt")
    with pytest.raises(ValueError, match="fewer than one encoder frame"):
        asr_bleu.main(argv + ["--rm-silence"], transcriber=FakeTranscriber())
    write_wav(d / "1_pred.wav", np.full(500, 0.1))
    tr, bleu = asr_bleu.main(argv + ["--rm-silence", "--transcripts_path", str(tmp_path / "t.txt")], transcriber=FakeTranscriber())
    assert tr == ["len 800", "len 500", "len 600"]
    assert (tmp_path / "t.txt").read_text() == "len 800\nlen 500\nlen 600\n"
    assert not (d / "pred.txt").exists()


def test_model_flags_refuse_downloads_and_other_languages():
    base = ["--audio_dirpath", ".", "--reference_path", "r", "--reference_format", "txt"]
    with pytest.raises(SystemExit, match="only the `en`"):
        asr_bleu.check_model_args(asr_bleu.parse_args(base + ["--lang", "fr"]))
    with pytest.raises(SystemExit, match="wav2vec_vox_960h_pl.pt"):
        asr_bleu.check_model_args(asr_bleu.parse_args(base + ["--lang", "en"]))
    with pytest.raises(SystemExit, match="dict.ltr.txt"):
        asr_bleu.check_model_args(asr_bleu.parse_args(base + ["--lang", "en", "--asr-model", "m.pt",
                                                             "--asr-dict", "https://dl.fbaipublicfiles.com/fairseq/wav2vec/dict.ltr.txt"]))


@pytest.mark.parametrize("rm", [False, True])
def test_unsupported_audio_is_refused_not_scored_empty(tmp_path, rm):
    d = tmp_path / "wavs"
    d.mkdir()
    write_wav(d / "0_pred.wav", np.full(800, 0.5))
    write_wav(d / "1_pred.wav", np.full(900, 0.5), rate=22050)
    (tmp_path / "ref.txt").write_text("a\nb\n")
    argv = ["--lang", "en", "--audio_dirpath", str(d), "--reference_path", str(tmp_path / "ref.txt"), "--reference_format", "txt"]
    with pytest.raises(AudioRefused, match="1_pred.wav: 22050 Hz"):
        asr_bleu.main(argv + (["--rm-silence"] if rm else []), transcriber=FakeTranscriber())
    write_wav(d / "1_pred.wav", np.full(900, 0.5), channels=2)
    with pytest.raises(AudioRefused, match="2 channels"):
        asr_bleu.main(argv + (["--rm-silence"] if rm else []), transcriber=FakeTranscriber())
    (d / "1_pred.wav").write_bytes(b"not a wav file at all")  # unreadable: the reference's torchaudio.load fails too
    if rm:
        with pytest.raises(ValueError, match="RIFF"):
            asr_bleu.main(argv + ["--rm-silence"], transcriber=FakeTranscriber())
    else:
        tr, _ = asr_bleu.main(argv, transcriber=FakeTranscriber())
        assert tr == ["len 800", ""]


def test_tsv_cells_pandas_would_not_read_as_text_are_refused(tmp_path):
    (tmp_path / "na.tsv").write_text("id\ttgt\n0\thello\n1\tNA\n")
    with pytest.raises(ValueError, match="NaN"):
        asr_bleu.extract_text_for_eval(str(tmp_path / "na.tsv"), "tsv", "tgt")
    (tmp_path / "num.tsv").write_text("id\ttgt\n0\t12\n1\t3.5\n")
    with pytest.raises(ValueError, match="only numbers"):
        asr_bleu.extract_text_for_eval(str(tmp_path / "num.tsv"), "tsv", "tgt")


def test_checkpoint_with_uninstalled_cfg_classes_still_loads(tmp_path, monkeypatch):
    import sys
    import types

    mod = types.ModuleType("fake_omegaconf_for_test")

    class DictConfig:
        def __init__(self):
            self.content = {"task": {"normalize": True}}

    DictConfig.__module__ = mod.__name__
    DictConfig.__qualname__ = "DictConfig"
    mod.DictConfig = DictConfig
    monkeypatch.setitem(sys.modules, mod.__name__, mod)
    w = {"w2v_encoder.proj.weight": torch.arange(6.0).view(2, 3)}
    torch.save({"model": w, "cfg": DictConfig()}, tmp_path / "ck.pt")
    ck, complete = load_checkpoint(str(tmp_path / "ck.pt"))
    assert complete and isinstance(ck["cfg"], DictConfig)
    monkeypatch.delitem(sys.modules, mod.__name__)
    ck, complete = load_checkpoint(str(tmp_path / "ck.pt"))  # the class is gone: the weights load, the cfg is opaque
    assert not complete and torch.equal(ck["model"]["w2v_encoder.proj.weight"], w["w2v_encoder.proj.weight"])
    assert parse_settings(["normalize=False", "extractor_mode=layer_norm"]) == {"normalize": False, "extractor_mode": "layer_norm"}
    with pytest.raises(ValueError, match="unknown setting"):
        parse_settings(["bogus=1"])
