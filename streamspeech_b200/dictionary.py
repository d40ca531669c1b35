"""fairseq `Dictionary` look-alike: index <-> symbol, specials <s>=0 <pad>=1 </s>=2 <unk>=3
(fairseq/data/dictionary.py; unit dictionary + <blank>: researches/ctc_unity/tasks/speech_to_speech_ctc.py:15-17)."""
from __future__ import annotations

import os
from typing import Dict, List


class Dictionary:
    def __init__(self, symbols: List[str]):
        self.symbols = ["<s>", "<pad>", "</s>", "<unk>"] + list(symbols)
        self.indices: Dict[str, int] = {s: i for i, s in enumerate(self.symbols)}
        self.bos_index, self.pad_index, self.eos_index, self.unk_index = 0, 1, 2, 3
        self.blank_index = self.indices.get("<blank>", None)

    def __len__(self):
        return len(self.symbols)

    def __getitem__(self, idx):
        idx = int(idx)
        return self.symbols[idx] if idx < len(self.symbols) else "<unk>"

    def index(self, sym):
        return self.indices.get(sym, self.unk_index)

    def bos(self):
        return self.bos_index

    def pad(self):
        return self.pad_index

    def eos(self):
        return self.eos_index

    def unk(self):
        return self.unk_index

    @classmethod
    def load(cls, path: str) -> "Dictionary":
        """`<symbol> <count>` per line (fairseq Dictionary.add_from_file)."""
        syms = []
        with open(path, encoding="utf-8") as f:
            for line in f:
                line = line.rstrip("\n")
                if not line:
                    continue
                sym = line.rsplit(" ", 1)[0] if " " in line else line
                syms.append(sym)
        return cls(syms)

    @classmethod
    def synthetic(cls, size: int) -> "Dictionary":
        """Deterministic stand-in for an SPM unigram vocabulary of `size` entries (incl. the 4 specials):
        every third piece starts a word (▁), so the whole-word logic of the agents has something to bite on."""
        return cls([("▁" if i % 3 == 0 else "") + f"w{i}" for i in range(size - 4)])

    @classmethod
    def units(cls, n_units: int, blank: bool = True) -> "Dictionary":
        """target dictionary of the S2UT task: "0".."n-1" then <blank> (speech_to_speech_ctc); UnitY's speech_to_speech task has no
        blank (fairseq/tasks/speech_to_speech.py: --target-code-size symbols after the specials)."""
        return cls([str(i) for i in range(n_units)] + (["<blank>"] if blank else []))

    @classmethod
    def load_multitask(cls, args, cfg):
        """dict paths from the multitask yaml (configs/<pair>/config_mtl_asr_st_ctcst.yaml) under --data-bin."""
        import yaml

        out = {"tgt": cls.units(cfg.unit_vocab - 4, blank=False) if cfg.unity else cls.units(cfg.unit_vocab - 5)}
        path = os.path.join(args.data_bin, args.multitask_config_yaml)
        with open(path) as f:
            mt = yaml.safe_load(f)
        for name, spec in mt.items():
            p = spec["dict"]
            if not os.path.exists(p):
                p = os.path.join(args.data_bin, os.path.basename(os.path.dirname(p)), os.path.basename(p))
            out[name] = cls.load(p)
        return out
