"""Compile the two native pieces of fairseq that the generate fixture pins against into oracle/_ref/ (build container only).

Run:  python -m oracle.build_ref_ext      (needs the reference tree, Cython and a C++ compiler)

  fairseq/data/data_utils_fast.pyx  -> oracle/_ref/data_utils_fast*.so   (batch_by_size_vec; Cython as C++: it uses libcpp.bool)
  fairseq/clib/libbleu/libbleu.cpp  -> oracle/_ref/libbleu.so            (the BLEU statistics fairseq's bleu scorer reads via ctypes)

Neither is part of the package: oracle/gen_golden_generate.py imports them to write tests/golden/offline_generate.npz.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "oracle", "_ref")


def build() -> str:
    import numpy as np
    from Cython.Build import cythonize

    os.makedirs(OUT, exist_ok=True)
    fq = os.path.join(ref_loader.REF, "fairseq", "fairseq")
    with tempfile.TemporaryDirectory() as tmp:
        pyx = os.path.join(tmp, "data_utils_fast.pyx")
        shutil.copy(os.path.join(fq, "data", "data_utils_fast.pyx"), pyx)
        cythonize([pyx], language="c++", quiet=True)
        ext = sysconfig.get_config_var("EXT_SUFFIX")
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-I" + sysconfig.get_paths()["include"], "-I" + np.get_include(),
                        "-DNPY_NO_DEPRECATED_API=NPY_1_7_API_VERSION", os.path.join(tmp, "data_utils_fast.cpp"), "-o",
                        os.path.join(OUT, "data_utils_fast" + ext)], check=True)
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", os.path.join(fq, "clib", "libbleu", "libbleu.cpp"), "-o",
                    os.path.join(OUT, "libbleu.so")], check=True)
    return OUT


if __name__ == "__main__":
    assert ref_loader.available(), "reference tree missing"
    print("built into", build())
