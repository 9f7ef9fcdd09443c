"""CPU tests: the C-ABI library loads, exports every symbol include/nano_b200.h declares, and refuses to
compute without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from nano_b200 import build as nb_build, engine as E, modelfile as mf


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "nano_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(nb200_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    out = subprocess.run(["nm", "-D", "--defined-only", nb_build.ENGINE_SO], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (nb200_\w+)", out))
    missing = [s for s in declared_symbols() if s not in exported]
    assert not missing, f"declared in include/nano_b200.h but not exported: {missing}"
    assert len(declared_symbols()) >= 20


def test_binding_covers_header():
    assert set(E.EXPORTS) == set(declared_symbols())
    L = E.lib()
    for s in E.EXPORTS:
        assert hasattr(L, s)


def test_sm90a_code_is_embedded():
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", nb_build.ENGINE_SO], capture_output=True, text=True).stdout
    assert "sm_90a" in out


@pytest.mark.skipif(E.device_count() > 0, reason="box has a GPU")
def test_no_cpu_fallback():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, mf.QUANT_Q80, 64)
    with pytest.raises(E.NB200Error, match="no CUDA device"):
        E.Engine(path, 16)
    with pytest.raises(E.NB200Error, match="no CUDA device"):
        E.op_q80_quantize(np.zeros(128, np.float32), 64)


def test_product_does_not_reference_oracle():
    """Nothing under nano_b200/ may import, link or dlopen anything under oracle/."""
    bad = []
    for dirpath, _d, files in os.walk(os.path.join(ROOT, "nano_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".c", ".h")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                if re.search(r"(from|import)\s+oracle|oracle/|libnano_oracle|libnano_ref_", txt):
                    bad.append(f)
    assert not bad, bad
    ldd = subprocess.run(["ldd", nb_build.ENGINE_SO], capture_output=True, text=True).stdout
    assert "oracle" not in ldd and "nano_ref" not in ldd
