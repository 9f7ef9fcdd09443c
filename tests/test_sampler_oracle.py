"""The oracle's restatement of one sampling step (nor_sample_top_p, oracle/nano_oracle.c) against the unmodified reference's
own softmax and sample_top_p (infer.c:616-634, 1062-1109), on the CPU.

The id and the six ids the observation hook reports (infer.c:1086-1095) must be equal on every input family of
sampler_cases.py, at vocabulary sizes on both sides of the device sampler's 4096-entry chunk and at the Nano-168M and
Qwen3 sizes.  n0 = 0 is left out: the reference reads probindex[-1] there.
"""
import ctypes as C

import numpy as np
import pytest

import sampler_cases as sc
from nano_b200 import modelfile as mf
from oracle import bindings as ob

needs_ref = pytest.mark.skipif(not ob.ref_available("strict"), reason="needs the unmodified reference (oracle/_ref)")


@pytest.fixture(scope="module")
def ref():
    path = mf.cached_model(mf.PRESETS["toy-nano"], mf.QUANT_Q80, 64)
    return ob.RefEngine(path, 8, "strict")           # only its context (observation hook) is used


def ref_sample(ref, logits, T, top_p, coin):
    L = ref.L
    p = (np.ascontiguousarray(logits, np.float32) / np.float32(T)).astype(np.float32)     # infer.c:1174-1176
    L.softmax(p.ctypes.data_as(ob.f32p), p.size)
    pi = (ob.ProbIndex * p.size)()
    return L.sample_top_p(ref.h, p.ctypes.data_as(ob.f32p), p.size, top_p, C.cast(pi, C.c_void_p), coin)


@needs_ref
@pytest.mark.parametrize("V", [4096, 4097, 16384, 151936])
def test_sample_top_p_matches_reference(ref, V):
    n = 0
    for label, lg, T, top_p, coin in sc.cases(V):
        tok, six, n0, last = ob.sample_top_p(lg, T, top_p, coin)
        assert n0 > 0, label
        rtok = ref_sample(ref, lg, T, top_p, coin)
        assert tok == rtok, f"V {V} {label}: oracle {tok}, reference {rtok} (n0 {n0}, last {last})"
        n += 1
    assert n > 60


@needs_ref
@pytest.mark.parametrize("V", [4096, 4097, 16384, 151936])
def test_observed_ids_match_reference(ref, V):
    """The six ids sample_top_p reports to the observation hook, read back through the harness (orh_last_sample)."""
    last_sample = ob.ref_last_sample("strict")
    if last_sample is None:
        pytest.skip("oracle/_ref was built from a harness without orh_last_sample; rebuild it from the reference tree")
    for label, lg, T, top_p, coin in sc.cases(V):
        _, six, n0, _ = ob.sample_top_p(lg, T, top_p, coin)
        ref_sample(ref, lg, T, top_p, coin)
        got = np.zeros(6, np.uint32)
        last_sample(got.ctypes.data_as(ob.u32p))
        assert six == got.tolist(), f"V {V} {label}: oracle {six}, reference {got.tolist()} (n0 {n0})"


def test_empty_nucleus_rule():
    """n0 = 0: the first index of the largest probability, six zero ids."""
    for V in (512, 4097, 151936):
        lg, T, top_p, want = sc.empty_nucleus_case(V)
        assert ob.sample_top_p(lg, T, top_p, 0.5) == (want, [0] * 6, 0, -1)
