"""The device sampler (nano_b200/csrc/sample.cu) and the classifier's penalty and first-max argmax at real vocabulary sizes.

* tests/sample_probe.cu runs sample_top_p_launch alone on host-given logits.  At V from 512 to 151936 (one to 38 chunks of
  the sequential scans) and on every input family of sampler_cases.py, the id, the six observed ids, n0, the n0 sorted
  probabilities (bit for bit) and their order equal the oracle's nor_sample_top_p; the oracle's probabilities are checked
  against a float64 softmax.  n0 = 0 returns the first-max argmax and six zero ids.
* Fast mode, streaming and multi-kernel: after next_sampled the logits are the raw logits of forward() with every seen id
  divided by the penalty, bit for bit, and (id, six ids) equal the oracle's sampler on them.  The history revisits
  positions with other ids, so the engine's seen-set is rebuilt.
* A classifier of 16 row classes, each first seen at a scattered index and copied after it: logits tie exactly, and the
  greedy pick (per call and in the device loop) is always the first copy, on every path; the sampler's six ids are the
  winning class's first six copies.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import sampler_cases as sc
from conftest import assert_bits_equal
from nano_b200 import build as nb_build, engine as E, modelfile as mf
from oracle import bindings as ob
from test_gpu_stream_matrix import MULTI, STREAM, assert_path, engine

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
Q80 = mf.QUANT_Q80


@pytest.fixture(scope="module")
def probe():
    d = tempfile.mkdtemp(prefix="nb200_sample_probe_")
    so = os.path.join(d, "libsample_probe.so")
    subprocess.run([nb_build.NVCC, *nb_build.GENCODE, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                    "-I" + nb_build.CSRC, os.path.join(HERE, "sample_probe.cu"), "-o", so], check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    lib = C.CDLL(so)
    lib.probe_sample.argtypes = [ob.f32p, C.c_uint32, C.c_float, C.c_float, C.c_float, ob.u32p, ob.f32p, ob.u32p]

    def run(logits, T, top_p, coin):
        lg = np.ascontiguousarray(logits, np.float32)
        out = np.zeros(9, np.uint32); keys = np.zeros(lg.size, np.float32); vals = np.zeros(lg.size, np.uint32)
        rc = lib.probe_sample(lg.ctypes.data_as(ob.f32p), lg.size, T, top_p, coin, out.ctypes.data_as(ob.u32p),
                              keys.ctypes.data_as(ob.f32p), vals.ctypes.data_as(ob.u32p))
        assert rc == 0, f"probe_sample returned {rc}"
        return out, keys, vals
    return run


def check_against_float64(logits, T, sp, si):
    """The oracle's probabilities against exp in float64 of the same float32 differences y - max: one common factor (the
    float32 normaliser's rounding, within its sequential-sum bound) and 4 ulp per probability."""
    y = (np.asarray(logits, np.float32) / np.float32(T)).astype(np.float32)
    d = (y - y.max()).astype(np.float32)
    e = np.exp(d.astype(np.float64))
    p64 = (e / e.sum())[si]
    big = sp > 1e-30
    c = float(np.median(sp[big] / p64[big]))
    assert abs(c - 1.0) <= y.size * 2.0 ** -24, f"normaliser off by {c - 1:.3e}"
    err = np.abs(sp.astype(np.float64) - c * p64) / np.spacing(sp).astype(np.float64)
    assert err.max() <= 4, f"{err.max():.1f} ulp from the float64 softmax at sorted index {int(np.argmax(err))}"


@pytest.mark.parametrize("V", [512, 4095, 4096, 4097, 8192, 8193, 16384, 151936])
def test_device_sampler_matches_oracle(probe, V):
    checked = set()
    for label, lg, T, top_p, coin in sc.cases(V):
        tok, six, n0, last, sp, si = ob.sample_top_p(lg, T, top_p, coin, sorted_out=True)
        out, keys, vals = probe(lg, T, top_p, coin)
        what = f"V {V} {label} (n0 {n0}, last {last})"
        assert int(out[7]) == n0, f"{what}: device n0 {out[7]}"
        assert_bits_equal(keys[:n0], sp, f"{what}: sorted probabilities")
        assert np.array_equal(vals[:n0], si), f"{what}: sorted order differs at {np.nonzero(vals[:n0] != si)[0][:8]}"
        assert np.all(keys[n0:] == -1.0), f"{what}: rejected keys"
        assert (int(out[0]), out[1:7].tolist()) == (tok, six), f"{what}: device {out[0]} {out[1:7].tolist()}, oracle {tok} {six}"
        key = (id(lg), T)
        if key not in checked:
            checked.add(key)
            _, _, _, _, sp1, si1 = ob.sample_top_p(lg, T, 1.0, 0.0, sorted_out=True)       # every probability
            check_against_float64(lg, T, sp1, si1)


@pytest.mark.parametrize("V", [512, 4097, 151936])
def test_empty_nucleus(probe, V):
    """n0 = 0 (the reference reads probindex[-1]): the first index of the largest probability, six zero ids."""
    lg, T, top_p, want = sc.empty_nucleus_case(V)
    out, _, _ = probe(lg, T, top_p, 0.5)
    assert int(out[7]) == 0
    assert (int(out[0]), out[1:7].tolist()) == (want, [0] * 6) == ob.sample_top_p(lg, T, top_p, 0.5)[:2]


def history(V, n, seed):
    """Ids 0 and V - 1, repeats, and ids on 32 / 64 / 128 / 4096-row boundaries, then random ids."""
    rng = np.random.default_rng(seed)
    edge = [0, V - 1, 5, 5, 127, 128, 0, 4095, 4096, 8191, V - 2, 5, V - 1, 1023, 1024, 63, 64, 31, 32, V // 2]
    if seed % 2:
        edge = edge[::-1]
    h = np.asarray(edge + rng.integers(0, V, n).tolist(), np.uint32)[:n + 1]
    return np.ascontiguousarray(h)


@pytest.mark.parametrize("want", [STREAM, MULTI])
@pytest.mark.parametrize("name,gs", [("v16k-nano", 128), ("v152k-qwen3", 64)])
def test_fast_mode_penalty_and_sampling(name, gs, want, monkeypatch):
    spec = mf.PRESETS[name]
    V, S, pen, T, top_p = spec.vocab, 24, 1.3, 0.7, 0.8
    path = mf.cached_model(spec, Q80, gs)
    eng = engine(path, S, 0 if want == STREAM else E.FLAG_NO_STREAM, monkeypatch)
    assert_path(eng, want)
    st = 39
    for seed in (1, 2):                          # the second history revisits every position with other ids
        ids = history(V, S, seed)
        for pos in range(S - 1):
            raw = eng.forward(int(ids[pos]), pos)
            coin, st = ob.random_f32(st)
            tok, six = eng.next_sampled(ids, pos, pen, T, top_p, float(coin))
            got = eng.logits()
            seen = np.unique(ids[:pos])
            exp = raw.copy()
            exp[seen] = (raw[seen] / np.float32(pen)).astype(np.float32)
            assert_bits_equal(got, exp, f"{want} history {seed} pos {pos}: penalised logits")
            otok, osix, n0, _ = ob.sample_top_p(got, T, top_p, float(coin))
            assert (tok, six) == (otok, osix), f"{want} history {seed} pos {pos} (n0 {n0}): engine {tok} {six}, oracle {otok} {osix}"
    eng.close()


TIE_FIRSTS = [0, 31, 32, 63, 64, 255, 256, 1023, 4096, 65536, 100003, 151936 - 129, 151936 - 128, 151936 - 33, 151936 - 2, 151936 - 1]


@pytest.fixture(scope="module")
def tie_model():
    """v152k-qwen3-untied with a classifier of 16 row classes: class c first appears at TIE_FIRSTS[c] (some in the last CTA,
    some on warp and tile boundaries); every other row is a copy of a class that has already appeared."""
    spec = mf.PRESETS["v152k-qwen3-untied"]
    L, E_, F, V, Q, K, hd = spec.n_layer, spec.n_embd, spec.n_hidden, spec.vocab, spec.q_dim, spec.kv_dim, spec.hd
    rng = np.random.default_rng(11)

    def normal(shape, std):
        return (rng.standard_normal(shape, dtype=np.float32) * np.float32(std)).astype(np.float32)
    firsts = np.asarray(TIE_FIRSTS)
    appeared = np.searchsorted(firsts, np.arange(V), side="right")
    cls_of = (rng.random(V) * appeared).astype(np.int64)
    cls_of[firsts] = np.arange(firsts.size)
    rows = normal((firsts.size, E_), 0.1)
    w = {"attn_norm": 1 + normal((L, E_), 0.02), "ffn_norm": 1 + normal((L, E_), 0.02), "final_norm": 1 + normal(E_, 0.02),
         "emb": normal((V, E_), 0.02), "wq": normal((L, Q, E_), 0.02), "wk": normal((L, K, E_), 0.02), "wv": normal((L, K, E_), 0.02),
         "wo": normal((L, E_, Q), 0.01), "w1": normal((L, F, E_), 0.02), "w2": normal((L, E_, F), 0.02), "w3": normal((L, F, E_), 0.01),
         "q_norm": 1 + normal((L, hd), 0.02), "k_norm": 1 + normal((L, hd), 0.02), "cls": rows[cls_of]}
    path = os.path.join(tempfile.mkdtemp(prefix="nb200_ties_"), "ties.bin")
    mf.write_model_from_weights(path, spec, Q80, 64, w)
    return path, cls_of, firsts


def class_margin(logits, cls_of, firsts):
    """Gap between the best and the second-best class logit."""
    top = np.sort(logits[firsts])
    return float(top[-1] - top[-2])


@pytest.mark.parametrize("mode", ["stream", "multi", "exact"])
def test_argmax_ties_pick_first_occurrence(tie_model, mode, monkeypatch):
    path, cls_of, firsts = tie_model
    S, P = 24, 4
    first_set = set(firsts.tolist())
    stream = np.random.default_rng(3).integers(0, cls_of.size, S + 1).astype(np.uint32)      # teacher-forced ids
    prompt = [7, 100000, 7, 65536]
    o = ob.NanoOracle(path, S)
    want_tf, margins = [], []
    for pos in range(S - 1):
        want_tf.append(o.next_greedy(stream, pos, 0, 1.0))
        margins.append(class_margin(o.logits(), cls_of, firsts))
    ids_o = np.zeros(S + 1, np.uint32); ids_o[:P] = prompt
    for pos in range(S - 1):
        ids_o[pos + 1] = o.next_greedy(ids_o, pos, 1 if pos < P - 1 else 0, 1.0)
    o.close()
    assert len(set(want_tf)) >= 6 and max(want_tf) > cls_of.size - 256       # many classes win, some first seen in the last CTA
    flags = {"stream": 0, "multi": E.FLAG_NO_STREAM, "exact": E.FLAG_EXACT}[mode]
    eng = engine(path, S, flags, monkeypatch)
    if mode != "exact":
        assert_path(eng, STREAM if mode == "stream" else MULTI)
    # teacher-forced: the first copy of the best class at every step; the oracle's id wherever its class margin is beyond
    # the fast-mode noise (every step in exact mode)
    for pos in range(S - 1):
        got = eng.next_greedy(stream, pos, 0, 1.0)
        assert got in first_set, f"{mode} pos {pos}: id {got} is a later copy of class {cls_of[got]} (first copy {firsts[cls_of[got]]})"
        if mode == "exact" or margins[pos] >= 0.05:
            assert got == want_tf[pos], f"{mode} pos {pos}: {got} vs oracle {want_tf[pos]} (class margin {margins[pos]:.3f})"
    # greedy decoding: per call and in the device loop
    a = np.zeros(S + 1, np.uint32); a[:P] = prompt
    for pos in range(S - 1):
        a[pos + 1] = eng.next_greedy(a, pos, 1 if pos < P - 1 else 0, 1.0)
    b = np.zeros(S + 1, np.uint32); b[:P] = prompt
    eng.decode_greedy(b, P, S, 1.0)
    assert a[:S].tolist() == b[:S].tolist(), f"{mode}: device loop differs from the per-call loop"
    assert set(a[P:S].tolist()) <= first_set, f"{mode}: a later copy won a tie: {a[P:S].tolist()}"
    if mode == "exact":
        assert a[:S].tolist() == ids_o[:S].tolist(), f"{mode}: {a[:S].tolist()} vs oracle {ids_o[:S].tolist()}"
    # the sampler's six ids: the winning class's first copies, in index order
    for pos in range(S - 1):
        tok, six = eng.next_sampled(stream, pos, 1.0, 0.7, 0.8, 0.0)
        lg = eng.logits()
        assert (tok, six) == ob.sample_top_p(lg, 0.7, 0.8, 0.0)[:2], f"{mode} pos {pos}"
        members = np.nonzero(cls_of == cls_of[six[0]])[0]
        assert six[0] in first_set
        if members.size >= 6:
            assert six == members[:6].tolist(), f"{mode} pos {pos}: six ids {six}, first copies {members[:6].tolist()}"
    eng.close()
