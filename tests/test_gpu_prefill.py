"""Batched prompt prefill (nb200_prefill, nano_b200/csrc/prefill.cuh).

Prefill runs the prompt in chunks of up to 16 positions per pass over the weights with the token path's own arithmetic, so its
K / V rows must equal, bit for bit, those nb200_forward writes position by position on the multi-kernel path of an engine with
the same flags (NB200_FLAG_NO_STREAM), and in exact mode those of the strict reference.  Covered here:
  * the bit identity over the toy shapes x F32 / Q80 (every group size) / Q4K x exact / fast, chunk boundaries and a prefill
    that starts mid-session, then the next position's logits and a greedy continuation with a repetition penalty;
  * exact mode against the oracle; every attention kernel of the token path, a 1 000+ position prefill and the BASELINE shapes;
  * a default (streaming) engine continuing after a prefill; rows outside the prefilled range; refusals; launch counts;
  * (CPU) no prefill kernel has a stack frame of its own.
"""
import math
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, assert_bits_equal
from nano_b200 import build as nb_build, engine as E, modelfile as mf

F32, Q80, Q4K = mf.QUANT_F32, mf.QUANT_Q80, mf.QUANT_Q4K
NS = (1, 15, 16, 17, 40)
PEN = 1.3


def quant_id(quant, gs):
    return {F32: "f32", Q80: f"q80g{gs}", Q4K: "q4k"}[quant]


def nostream(path, S, flags=0, monkeypatch=None, **env):
    if monkeypatch is not None and env:
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, str(v))
            eng = E.Engine(path, S, flags=flags | E.FLAG_NO_STREAM)
    else:
        eng = E.Engine(path, S, flags=flags | E.FLAG_NO_STREAM)
    assert eng.path.startswith("multi-kernel"), eng.path
    return eng


def kv_rows(eng, kv_dim, upto, lo=0):
    """K and V rows [L][upto - lo][kv_dim] of positions lo .. upto-1."""
    k = np.stack([np.stack([eng.read(E.F_KROW, kv_dim, l, p) for p in range(lo, upto)]) for l in range(eng.n_layer)])
    v = np.stack([np.stack([eng.read(E.F_VROW, kv_dim, l, p) for p in range(lo, upto)]) for l in range(eng.n_layer)])
    return k, v


def assert_rows_equal(a, b, upto, what, lo=0):
    ka, va = kv_rows(a, a.kv_dim, upto, lo)
    kb, vb = kv_rows(b, b.kv_dim, upto, lo)
    assert_bits_equal(ka, kb, f"{what}: K rows {lo}..{upto - 1}")
    assert_bits_equal(va, vb, f"{what}: V rows {lo}..{upto - 1}")


def token_path(eng, toks, upto):
    for p in range(upto):
        eng.forward_nolog(int(toks[p]), p)


def greedy(eng, toks, p0, steps=16):
    ids = np.zeros(p0 + steps + 2, np.uint32)
    ids[: p0 + 1] = toks[: p0 + 1]
    for pos in range(p0, p0 + steps):
        ids[pos + 1] = eng.next_greedy(ids, pos, 0, PEN)
    return ids[p0 + 1: p0 + steps + 1].tolist()


def file_variants(name):
    return [(F32, 128), (Q80, 32), (Q80, 64), (Q80, 128), (Q80, 256), (Q4K, 128)]


# ------------------------------------------------------------------------------------------------ 1. bit identity
ID_CASES = [(n, q, g, x) for n in ("toy-nano", "toy-qwen3", "mini-qwen3", "toy-qwen2") for q, g in file_variants(n)
            for x in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,exact", ID_CASES,
                         ids=[f"{c[0]}-{quant_id(c[1], c[2])}-{'exact' if c[3] else 'fast'}" for c in ID_CASES])
def test_prefill_bit_identical_to_token_path(name, quant, gs, exact):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = 64
    flags = E.FLAG_EXACT if exact else 0
    toks = mf.teacher_tokens(S, spec.vocab)
    ref, pre = nostream(path, S, flags), nostream(path, S, flags)
    for pos0 in (0, 5):
        for n in NS:
            p0 = pos0 + n
            what = f"{name} {quant_id(quant, gs)} {'exact' if exact else 'fast'} prefill [{pos0}, {p0})"
            token_path(ref, toks, p0)
            token_path(pre, toks, pos0)
            pre.prefill(toks, pos0, n)
            assert_rows_equal(pre, ref, p0, what)
            assert_bits_equal(pre.forward(int(toks[p0]), p0), ref.forward(int(toks[p0]), p0), f"{what}: logits at {p0}")
            assert greedy(pre, toks, p0) == greedy(ref, toks, p0), f"{what}: greedy continuation differs"
    assert pre.prefill_info() == {"chunk": 16, "attention": "exact" if exact else ref.kernels()["attention"]}, pre.prefill_info()
    ref.close(); pre.close()


# ------------------------------------------------------------------------------------------------ 2. exact mode vs the oracle
ORACLE_CASES = [(n, q, g) for n in ("toy-nano", "toy-qwen3", "mini-qwen3", "toy-qwen2") for q, g in file_variants(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", ORACLE_CASES, ids=[f"{c[0]}-{quant_id(c[1], c[2])}" for c in ORACLE_CASES])
def test_exact_prefill_equals_strict_reference(name, quant, gs):
    from oracle import bindings as ob
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S, n = 64, 37
    toks = mf.teacher_tokens(S, spec.vocab)
    o = ob.NanoOracle(path, S)
    for p in range(n):
        o.forward(int(toks[p]), p)
    want_logits = o.forward(int(toks[n]), n)
    ok, ov = (a.copy() for a in o.kv())
    o.close()
    eng = nostream(path, S, E.FLAG_EXACT)
    eng.prefill(toks, 0, n)
    k, v = kv_rows(eng, spec.kv_dim, n)
    assert_bits_equal(k, ok[:, :n], "K rows vs the oracle")
    assert_bits_equal(v, ov[:, :n], "V rows vs the oracle")
    assert_bits_equal(eng.forward(int(toks[n]), n), want_logits, f"logits at {n} vs the oracle")
    eng.close()


# ------------------------------------------------------------------------------------------------ 3. attention kernels
ATTN_WANT = {"kvm1-nano": "fast<1>", "kvm4-qwen3-hd64": "fast<4>", "kvm4-qwen3-hd128": "fast<4>", "kvm8-qwen3": "fast<8>",
             "kvm3-qwen3": "generic", "kvm5-qwen3": "generic", "kvm7-nano": "generic", "mqa-qwen3": "generic",
             "hd96-qwen3": "generic", "hd192-nano": "generic", "hd512-qwen3": "generic"}
ATTN_CASES = ([(n, w, {}) for n, w in ATTN_WANT.items()] +
              [(n, "generic", {"NB200_GENERIC_ATTN": 1}) for n in ("kvm1-nano", "kvm4-qwen3-hd64", "kvm4-qwen3-hd128")])


@pytest.mark.gpu
@pytest.mark.parametrize("name,want,env", ATTN_CASES, ids=[c[0] + ("-generic-env" if c[2] else "") for c in ATTN_CASES])
def test_prefill_attention_kernels(name, want, env, monkeypatch):
    """Every attention kernel the token path selects, in fast and exact mode, over 100 positions (up to four splits)."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S, n = 128, 100
    toks = mf.teacher_tokens(S, spec.vocab)
    for flags in (0, E.FLAG_EXACT):
        ref = nostream(path, S, flags, monkeypatch, **env)
        pre = nostream(path, S, flags, monkeypatch, **env)
        token_path(ref, toks, n)
        pre.prefill(toks, 0, n)
        kind = "exact" if flags else want
        assert ref.kernels()["attention"] == kind and pre.prefill_info()["attention"] == kind, (ref.kernels(), pre.prefill_info())
        assert_rows_equal(pre, ref, n, f"{name} {kind}")
        assert_bits_equal(pre.forward(int(toks[n]), n), ref.forward(int(toks[n]), n), f"{name} {kind}: logits at {n}")
        ref.close(); pre.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["long-nano", "long-qwen3"])
def test_long_prefill(name):
    """One prefill of 1 040 positions: the late positions attend across many splits of the cache."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S, n = 1100, 1040
    toks = mf.teacher_tokens(S, spec.vocab)
    ref, pre = nostream(path, S), nostream(path, S)
    token_path(ref, toks, n)
    pre.prefill(toks, 0, n)
    assert_rows_equal(pre, ref, n, f"{name} prefill of {n}")
    assert_bits_equal(pre.forward(int(toks[n]), n), ref.forward(int(toks[n]), n), f"{name}: logits at {n}")
    ref.close(); pre.close()


# ------------------------------------------------------------------------------------------------ 4. BASELINE shapes
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,n", [("nano-168m", Q80, 128, 496), ("qwen3-0.6b", Q4K, 128, 512)])
def test_prefill_baseline_shapes(name, quant, gs, n):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = n + 16
    toks = mf.teacher_tokens(S, spec.vocab)
    ref = nostream(path, S)
    token_path(ref, toks, n)
    want = kv_rows(ref, spec.kv_dim, n)
    want_logits = ref.forward(int(toks[n]), n)
    ref.close()
    pre = nostream(path, S)
    ms = pre.prefill(toks, 0, n)
    got = kv_rows(pre, spec.kv_dim, n)
    assert_bits_equal(got[0], want[0], f"{name}: K rows")
    assert_bits_equal(got[1], want[1], f"{name}: V rows")
    assert_bits_equal(pre.forward(int(toks[n]), n), want_logits, f"{name}: logits at {n}")
    print(f"{name} {quant_id(quant, gs)}: prefill of {n} positions {ms:.2f} ms, chunk {pre.prefill_info()['chunk']}")
    pre.close()


# ------------------------------------------------------------------------------------------------ 5. default path
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", [("toy-nano", Q80, 64), ("toy-qwen3", Q80, 64), ("toy-qwen3", Q4K, 128)])
def test_default_engine_continues_after_prefill(name, quant, gs):
    """Prefill does not depend on the execution path: a default engine's prefilled rows equal the multi-kernel engine's.  Its
    own decode then continues from them within the noise-floor policy of the engine tests, teacher-forced against the oracle."""
    from oracle import bindings as ob
    from test_gpu_engine import TOL, reference_noise_floor
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S, P = 40, 24
    toks = mf.teacher_tokens(S, spec.vocab)
    dflt = E.Engine(path, S)
    assert dflt.path.startswith("streaming"), dflt.path
    multi = nostream(path, S)
    dflt.prefill(toks, 0, P)
    multi.prefill(toks, 0, P)
    assert_rows_equal(dflt, multi, P, f"{name} default vs multi-kernel prefill")
    multi.close()
    limit = max(TOL[quant], 1.5 * reference_noise_floor(name, quant, gs, path, S))
    o = ob.NanoOracle(path, S)
    for p in range(P):
        o.forward(int(toks[p]), p)
    worst = 0.0
    for p in range(P, S):
        a = dflt.forward(int(toks[p]), p); b = o.forward(int(toks[p]), p)
        worst = max(worst, float(np.abs(a - b).max()))
        top2 = np.partition(b, -2)[-2:]
        if float(top2[1] - top2[0]) > 2 * limit:
            assert int(np.argmax(a)) == int(np.argmax(b)), f"{name} pos {p}: argmax differs, margin {top2[1] - top2[0]}"
    o.close()
    assert worst <= limit, f"{name}: max|dlogit| {worst} > {limit}"
    ids = greedy(dflt, toks, P - 1, 8)
    assert all(0 <= i < spec.vocab for i in ids)
    print(f"{name} {quant_id(quant, gs)} [{dflt.path[:24]}]: max|dlogit| {worst:.3e} (limit {limit:.3e}), greedy {ids}")
    dflt.close()


# ------------------------------------------------------------------------------------------------ 6. untouched rows
@pytest.mark.gpu
@pytest.mark.parametrize("exact", [False, True])
def test_prefill_leaves_other_rows_alone(exact):
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    S = 64
    toks = mf.teacher_tokens(S, spec.vocab)
    eng = nostream(path, S, E.FLAG_EXACT if exact else 0)
    token_path(eng, toks, 61)
    before = kv_rows(eng, spec.kv_dim, 61, 20)
    other = toks.copy(); other[:20] = (other[:20] + 7) % spec.vocab
    eng.prefill(other, 0, 20)
    after = kv_rows(eng, spec.kv_dim, 61, 20)
    assert_bits_equal(after[0], before[0], "K rows 20..60")
    assert_bits_equal(after[1], before[1], "V rows 20..60")
    eng.close()


# ------------------------------------------------------------------------------------------------ 7. refusals
def _cache(eng, spec, upto):
    return kv_rows(eng, spec.kv_dim, upto)


@pytest.mark.gpu
def test_prefill_refusals():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    S = 48                                               # below block_size 64: the limit is max_seq_len
    toks = mf.teacher_tokens(S + 8, spec.vocab)
    eng = nostream(path, S)
    token_path(eng, toks, S)
    before = _cache(eng, spec, S)
    bad = toks.copy(); bad[10] = spec.vocab
    for args, msg in [((toks, 0, 0), "empty"), ((toks, 40, 9), "past"), ((toks, S, 1), "past"), ((bad, 0, 20), "out of range")]:
        with pytest.raises(E.NB200Error, match=msg):
            eng.prefill(*args)
        k, v = _cache(eng, spec, S)
        assert_bits_equal(k, before[0], f"K rows after refusing {args[1:]}"); assert_bits_equal(v, before[1], f"V rows after {args[1:]}")
    eng.prefill(toks, 40, 8)                             # exactly up to the limit is accepted
    eng.close()

    eng = nostream(path, S)
    token_path(eng, toks, 8)
    before = _cache(eng, spec, 8)
    eng.lora_load(mf.write_lora(spec))
    with pytest.raises(E.NB200Error, match="LoRA"):
        eng.prefill(toks, 0, 8)
    k, v = _cache(eng, spec, 8)
    assert_bits_equal(k, before[0], "K rows after refusing LoRA"); assert_bits_equal(v, before[1], "V rows after refusing LoRA")
    eng.lora_enable(False)
    eng.prefill(toks, 0, 8)
    eng.close()


@pytest.mark.gpu
@pytest.mark.skipif(E.device_count() < 2, reason="tensor parallelism needs 2 GPUs")
def test_prefill_refuses_tensor_parallel():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    g = E.TpGroup(path, 32, 2)
    toks = mf.teacher_tokens(32, spec.vocab)
    for r in g.ranks:
        with pytest.raises(E.NB200Error, match="tensor-parallel"):
            r.prefill(toks, 0, 8)
    g.close()


# ------------------------------------------------------------------------------------------------ 8. launch count
@pytest.mark.gpu
@pytest.mark.parametrize("n", [16, 40])
def test_prefill_launch_count(n):
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    eng = nostream(path, 64)
    assert eng.prefill_info()["chunk"] == 0
    toks = mf.teacher_tokens(64, spec.vocab)
    before = eng.launches
    eng.prefill(toks, 0, n)
    M = eng.prefill_info()["chunk"]
    assert M == 16
    got = eng.launches - before
    assert got == math.ceil(n / M) * (1 + 6 * spec.n_layer), got      # embed, then QKV, K rows, attention, O, W1|W3, W2 per layer
    assert got * 4 < n * eng.launches_per_token, (got, n * eng.launches_per_token)
    eng.close()


# ------------------------------------------------------------------------------------------------ CPU: stack frames
def test_prefill_kernels_have_no_stack_frame():
    """Every k_prefill_* kernel keeps its state in registers.  The one exception is allowed only where the token path's own
    attention body has a frame (k_attention_fast<8>, wrapped unchanged by k_prefill_attention_fast<8>): no larger than it."""
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", nb_build.ENGINE_SO],
                         capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    stack = {}
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            st = re.search(r"STACK:(\d+)", lines[i + 1])
            stack[m.group(1)] = int(st.group(1)) if st else 0
    prefill = {f: s for f, s in stack.items() if "k_prefill_" in f}
    # matvec: Q80 (4 group sizes) / F32 / Q4K / exact F32 x 3 epilogues; embed, K rows, attention fast<1|2|4|8> / generic / exact
    assert len(prefill) == 29, sorted(prefill)
    token_fast8 = [s for f, s in stack.items() if re.search(r"16k_attention_fastILi8ELb0E", f)]
    assert len(token_fast8) == 1
    bad = {}
    for f, s in prefill.items():
        allowed = token_fast8[0] if re.search(r"24k_prefill_attention_fastILi8EE", f) else 0
        if s > allowed:
            bad[f] = s
    assert not bad, f"stack bytes per thread: {bad}"
