"""Every kernel variant of the multi-kernel path (run_token: k_matvec<QUANT, EPI, RB, LPG>, the split-KV attention kernels),
on 2-layer models whose shapes select them, against the oracle and against a float64 restatement of the forward pass
(tests/ref64.py).  The multi-kernel path is the only one in exact mode, with a LoRA plug-in and under tensor parallelism,
and it runs every shape the streaming kernel declines.

* The generic split-KV attention `k_attention` (kv_mul outside {1, 2, 4, 8}, head_dim > 128, a Qwen3 head_dim that is not
  a power of two) and `k_attention_fast<8>` where the merge's shared-memory cap cuts the split count.
* The matvec row-block variants, forced with NB200_MATVEC_RB on a model whose classifier ends in a partial row block,
  for F32, Q4K and Q80 with groups of 32, 64, 128 and 256; at op level the 12 Q80 store variants.
* Every engine case asserts the kernels it ran (Engine.kernels()): a shape that selects another kernel fails, it does
  not pass silently.
* Fast mode within twice the reference's noise floors (fast_limit; argmax agreement where the oracle's margin is real, K / V rows of every
  layer), exact mode bit-identical; F32 within 4x the oracle's own distance from float64 at S = 512 and 2048.
"""
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, assert_bits_equal
from nano_b200 import build as nb_build, engine as E, modelfile as mf
from oracle import bindings as ob
from test_gpu_engine import reference_noise_floor
from test_gpu_ops import edgey, o_q4k_quant, o_q80_matvec, oracle
from test_gpu_stream_matrix import S_FAST, S_LONG, TIGHT_SHAPES, TOL, oracle_run, tight_check

sys.path.insert(0, GOLDEN)
from make_golden import MULTI_ATTN_PRESETS, MULTI_CASES  # noqa: E402
sys.path.remove(GOLDEN)

F32, Q80, Q4K = mf.QUANT_F32, mf.QUANT_Q80, mf.QUANT_Q4K
RBS = (1, 2, 4)

# the attention kernel each preset selects in fast mode
ATTN_WANT = {"kvm3-qwen3": "generic", "kvm5-qwen3": "generic", "kvm7-nano": "generic", "mqa-qwen3": "generic",
             "hd96-qwen3": "generic", "hd192-nano": "generic", "hd512-qwen3": "generic", "kvm8-qwen3": "fast<8>",
             "kvm1-nano": "fast<1>", "kvm4-qwen3-hd64": "fast<4>", "mv-nano": "fast<2>"}
ATTN_CASES = ([c for c in MULTI_CASES if c[0] in MULTI_ATTN_PRESETS] +
              [("kvm1-nano", F32, 128), ("kvm4-qwen3-hd64", F32, 128)])       # the other specialisations of the split-KV kernel
MV_CASES = [c for c in MULTI_CASES if c[0] == "mv-nano"]


def case_id(c):
    return f"{c[0]}-{ {F32: 'f32', Q80: 'q80g', Q4K: 'q4k'}[c[1]] }{c[2] if c[1] == Q80 else ''}"


def multi_engine(path, S, flags, monkeypatch, **env):
    """An engine on the multi-kernel path (NB200_FLAG_NO_STREAM) with the given NB200_* knobs."""
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, str(v))
        eng = E.Engine(path, S, flags=flags | E.FLAG_NO_STREAM)
    assert eng.path.startswith("multi-kernel"), eng.path
    return eng


def expected_matvec(quant, rb, exact):
    """(epilogue, RB) of every k_matvec launch of one token under NB200_MATVEC_RB=rb.  RB = 1 exists for Q80 only, and
    not for W1|W3 (SwiGLU pairs rows); the exact-mode F32 path has its own kernel (k_matvec_f32_exact)."""
    if quant == F32 and exact:
        return set()
    r1 = rb if quant == Q80 else max(rb, 2)
    return {("qkv", r1), ("resid", r1), ("cls", r1), ("swiglu", max(rb, 2))}


def fast_limit(name, quant, gs, path, S):
    """max(tolerance, 2 x the reference's own fast-vs-strict noise floor).  In fast mode a quantised file's deviation is set by
    which activation codes flip (a 1-ulp difference before quantisation moves a whole group's dot product), and the floor
    is one sample of that from two compiler builds.  On an H100 (400 W), over the 36 quantised files here, the
    worst deviation was 1.65 x the floor (kvm5-qwen3 Q80 g128: 0.0203 against 0.0127) while the same kernels were bit-identical
    in exact mode and, in F32, within 0.65 x the oracle's own distance from float64: the arithmetic is pinned there, and
    this bound catches what flips cannot explain."""
    return max(TOL[quant], 2.0 * reference_noise_floor(name, quant, gs, path, S))


def fast_check(eng, spec, S, ref, ok, ov, limit, what, causal=1):
    """Logits within `limit` at every position (argmax agreement where the oracle's margin is real), K / V rows of every
    layer within the same bound."""
    toks = mf.teacher_tokens(S, spec.vocab)
    worst = 0.0
    for pos in range(S):
        a = eng.forward(toks[pos], pos, causal); b = ref[pos]
        worst = max(worst, float(np.abs(a - b).max()))
        top2 = np.partition(b, -2)[-2:]
        if float(top2[1] - top2[0]) > 2 * limit:
            assert int(np.argmax(a)) == int(np.argmax(b)), f"{what} pos {pos}: argmax differs, margin {top2[1] - top2[0]}"
    assert worst <= limit, f"{what}: max|dlogit| {worst} > {limit}"
    for l in range(spec.n_layer):
        for pos in (0, 1, S // 2, S - 1):
            dk = np.abs(eng.read(E.F_KROW, spec.kv_dim, l, pos) - ok[l, pos]).max()
            dv = np.abs(eng.read(E.F_VROW, spec.kv_dim, l, pos) - ov[l, pos]).max()
            assert max(dk, dv) <= limit, f"{what} layer {l} pos {pos}: max|dK| {dk}, max|dV| {dv} > {limit}"
    print(f"{what}: max|dlogit| {worst:.3e} (limit {limit:.3e})")


def exact_check(eng, spec, S, ref, ok, ov, what, causal=1):
    toks = mf.teacher_tokens(S, spec.vocab)
    for pos in range(S):
        assert_bits_equal(eng.forward(toks[pos], pos, causal), ref[pos], f"{what} pos {pos}")
    for l in range(spec.n_layer):
        for pos in (0, 1, S // 2, S - 1):
            assert_bits_equal(eng.read(E.F_KROW, spec.kv_dim, l, pos), ok[l, pos], f"{what} K row {l}/{pos}")
            assert_bits_equal(eng.read(E.F_VROW, spec.kv_dim, l, pos), ov[l, pos], f"{what} V row {l}/{pos}")


def greedy_check(eng, path, spec, S=40, pen=1.3):
    """Greedy ids with a repetition penalty: the per-call loop and the device-resident loop agree; in exact mode both
    equal the oracle's ids."""
    P = 6
    prompt = [5, 9, 5, 3, 9, 5]
    a = np.zeros(S + 1, np.uint32); a[:P] = prompt
    for pos in range(S - 1):
        a[pos + 1] = eng.next_greedy(a, pos, 1 if pos < P - 1 else 0, pen)
    b = np.zeros(S + 1, np.uint32); b[:P] = prompt
    eng.decode_greedy(b, P, S, pen)
    assert a[:S].tolist() == b[:S].tolist(), "decode_greedy differs from the per-call loop"
    o = ob.NanoOracle(path, S)
    ids_o = np.zeros(S + 1, np.uint32); ids_o[:P] = prompt
    for pos in range(S - 1):
        ids_o[pos + 1] = o.next_greedy(ids_o, pos, 1 if pos < P - 1 else 0, pen)
    o.close()
    return a[:S].tolist() == ids_o[:S].tolist()


# ------------------------------------------------------------------------------------------------ §1 attention matrix
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", ATTN_CASES, ids=[case_id(c) for c in ATTN_CASES])
def test_attention_matrix(name, quant, gs, monkeypatch):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = S_FAST
    ref, ok, ov = oracle_run(path, S, spec.vocab)
    limit = fast_limit(name, quant, gs, path, S)
    eng = multi_engine(path, S, 0, monkeypatch)
    assert eng.kernels()["attention"] == ATTN_WANT[name], eng.kernels()
    fast_check(eng, spec, S, ref, ok, ov, limit, f"{case_id((name, quant, gs))} fast, attention {ATTN_WANT[name]}")
    eng.close()
    eng = multi_engine(path, S, E.FLAG_EXACT, monkeypatch)
    assert eng.kernels()["attention"] == "exact", eng.kernels()
    exact_check(eng, spec, S, ref, ok, ov, "exact")
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", MULTI_ATTN_PRESETS)
def test_attention_greedy_with_penalty(name, monkeypatch):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    for flags in (E.FLAG_EXACT, 0):
        eng = multi_engine(path, 40, flags, monkeypatch)
        same = greedy_check(eng, path, spec)
        assert eng.kernels()["attention"] == ("exact" if flags else ATTN_WANT[name]), eng.kernels()
        if flags == E.FLAG_EXACT:
            assert same, "exact-mode greedy ids differ from the oracle's"
        eng.close()


# ------------------------------------------------------------------------------------------------ §2 F32 against float64
@pytest.mark.gpu
@pytest.mark.parametrize("S", [512, S_LONG])
@pytest.mark.parametrize("name", MULTI_ATTN_PRESETS)
def test_f32_attention_tight_vs_float64(name, S, monkeypatch):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, F32, 128)
    eng = multi_engine(path, S, 0, monkeypatch)
    tight_check(eng, spec, path, S, f"{name} multi-kernel {ATTN_WANT[name]} S {S}")
    assert eng.kernels()["attention"] == ATTN_WANT[name], eng.kernels()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [512, S_LONG])
@pytest.mark.parametrize("name", TIGHT_SHAPES)
def test_f32_generic_attention_on_fast_shapes(name, S, monkeypatch):
    """NB200_GENERIC_ATTN=1 runs the generic kernel on the shapes of the specialised one: hd 52 / 64 / 128, Nano RoPE,
    kv_mul 1 / 2 / 4."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, F32, 128)
    eng = multi_engine(path, S, 0, monkeypatch, NB200_GENERIC_ATTN=1)
    tight_check(eng, spec, path, S, f"{name} multi-kernel generic S {S}")
    assert eng.kernels()["attention"] == "generic", eng.kernels()
    eng.close()


# ------------------------------------------------------------------------------------------------ §3 matvec matrix
@pytest.mark.gpu
@pytest.mark.parametrize("rb", RBS)
@pytest.mark.parametrize("name,quant,gs", MV_CASES, ids=[case_id(c) for c in MV_CASES])
def test_matvec_matrix(name, quant, gs, rb, monkeypatch):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = S_FAST
    ref, ok, ov = oracle_run(path, S, spec.vocab)
    what = f"{case_id((name, quant, gs))} RB {rb}"
    eng = multi_engine(path, S, E.FLAG_EXACT, monkeypatch, NB200_MATVEC_RB=rb)
    exact_check(eng, spec, S, ref, ok, ov, f"{what} exact")
    assert greedy_check(eng, path, spec), f"{what}: exact-mode greedy ids differ from the oracle's"
    assert eng.kernels()["matvec"] == expected_matvec(quant, rb, True), eng.kernels()
    eng.close()
    limit = fast_limit(name, quant, gs, path, S)
    eng = multi_engine(path, S, 0, monkeypatch, NB200_MATVEC_RB=rb)
    fast_check(eng, spec, S, ref, ok, ov, limit, f"{what} fast")
    greedy_check(eng, path, spec)
    assert eng.kernels() == {"matvec": expected_matvec(quant, rb, False), "attention": ATTN_WANT[name]}, eng.kernels()
    print(f"{what}: kernels {sorted(eng.kernels()['matvec'])}")
    eng.close()
    if quant == F32:
        eng = multi_engine(path, 64, 0, monkeypatch, NB200_MATVEC_RB=rb)
        tight_check(eng, spec, path, 64, f"{what} fast", n_ref=64)
        eng.close()


# ------------------------------------------------------------------------------------------------ §4 op level
Q80_OP_SHAPES = [(256, 7, 64), (256, 33, 32), (768, 64, 128), (1024, 1000, 128), (1024, 130, 64), (3072, 257, 128),
                 (2048, 96, 256), (2560, 50, 128), (9728, 40, 128), (896, 2051, 32),
                 (5376, 103, 32)]      # 49072 B of dynamic shared memory: under 48 KB alone, over it with the static part


@pytest.mark.gpu
@pytest.mark.parametrize("rb", RBS)
@pytest.mark.parametrize("n,d,gs", Q80_OP_SHAPES)
def test_q80_matvec_forced_rb_bit_exact(n, d, gs, rb, monkeypatch):
    """nb200_op_q80_matvec (k_matvec<Q80, EPI_STORE, RB, gs / 16>, the ordered group sum) under each row block."""
    rng = np.random.default_rng(n * 7 + d)
    x = edgey(rng, n)
    wq, ws = mf.quantize_q80(rng.standard_normal((d, n), dtype=np.float32) * np.float32(0.02), gs)
    monkeypatch.setenv("NB200_MATVEC_RB", str(rb))
    assert_bits_equal(E.op_q80_matvec(x, wq, ws, n, d, gs), o_q80_matvec(x, wq, ws, n, d, gs), f"q80 matvec RB {rb}")


@pytest.mark.gpu
@pytest.mark.parametrize("rb", [2, 4])
@pytest.mark.parametrize("n,d", [(768, 100), (2048, 771), (5376, 45)])
def test_f32_q4k_matvec_forced_rb(n, d, rb, monkeypatch):
    """The F32 and Q4K store variants (op level) under both row blocks: Q4K bit-exact, F32 within the fp32 tree bound."""
    rng = np.random.default_rng(n + d)
    x = edgey(rng, n)
    W = (rng.standard_normal((d, n), dtype=np.float32) * np.float32(0.05)).astype(np.float32)
    monkeypatch.setenv("NB200_MATVEC_RB", str(rb))
    wb = mf.quantize_q4k_blocks(W).reshape(-1)
    xb = o_q4k_quant(x)
    want = np.zeros(d, np.float32)
    oracle().nor_matvec_q4k(want.ctypes.data_as(ob.f32p), xb.ctypes.data_as(ob.u8p), wb.ctypes.data_as(ob.u8p), 0, d, n)
    assert_bits_equal(E.op_q4k_matvec(x, wb, n, d), want, f"q4k matvec RB {rb}")
    oracle().nor_matvec_f32(want.ctypes.data_as(ob.f32p), x.ctypes.data_as(ob.f32p), W.ctypes.data, n, d)
    got = E.op_f32_matvec(x, W, n, d, exact=0)
    assert np.abs(got - want).max() <= 2e-6 * np.abs(W).max() * np.abs(x).max() * n ** 0.5 + 1e-7


# ------------------------------------------------------------------------------------------------ §5 non-causal
@pytest.mark.gpu
@pytest.mark.parametrize("quant", [F32, Q80])
@pytest.mark.parametrize("name", ["kvm5-qwen3", "kvm8-qwen3"])
def test_non_causal(name, quant, monkeypatch):
    """forward(tok, pos, 0), as seq2seq runs it: every position attends to all max_seq cache rows.  Exact mode bit-identical;
    F32 fast mode within the F32 tolerance."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, 128)
    S = S_FAST
    toks = mf.teacher_tokens(S, spec.vocab)
    o = ob.NanoOracle(path, S)
    ref = np.stack([o.forward(toks[p], p, 0) for p in range(S)])
    ok, ov = (a.copy() for a in o.kv())
    o.close()
    eng = multi_engine(path, S, E.FLAG_EXACT, monkeypatch)
    exact_check(eng, spec, S, ref, ok, ov, "exact non-causal", causal=0)
    eng.close()
    if quant == F32:
        eng = multi_engine(path, S, 0, monkeypatch)
        fast_check(eng, spec, S, ref, ok, ov, TOL[F32], f"{name} fast non-causal", causal=0)
        assert eng.kernels()["attention"] == ATTN_WANT[name], eng.kernels()
        eng.close()


# ------------------------------------------------------------------------------------------------ §6 coverage guard (CPU)
EPI_NUM = {n: i for i, n in enumerate(E.MATVEC_EPILOGUES)}


def declared_matvec():
    """(QUANT, EPI, RB, LPG) of every single-GPU k_matvec instantiation a case above runs."""
    out = set()
    for _name, quant, gs in MV_CASES:
        lpg = gs // 16 if quant == Q80 else 8
        for rb in RBS:
            for exact in (True, False):
                out |= {(quant, EPI_NUM[e], r, lpg) for e, r in expected_matvec(quant, rb, exact)}
    for _n, _d, gs in Q80_OP_SHAPES:
        out |= {(Q80, EPI_NUM["store"], rb, gs // 16) for rb in RBS}
    out |= {(q, EPI_NUM["store"], rb, 8) for q in (F32, Q4K) for rb in (2, 4)}
    return out


def declared_attention():
    return {ATTN_WANT[c[0]] for c in ATTN_CASES + MV_CASES} | {"exact"}


def test_every_single_gpu_multikernel_variant_has_a_case():
    """The k_matvec and attention kernels in the built library (tensor-parallel variants aside) are exactly the ones the
    cases above run: a new instantiation without a case, or a case dropped from the matrix, fails here."""
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", nb_build.ENGINE_SO],
                         capture_output=True, text=True, check=True).stdout
    matvec, attention = set(), set()
    for name in re.findall(r"Function (\S+):", out):
        m = re.search(r"8k_matvecILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])E", name)
        if m and m.group(5) == "0":
            matvec.add((int(m.group(1)), int(m.group(2)), int(m.group(3)), int(m.group(4))))
        m = re.search(r"16k_attention_fastILi(\d+)ELb([01])E", name)
        if m and m.group(2) == "0":
            attention.add(f"fast<{m.group(1)}>")
        if re.search(r"11k_attentionE", name):
            attention.add("generic")
        if re.search(r"17k_attention_exactE", name):
            attention.add("exact")
    assert len(matvec) == 76, len(matvec)
    assert matvec == declared_matvec(), (f"no case: {sorted(matvec - declared_matvec())}; "
                                         f"not in the library: {sorted(declared_matvec() - matvec)}")
    assert attention == declared_attention(), (attention, declared_attention())
