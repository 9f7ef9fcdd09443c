"""Every instantiation of the streaming decode kernel (k_decode_stream<QUANT, LPG, KVM>) and of the multi-kernel split-KV
attention (k_attention_fast<KVM>), on 2-layer models whose shapes select them, against the oracle and against a float64
restatement of the forward pass (tests/ref64.py).

* KVM = n_head / n_kv_head in {1, 2, 4}; hd 128, 64 and 52 (hd % 16 != 0: the unrotated score loop).
* Activation-prologue widths around its poll batches and slots: n = 3840 (one full batch of 15 warps x 2 slots x 128),
  3968 (one slot into the second batch), 11520 (st_prep_max_n for Q80 / F32); Q4K 4096 (second warp slot) and 7680
  (its st_prep_max_n); one group / block past each limit takes the multi-kernel path.
* Every case asserts the path it claims to run: setup_stream declines a shape without an error.
* F32 at tight tolerance: at every position, max|gpu - ref64| <= 4 max|oracle - ref64| + 1e-6 max|ref64|, for the
  logits and for the K / V rows of every layer, over long contexts (many splits, several ring segments per split, the
  split-0 merge) and over the knobs that move the ring and split geometry.
"""
import numpy as np
import pytest

import ref64
from conftest import assert_bits_equal
from nano_b200 import engine as E, modelfile as mf
from oracle import bindings as ob
from test_gpu_engine import reference_noise_floor

F32, Q80, Q4K = mf.QUANT_F32, mf.QUANT_Q80, mf.QUANT_Q4K
STREAM, MULTI = "stream", "multi"
ALL4 = [(F32, 128), (Q80, 128), (Q80, 64), (Q4K, 128)]

# (preset, quant, gs, path the fast mode must take by default when streaming is forced)
CASES = ([("kvm1-nano", q, g, STREAM) for q, g in ALL4] +
         [("kvm4-qwen3-hd128", q, g, STREAM) for q, g in ALL4] +
         [("kvm4-qwen3-hd64", q, g, STREAM) for q, g in ALL4] +
         [("hd52-nano", F32, 128, STREAM), ("qwen3-4b-2l", Q80, 128, STREAM)] +
         [("ffn3840-nano", q, g, STREAM) for q, g in ALL4[1:]] +
         # F32 rows of 3840+ floats (15 KB) leave no room for the ring's 12 stages beside two activation operands: setup_stream
         # declines them, so the F32 prologue never runs past its first poll batch
         [("ffn3840-nano", F32, 128, MULTI), ("ffn11520-nano", F32, 128, MULTI),
          ("ffn3968-nano", Q80, 128, STREAM), ("ffn3968-nano", Q80, 64, STREAM),
          ("ffn4096-nano", Q4K, 128, STREAM), ("ffn4096-nano", Q80, 64, STREAM),
          ("ffn7680-nano", Q4K, 128, STREAM), ("ffn7680-nano", Q80, 128, STREAM),
          ("ffn11520-nano", Q80, 128, STREAM), ("ffn11520-nano", Q80, 64, STREAM),
          ("ffn7936-nano", Q4K, 128, MULTI), ("ffn7936-nano", Q80, 128, STREAM),
          ("ffn11648-nano", Q80, 128, MULTI), ("ffn11648-nano", F32, 128, MULTI)])
TOL = {F32: 1e-4, Q80: 1e-2, Q4K: 1e-2}
S_FAST = 40                  # the sequence length of the committed noise floors


def case_id(c):
    return f"{c[0]}-{ {F32: 'f32', Q80: 'q80g', Q4K: 'q4k'}[c[1]] }{c[2] if c[1] == Q80 else ''}"


def assert_path(eng, want):
    if want == STREAM:
        assert eng.path.startswith("streaming"), f"expected the streaming kernel, engine runs: {eng.path}"
    else:
        assert eng.path.startswith("multi-kernel"), f"expected the multi-kernel path, engine runs: {eng.path}"


def engine(path, S, flags, monkeypatch, **env):
    """An engine created with NB200_STREAM=1 (streaming wherever the shape allows it) and the given NB200_* knobs."""
    with monkeypatch.context() as m:
        m.setenv("NB200_STREAM", "1")
        for k, v in env.items():
            m.setenv(k, str(v))
        return E.Engine(path, S, flags=flags)


_ORACLE = {}


def oracle_run(path, S, vocab):
    """Teacher-forced oracle logits [S, V] and K / V caches (cached per file and length)."""
    key = (path, S)
    if key not in _ORACLE:
        o = ob.NanoOracle(path, S)
        toks = mf.teacher_tokens(S, vocab)
        lg = np.stack([o.forward(toks[p], p) for p in range(S)])
        k, v = o.kv()
        _ORACLE[key] = (lg, k.copy(), v.copy())
        o.close()
    return _ORACLE[key]


# ------------------------------------------------------------------------------------------------ §1 every instantiation
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,want", CASES, ids=[case_id(c) for c in CASES])
def test_instantiation_matrix(name, quant, gs, want, monkeypatch):
    """Fast mode on the selected path and on the multi-kernel path: logits within the floor policy (argmax agreement
    where the oracle's margin is real) and K / V rows of every layer within the same bound; exact mode bit-identical,
    logits and K / V rows."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = S_FAST
    toks = mf.teacher_tokens(S, spec.vocab)
    ref, ok, ov = oracle_run(path, S, spec.vocab)
    limit = max(TOL[quant], 1.5 * reference_noise_floor(name, quant, gs, path, S))
    kv_pos = (0, 1, S // 2, S - 1)
    for flags, expect in ((0, want), (E.FLAG_NO_STREAM, MULTI)):
        eng = engine(path, S, flags, monkeypatch)
        assert_path(eng, expect)
        worst = 0.0
        for pos in range(S):
            a = eng.forward(toks[pos], pos); b = ref[pos]
            worst = max(worst, float(np.abs(a - b).max()))
            top2 = np.partition(b, -2)[-2:]
            if float(top2[1] - top2[0]) > 2 * limit:
                assert int(np.argmax(a)) == int(np.argmax(b)), f"{expect} pos {pos}: argmax differs, margin {top2[1] - top2[0]}"
        assert worst <= limit, f"{expect}: max|dlogit| {worst} > {limit}"
        for l in range(spec.n_layer):
            for pos in kv_pos:
                dk = np.abs(eng.read(E.F_KROW, spec.kv_dim, l, pos) - ok[l, pos]).max()
                dv = np.abs(eng.read(E.F_VROW, spec.kv_dim, l, pos) - ov[l, pos]).max()
                assert max(dk, dv) <= limit, f"{expect} layer {l} pos {pos}: max|dK| {dk}, max|dV| {dv} > {limit}"
        print(f"{name} {quant:#x} gs {gs} {expect}: max|dlogit| {worst:.3e} (limit {limit:.3e})")
        eng.close()
    eng = engine(path, S, E.FLAG_EXACT, monkeypatch)
    for pos in range(S):
        assert_bits_equal(eng.forward(toks[pos], pos), ref[pos], f"exact pos {pos}")
    for l in range(spec.n_layer):
        for pos in kv_pos:
            assert_bits_equal(eng.read(E.F_KROW, spec.kv_dim, l, pos), ok[l, pos], f"exact K row {l}/{pos}")
            assert_bits_equal(eng.read(E.F_VROW, spec.kv_dim, l, pos), ov[l, pos], f"exact V row {l}/{pos}")
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kvm1-nano", "kvm4-qwen3-hd128", "kvm4-qwen3-hd64"])
def test_device_loop_kvm1_kvm4(name, monkeypatch):
    """Greedy ids with a repetition penalty: exact mode equals the oracle, per call and in the device-resident loop; on the
    streaming kernel the device-resident loop reproduces the per-call loop."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S, P, pen = 40, 6, 1.3
    prompt = [5, 9, 5, 3, 9, 5]
    o = ob.NanoOracle(path, S)
    ids_o = np.zeros(S + 1, np.uint32); ids_o[:P] = prompt
    for pos in range(S - 1):
        ids_o[pos + 1] = o.next_greedy(ids_o, pos, 1 if pos < P - 1 else 0, pen)
    o.close()
    for flags in (E.FLAG_EXACT, 0):
        eng = engine(path, S, flags, monkeypatch)
        if flags == 0:
            assert_path(eng, STREAM)
        a = np.zeros(S + 1, np.uint32); a[:P] = prompt
        for pos in range(S - 1):
            a[pos + 1] = eng.next_greedy(a, pos, 1 if pos < P - 1 else 0, pen)
        b = np.zeros(S + 1, np.uint32); b[:P] = prompt
        eng.decode_greedy(b, P, S, pen)
        assert a[:S].tolist() == b[:S].tolist(), eng.path
        if flags == E.FLAG_EXACT:
            assert a[:S].tolist() == ids_o[:S].tolist()
        eng.close()


# ------------------------------------------------------------------------------------------------ §2 F32 against float64
_REF64 = {}


def ref64_run(path, S, vocab):
    key = (path, S)
    if key not in _REF64:
        spec, p = ref64.load_f32(path)
        _REF64[key] = ref64.forward(spec, p, mf.teacher_tokens(S, vocab))
    return _REF64[key]


def test_ref64_matches_oracle_on_cpu():
    """The float64 restatement is itself checked against the C oracle (no GPU): fp32 noise only, on the toy files and on
    the F32 shapes of the tight tests.  Qwen3 at S = 512 as well: a RoPE frequency one ulp off the engines' fp32 table moves
    the late positions' K rows by ~2e-5 relative, ten times the fp32 noise seen here."""
    for name, S in (("toy-nano", 24), ("toy-qwen3", 24), ("kvm1-nano", 24), ("kvm4-qwen3-hd128", 24), ("kvm4-qwen3-hd64", 24),
                    ("hd52-nano", 24), ("long-qwen3", 512)):
        spec = mf.PRESETS[name]
        path = mf.cached_model(spec, F32, 128)
        lg, k, v = ref64_run(path, S, spec.vocab)
        ora, ok, ov = oracle_run(path, S, spec.vocab)
        scale = np.abs(lg).max()
        assert np.abs(ora - lg).max() <= 1e-5 * scale, (name, np.abs(ora - lg).max(), scale)
        for l in range(spec.n_layer):
            assert np.abs(ok[l, :S] - k[l]).max() <= 1e-5 * np.abs(k[l]).max(), (name, l, "K")
            assert np.abs(ov[l, :S] - v[l]).max() <= 1e-5 * np.abs(v[l]).max(), (name, l, "V")


def test_session64_matches_oracle_on_cpu():
    """The float64 session (ref64.Session64) against the C oracle driven through the same calls: a teacher-forced run, a
    rewind, a non-causal sweep over all rows (some never written) and a second session over stale rows.  fp32 noise only."""
    for name in ("toy-nano", "toy-qwen3"):
        spec = mf.PRESETS[name]
        path = mf.cached_model(spec, F32, 128)
        S = 32
        o = ob.NanoOracle(path, S); s = ref64.Session64(*ref64.load_f32(path), S)
        a, b = mf.teacher_tokens(S, spec.vocab), mf.teacher_tokens(S, spec.vocab, seed=7)
        script = ([(a[p], p, 1) for p in range(24)] + [(b[p], p, 1) for p in range(8, 20)] +
                  [(a[p], p, 0) for p in range(S)] + [(b[p], p, 1) for p in range(6)])
        for tok, pos, causal in script:
            lg32, lg64 = o.forward(tok, pos, causal), s.forward(tok, pos, causal)
            assert np.abs(lg32 - lg64).max() <= 1e-5 * np.abs(lg64).max(), (name, pos, causal)
        ok, ov = o.kv()
        for l in range(spec.n_layer):
            assert np.abs(ok[l] - s.k[l]).max() <= 1e-5 * np.abs(s.k[l]).max(), (name, l, "K")
            assert np.abs(ov[l] - s.v[l]).max() <= 1e-5 * np.abs(s.v[l]).max(), (name, l, "V")
        o.close()


TIGHT_SHAPES = ["kvm1-nano", "long-qwen3", "hd52-nano", "kvm4-qwen3-hd128", "kvm4-qwen3-hd64"]     # KVM 1, 2, 2, 4, 4
S_LONG = 2048
# NB200_STAGE_KB=1: setup_stream raises the stage to the smallest one that holds a row unit of the widest matrix, so this is the
# smallest stage each shape allows -- K/V rows per tile: hd52-nano 4 (the minimum), kvm1-nano 8, kvm4-qwen3-hd128 8,
# long-qwen3 12 (its 12 KB W2 rows), against 36 / 32 / 16 / 16 at the default 16 KB
KNOBS = {"chunk8": {"NB200_ATTN_CHUNK": 8}, "chunk64": {"NB200_ATTN_CHUNK": 64}, "stages12": {"NB200_STAGES": 12},
         "min_stage": {"NB200_STAGE_KB": 1}, "owned2": {"NB200_OWNED_ROWS": 2}}


def tight_check(eng, spec, path, S, what, n_ref=S_LONG):
    """Run S teacher-forced positions; every position's logits, and K / V rows of every layer at a stride of positions,
    must be as close to float64 as the oracle's fp32 within 4x (+ 1e-6 of the largest value).  Prints the worst
    |gpu - ref64| / |oracle - ref64| and the worst share of the bound used.  The references run n_ref >= S positions
    (one cached run serves every S of a file)."""
    lg64, k64, v64 = ref64_run(path, n_ref, spec.vocab)
    ora, ok, ov = oracle_run(path, n_ref, spec.vocab)
    toks = mf.teacher_tokens(S, spec.vocab)
    worst, share = 0.0, 0.0

    def check(got, o32, r64, where):
        nonlocal worst, share
        err, oerr, slack = np.abs(got - r64).max(), np.abs(o32 - r64).max(), 1e-6 * np.abs(r64).max()
        assert err <= 4 * oerr + slack, f"{what} {where}: max|gpu - ref64| {err:.3e} > 4 x {oerr:.3e} + {slack:.1e}"
        worst = max(worst, err / oerr if oerr > 0 else 0.0)
        share = max(share, err / (4 * oerr + slack))
    for pos in range(S):
        check(eng.forward(toks[pos], pos), ora[pos], lg64[pos], f"pos {pos} logits")
    for pos in sorted({0, 1, S // 2, S - 2, S - 1} | set(range(127, S, 256))):
        for l in range(spec.n_layer):
            check(eng.read(E.F_KROW, spec.kv_dim, l, pos), ok[l, pos], k64[l, pos], f"pos {pos} layer {l} K")
            check(eng.read(E.F_VROW, spec.kv_dim, l, pos), ov[l, pos], v64[l, pos], f"pos {pos} layer {l} V")
    print(f"{what}: worst |gpu - ref64| / |oracle - ref64| = {worst:.3f}, worst share of the bound {share:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("S", [512, S_LONG])
@pytest.mark.parametrize("which", [STREAM, MULTI])
@pytest.mark.parametrize("name", TIGHT_SHAPES)
def test_f32_tight_vs_float64(name, which, S, monkeypatch):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, F32, 128)
    eng = engine(path, S, 0 if which == STREAM else E.FLAG_NO_STREAM, monkeypatch)
    assert_path(eng, which)
    tight_check(eng, spec, path, S, f"{name} {which} S {S}")
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("knob", list(KNOBS))
@pytest.mark.parametrize("name", ["kvm1-nano", "hd52-nano", "long-qwen3", "kvm4-qwen3-hd128"])
def test_f32_tight_ring_and_split_knobs(name, knob, monkeypatch):
    """The streaming kernel with the knobs that move its ring and split geometry: many splits (up to nsplit_max), the
    minimum ring (kStSegTiles + 4 stages), small stages (few K/V rows per tile, more segments), warp-owned tiles."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, F32, 128)
    eng = engine(path, S_LONG, 0, monkeypatch, **KNOBS[knob])
    assert_path(eng, STREAM)
    tight_check(eng, spec, path, S_LONG, f"{name} stream {knob}")
    eng.close()
