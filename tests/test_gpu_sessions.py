"""The engine across whole sessions: one script of calls applied to the engine and to its references in lockstep.

The engine keeps state between calls, and the reference's own callers use it: a new chat turn starts again at pos 0 on the
same context, seq2seq runs n_layer non-causal sweeps over all max_seq positions (each position then attends to rows an
earlier sweep wrote, or to rows that are still zero), llm_forward takes the LoRA plug-in per call, and the repetition penalty's
`seen` set is mirrored on the host across calls.  Every step is checked:

* exact mode: logits and ids bit-identical to the oracle (to the strict reference in the LoRA scripts);
* fast paths: logits within the fast_limit policy, ids equal wherever the oracle's top-1 / top-2 margin is real;
* F32 files: max|gpu - ref64| <= 4 max|oracle - ref64| + 1e-6 max|ref64| against the float64 session (tests/ref64.py);
* steps with a penalty compare the engine's post-penalty logits with the reference's raw logits, every id of ids[0..pos)
  divided by the penalty.

At every checkpoint the whole K / V cache of every layer, all max_seq rows, is compared: stale rows of abandoned branches and
earlier sessions, and rows never written, which must be exactly 0.
"""
import os

import numpy as np
import pytest

import ref64
from conftest import assert_bits_equal
from nano_b200 import engine as E, modelfile as mf
from oracle import bindings as ob
from test_gpu_multikernel_matrix import fast_limit
from test_gpu_stream_matrix import S_FAST

pytestmark = pytest.mark.gpu

F32, Q80, Q4K = mf.QUANT_F32, mf.QUANT_Q80, mf.QUANT_Q4K
# (flags, environment, path the engine must report)
PATHS = {"stream": (0, {"NB200_STREAM": "1"}, "streaming"),
         "stream-owned-tiles": (0, {"NB200_STREAM": "1", "NB200_OWNED_ROWS": "2"}, "streaming"),
         "multikernel": (E.FLAG_NO_STREAM, {}, "multi-kernel"),
         "exact": (E.FLAG_EXACT, {}, "multi-kernel")}
# toy shapes in every file kind; the tight shapes select the streaming kernel at KVM 1 / 2 / 4 and k_attention_fast<1|2|4>
# (hd52-nano has n_embd 208: no Q80 group size of the engine divides it)
FILES = ([(n, q, g) for n in ("toy-nano", "toy-qwen3") for q, g in ((F32, 128), (Q80, 64), (Q4K, 128))] +
         [("kvm1-nano", F32, 128), ("kvm1-nano", Q80, 128), ("hd52-nano", F32, 128),
          ("kvm4-qwen3-hd64", F32, 128), ("kvm4-qwen3-hd64", Q80, 128)])
PEN = 1.3


def session_limit(name, quant, gs):
    """The fast-mode bound of a session: fast_limit, doubled for quantised files.  fast_limit rests on the reference's own
    fast-vs-strict floor over 40 causal positions; a session runs several hundred steps, and the n_layer non-causal sweeps of
    seq2seq carry one step's activation-code flips into every later row.  On an H100 (700 W power limit) the quantised files
    reached 1.46x fast_limit (K rows at the end of the context-end script) while exact mode was bit-identical on the same
    scripts; F32 files keep fast_limit and the float64 bound."""
    lim = fast_limit(name, quant, gs, mf.cached_model(mf.PRESETS[name], quant, gs), S_FAST)
    return lim if quant == F32 else 2.0 * lim


def file_id(f):
    return f"{f[0]}-{ {F32: 'f32', Q80: 'q80g', Q4K: 'q4k'}[f[1]] }{f[2] if f[1] == Q80 else ''}"


def kv_all(eng, spec, S):
    """The engine's whole K / V cache: [L, S, kv_dim] each."""
    k = np.stack([np.stack([eng.read(E.F_KROW, spec.kv_dim, l, p) for p in range(S)]) for l in range(spec.n_layer)])
    v = np.stack([np.stack([eng.read(E.F_VROW, spec.kv_dim, l, p) for p in range(S)]) for l in range(spec.n_layer)])
    return k, v


def penalised(logits, ids, pos, pen):
    """generate_next_token's repetition penalty: every id of ids[0..pos) divided by the penalty (infer.c:1140-1145)."""
    out = logits.copy()
    if pen != 1.0 and pos > 0:
        seen = np.unique(np.asarray(ids[:pos], np.int64))
        out[seen] = out[seen] / (np.float32(pen) if out.dtype == np.float32 else pen)
    return out


def new_engine(path, S, which, monkeypatch, **env):
    flags, penv, want = PATHS[which]
    with monkeypatch.context() as m:
        for k, v in {**penv, **env}.items():
            m.setenv(k, str(v))
        eng = E.Engine(path, S, flags=flags)
    # setup_stream declines a shape without an error: a case must fail, not quietly test the other path
    assert eng.path.startswith(want), f"{which}: engine runs {eng.path}"
    return eng


class RefLora:
    """The strict reference with a plug-in that is passed per call, as llm_forward takes it."""

    def __init__(self, path, S, image):
        self.r = ob.RefEngine(path, S, "strict")
        self.r.load_lora(image)
        self.on = True

    def forward(self, tok, pos, causal=1):
        return self.r.forward(tok, pos, causal, lora=self.on)

    def kv(self):
        return self.r.kv()

    def close(self):
        self.r.close()


class Lockstep:
    """One script applied to an engine and its references.  ids arrays are shared: where a fast path picks another id
    (allowed only where the oracle's margin is within noise), the references are teacher-forced with the engine's choice."""

    def __init__(self, name, quant, gs, S, which, monkeypatch, ref=None, limit=None):
        self.spec = mf.PRESETS[name]
        self.path = mf.cached_model(self.spec, quant, gs)
        self.S, self.which, self.exact = S, which, which == "exact"
        self.eng = new_engine(self.path, S, which, monkeypatch)
        self.ref = ref if ref is not None else ob.NanoOracle(self.path, S)
        self.r64 = ref64.Session64(*ref64.load_f32(self.path), S) if quant == F32 and ref is None else None
        self.limit = 0.0 if self.exact else (limit if limit is not None else session_limit(name, quant, gs))
        self.worst64 = 0.0          # worst |gpu - ref64| / |oracle - ref64|
        self.worst = 0.0            # worst max|gpu - reference| in fast mode

    def close(self):
        self.eng.close(); self.ref.close()

    def _f64(self, got, o32, r64, what):
        err, oerr, slack = np.abs(got - r64).max(), np.abs(o32 - r64).max(), 1e-6 * np.abs(r64).max()
        assert err <= 4 * oerr + slack, f"{what}: max|gpu - ref64| {err:.3e} > 4 x {oerr:.3e} + {slack:.1e}"
        self.worst64 = max(self.worst64, err / oerr if oerr > 0 else 0.0)

    def _logits(self, got, want, want64, what):
        if self.exact:
            assert_bits_equal(got, want, what)
        else:
            d = float(np.abs(got - want).max())
            self.worst = max(self.worst, d)
            assert d <= self.limit, f"{what}: max|dlogit| {d} > {self.limit}"
            top2 = np.partition(want, -2)[-2:]
            if float(top2[1] - top2[0]) > 2 * self.limit:
                assert int(np.argmax(got)) == int(np.argmax(want)), f"{what}: argmax differs, margin {top2[1] - top2[0]}"
        if want64 is not None:
            self._f64(got, want, want64, what)

    def _refs(self, tok, pos, causal=1):
        return self.ref.forward(tok, pos, causal), (self.r64.forward(tok, pos, causal) if self.r64 else None)

    def forward(self, tok, pos, causal=1):
        got = self.eng.forward(tok, pos, causal)
        want, w64 = self._refs(tok, pos, causal)
        self._logits(got, want, w64, f"{self.which} forward({tok}, {pos}, causal={causal})")
        return got

    def _step(self, ids, pos, prefilling, pen, got, nxt, what):
        """References for one generate_next_token step; returns the id the script continues with."""
        p = 1.0 if prefilling else pen
        raw, raw64 = self._refs(ids[pos], pos)
        want = penalised(raw, ids, pos, p)
        self._logits(got, want, None if raw64 is None else penalised(raw64, ids, pos, p), f"{self.which} {what} pos {pos}")
        if prefilling:
            assert nxt == ids[pos + 1]
        elif self.exact and what != "next_sampled":
            assert nxt == int(np.argmax(want)), f"{what} pos {pos}: id {nxt}, reference {int(np.argmax(want))}"
        return nxt

    def next_greedy(self, ids, pos, prefilling, pen=PEN):
        nxt = self.eng.next_greedy(ids, pos, prefilling, pen)
        return self._step(ids, pos, prefilling, pen, self.eng.logits(), nxt, "next_greedy")

    def next_sampled(self, ids, pos, pen=PEN, temperature=0.7, top_p=0.8, coin=0.37):
        nxt, _ = self.eng.next_sampled(ids, pos, pen, temperature, top_p, coin)
        got = self.eng.logits()
        assert nxt == ob.sample_top_p(got, temperature, top_p, coin)[0], f"next_sampled pos {pos}"
        return self._step(ids, pos, 0, pen, got, nxt, "next_sampled")

    def decode_greedy(self, ids, n_prompt, n_total, pen=PEN):
        """The device loop, then the references over the same positions, teacher-forced with the engine's ids.  The device
        loop divides by the penalty at every step, teacher-forced ones included (only their ids are specified)."""
        self.eng.decode_greedy(ids, n_prompt, n_total, pen)
        last = self.eng.logits()
        for pos in range(n_total - 1):
            pre = pos < n_prompt - 1
            raw, raw64 = self._refs(ids[pos], pos)
            want = penalised(raw, ids, pos, pen)
            if pos == n_total - 2:
                self._logits(last, want, None if raw64 is None else penalised(raw64, ids, pos, pen),
                             f"{self.which} decode_greedy last pos {pos}")
            if not pre:
                top2 = np.partition(want, -2)[-2:]
                if self.exact or float(top2[1] - top2[0]) > 2 * self.limit:
                    assert ids[pos + 1] == int(np.argmax(want)), f"decode_greedy pos {pos}: id {ids[pos + 1]}"

    def lora(self, on):
        self.eng.lora_enable(on)
        self.ref.on = on

    def checkpoint(self, what):
        ek, ev = kv_all(self.eng, self.spec, self.S)
        rk, rv = self.ref.kv()
        for got, want, nm in ((ek, rk, "K"), (ev, rv, "V")):
            unwritten = ~want.any(axis=2)
            assert not got[unwritten].any(), f"{what}: {nm} rows the reference never wrote are not zero in the engine"
            if self.exact:
                assert_bits_equal(got, want, f"{what}: {nm} cache")
            else:
                d = float(np.abs(got - want).max())
                assert d <= self.limit, f"{what}: {nm} cache max|d| {d} > {self.limit}"
        if self.r64 is not None:
            for l in range(self.spec.n_layer):
                self._f64(ek[l], rk[l], self.r64.k[l], f"{what}: K cache layer {l}")
                self._f64(ev[l], rv[l], self.r64.v[l], f"{what}: V cache layer {l}")

    def report(self, what):
        print(f"{what}: worst |gpu - ref64| / |oracle - ref64| {self.worst64:.3f}, worst fast max|dlogit| {self.worst:.3e}")


# ------------------------------------------------------------------------------------------------ scripts
def script_rewind(d):
    """Teacher-force 0..S-1; rewind to S/3 and regenerate with other tokens; a new, shorter session from 0."""
    S, V = d.S, d.spec.vocab
    a, b = mf.teacher_tokens(S, V), mf.teacher_tokens(S, V, seed=7)
    for p in range(S):
        d.forward(a[p], p)
    d.checkpoint("teacher-forced")
    for p in range(S // 3, S):
        d.forward(b[p], p)
    d.checkpoint("rewound to S/3")
    for p in range(S // 2):
        d.forward(b[S - 1 - p], p)
    d.checkpoint("second session, stale rows above S/2")


def seq2seq(d, toks):
    """The shim's seq2seq loop (infer.c:1365-1402): n_layer non-causal sweeps, then the argmax sweep."""
    n = len(toks)
    for _ in range(d.spec.n_layer):
        for p in range(n):
            d.forward(toks[p], p, 0)
    return [int(np.argmax(d.forward(toks[p], p, 0))) for p in range(n)]


def script_seq2seq(d):
    """seq2seq over every position the model's RoPE table allows (all max_seq rows are attended to), a causal session on
    the same engine, and another sweep."""
    n = min(d.S, d.spec.block_size)
    toks = mf.teacher_tokens(n, d.spec.vocab, seed=11)
    seq2seq(d, toks)
    d.checkpoint("seq2seq")
    c = mf.teacher_tokens(n, d.spec.vocab, seed=5)
    for p in range(n // 2):
        d.forward(c[p], p)
    d.checkpoint("causal session after seq2seq")
    seq2seq(d, toks[::-1].copy())
    d.checkpoint("second seq2seq")


def script_penalty(d):
    """Per-call sessions with a repetition penalty that walk every branch of the host mirror of the device `seen` set."""
    S = d.S
    P = 6
    A = np.zeros(S + 1, np.uint32); A[:P] = [5, 9, 5, 3, 9, 5]
    for pos in range(40):                                   # A, with one sampled step
        A[pos + 1] = (d.next_sampled(A, pos) if pos == 30 else d.next_greedy(A, pos, 1 if pos < P - 1 else 0))
    d.checkpoint("session A")
    B = np.zeros(S + 1, np.uint32); B[:12] = A[:12]; B[12:16] = [(int(A[12]) + 1) % d.spec.vocab, 7, 8, 2]
    for pos in range(24):                                   # B: shorter than the mirror -> reset
        B[pos + 1] = d.next_greedy(B, pos, 1 if pos < 15 else 0)
    d.checkpoint("session B")
    Cc = np.zeros(S + 1, np.uint32); Cc[:24] = B[:24]; Cc[24:30] = [11, 12, 13, 11, 12, 13]
    for pos in range(36):                                   # C: starts with B's history -> the mirror's prefix is reused
        Cc[pos + 1] = d.next_greedy(Cc, pos, 1 if pos < 29 else 0)
    d.checkpoint("session C")
    D = np.zeros(S + 1, np.uint32); D[:37] = Cc[:37]
    fresh = next(t for t in range(d.spec.vocab) if t not in set(Cc[:S].tolist()))
    D[:37][D[:37] == D[3]] = fresh                          # D: longer than C's history, differs from it at index 3 -> reset
    for pos in range(44):
        D[pos + 1] = d.next_greedy(D, pos, 1 if pos < 36 else 0)
    d.checkpoint("session D")
    F = np.zeros(S + 1, np.uint32); F[:5] = [9, 8, 7, 9, 8]
    d.decode_greedy(F, 5, 40)
    d.checkpoint("decode_greedy")
    G = np.zeros(S + 1, np.uint32); G[:5] = F[:5]
    for pos in range(39):                                   # E: per call again, the same prompt
        G[pos + 1] = d.next_greedy(G, pos, 1 if pos < 4 else 0)
    assert G[:40].tolist() == F[:40].tolist(), "the per-call loop and the device loop disagree"
    d.checkpoint("session E")


def script_context_end(d):
    """The last position of the context, in the device loop and per call."""
    S = d.S
    ids = np.zeros(S + 1, np.uint32); ids[:5] = [9, 8, 7, 9, 8]
    d.decode_greedy(ids, 5, S + 1)                          # the last step decodes pos S-1
    d.checkpoint("decode_greedy to max_seq + 1")
    ids = np.zeros(S + 1, np.uint32); ids[:] = mf.teacher_tokens(S + 1, d.spec.vocab, seed=3)
    d.decode_greedy(ids, S + 1, S + 1)
    d.checkpoint("decode_greedy, all prompt")
    ids = np.zeros(S + 1, np.uint32); ids[0] = 17
    d.decode_greedy(ids, 1, S + 1)
    d.checkpoint("decode_greedy, one prompt id")
    ids = np.zeros(S + 1, np.uint32); ids[:S] = mf.teacher_tokens(S, d.spec.vocab, seed=13)
    for pos in range(S):
        ids[pos + 1] = d.next_greedy(ids, pos, 1 if pos < S - 1 else 0)
    d.checkpoint("next_greedy at max_seq - 1")


SCRIPTS = {"rewind": (script_rewind, 48), "seq2seq-64": (script_seq2seq, 64), "seq2seq-512": (script_seq2seq, 512),
           "penalty": (script_penalty, 64), "context-end": (script_context_end, 48)}


@pytest.mark.parametrize("which", list(PATHS))
@pytest.mark.parametrize("script", list(SCRIPTS))
@pytest.mark.parametrize("name,quant,gs", FILES, ids=[file_id(f) for f in FILES])
def test_session_scripts(name, quant, gs, script, which, monkeypatch):
    fn, S = SCRIPTS[script]
    d = Lockstep(name, quant, gs, S, which, monkeypatch)
    fn(d)
    d.report(f"{name} {quant:#x} gs {gs} {script} {which}")
    d.close()


# ------------------------------------------------------------------------------------------------ LoRA per call
LORA_FILES = [("toy-nano", F32, 128), ("toy-nano", Q80, 64), ("toy-nano", Q4K, 128), ("mini-nano", Q80, 128)]


@pytest.mark.skipif(not ob.ref_available("strict"), reason="needs the unmodified reference (oracle/_ref)")
@pytest.mark.parametrize("which", ["exact", "stream"])
@pytest.mark.parametrize("rank", [1, 8, 64])
@pytest.mark.parametrize("name,quant,gs", LORA_FILES, ids=[file_id(f) for f in LORA_FILES])
def test_lora_toggled_mid_session(name, quant, gs, rank, which, monkeypatch):
    """The plug-in off for positions 0-9, on for 10-29, off again; then a non-causal sweep with it loaded but off (what
    seq2seq passes).  The K / V cache is shared by the streaming and the multi-kernel path, which the toggles switch."""
    if not ob.ref_has_forward_lora():
        pytest.skip("the reference harness in oracle/_ref predates orh_forward_lora (llm_forward without the plug-in)")
    spec = mf.PRESETS[name]
    S = 40
    image = mf.write_lora(spec, rank, 2 * rank, seed=7)
    ref = RefLora(mf.cached_model(spec, quant, gs), S, image)
    d = Lockstep(name, quant, gs, S, which, monkeypatch, ref=ref, limit=session_limit(name, quant, gs))
    base = d.eng.path
    d.eng.lora_load(image)
    assert d.eng.path.startswith("multi-kernel"), d.eng.path
    toks = mf.teacher_tokens(S, spec.vocab)
    for lo, hi, on in ((0, 10, False), (10, 30, True), (30, S, False)):
        d.lora(on)
        assert d.eng.path.startswith("multi-kernel") if on else d.eng.path == base, d.eng.path
        for p in range(lo, hi):
            d.forward(toks[p], p)
        d.checkpoint(f"plug-in {'on' if on else 'off'} for {lo}..{hi - 1}")
    assert d.eng.path == base
    seq2seq(d, mf.teacher_tokens(S, spec.vocab, seed=11))
    d.checkpoint("seq2seq with the plug-in loaded but off")
    d.report(f"{name} {quant:#x} gs {gs} rank {rank} {which}")
    d.close()


# ------------------------------------------------------------------------------------------------ as created, calibration
def assert_as_created(eng, spec, S, what):
    k, v = kv_all(eng, spec, S)
    assert not k.any() and not v.any(), f"{what}: K/V rows are not zero after creation"
    assert not eng.logits().any(), f"{what}: logits are not zero after creation"


@pytest.mark.parametrize("which", list(PATHS))
@pytest.mark.parametrize("name", ["toy-nano", "toy-qwen3"])
def test_as_created(name, which, monkeypatch):
    spec = mf.PRESETS[name]
    eng = new_engine(mf.cached_model(spec, Q80, 64), 64, which, monkeypatch)
    assert_as_created(eng, spec, 64, which)
    eng.close()


def calib_model():
    return mf.cached_model(mf.PRESETS["calib-qwen3"], Q80, 128, fast=True)


def test_calibration_leaves_no_state(monkeypatch):
    """A Q80 engine of 256 MiB of weights or more times both fast paths at creation, from the middle of its context.  It must
    then compute what an engine forced onto the same path (which skips the timing) computes: the first seq2seq sweep attends
    to every cache row, including the rows the timing steps wrote."""
    spec = mf.PRESETS["calib-qwen3"]
    path, S = calib_model(), 64
    eng = E.Engine(path, S)
    assert eng.calibration is not None, "the engine no longer calibrates: this case would test nothing"
    assert_as_created(eng, spec, S, "calibrated engine")
    with monkeypatch.context() as m:
        m.setenv("NB200_STREAM", "1" if eng.path.startswith("streaming") else "0")
        ctl = E.Engine(path, S)
    assert ctl.calibration is None and ctl.path == eng.path, (ctl.path, eng.path)
    toks = mf.teacher_tokens(S, spec.vocab)
    for p in range(8):                                       # control: the two engines compute identically
        assert_bits_equal(eng.forward(toks[p], p), ctl.forward(toks[p], p), f"causal pos {p}")
    for sweep in range(spec.n_layer + 1):
        for p in range(S):
            assert_bits_equal(eng.forward(toks[p], p, 0), ctl.forward(toks[p], p, 0), f"seq2seq sweep {sweep} pos {p}")
    eng.close(); ctl.close()


# ------------------------------------------------------------------------------------------------ block_size
def test_positions_stop_at_block_size():
    """The RoPE table has block_size rows: a context longer than that is legal (nano_cli creates one), but every entry
    point refuses a position at or past block_size."""
    spec = mf.PRESETS["toy-nano"]                            # block 64
    path, S = mf.cached_model(spec, F32, 128), 128
    eng = E.Engine(path, S, flags=E.FLAG_EXACT); o = ob.NanoOracle(path, S)
    toks = mf.teacher_tokens(64, spec.vocab)
    for p in range(64):
        assert_bits_equal(eng.forward(toks[p], p), o.forward(toks[p], p), f"pos {p}")
    o.close(); eng.close()
    eng = E.Engine(path, S)
    ids = np.zeros(S + 1, np.uint32); ids[:66] = mf.teacher_tokens(66, spec.vocab)
    with pytest.raises(E.NB200Error):
        eng.forward(1, 64)
    with pytest.raises(E.NB200Error):
        eng.next_greedy(ids, 64, 0, PEN)
    with pytest.raises(E.NB200Error):
        eng.next_sampled(ids, 64, PEN, 0.7, 0.8, 0.5)
    with pytest.raises(E.NB200Error):
        eng.decode_greedy(ids.copy(), 5, 66)
    eng.decode_greedy(ids, 5, 65)                            # the last step decodes pos 63
    eng.close()


def test_calibration_stays_inside_the_rope_table():
    """max_seq 1024 on a 256-row table: the timing steps start inside the table, and leave nothing behind."""
    spec = mf.PRESETS["calib-qwen3"]
    eng = E.Engine(calib_model(), 1024)
    assert eng.calibration is not None
    assert_as_created(eng, spec, 1024, "max_seq 1024")
    eng.close()


@pytest.mark.skipif(not os.path.exists(ob.REFHOST_SO), reason="needs the reference's tokenizer/utils objects")
def test_shim_session_ends_at_block_size():
    """llm_session_step ends a session at block_size with NANO_STOP_ERROR, as it does at max_seq_len."""
    from test_gpu_shim import shim
    L = shim()
    ctx = L.llm_context_init(mf.cached_model(mf.PRESETS["toy-nano"], Q80, 64).encode(), None, 128, 1.0, 0.0, 0.8, 20, 39)
    s = L.llm_session_init(ctx, "0123456789" * 7, 128, 0)
    statuses = []
    for _ in range(100):
        statuses.append(L.llm_session_step(ctx, s))
        if statuses[-1] <= 0:
            break
    assert statuses[-1] == -20 and s.contents.pos == 64, (statuses[-3:], s.contents.pos)
    L.llm_session_free(s)
    L.llm_context_free(ctx)
