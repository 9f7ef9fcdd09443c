"""Batched multi-session decode (nb200_batch_*, nano_b200/csrc/batch.cuh).

A batch runs one decode step of up to M sessions ("slots") per pass over the weights with the multi-kernel token path's own
arithmetic, so every slot's next ids, logits and K / V rows must equal, bit for bit, those of an engine created with the same
flags plus NB200_FLAG_NO_STREAM running that session alone (nb200_prefill + nb200_next_greedy), and in exact mode those of the
strict reference.  Covered here:
  * the bit identity over the toy shapes x F32 / Q80 (every group size) / Q4K x exact / fast: five sessions, some prefilled
    through the batch and some started token by token, penalties 1.3 and 1.0, a different set of slots in every call;
  * exact mode against the oracle; every attention kernel, long slots sharing a pass with short ones; the classifier shapes
    (partial last row block, M < 16, untied, exact ties); pass shapes; the BASELINE shapes;
  * the engine's own session untouched by batch traffic; refusals; launch counts;
  * (CPU) no batch kernel has a stack frame of its own.
"""
import re
import subprocess

import numpy as np
import pytest

from conftest import assert_bits_equal
from nano_b200 import build as nb_build, engine as E, modelfile as mf
from test_gpu_sampler import tie_model  # noqa: F401  (the tied-classifier model file, a module fixture)

F32, Q80, Q4K = mf.QUANT_F32, mf.QUANT_Q80, mf.QUANT_Q4K
PEN = 1.3


def quant_id(quant, gs):
    return {F32: "f32", Q80: f"q80g{gs}", Q4K: "q4k"}[quant]


def nostream(path, S, flags=0, monkeypatch=None, **env):
    if monkeypatch is not None and env:
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, str(v))
            return E.Engine(path, S, flags=flags | E.FLAG_NO_STREAM)
    return E.Engine(path, S, flags=flags | E.FLAG_NO_STREAM)


def engine_kv(eng, upto):
    k = np.stack([np.stack([eng.read(E.F_KROW, eng.kv_dim, l, p) for p in range(upto)]) for l in range(eng.n_layer)])
    v = np.stack([np.stack([eng.read(E.F_VROW, eng.kv_dim, l, p) for p in range(upto)]) for l in range(eng.n_layer)])
    return k, v


def slot_kv(batch, slot, upto):
    eng = batch.engine
    k = np.stack([np.stack([batch.read(E.F_KROW, eng.kv_dim, slot, l, p) for p in range(upto)]) for l in range(eng.n_layer)])
    v = np.stack([np.stack([batch.read(E.F_VROW, eng.kv_dim, slot, l, p) for p in range(upto)]) for l in range(eng.n_layer)])
    return k, v


class Session:
    """One session in a batch slot and, beside it, the same session alone on its own multi-kernel engine."""

    def __init__(self, batch, slot, ref, prompt, penalty, S, prefill):
        self.batch, self.slot, self.ref, self.penalty = batch, slot, ref, penalty
        self.prompt = np.asarray(prompt, np.uint32)
        self.ids = np.zeros(S + 1, np.uint32)
        self.ids[: len(prompt)] = self.prompt
        self.pos = 0
        if prefill and len(prompt) > 1:           # the prompt's K / V rows in one call, then decode from its last position
            n = len(prompt) - 1
            batch.prefill(slot, self.ids, 0, n)
            ref.prefill(self.ids, 0, n)
            self.pos = n

    def entry(self):
        return self.slot, self.ids, self.pos, self.penalty

    def advance(self, got, what):
        """The batch's id for this slot from the last call: compare with the engine's step at the same position."""
        want = self.ref.next_greedy(self.ids, self.pos, 0, self.penalty)
        assert got == want, f"{what} slot {self.slot} pos {self.pos}: id {got} vs {want}"
        assert_bits_equal(self.batch.logits(self.slot), self.ref.logits(), f"{what} slot {self.slot} pos {self.pos}: logits")
        if self.pos + 1 >= len(self.prompt):      # past the prompt: the session continues with its greedy id
            self.ids[self.pos + 1] = got
        self.pos += 1

    def check_cache(self, what):
        k, v = slot_kv(self.batch, self.slot, self.pos)
        rk, rv = engine_kv(self.ref, self.pos)
        assert_bits_equal(k, rk, f"{what} slot {self.slot}: K rows 0..{self.pos - 1}")
        assert_bits_equal(v, rv, f"{what} slot {self.slot}: V rows 0..{self.pos - 1}")


def step(batch, sessions, what):
    entries = [s.entry() for s in sessions]
    got = batch.next_greedy([e[0] for e in entries], [e[1] for e in entries], [e[2] for e in entries], [e[3] for e in entries])
    for s, g in zip(sessions, got):
        s.advance(g, what)
    return got


def run_sessions(path, S, flags, prompts, prefilled, penalties, steps, what, batch_flags=None, n_slots=None, seed=5):
    """The sessions side by side in one batch on an engine with batch_flags (default: flags, default path), each checked
    after every call against its own NO_STREAM engine; the set and order of the slots in a call change from call to call."""
    eng = E.Engine(path, S, flags=flags if batch_flags is None else batch_flags)
    batch = eng.batch(n_slots or len(prompts))
    refs = [nostream(path, S, flags) for _ in prompts]
    sess = [Session(batch, i, refs[i], prompts[i], penalties[i], S, prefilled[i]) for i in range(len(prompts))]
    rng = np.random.default_rng(seed)
    done = {i: 0 for i in range(len(sess))}
    target = {i: len(prompts[i]) - 1 - sess[i].pos + steps for i in range(len(sess))}     # prompt positions left + steps
    while any(done[i] < target[i] for i in done):
        live = [i for i in done if done[i] < target[i]]
        pick = [i for i in live if rng.random() < 0.7] or live[:1]
        rng.shuffle(pick)
        step(batch, [sess[i] for i in pick], what)
        for i in pick:
            done[i] += 1
    for s in sess:
        s.check_cache(what)
    info = batch.info()
    for r in refs:
        r.close()
    eng.close()
    return info


def prompts_for(vocab, lens, seed=39):
    return [mf.teacher_tokens(n, vocab, seed + i)[:n] for i, n in enumerate(lens)]


def file_variants(name):
    return [(F32, 128), (Q80, 32), (Q80, 64), (Q80, 128), (Q80, 256), (Q4K, 128)]


# ------------------------------------------------------------------------------------------------ 1. bit identity
ID_CASES = [(n, q, g, x) for n in ("toy-nano", "toy-qwen3", "mini-qwen3", "toy-qwen2") for q, g in file_variants(n)
            for x in (False, True)]
LENS = (1, 7, 16, 23, 40)


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,exact", ID_CASES,
                         ids=[f"{c[0]}-{quant_id(c[1], c[2])}-{'exact' if c[3] else 'fast'}" for c in ID_CASES])
def test_batch_bit_identical_to_single_sessions(name, quant, gs, exact):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    flags = E.FLAG_EXACT if exact else 0
    info = run_sessions(path, 64, flags, prompts_for(spec.vocab, LENS), [False, True, False, True, True],
                        [PEN, 1.0, PEN, 1.0, PEN], 20, f"{name} {quant_id(quant, gs)} {'exact' if exact else 'fast'}")
    assert info["chunk"] == 16 and info["slots"] == 5, info


# ------------------------------------------------------------------------------------------------ 2. exact mode vs the oracle
ORACLE_CASES = [(n, q, g) for n in ("toy-nano", "toy-qwen3", "mini-qwen3", "toy-qwen2") for q, g in file_variants(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", ORACLE_CASES, ids=[f"{c[0]}-{quant_id(c[1], c[2])}" for c in ORACLE_CASES])
def test_exact_batch_equals_strict_reference(name, quant, gs):
    from oracle import bindings as ob
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = 64
    eng = E.Engine(path, S, flags=E.FLAG_EXACT)
    batch = eng.batch(3)
    lens = (37, 5, 20)
    toks = prompts_for(spec.vocab, [n + 1 for n in lens])
    for slot in (0, 2):
        batch.prefill(slot, toks[slot], 0, lens[slot])
    for p in range(lens[1]):                                  # slot 1 token by token, in passes shared with nothing
        batch.next_greedy([1], [toks[1]], [p], [1.0])
    batch.next_greedy([2, 0, 1], [toks[2], toks[0], toks[1]], [lens[2], lens[0], lens[1]], [1.0, 1.0, 1.0])
    for slot, n in enumerate(lens):
        o = ob.NanoOracle(path, S)
        for p in range(n):
            o.forward(int(toks[slot][p]), p)
        want = o.forward(int(toks[slot][n]), n)
        ok, ov = (a.copy() for a in o.kv())
        o.close()
        k, v = slot_kv(batch, slot, n + 1)
        assert_bits_equal(k, ok[:, : n + 1], f"slot {slot}: K rows vs the oracle")
        assert_bits_equal(v, ov[:, : n + 1], f"slot {slot}: V rows vs the oracle")
        assert_bits_equal(batch.logits(slot), want, f"slot {slot}: logits at {n} vs the oracle")
    eng.close()


# ------------------------------------------------------------------------------------------------ 3. attention kernels
ATTN_WANT = {"kvm1-nano": "fast<1>", "kvm4-qwen3-hd64": "fast<4>", "kvm4-qwen3-hd128": "fast<4>", "kvm8-qwen3": "fast<8>",
             "kvm3-qwen3": "generic", "kvm5-qwen3": "generic", "kvm7-nano": "generic", "mqa-qwen3": "generic",
             "hd96-qwen3": "generic", "hd192-nano": "generic", "hd512-qwen3": "generic"}
ATTN_CASES = ([(n, w, {}) for n, w in ATTN_WANT.items()] +
              [(n, "generic", {"NB200_GENERIC_ATTN": 1}) for n in ("kvm1-nano", "kvm4-qwen3-hd64", "kvm4-qwen3-hd128")])


@pytest.mark.gpu
@pytest.mark.parametrize("name,want,env", ATTN_CASES, ids=[c[0] + ("-generic-env" if c[2] else "") for c in ATTN_CASES])
def test_batch_attention_kernels(name, want, env, monkeypatch):
    """Every attention kernel, fast and exact: slots at positions spread over one to four splits share each pass."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S = 128
    for flags in (0, E.FLAG_EXACT):
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, str(v))
            eng = E.Engine(path, S, flags=flags)
            refs = [E.Engine(path, S, flags=flags | E.FLAG_NO_STREAM) for _ in range(4)]
        batch = eng.batch(4)
        kind = "exact" if flags else want
        assert batch.info()["attention"] == kind and refs[0].kernels()["attention"] in (None, kind), batch.info()
        prompts = prompts_for(spec.vocab, (100, 40, 3, 70))
        sess = [Session(batch, i, refs[i], prompts[i], [PEN, 1.0, PEN, 1.0][i], S, True) for i in range(4)]
        for _ in range(4):
            step(batch, sess, f"{name} {kind}")
        assert refs[0].kernels()["attention"] == kind
        for s in sess:
            s.check_cache(f"{name} {kind}")
        for r in refs:
            r.close()
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["long-nano", "long-qwen3"])
def test_long_slot_shares_passes_with_short_ones(name):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S = 1100
    run_sessions(path, S, 0, prompts_for(spec.vocab, (1041, 3, 30)), [True, False, True], [PEN, 1.0, PEN], 4, f"{name} long slot")


# ------------------------------------------------------------------------------------------------ 4. classifier shapes
CLS_CASES = ([("mv-nano", q, g) for q, g in [(F32, 128), (Q80, 32), (Q80, 256), (Q4K, 128)]] +
             [("toy-nano-untied", Q80, 64), ("toy-qwen3-untied", Q80, 128), ("v152k-qwen3-untied", Q80, 64)])


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", CLS_CASES, ids=[f"{c[0]}-{quant_id(c[1], c[2])}" for c in CLS_CASES])
@pytest.mark.parametrize("exact", [False, True], ids=["fast", "exact"])
def test_batch_classifier_shapes(name, quant, gs, exact):
    """mv-nano: V = 4099 ends in a partial row block, F = 5376 gives M < 16 for F32; the untied classifiers."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    info = run_sessions(path, 48, E.FLAG_EXACT if exact else 0, prompts_for(spec.vocab, (9, 1, 17)), [True, False, True],
                        [PEN, PEN, 1.0], 6, f"{name} {quant_id(quant, gs)}")
    if name == "mv-nano" and quant == F32:
        assert info["chunk"] < 16, info


@pytest.mark.gpu
@pytest.mark.parametrize("exact", [False, True], ids=["fast", "exact"])
def test_batch_argmax_ties_pick_first_copy(tie_model, exact):
    """Exactly tied classifier rows: every slot's greedy id is the first copy, as on the token path."""
    path, cls_of, firsts = tie_model
    spec = mf.PRESETS["v152k-qwen3-untied"]
    S = 24
    first_set = set(firsts.tolist())
    prompts = [np.random.default_rng(3 + i).integers(0, spec.vocab, 6).astype(np.uint32) for i in range(3)]
    flags = E.FLAG_EXACT if exact else 0
    eng = E.Engine(path, S, flags=flags)
    batch = eng.batch(3)
    refs = [nostream(path, S, flags) for _ in range(3)]
    sess = [Session(batch, i, refs[i], prompts[i], 1.0, S, i != 1) for i in range(3)]
    for _ in range(10):
        got = step(batch, sess, "ties")
        for s, g in zip(sess, got):
            if s.pos > len(s.prompt):
                assert g in first_set, f"slot {s.slot}: id {g} is a later copy of class {cls_of[g]}"
    for r in refs:
        r.close()
    eng.close()


# ------------------------------------------------------------------------------------------------ 5. pass shapes
@pytest.mark.gpu
def test_pass_shapes():
    """n = 1, M - 1, M, M + 1 and n_slots > M (two passes per call); then a slot reused for a new session over stale rows."""
    spec = mf.PRESETS["toy-qwen3"]
    path = mf.cached_model(spec, Q80, 64)
    S = 64
    eng = E.Engine(path, S)
    batch = eng.batch(20)
    M = batch.info()["chunk"]
    assert M == 16
    refs = [nostream(path, S) for _ in range(20)]
    prompts = prompts_for(spec.vocab, [2 + (i * 7) % 19 for i in range(20)])
    sess = [Session(batch, i, refs[i], prompts[i], PEN if i % 2 else 1.0, S, i % 3 != 0) for i in range(20)]
    order = list(range(20))[::-1]
    for n in (1, M - 1, M, M + 1, 20, 20):
        step(batch, [sess[i] for i in order[:n]], f"n={n}")
        order = order[3:] + order[:3]
    for s in sess:
        s.check_cache("pass shapes")
    # slot 4 starts a new, shorter session over the longer one's rows (prefilled), slot 7 token by token
    for slot, pre in ((4, True), (7, False)):
        refs[slot].close()
        refs[slot] = nostream(path, S)
        sess[slot] = Session(batch, slot, refs[slot], prompts_for(spec.vocab, [5], 77 + slot)[0], PEN, S, pre)
    for _ in range(8):
        step(batch, [sess[4], sess[7], sess[0]], "reused slot")
    for slot in (4, 7):
        sess[slot].check_cache("reused slot")
    for r in refs:
        r.close()
    eng.close()


# ------------------------------------------------------------------------------------------------ 6. BASELINE shapes
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,nses", [("nano-168m", Q80, 128, 16), ("qwen3-0.6b", Q4K, 128, 4)])
def test_batch_baseline_shapes(name, quant, gs, nses):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = 64
    eng = E.Engine(path, S)
    batch = eng.batch(nses)
    ref = nostream(path, S)
    prompts = prompts_for(spec.vocab, [16] * nses)
    ids = [np.zeros(S + 1, np.uint32) for _ in range(nses)]
    for i in range(nses):
        ids[i][:16] = prompts[i]
        batch.prefill(i, ids[i], 0, 15)
    pos = 15
    for _ in range(3):
        got = batch.next_greedy(list(range(nses)), ids, [pos] * nses, [PEN] * nses)
        for i in range(nses):
            ids[i][pos + 1] = got[i]
        pos += 1
    for i in range(nses):                        # one NO_STREAM engine replays every session in turn
        ref.prefill(ids[i], 0, 15)
        for p in range(15, pos):
            assert ref.next_greedy(ids[i], p, 0, PEN) == int(ids[i][p + 1]), f"{name} session {i} pos {p}"
        assert_bits_equal(batch.logits(i), ref.logits(), f"{name} session {i}: logits at {pos - 1}")
        if i in (0, nses - 1):
            k, v = slot_kv(batch, i, pos)
            rk, rv = engine_kv(ref, pos)
            assert_bits_equal(k, rk, f"{name} session {i}: K rows"); assert_bits_equal(v, rv, f"{name} session {i}: V rows")
    ref.close(); eng.close()


# ------------------------------------------------------------------------------------------------ 7. isolation
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", [("toy-nano", Q80, 64), ("toy-qwen3", Q4K, 128)])
def test_engine_session_untouched_by_batch(name, quant, gs):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S, P = 48, 12
    toks = mf.teacher_tokens(S, spec.vocab)

    def run(eng, batch):
        ids = np.zeros(S + 1, np.uint32); ids[:P] = toks[:P]
        out, logits = [], []
        other = prompts_for(spec.vocab, [S], 90)[0]
        for pos in range(S - 1):
            ids[pos + 1] = eng.next_greedy(ids, pos, 1 if pos < P - 1 else 0, PEN)
            logits.append(eng.logits())
            if batch is not None:
                batch.next_greedy([pos % 2], [other], [pos // 2], [PEN])
                if pos == 20:
                    batch.prefill(1, other, 0, 30)
        cfg = E.Config()
        E._check(E.lib().nb200_get_config(eng.h, E.C.byref(cfg)))
        return ids, np.stack(logits), engine_kv(eng, S - 1), list(cfg.reserved)[3:7]

    alone = E.Engine(path, S)
    want = run(alone, None)
    alone.close()
    eng = E.Engine(path, S)
    batch = eng.batch(2)
    got = run(eng, batch)
    assert got[3] == want[3], (got[3], want[3])        # nb200_config.reserved[3..6]
    assert got[0].tolist() == want[0].tolist()
    assert_bits_equal(got[1], want[1], "the engine's logits")
    assert_bits_equal(got[2][0], want[2][0], "the engine's K rows"); assert_bits_equal(got[2][1], want[2][1], "the engine's V rows")
    eng.close()
    assert batch.h is None                       # Engine.close closed its batch first


# ------------------------------------------------------------------------------------------------ 8. refusals
@pytest.mark.gpu
def test_batch_refusals():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    S = 48                                               # below block_size 64: the limit is max_seq_len
    eng = nostream(path, S)
    with pytest.raises(E.NB200Error, match="at least one slot"):
        eng.batch(0)
    batch = eng.batch(3)
    toks = [mf.teacher_tokens(S + 1, spec.vocab, 50 + i) for i in range(3)]
    batch.prefill(0, toks[0], 0, 20)
    batch.prefill(1, toks[1], 0, 10)
    batch.next_greedy([0, 1], toks[:2], [20, 10], [PEN, PEN])

    def state():
        return [slot_kv(batch, s, S) for s in range(3)] + [batch.logits(s) for s in range(3)]
    before = state()
    bad = toks[0].copy(); bad[5] = spec.vocab
    bad_now = toks[0].copy(); bad_now[21] = spec.vocab
    cases = [
        (lambda: batch.next_greedy([], [], [], []), "no entries"),
        (lambda: batch.next_greedy([3], toks[:1], [21], [1.0]), "slot 3"),
        (lambda: batch.next_greedy([0, 0], toks[:2], [21, 11], [1.0, 1.0]), "twice"),
        (lambda: batch.next_greedy([0, 1], toks[:2], [21, S], [1.0, 1.0]), "past"),
        (lambda: batch.next_greedy([1, 0], [toks[1], bad_now], [11, 21], [1.0, 1.0]), "out of range"),
        (lambda: batch.next_greedy([1, 0], [toks[1], bad], [11, 21], [1.0, PEN]), "out of range"),
        (lambda: batch.prefill(3, toks[0], 0, 4), "slot 3"),
        (lambda: batch.prefill(2, toks[0], 0, 0), "empty"),
        (lambda: batch.prefill(2, toks[0], 40, 9), "past"),
        (lambda: batch.prefill(2, bad, 0, 8), "out of range"),
    ]
    for fn, msg in cases:
        with pytest.raises(E.NB200Error, match=msg):
            fn()
        after = state()
        for a, b in zip(before, after):
            if isinstance(a, tuple):
                assert_bits_equal(a[0], b[0], f"K rows after refusing '{msg}'"); assert_bits_equal(a[1], b[1], f"V rows after '{msg}'")
            else:
                assert_bits_equal(a, b, f"logits after refusing '{msg}'")
    batch.prefill(2, toks[2], 40, 8)                     # exactly up to the limit is accepted
    batch.next_greedy([2], toks[2:], [S - 1], [1.0])
    # an active LoRA plug-in: refused at every call, also when it is enabled after the batch was created
    eng.lora_load(mf.write_lora(spec))
    for fn in (lambda: batch.next_greedy([0], toks[:1], [21], [1.0]), lambda: batch.prefill(0, toks[0], 0, 4), lambda: eng.batch(1)):
        with pytest.raises(E.NB200Error, match="LoRA"):
            fn()
    k, v = slot_kv(batch, 0, S)
    assert_bits_equal(k, before[0][0], "K rows after refusing LoRA"); assert_bits_equal(v, before[0][1], "V rows after refusing LoRA")
    eng.lora_enable(False)
    batch.next_greedy([0], toks[:1], [21], [1.0])
    eng.close()


@pytest.mark.gpu
@pytest.mark.skipif(E.device_count() < 2, reason="tensor parallelism needs 2 GPUs")
def test_batch_refuses_tensor_parallel():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    g = E.TpGroup(path, 32, 2)
    for r in g.ranks:
        with pytest.raises(E.NB200Error, match="tensor-parallel"):
            r.batch(2)
    g.close()


# ------------------------------------------------------------------------------------------------ 9. launch count
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 16, 17])
def test_batch_launch_count(n):
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    eng = E.Engine(path, 64)
    batch = eng.batch(17)
    toks = [mf.teacher_tokens(64, spec.vocab, 60 + i) for i in range(n)]
    before = eng.launches
    batch.next_greedy(list(range(n)), toks, [3] * n, [1.0] * n)        # penalty 1.0: no seen-set update
    got = eng.launches - before
    passes = -(-n // batch.info()["chunk"])
    assert got == passes * (1 + 5 * spec.n_layer + 2), got      # embed; QKV, attention, O, W1|W3, W2 per layer; classifier, argmax
    eng.close()


# ------------------------------------------------------------------------------------------------ CPU: stack frames
def test_batch_kernels_have_no_stack_frame():
    """Every k_batch_* kernel keeps its state in registers.  The one exception is allowed only where the token path's own
    attention body has a frame (k_attention_fast<8>, wrapped by k_batch_attention_fast<8>): no larger than it."""
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", nb_build.ENGINE_SO],
                         capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    stack = {}
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            st = re.search(r"STACK:(\d+)", lines[i + 1])
            stack[m.group(1)] = int(st.group(1)) if st else 0
    batch = {f: s for f, s in stack.items() if "k_batch_" in f}
    # matvec: Q80 (4 group sizes) / F32 / Q4K / exact F32 x {QKV, classifier}; attention fast<1|2|4|8> / generic / exact; argmax
    assert len(batch) == 21, sorted(batch)
    token_fast8 = [s for f, s in stack.items() if re.search(r"16k_attention_fastILi8ELb0E", f)]
    assert len(token_fast8) == 1
    bad = {}
    for f, s in batch.items():
        allowed = token_fast8[0] if re.search(r"22k_batch_attention_fastILi8EE", f) else 0
        if s > allowed:
            bad[f] = s
    assert not bad, f"stack bytes per thread: {bad}"
