"""Batched speculative greedy decoding (nb200_batch_verify_greedy).

Entry i of a call must do in its slot exactly what nb200_verify_greedy does on an engine created with the same flags plus
NB200_FLAG_NO_STREAM running that session alone: the same accepted count, corrected ids, logits and whole K / V cache (the rows
past the accepted ones restored), whatever the packing of the entries into passes.  Each session here runs beside its own
NO_STREAM engine calling nb200_verify_greedy with the same drafts.  Covered here:
  * the toy shapes x F32 / Q80 (every group size) / Q4K x exact / fast at penalties 1.0 and 1.3: four sessions of different
    prompt lengths; drafts all correct, wrong at index k, first wrong, random, recurring; n_pos sums below M, exactly M, above M
    (two, three and four passes), an entry of n_pos = M alone, n_pos = 1 entries; a rewind over older rows; then
    Batch.next_greedy and Batch.next_sampled steps;
  * n_pos = 1 everywhere against nb200_batch_next_greedy on a second batch; exact mode against the oracle; every attention
    kernel and a slot near position 1040 sharing passes with short ones; penalty 50 with recurring drafts; classifier ties;
  * the engine's own session and the slots not in a call untouched; refusals; launch counts;
  * (CPU) the new kernels exist and have no stack frame and no local memory.
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


def nostream(path, S, flags=0):
    return E.Engine(path, S, flags=flags | E.FLAG_NO_STREAM)


def limit(eng):
    return min(eng.max_seq_len, eng.block_size)


def engine_kv(eng, S):
    k = np.stack([np.stack([eng.read(E.F_KROW, eng.kv_dim, l, p) for p in range(S)]) for l in range(eng.n_layer)])
    v = np.stack([np.stack([eng.read(E.F_VROW, eng.kv_dim, l, p) for p in range(S)]) for l in range(eng.n_layer)])
    return k, v


def slot_kv(batch, slot, S):
    eng = batch.engine
    k = np.stack([np.stack([batch.read(E.F_KROW, eng.kv_dim, slot, l, p) for p in range(S)]) for l in range(eng.n_layer)])
    v = np.stack([np.stack([batch.read(E.F_VROW, eng.kv_dim, slot, l, p) for p in range(S)]) for l in range(eng.n_layer)])
    return k, v


def truth(T, prompt, lim, penalty):
    """The greedy session of `prompt` on the NO_STREAM engine T: ids[0..lim] (prompt teacher-forced)."""
    ids = np.zeros(lim + 1, np.uint32)
    P = len(prompt)
    ids[:P] = prompt
    if P > 1:
        T.prefill(ids, 0, P - 1)
    for p in range(P - 1, lim):
        ids[p + 1] = T.next_greedy(ids, p, 0, penalty)
    return ids


def drafts_for(tr, pos, n, form, rng, vocab):
    d = tr[pos + 1: pos + n].copy()
    if n == 1:
        return d
    if form == "first":
        d[0] = (d[0] + 1) % vocab
    elif isinstance(form, int):           # wrong at index form
        d[min(form, n - 2)] = (d[min(form, n - 2)] + 1 + rng.integers(vocab - 1)) % vocab
    elif form == "random":
        d = rng.integers(0, vocab, n - 1).astype(np.uint32)
    elif form == "recur":                 # the first draft again at every later index
        d[1:] = d[0]
    return d


class Sess:
    """One greedy session in a batch slot and, beside it, the same session on its own NO_STREAM engine R (verify calls there
    with the same drafts).  tr: the session's greedy ids, from the truth engine T."""

    def __init__(self, batch, slot, R, T, S, penalty, what):
        self.batch, self.slot, self.R, self.T, self.S, self.penalty, self.what = batch, slot, R, T, S, penalty, what
        self.lim = limit(R)

    def start(self, prompt):
        self.tr = truth(self.T, prompt, self.lim, self.penalty)
        self.pos = len(prompt) - 1
        if self.pos:
            self.batch.prefill(self.slot, self.tr, 0, self.pos)
            self.R.prefill(self.tr, 0, self.pos)

    def room(self, n):
        return max(1, min(n, self.lim - self.pos))


def verify_call(batch, plan, rng, what, check=True):
    """plan: [(session, n_pos, draft form)].  One batch call; every entry against its session's own engine."""
    plan = [(s, s.room(n), f) for s, n, f in plan]
    arrs, want = [], []
    for s, n, form in plan:
        d = drafts_for(s.tr, s.pos, n, form, rng, batch.engine.vocab)
        ids = s.tr.copy()
        ids[s.pos + 1: s.pos + n] = d
        arrs.append(ids)
        a = 0
        while a < n - 1 and d[a] == s.tr[s.pos + 1 + a]:
            a += 1
        want.append((a, d))
    pens = [s.penalty for s, _, _ in plan]
    got = batch.verify_greedy([s.slot for s, _, _ in plan], arrs, [s.pos for s, _, _ in plan], [n for _, n, _ in plan], pens)
    for (s, n, form), ids, (wa, d), a in zip(plan, arrs, want, got):
        tag = f"{what} {s.what} slot {s.slot} pos {s.pos} n {n} drafts {form}"
        ref = s.tr.copy()
        ref[s.pos + 1: s.pos + n] = d
        ra = s.R.verify_greedy(ref, s.pos, n, s.penalty)
        assert a == wa == ra, f"{tag}: accepted {a}, want {wa}, the engine's {ra}"
        assert ids.tolist() == ref.tolist(), f"{tag}: ids"
        assert ids[: s.pos + a + 2].tolist() == s.tr[: s.pos + a + 2].tolist(), f"{tag}: ids vs the greedy session"
        if check:
            assert_bits_equal(batch.logits(s.slot), s.R.logits(), f"{tag}: logits")
            k, v = slot_kv(batch, s.slot, s.S)
            rk, rv = engine_kv(s.R, s.S)
            assert_bits_equal(k, rk, f"{tag}: K cache")
            assert_bits_equal(v, rv, f"{tag}: V cache")
        s.pos += a + 1
    return got


def continue_steps(batch, sess, rng, what, greedy=2, sampled=2):
    """Batch.next_greedy, then Batch.next_sampled steps of every session, against its engine's next_greedy / next_sampled."""
    live = [s for s in sess if s.pos + greedy + sampled < s.lim]
    ids = {s.slot: s.tr.copy() for s in live}
    for _ in range(greedy):
        got = batch.next_greedy([s.slot for s in live], [ids[s.slot] for s in live], [s.pos for s in live], [s.penalty for s in live])
        for s, g in zip(live, got):
            want = s.R.next_greedy(ids[s.slot], s.pos, 0, s.penalty)
            assert g == want == ids[s.slot][s.pos + 1], f"{what} slot {s.slot}: next_greedy at {s.pos} after verify"
            assert_bits_equal(batch.logits(s.slot), s.R.logits(), f"{what} slot {s.slot}: logits of next_greedy at {s.pos}")
            s.pos += 1
    for _ in range(sampled):
        coins = rng.random(len(live)).astype(np.float32).tolist()
        got, _ = batch.next_sampled([s.slot for s in live], [ids[s.slot] for s in live], [s.pos for s in live],
                                    [s.penalty for s in live], [0.8] * len(live), [0.9] * len(live), coins)
        for s, g, c in zip(live, got, coins):
            want, _ = s.R.next_sampled(ids[s.slot], s.pos, s.penalty, 0.8, 0.9, c)
            assert g == want, f"{what} slot {s.slot}: next_sampled at {s.pos} after verify: {g} vs {want}"
            ids[s.slot][s.pos + 1] = g
            s.pos += 1


def make(path, S, flags, penalties, what, n_slots=None, batch_flags=None):
    eng = E.Engine(path, S, flags=flags if batch_flags is None else batch_flags)
    batch = eng.batch(n_slots or len(penalties))
    T = nostream(path, S, flags)
    sess = [Sess(batch, i, nostream(path, S, flags), T, S, p, what) for i, p in enumerate(penalties)]
    return eng, batch, T, sess


def close(eng, T, sess):
    for s in sess:
        s.R.close()
    T.close()
    eng.close()


def file_variants():
    return [(F32, 128), (Q80, 32), (Q80, 64), (Q80, 128), (Q80, 256), (Q4K, 128)]


# ------------------------------------------------------------------------------------------------ 1. bit identity
ID_CASES = [(n, q, g, x) for n in ("toy-nano", "toy-qwen3", "mini-qwen3", "toy-qwen2") for q, g in file_variants()
            for x in (False, True)]


def scenario(path, S, flags, penalty, vocab, what):
    eng, batch, T, sess = make(path, S, flags, [penalty] * 4, what)
    assert batch.info()["chunk"] == 16
    for s, P, seed in zip(sess, (1, 6, 12, 20), (39, 40, 41, 42)):
        s.start(mf.teacher_tokens(P, vocab, seed)[:P])
    s0, s1, s2, s3 = sess
    rng = np.random.default_rng(17)
    plans = [
        [(s0, 4, "correct"), (s1, 4, 2), (s2, 3, "first"), (s3, 1, None)],                                      # 12 rows < M
        [(s0, 4, "recur"), (s1, 4, "correct"), (s2, 4, 1), (s3, 4, "first")],                                  # exactly M
        [(s3, 8, "correct"), (s1, 6, 3), (s0, 5, "random"), (s2, 7, "correct")],                               # two passes
        [(s2, 16, "correct")],                                                                                  # M alone
        [(s0, 1, None), (s1, 1, None), (s3, 1, None), (s2, 1, None)],                                          # n_pos = 1
        [(s0, 12, "correct"), (s1, 4, "recur"), (s2, 10, 6), (s3, 10, "correct")],                              # three passes
        [(s1, 10, "correct"), (s3, 10, 4), (s0, 7, "first"), (s2, 12, "random")],                               # four passes
    ]
    for k, plan in enumerate(plans):
        verify_call(batch, plan, rng, f"call {k}")
    # a new session in slot 1 over its older, longer rows: the rejected rows must come back as the old session wrote them
    s1.start(mf.teacher_tokens(12, vocab, 77)[:12])
    verify_call(batch, [(s1, 16, 3), (s0, 2, "correct")], rng, "rewind")
    verify_call(batch, [(s3, 2, "random"), (s1, 15, "correct")], rng, "rewind")
    continue_steps(batch, sess, rng, what)
    close(eng, T, sess)


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,exact", ID_CASES,
                         ids=[f"{c[0]}-{quant_id(c[1], c[2])}-{'exact' if c[3] else 'fast'}" for c in ID_CASES])
def test_batch_verify_bit_identical_to_verify_greedy(name, quant, gs, exact):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    for penalty in (1.0, PEN):
        scenario(path, 64, E.FLAG_EXACT if exact else 0, penalty, spec.vocab,
                 f"{name} {quant_id(quant, gs)} {'exact' if exact else 'fast'} penalty {penalty}")


# ------------------------------------------------------------------------------------------------ 2. n_pos = 1 everywhere
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,exact", [("toy-qwen3", Q80, 64, False), ("toy-nano", Q4K, 128, False),
                                                 ("mini-qwen3", F32, 128, True)])
def test_single_position_entries_equal_next_greedy(name, quant, gs, exact):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S, n = 48, 20                                             # 20 slots: two passes per call
    eng = E.Engine(path, S, flags=E.FLAG_EXACT if exact else 0)
    A, B = eng.batch(n), eng.batch(n)
    ids = [mf.teacher_tokens(S + 1, spec.vocab, 5 + i) for i in range(n)]
    pens = [PEN if i % 2 else 1.0 for i in range(n)]
    pos = [i % 7 if i % 3 else 0 for i in range(n)]
    for i in range(n):
        if pos[i]:
            A.prefill(i, ids[i], 0, pos[i])
            B.prefill(i, ids[i], 0, pos[i])
    for step in range(6):
        order = [(i * 7 + step) % n for i in range(n)][: n - step]
        ga = [x.copy() for x in ids]
        acc = A.verify_greedy(order, [ga[i] for i in order], [pos[i] for i in order], [1] * len(order), [pens[i] for i in order])
        gb = B.next_greedy(order, [ids[i] for i in order], [pos[i] for i in order], [pens[i] for i in order])
        assert acc == [0] * len(order)
        for i, g in zip(order, gb):
            assert int(ga[i][pos[i] + 1]) == g, f"slot {i} pos {pos[i]}"
            ids[i][pos[i] + 1] = g
            assert_bits_equal(A.logits(i), B.logits(i), f"slot {i} pos {pos[i]}: logits")
            pos[i] += 1
    for i in (0, 7, n - 1):
        ka, va = slot_kv(A, i, S)
        kb, vb = slot_kv(B, i, S)
        assert_bits_equal(ka, kb, f"slot {i}: K cache"); assert_bits_equal(va, vb, f"slot {i}: V cache")
    eng.close()


# ------------------------------------------------------------------------------------------------ 3. exact mode vs the oracle
ORACLE_CASES = [("toy-qwen3", F32, 128), ("toy-nano", Q80, 64), ("mini-qwen3", Q80, 128), ("toy-qwen2", Q4K, 128)]


def penalised(raw, ids, pos, penalty):
    out = raw.copy()
    if penalty != 1.0:
        for i in set(int(t) for t in ids[:pos]):
            out[i] = np.float32(out[i]) / np.float32(penalty)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", ORACLE_CASES, ids=[f"{c[0]}-{quant_id(c[1], c[2])}" for c in ORACLE_CASES])
@pytest.mark.parametrize("penalty", [1.0, PEN])
def test_exact_batch_verify_equals_oracle(name, quant, gs, penalty):
    from oracle import bindings as ob
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S, P = 48, 9
    o = ob.NanoOracle(path, S)
    tr = np.zeros(S + 1, np.uint32)
    tr[:P] = mf.teacher_tokens(P, spec.vocab, 21)
    want_logits = {}
    for p in range(S - 1):
        raw = o.forward(int(tr[p]), p)
        if p >= P - 1:
            want_logits[p] = penalised(raw, tr, p, penalty)
            tr[p + 1] = int(np.argmax(want_logits[p]))
    ok, ov = (a.copy() for a in o.kv())
    o.close()
    eng = E.Engine(path, S, flags=E.FLAG_EXACT)
    batch = eng.batch(2)
    other = mf.teacher_tokens(S + 1, spec.vocab, 3)
    batch.prefill(0, tr, 0, P - 1)
    batch.prefill(1, other, 0, 4)
    pos, opos = P - 1, 4
    rng = np.random.default_rng(2)
    for n, form in ((16, "correct"), (10, 6), (5, "first"), (15, "correct")):
        ids = tr.copy()
        ids[pos + 1: pos + n] = drafts_for(tr, pos, n, form, rng, spec.vocab)
        o_ids = other.copy()
        oa, a = batch.verify_greedy([1, 0], [o_ids, ids], [opos, pos], [16 - n + 1, n], [1.0, penalty])
        assert ids[: pos + a + 2].tolist() == tr[: pos + a + 2].tolist(), f"ids vs the oracle, verify at {pos}"
        assert_bits_equal(batch.logits(0), want_logits[pos + a], f"logits at {pos + a} vs the oracle")
        pos += a + 1
        opos += oa + 1
    k, v = slot_kv(batch, 0, pos)
    assert_bits_equal(k, ok[:, :pos], "K rows vs the oracle")
    assert_bits_equal(v, ov[:, :pos], "V rows vs the oracle")
    eng.close()


# ------------------------------------------------------------------------------------------------ 4. attention kernels
ATTN_WANT = {"kvm1-nano": "fast<1>", "kvm4-qwen3-hd64": "fast<4>", "kvm8-qwen3": "fast<8>", "kvm3-qwen3": "generic",
             "mqa-qwen3": "generic", "hd96-qwen3": "generic", "hd192-nano": "generic"}
ATTN_CASES = ([(n, w, {}) for n, w in ATTN_WANT.items()] +
              [(n, "generic", {"NB200_GENERIC_ATTN": 1}) for n in ("kvm1-nano", "kvm4-qwen3-hd64")])


@pytest.mark.gpu
@pytest.mark.parametrize("name,want,env", ATTN_CASES, ids=[c[0] + ("-generic-env" if c[2] else "") for c in ATTN_CASES])
def test_batch_verify_attention_kernels(name, want, env, monkeypatch):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S = 96
    for flags in (0, E.FLAG_EXACT):
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, str(v))
            eng, batch, T, sess = make(path, S, flags, [PEN, 1.0, PEN], f"{name}")
        kind = "exact" if flags else want
        assert batch.info()["attention"] == kind, batch.info()
        for s, P, seed in zip(sess, (70, 3, 40), (4, 5, 6)):
            s.start(mf.teacher_tokens(P, spec.vocab, seed)[:P])
        rng = np.random.default_rng(1)
        verify_call(batch, [(sess[0], 8, 5), (sess[1], 5, "correct"), (sess[2], 3, "correct")], rng, kind)
        verify_call(batch, [(sess[2], 6, 2), (sess[0], 16, "correct"), (sess[1], 9, "correct")], rng, kind)
        assert sess[0].R.prefill_info()["attention"] == kind
        continue_steps(batch, sess, rng, kind, sampled=0)
        close(eng, T, sess)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["long-nano", "long-qwen3"])
def test_batch_verify_near_position_1040(name):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S = 1072
    eng, batch, T, sess = make(path, S, 0, [PEN, 1.0, PEN], f"{name} long")
    for s, P, seed in zip(sess, (1036, 3, 30), (4, 5, 6)):
        s.start(mf.teacher_tokens(P, spec.vocab, seed)[:P])
    rng = np.random.default_rng(3)
    for plan in ([(sess[1], 4, "correct"), (sess[0], 8, "correct"), (sess[2], 4, 1)],
                 [(sess[0], 16, 3), (sess[2], 5, "correct"), (sess[1], 1, None)]):
        verify_call(batch, plan, rng, "long", check=False)
        for s in sess:
            assert_bits_equal(batch.logits(s.slot), s.R.logits(), f"{name} slot {s.slot}: logits")
    lo = 1030
    for l in range(eng.n_layer):
        for p in range(lo, S):
            for f in (E.F_KROW, E.F_VROW):
                assert_bits_equal(batch.read(f, eng.kv_dim, 0, l, p), sess[0].R.read(f, eng.kv_dim, l, p), f"{name}: layer {l} row {p}")
    for s in sess[1:]:
        k, v = slot_kv(batch, s.slot, 48)
        rk, rv = engine_kv(s.R, 48)
        assert_bits_equal(k, rk, f"{name} slot {s.slot}: K rows"); assert_bits_equal(v, rv, f"{name} slot {s.slot}: V rows")
    continue_steps(batch, sess, rng, "long", sampled=0)
    close(eng, T, sess)


# ------------------------------------------------------------------------------------------------ 5. penalty through drafts, ties
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", [("toy-nano", Q80, 64), ("toy-qwen3", Q4K, 128), ("mini-qwen3", F32, 128)])
@pytest.mark.parametrize("exact", [False, True], ids=["fast", "exact"])
def test_batch_verify_penalty_50(name, quant, gs, exact):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = 48
    eng, batch, T, sess = make(path, S, E.FLAG_EXACT if exact else 0, [50.0, 50.0, 1.0], f"{name} penalty 50")
    for s, P, seed in zip(sess, (6, 9, 4), (8, 9, 10)):
        s.start(mf.teacher_tokens(P, spec.vocab, seed)[:P])
    rng = np.random.default_rng(4)
    for plan in ([(sess[0], 8, "recur"), (sess[1], 8, "recur")], [(sess[0], 16, "correct")],
                 [(sess[1], 9, "recur"), (sess[2], 4, "recur"), (sess[0], 3, "recur")], [(sess[0], 10, 2), (sess[1], 6, "correct")]):
        verify_call(batch, plan, rng, "penalty 50")
    close(eng, T, sess)


@pytest.mark.gpu
@pytest.mark.parametrize("exact", [False, True], ids=["fast", "exact"])
def test_batch_verify_ties_pick_first_copy(tie_model, exact):
    path, cls_of, firsts = tie_model
    spec = mf.PRESETS["v152k-qwen3-untied"]
    S = 40
    eng, batch, T, sess = make(path, S, E.FLAG_EXACT if exact else 0, [1.0, 1.0], "ties")
    for i, s in enumerate(sess):
        s.start(np.random.default_rng(3 + i).integers(0, spec.vocab, 6).astype(np.uint32))
    rng = np.random.default_rng(5)
    for plan in ([(sess[0], 8, "correct"), (sess[1], 8, 4)], [(sess[1], 16, "correct")], [(sess[0], 8, "first"), (sess[1], 4, "correct")]):
        verify_call(batch, plan, rng, "ties")
    first_set = set(firsts.tolist())
    for s in sess:
        assert all(int(i) in first_set for i in s.tr[6: s.pos + 1]), "a greedy id is a later copy of its class"
    close(eng, T, sess)


# ------------------------------------------------------------------------------------------------ 6. isolation
@pytest.mark.gpu
def test_batch_verify_leaves_engine_and_other_slots_alone():
    spec = mf.PRESETS["toy-qwen3"]
    path = mf.cached_model(spec, Q80, 64)
    S = 48
    eng = E.Engine(path, S)
    batch = eng.batch(3)
    toks = [mf.teacher_tokens(S + 1, spec.vocab, 30 + i) for i in range(4)]
    for p in range(12):                                       # the engine's own session
        eng.next_greedy(toks[3], p, 0, PEN)
    batch.prefill(2, toks[2], 0, 10)
    batch.next_greedy([2], [toks[2]], [10], [PEN])
    cfg = E.Config()

    def engine_state():
        E._check(E.lib().nb200_get_config(eng.h, E.C.byref(cfg)))
        return engine_kv(eng, S) + (eng.logits(), list(cfg.reserved)[3:7])

    def slot2():
        return slot_kv(batch, 2, S) + (batch.logits(2),)
    e0, s0 = engine_state(), slot2()
    for pos in (0, 16):
        batch.verify_greedy([1, 0], [toks[1].copy(), toks[0].copy()], [pos, pos + 3], [16, 9], [PEN, 1.0])
    e1, s1 = engine_state(), slot2()
    assert e1[3] == e0[3], (e1[3], e0[3])
    for a, b in zip(e0[:3], e1[:3]):
        assert_bits_equal(a, b, "the engine's own state")
    for a, b in zip(s0, s1):
        assert_bits_equal(a, b, "slot 2, not in the calls")
    eng.close()


# ------------------------------------------------------------------------------------------------ 7. refusals
@pytest.mark.gpu
def test_batch_verify_refusals():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    S = 48                                                    # below block_size 64: the limit is max_seq_len
    eng = nostream(path, S)
    batch = eng.batch(3)
    toks = [mf.teacher_tokens(S + 20, spec.vocab, 50 + i) for i in range(3)]
    batch.prefill(0, toks[0], 0, 20)
    batch.prefill(1, toks[1], 0, 10)
    batch.verify_greedy([0, 1], [toks[0].copy(), toks[1].copy()], [20, 10], [4, 3], [PEN, PEN])

    def state():
        return [slot_kv(batch, s, S) for s in range(3)] + [batch.logits(s) for s in range(3)]
    before = state()
    bad_draft = toks[0].copy(); bad_draft[24] = spec.vocab
    bad_past = toks[0].copy(); bad_past[3] = spec.vocab
    t0, t1 = toks[0], toks[1]
    cases = [
        (([], [], [], [], []), "no entries"),
        (([3], [t0], [22], [2], [1.0]), "slot 3"),
        (([0, 0], [t0, t1], [22, 11], [2, 2], [1.0, 1.0]), "twice"),
        (([1, 0], [t1, t0], [11, 22], [2, 0], [1.0, 1.0]), "1 .. M = 16"),
        (([1, 0], [t1, t0], [11, 22], [2, 17], [1.0, 1.0]), "1 .. M = 16"),
        (([1, 0], [t1, t0], [11, 40], [2, 9], [1.0, 1.0]), "past"),
        (([1, 0], [t1, t0], [11, 48], [2, 1], [1.0, 1.0]), "past"),
        (([1, 0], [t1, bad_draft], [11, 22], [2, 4], [1.0, 1.0]), "out of range"),
        (([1, 0], [t1, bad_past], [11, 22], [2, 4], [1.0, PEN]), "out of range"),
    ]
    for args, msg in cases:
        arrs = [a.copy() for a in args[1]]
        with pytest.raises(E.NB200Error, match=re.escape(msg)):
            batch.verify_greedy(args[0], arrs, *args[2:])
        for a, b in zip(arrs, args[1]):
            assert a.tolist() == b.tolist(), f"ids after refusing '{msg}'"
        after = state()
        for a, b in zip(before, after):
            if isinstance(a, tuple):
                assert_bits_equal(a[0], b[0], f"K rows after refusing '{msg}'"); assert_bits_equal(a[1], b[1], f"V rows after '{msg}'")
            else:
                assert_bits_equal(a, b, f"logits after refusing '{msg}'")
    batch.verify_greedy([2], [bad_past.copy()], [40], [8], [1.0])     # penalty 1 reads no earlier ids; exactly up to the limit
    eng.lora_load(mf.write_lora(spec))
    with pytest.raises(E.NB200Error, match="LoRA"):
        batch.verify_greedy([0], [t0.copy()], [22], [4], [1.0])
    eng.lora_enable(False)
    batch.verify_greedy([0], [t0.copy()], [22], [4], [1.0])
    eng.close()


# ------------------------------------------------------------------------------------------------ 8. launch counts
@pytest.mark.gpu
def test_batch_verify_launch_counts():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    L = spec.n_layer
    eng = E.Engine(path, 64)
    batch = eng.batch(4)
    toks = [mf.teacher_tokens(64, spec.vocab, 60 + i) for i in range(4)]
    chunk = 1 + 6 * L + 3
    cases = [
        # (n_pos, penalties, launches): per pass the chunk, classifier, argmax, accept; + save where a pass drafts; + seen rows
        # where it has a penalty != 1; + one seen-set update per penalised slot with new ids
        ([1, 1], [1.0, 1.0], chunk),
        ([8, 8], [1.0, 1.0], chunk + 1),
        ([8, 1], [PEN, 1.0], chunk + 1 + 1 + 1),
        ([8, 1], [PEN, 1.0], chunk + 1 + 1),                  # slot 0's seen set already holds ids[0..5)
        ([16, 1, 1, 1], [1.0, 1.0, 1.0, 1.0], 2 * chunk + 1),   # passes 16 | 1+1+1: the first drafts
        ([10, 7, 1, 16], [1.0, 1.0, 1.0, 1.0], 3 * chunk + 3),  # passes 10 | 7+1 | 16: each drafts
        ([12, 1, 1, 2], [1.0, PEN, 1.0, 1.0], chunk + 1 + 1 + 1),
    ]
    for n_pos, pens, want in cases:
        before = eng.launches
        batch.verify_greedy(list(range(len(n_pos))), [t.copy() for t in toks[: len(n_pos)]], [5] * len(n_pos), n_pos, pens)
        assert eng.launches - before == want, (n_pos, pens, eng.launches - before, want)
    eng.close()


# ------------------------------------------------------------------------------------------------ CPU: the new kernels
def test_batch_verify_kernels_have_no_stack_frame():
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", nb_build.ENGINE_SO],
                         capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = {}
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m and "k_vbatch_" in m.group(1):
            found[m.group(1)] = lines[i + 1]
    names = sorted(re.search(r"k_vbatch_\w+?(?=E|N)", f).group(0) for f in found)
    assert names == ["k_vbatch_accept", "k_vbatch_krow", "k_vbatch_save", "k_vbatch_seen"], names
    for f, res in found.items():
        st = re.search(r"STACK:(\d+)", res)
        loc = re.search(r"LOCAL:(\d+)", res)
        assert st and int(st.group(1)) == 0, (f, res)
        assert loc and int(loc.group(1)) == 0, (f, res)
