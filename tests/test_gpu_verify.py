"""Speculative greedy decoding (nb200_verify_greedy, nb200_decode_lookup).

A verify pass runs the consumed id and n-1 drafted ids as one prefill chunk, then the batch's classifier and argmax on every
position, so the greedy id at each position must equal, bit for bit, what nb200_next_greedy returns there on an engine created
with the same flags plus NB200_FLAG_NO_STREAM; the accepted count, the correction, the logits and the whole K / V cache
(rejected rows restored) must then be what that engine has after stepping through the accepted positions.  Covered here:
  * the toy shapes x F32 / Q80 (every group size) / Q4K x exact / fast at penalties 1.0 and 1.3: drafts from a reference
    session, all correct, wrong at index k, first wrong, random, recurring; n = 1, M-1, M at pos 0, mid-context and limit-n,
    a rewind over an older session's rows; three more next_greedy steps afterwards;
  * penalty 50 with recurring drafted ids; exact classifier ties; exact mode against the oracle; every attention kernel and
    a pass near position 1040;
  * the prompt-lookup driver against nb200_decode_greedy (ids, cache, the drafting rule's counts), also on a streaming engine;
  * refusals; launch counts; (CPU) the seen-row kernel has no stack frame and no local memory.
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


def whole_kv(eng, S):
    """The whole K and V cache [L][S][kv_dim], written rows or not."""
    k = np.stack([np.stack([eng.read(E.F_KROW, eng.kv_dim, l, p) for p in range(S)]) for l in range(eng.n_layer)])
    v = np.stack([np.stack([eng.read(E.F_VROW, eng.kv_dim, l, p) for p in range(S)]) for l in range(eng.n_layer)])
    return k, v


def assert_same_state(a, b, S, what):
    assert_bits_equal(a.logits(), b.logits(), f"{what}: logits")
    ka, va = whole_kv(a, S)
    kb, vb = whole_kv(b, S)
    assert_bits_equal(ka, kb, f"{what}: K cache")
    assert_bits_equal(va, vb, f"{what}: V cache")


def limit(eng):
    return min(eng.max_seq_len, eng.block_size)


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
        d[form] = (d[form] + 1 + rng.integers(vocab - 1)) % vocab
    elif form == "random":
        d = rng.integers(0, vocab, n - 1).astype(np.uint32)
    elif form == "recur":                 # the first draft again at every later index
        d[1:] = d[0]
    return d


class Pair:
    """The engine under test V (verify calls) and the reference R (NO_STREAM, nb200_next_greedy), kept in lock-step on one
    greedy session whose ids are `tr` (from the truth engine T)."""

    def __init__(self, V, R, T, S, penalty, what):
        self.V, self.R, self.T, self.S, self.penalty, self.what = V, R, T, S, penalty, what
        self.lim = limit(V)
        self.rng = np.random.default_rng(17)

    def start(self, prompt, upto):
        """A session of `prompt`, positions 0 .. upto-1 prefilled on both engines."""
        self.tr = truth(self.T, prompt, self.lim, self.penalty)
        if upto:
            self.V.prefill(self.tr, 0, upto)
            self.R.prefill(self.tr, 0, upto)
        self.pos = upto

    def verify(self, n, form, check=True):
        pos, tr = self.pos, self.tr
        d = drafts_for(tr, pos, n, form, self.rng, self.V.vocab)
        ids = tr.copy()
        ids[pos + 1: pos + n] = d
        want_a = 0
        while want_a < n - 1 and d[want_a] == tr[pos + 1 + want_a]:
            want_a += 1
        a = self.V.verify_greedy(ids, pos, n, self.penalty)
        what = f"{self.what} verify pos {pos} n {n} drafts {form}"
        assert a == want_a, f"{what}: accepted {a}, want {want_a}"
        assert ids[: pos + a + 2].tolist() == tr[: pos + a + 2].tolist(), f"{what}: ids"
        assert ids[pos + a + 2: pos + n].tolist() == d[a + 1:].tolist(), f"{what}: ids past the correction"
        ref = tr.copy()
        for p in range(pos, pos + a + 1):
            g = self.R.next_greedy(ref, p, 0, self.penalty)
            assert g == tr[p + 1], f"{what}: reference id at {p}"
        if check:
            assert_same_state(self.V, self.R, self.S, what)
        self.pos = pos + a + 1
        return a

    def continue_greedy(self, steps=3):
        ids = self.tr.copy()
        for p in range(self.pos, min(self.pos + steps, self.lim - 1)):
            gv = self.V.next_greedy(ids, p, 0, self.penalty)
            gr = self.R.next_greedy(ids, p, 0, self.penalty)
            assert gv == gr == ids[p + 1], f"{self.what}: next_greedy at {p} after verify: {gv} vs {gr}"
            assert_bits_equal(self.V.logits(), self.R.logits(), f"{self.what}: logits of next_greedy at {p} after verify")


def scenario(path, S, flags, penalty, vocab, what, prompt_seed=39):
    """pos 0 to the limit with every n and draft form, then a rewind onto the older rows; three greedy steps after each."""
    V, R, T = nostream(path, S, flags), nostream(path, S, flags), nostream(path, S, flags)
    pr = Pair(V, R, T, S, penalty, what)
    M = 16
    pr.start(mf.teacher_tokens(1, vocab, prompt_seed), 0)
    pr.verify(M, "correct")                   # pos 0, a = M - 1
    pr.verify(M - 1, 5)
    pr.verify(1, None)
    pr.verify(M, "first")
    pr.verify(M - 1, "random")
    pr.verify(8, 6)
    pr.verify(M, "recur")
    assert V.prefill_info()["chunk"] == M
    lim = pr.lim
    if pr.pos < lim - M:                      # prefill to limit - M
        pr.V.prefill(pr.tr, pr.pos, lim - M - pr.pos)
        pr.R.prefill(pr.tr, pr.pos, lim - M - pr.pos)
        pr.pos = lim - M
    pr.verify(lim - pr.pos, "correct")        # up to the limit: the bonus id lands at ids[limit]
    # a new session over the old one's rows: the rejected rows must come back as the old session wrote them
    prompt = mf.teacher_tokens(12, vocab, prompt_seed + 1)
    pr.start(prompt, 11)
    pr.verify(M, 3)
    pr.verify(M - 1, "correct")
    pr.continue_greedy()
    for e in (V, R, T):
        e.close()


def file_variants():
    return [(F32, 128), (Q80, 32), (Q80, 64), (Q80, 128), (Q80, 256), (Q4K, 128)]


# ------------------------------------------------------------------------------------------------ 1. verify, unit
ID_CASES = [(n, q, g, x) for n in ("toy-nano", "toy-qwen3", "mini-qwen3", "toy-qwen2") for q, g in file_variants()
            for x in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,exact", ID_CASES,
                         ids=[f"{c[0]}-{quant_id(c[1], c[2])}-{'exact' if c[3] else 'fast'}" for c in ID_CASES])
def test_verify_bit_identical_to_next_greedy(name, quant, gs, exact):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    for penalty in (1.0, PEN):
        scenario(path, 64, E.FLAG_EXACT if exact else 0, penalty, spec.vocab,
                 f"{name} {quant_id(quant, gs)} {'exact' if exact else 'fast'} penalty {penalty}")


# ------------------------------------------------------------------------------------------------ 2. penalty through drafts, ties
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", [("toy-nano", Q80, 64), ("toy-qwen3", Q4K, 128), ("mini-qwen3", F32, 128)])
@pytest.mark.parametrize("exact", [False, True], ids=["fast", "exact"])
def test_penalty_reads_each_positions_drafts(name, quant, gs, exact):
    """Penalty 50: a drafted id that recurs, or that the greedy id would repeat, decides the argmax of the later positions."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = 48
    flags = E.FLAG_EXACT if exact else 0
    V, R, T = nostream(path, S, flags), nostream(path, S, flags), nostream(path, S, flags)
    pr = Pair(V, R, T, S, 50.0, f"{name} penalty 50")
    pr.start(mf.teacher_tokens(6, spec.vocab, 8), 5)
    for n, form in ((16, "recur"), (16, "correct"), (9, "recur"), (16, 2)):
        pr.verify(n, form)
    # the unpenalised continuation as drafts: wherever it repeats an id, penalty 50 rejects it at that position only
    pos = pr.pos
    n = min(16, pr.lim - pos)
    ids = np.concatenate([pr.tr, np.zeros(17, np.uint32)])
    base = truth(T, ids[: pos + 1], pr.lim, 1.0)
    ids[pos + 1: pos + n] = base[pos + 1: pos + n]
    want = 0
    while want < n - 1 and ids[pos + 1 + want] == pr.tr[pos + 1 + want]:
        want += 1
    assert V.verify_greedy(ids, pos, n, 50.0) == want
    assert ids[pos + want + 1] == pr.tr[pos + want + 1]
    for e in (V, R, T):
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("exact", [False, True], ids=["fast", "exact"])
def test_verify_ties_pick_first_copy(tie_model, exact):
    path, cls_of, firsts = tie_model
    spec = mf.PRESETS["v152k-qwen3-untied"]
    S = 40
    flags = E.FLAG_EXACT if exact else 0
    V, R, T = nostream(path, S, flags), nostream(path, S, flags), nostream(path, S, flags)
    pr = Pair(V, R, T, S, 1.0, "ties")
    pr.start(np.random.default_rng(3).integers(0, spec.vocab, 6).astype(np.uint32), 5)
    for n, form in ((16, "correct"), (16, 4), (8, "first")):
        pr.verify(n, form)
    first_set = set(firsts.tolist())
    assert all(int(i) in first_set for i in pr.tr[6: pr.pos + 1]), "a greedy id is a later copy of its class"
    for e in (V, R, T):
        e.close()


# ------------------------------------------------------------------------------------------------ 3. exact mode vs the oracle
ORACLE_CASES = [("toy-qwen3", F32, 128), ("toy-nano", Q80, 64), ("mini-qwen3", Q80, 128), ("toy-qwen2", Q4K, 128)]


def penalised(raw, ids, pos, penalty):
    """generate_next_token's repetition penalty over ids[0..pos) (division by the penalty, in fp32)."""
    out = raw.copy()
    if penalty != 1.0:
        for i in set(int(t) for t in ids[:pos]):
            out[i] = np.float32(out[i]) / np.float32(penalty)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", ORACLE_CASES, ids=[f"{c[0]}-{quant_id(c[1], c[2])}" for c in ORACLE_CASES])
@pytest.mark.parametrize("penalty", [1.0, PEN])
def test_exact_verify_equals_oracle(name, quant, gs, penalty):
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
    eng = nostream(path, S, E.FLAG_EXACT)
    eng.prefill(tr, 0, P - 1)
    pos = P - 1
    rng = np.random.default_rng(2)
    for n, form in ((16, "correct"), (16, 6), (5, "first"), (15, "correct")):
        ids = tr.copy()
        ids[pos + 1: pos + n] = drafts_for(tr, pos, n, form, rng, spec.vocab)
        a = eng.verify_greedy(ids, pos, n, penalty)
        assert ids[: pos + a + 2].tolist() == tr[: pos + a + 2].tolist(), f"ids vs the oracle, verify at {pos}"
        assert_bits_equal(eng.logits(), want_logits[pos + a], f"logits at {pos + a} vs the oracle")
        pos += a + 1
    k, v = whole_kv(eng, pos)
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
def test_verify_attention_kernels(name, want, env, monkeypatch):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S = 96
    for flags in (0, E.FLAG_EXACT):
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, str(v))
            V, R, T = nostream(path, S, flags), nostream(path, S, flags), nostream(path, S, flags)
        kind = "exact" if flags else want
        pr = Pair(V, R, T, S, PEN, f"{name} {kind}")
        pr.start(mf.teacher_tokens(70, spec.vocab, 4), 69)
        pr.verify(16, 9)
        pr.verify(16, "correct")
        assert V.prefill_info()["attention"] == kind, V.prefill_info()
        pr.continue_greedy()
        assert R.kernels()["attention"] == kind
        for e in (V, R, T):
            e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["long-nano", "long-qwen3"])
def test_verify_near_position_1040(name):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, 128)
    S = 1072
    V, R, T = nostream(path, S), nostream(path, S), nostream(path, S)
    pr = Pair(V, R, T, S, PEN, f"{name} long")
    pr.start(mf.teacher_tokens(1036, spec.vocab, 4), 1035)
    pr.verify(16, "correct", check=False)
    pr.verify(16, 3, check=False)
    assert_bits_equal(V.logits(), R.logits(), f"{name}: logits")
    lo = 1030
    for l in range(V.n_layer):
        for p in range(lo, S):
            for f in (E.F_KROW, E.F_VROW):
                assert_bits_equal(V.read(f, V.kv_dim, l, p), R.read(f, R.kv_dim, l, p), f"{name}: layer {l} row {p}")
    pr.continue_greedy()
    for e in (V, R, T):
        e.close()


# ------------------------------------------------------------------------------------------------ 5. the prompt-lookup driver
def lookup_stats(ids, n_prompt, n_total, ngram_max, draft_max, M, lim):
    """The drafting rule of nb200_decode_lookup replayed on the final (greedy) ids: [passes, no-draft steps, drafted, accepted]."""
    ids = [int(i) for i in ids[:n_total]]
    st = [0, 0, 0, 0]
    p = n_prompt - 1
    while p + 1 < n_total:
        cap = min(draft_max, M - 1, n_total - 2 - p, lim - 1 - p)
        k, src = 0, 0
        for g in range(min(ngram_max, p), 0, -1):
            s = next((s for s in range(p - g, -1, -1) if ids[s: s + g] == ids[p - g + 1: p + 1]), None)
            if s is None:
                continue
            k = min(cap, p + 1 - (s + g))
            if k >= 1:
                src = s + g
                break
        if k:
            a = 0
            while a < k and ids[src + a] == ids[p + 1 + a]:
                a += 1
            st[0] += 1; st[2] += k; st[3] += a
            p += a + 1
        else:
            st[1] += 1
            p += 1
    return st


def run_driver(path, S, flags, P, N, vocab, combos, what, check_cache=True, lookup_flags=None, prompt=None):
    ref = nostream(path, S, flags)
    lim = limit(ref)
    prompt = mf.teacher_tokens(P, vocab) if prompt is None else prompt
    P = len(prompt)
    want = {}
    for penalty in sorted({c[0] for c in combos}):
        w = np.zeros(N, np.uint32); w[:P] = prompt
        r = nostream(path, S, flags)
        r.decode_greedy(w, P, N, penalty)
        want[penalty] = (w, whole_kv(r, S) if check_cache else None)
        r.close()
    ref.close()
    seen = []
    for penalty, ngram_max, draft_max in combos:
        eng = E.Engine(path, S, flags=flags | E.FLAG_NO_STREAM) if lookup_flags is None else E.Engine(path, S, flags=lookup_flags)
        ids = np.zeros(N, np.uint32); ids[:P] = prompt
        stats, _, _ = eng.decode_lookup(ids, P, N, penalty, ngram_max, draft_max)
        tag = f"{what} penalty {penalty} ngram_max {ngram_max} draft_max {draft_max}"
        w, kv = want[penalty]
        assert ids.tolist() == w.tolist(), f"{tag}: ids differ from decode_greedy"
        M = eng.prefill_info()["chunk"]
        assert stats == lookup_stats(w, P, N, ngram_max, draft_max if draft_max is not None else M - 1, M, lim), f"{tag}: {stats}"
        if check_cache and kv is not None:
            k, v = whole_kv(eng, S)
            assert_bits_equal(k, kv[0], f"{tag}: K cache"); assert_bits_equal(v, kv[1], f"{tag}: V cache")
        seen.append(stats)
        eng.close()
    return seen


DRIVER_COMBOS = [(pen, g, dm) for pen in (1.0, PEN) for g in (1, 3) for dm in (1, 4, 15)]
DRIVER_TOY = [("toy-nano", Q80, 64, False), ("toy-qwen3", Q4K, 128, False), ("mini-qwen3", F32, 128, True),
              ("toy-qwen2", Q80, 32, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,exact", DRIVER_TOY,
                         ids=[f"{c[0]}-{quant_id(c[1], c[2])}-{'exact' if c[3] else 'fast'}" for c in DRIVER_TOY])
def test_decode_lookup_equals_decode_greedy(name, quant, gs, exact):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    seen = run_driver(path, 64, E.FLAG_EXACT if exact else 0, 8, 65, spec.vocab, DRIVER_COMBOS, name)
    assert any(s[0] for s in seen), f"{name}: no combination drafted anything: {seen}"


@pytest.mark.gpu
def test_decode_lookup_accepts_and_rejects():
    """A prompt ending in a trigram it holds earlier with a random continuation: the lookup drafts that continuation (the
    model's greedy ids are something else), and later drafts from the model's own repetitive output are accepted."""
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    seen = []
    for seed in range(3):
        r = np.random.default_rng(seed).integers(0, spec.vocab, 12).astype(np.uint32)
        prompt = np.concatenate([r[:4], r[4:7], r[7:12], r[4:7]])          # ... A B C X Y Z W V A B C
        for flags in (0, E.FLAG_EXACT):
            seen += run_driver(path, 64, flags, 0, 65, spec.vocab, [(1.0, 3, 15), (1.0, 1, 4)], "accept/reject",
                               check_cache=False, prompt=prompt)
    assert any(s[3] > 0 for s in seen) and any(s[3] < s[2] for s in seen), seen
    assert any(0 < s[3] < s[2] for s in seen), f"no run with both accepted and rejected drafts: {seen}"


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,S,N", [("nano-168m", Q80, 128, 192, 160), ("qwen3-0.6b", Q4K, 128, 192, 160)])
def test_decode_lookup_baseline_shapes(name, quant, gs, S, N):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    combos = [(1.0, 3, None), (PEN, 3, 4), (1.0, 1, 1), (PEN, 1, 15)]
    run_driver(path, S, 0, 16, N, spec.vocab, combos, name, check_cache=(name == "nano-168m"))
    # the default (streaming) engine runs the driver's steps on the multi-kernel path: the NO_STREAM ids again
    run_driver(path, S, 0, 16, N, spec.vocab, [(1.0, 3, None)], f"{name} streaming engine", check_cache=False, lookup_flags=0)


# ------------------------------------------------------------------------------------------------ 6. refusals
@pytest.mark.gpu
def test_verify_refusals():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    S = 48                                                # below block_size 64: the limit is max_seq_len
    eng = nostream(path, S)
    toks = mf.teacher_tokens(S + 20, spec.vocab, 50)      # room for the drafts of the calls past the limit
    eng.prefill(toks, 0, 20)
    eng.verify_greedy(toks.copy(), 20, 4, PEN)

    def state():
        return whole_kv(eng, S) + (eng.logits(),)
    before = state()
    bad_draft = toks.copy(); bad_draft[24] = spec.vocab
    bad_past = toks.copy(); bad_past[3] = spec.vocab
    cases = [
        (toks, 22, 0, 1.0, "1 .. M = 16"),
        (toks, 22, 17, 1.0, "1 .. M = 16"),
        (toks, 40, 9, 1.0, "past"),
        (toks, 48, 1, 1.0, "past"),
        (bad_draft, 22, 4, 1.0, "out of range"),
        (bad_past, 22, 4, PEN, "out of range"),
    ]
    for ids, pos, n, pen, msg in cases:
        arg = ids.copy()
        with pytest.raises(E.NB200Error, match=re.escape(msg)):
            eng.verify_greedy(arg, pos, n, pen)
        assert arg.tolist() == ids.tolist(), f"ids after refusing '{msg}'"
        after = state()
        for a, b in zip(before, after):
            assert_bits_equal(a, b, f"state after refusing '{msg}'")
    ids = toks.copy()
    with pytest.raises(E.NB200Error, match="ngram_max"):
        eng.decode_lookup(ids, 4, 20, 1.0, 0, 4)
    with pytest.raises(E.NB200Error, match="ngram_max"):
        eng.decode_lookup(ids, 4, 20, 1.0, 3, 0)
    assert ids.tolist() == toks.tolist()
    eng.verify_greedy(bad_past.copy(), 40, 8, 1.0)         # penalty 1 reads no earlier ids; exactly up to the limit
    eng.lora_load(mf.write_lora(spec))
    before = state()
    for fn in (lambda: eng.verify_greedy(toks.copy(), 20, 4, 1.0), lambda: eng.decode_lookup(toks.copy(), 4, 20)):
        with pytest.raises(E.NB200Error, match="LoRA"):
            fn()
    for a, b in zip(before, state()):
        assert_bits_equal(a, b, "state after refusing LoRA")
    eng.lora_enable(False)
    eng.verify_greedy(toks.copy(), 20, 4, 1.0)
    eng.close()


@pytest.mark.gpu
@pytest.mark.skipif(E.device_count() < 2, reason="tensor parallelism needs 2 GPUs")
def test_verify_refuses_tensor_parallel():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    g = E.TpGroup(path, 32, 2)
    toks = mf.teacher_tokens(33, spec.vocab, 50)
    for r in g.ranks:
        with pytest.raises(E.NB200Error, match="tensor-parallel"):
            r.verify_greedy(toks.copy(), 0, 4)
    g.close()


# ------------------------------------------------------------------------------------------------ 7. launch counts
@pytest.mark.gpu
@pytest.mark.parametrize("flags", [0, E.FLAG_NO_GRAPH], ids=["graph", "direct"])
def test_verify_launch_counts(flags):
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    L = spec.n_layer
    eng = nostream(path, 64, flags)
    toks = mf.teacher_tokens(64, spec.vocab, 60)
    for n, pen, extra in ((16, 1.0, 0), (1, 1.0, 0), (8, PEN, 2), (8, PEN, 1)):    # seen rows; + the seen-set update once
        before = eng.launches
        eng.verify_greedy(toks.copy(), 5, n, pen)
        assert eng.launches - before == 1 + 6 * L + 2 + extra, (n, pen, eng.launches - before)
    per_token = eng.launches_per_token
    assert per_token == 2 + 5 * L
    ids = toks.copy()
    before = eng.launches
    stats, _, _ = eng.decode_lookup(ids, 1, 2)              # one step without a draft (nothing to look up at position 0)
    assert stats == [0, 1, 0, 0]
    assert eng.launches - before == per_token
    eng.close()


# ------------------------------------------------------------------------------------------------ CPU: the new kernel's frame
def test_verify_seen_kernel_has_no_stack_frame():
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", nb_build.ENGINE_SO],
                         capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = []
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m and "k_verify_seen" in m.group(1):
            res = lines[i + 1]
            found.append(res)
            st = re.search(r"STACK:(\d+)", res)
            loc = re.search(r"LOCAL:(\d+)", res)
            assert st and int(st.group(1)) == 0, res
            assert loc and int(loc.group(1)) == 0, res
    assert len(found) == 1, found
