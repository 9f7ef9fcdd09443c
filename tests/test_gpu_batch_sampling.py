"""Batched temperature / top-p sampling (nb200_batch_next_sampled; sample_rows_launch in nano_b200/csrc/sample.cu).

Entry i of a call with temperature[i] > 0 does what nb200_next_sampled does in its slot, and with temperature[i] == 0 what
nb200_batch_next_greedy's entry does (six zero ids), so greedy and sampled sessions share passes.  Covered here:
  * the several-row sampler alone on host-given rows (tests/batch_sample_probe.cu): calls of 1, 5 and 16 rows mixing every case
    of sampler_cases.py, checked row by row against the oracle's sampler (id, six ids, n0, sorted probabilities bit for bit,
    their order, the rejected keys); empty-nucleus rows beside normal ones; NaN / +-inf rows and sixteen copies of one row
    against the single-row sampler;
  * bit identity through the engine: every slot's (id, six ids) and logits after every call, and its K / V rows at the end,
    equal its own NB200_FLAG_NO_STREAM engine's next_sampled / next_greedy; toy shapes x F32 / Q80 / Q4K x exact / fast, and
    the real vocabularies with one full pass and a second pass holding one sampled entry;
  * exact mode against the oracle and the unmodified strict reference; exact ties; the engine's own session untouched;
    refusals; launch counts;
  * (CPU) the sampler's row kernels have no stack frame and no spills.
"""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import sampler_cases as sc
from conftest import assert_bits_equal
from nano_b200 import build as nb_build, engine as E, modelfile as mf
from oracle import bindings as ob
from test_gpu_batch import engine_kv, file_variants, nostream, prompts_for, quant_id, slot_kv
from test_gpu_sampler import probe, tie_model  # noqa: F401  (module fixtures: the single-row probe, the tied-classifier model)

HERE = os.path.dirname(os.path.abspath(__file__))
F32, Q80, Q4K = mf.QUANT_F32, mf.QUANT_Q80, mf.QUANT_Q4K
PEN = 1.3


# ------------------------------------------------------------------------------------------------ 1. the sampler alone
@pytest.fixture(scope="module")
def rows_probe():
    d = tempfile.mkdtemp(prefix="nb200_batch_sample_probe_")
    so = os.path.join(d, "libbatch_sample_probe.so")
    subprocess.run([nb_build.NVCC, *nb_build.GENCODE, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                    "-I" + nb_build.CSRC, os.path.join(HERE, "batch_sample_probe.cu"), "-o", so], check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    lib = C.CDLL(so)
    lib.probe_sample_rows.argtypes = [ob.f32p, C.c_uint32, C.c_uint32, C.c_uint32, ob.u32p, ob.u32p, ob.f32p, ob.f32p, ob.f32p,
                                      ob.u32p, ob.u32p, ob.f32p, ob.u32p]

    def run(rows, slot, entry, T, top_p, coin):
        """rows [n_rows][V]; row j of the call samples rows[slot[j]] and reports under entry[j].  Returns res [16][16],
        next [16] (by entry) and the sorted keys / values [n][V] by row."""
        lg = np.ascontiguousarray(rows, np.float32)
        n, V = len(slot), lg.shape[1]
        u = lambda a: np.ascontiguousarray(a, np.uint32)             # noqa: E731
        f = lambda a: np.ascontiguousarray(a, np.float32)            # noqa: E731
        slot, entry, T, top_p, coin = u(slot), u(entry), f(T), f(top_p), f(coin)
        res = np.zeros((16, 16), np.uint32); nxt = np.zeros(16, np.uint32)
        keys = np.zeros((n, V), np.float32); vals = np.zeros((n, V), np.uint32)
        rc = lib.probe_sample_rows(lg.ctypes.data_as(ob.f32p), lg.shape[0], V, n, slot.ctypes.data_as(ob.u32p),
                                   entry.ctypes.data_as(ob.u32p), T.ctypes.data_as(ob.f32p), top_p.ctypes.data_as(ob.f32p),
                                   coin.ctypes.data_as(ob.f32p), res.ctypes.data_as(ob.u32p), nxt.ctypes.data_as(ob.u32p),
                                   keys.ctypes.data_as(ob.f32p), vals.ctypes.data_as(ob.u32p))
        assert rc == 0, f"probe_sample_rows returned {rc}"
        return res, nxt, keys, vals
    return run


def groups(items, sizes, seed):
    """items in calls of the given sizes (cycled), each call's order shuffled."""
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(items)).tolist()
    out, k = [], 0
    while order:
        n = sizes[k % len(sizes)]
        out.append([items[i] for i in order[:n]])
        order = order[n:]
        k += 1
    return out


def run_call(rows_probe, call, seed):
    """One call over a list of (label, logits, T, top_p, coin): the rows go to shuffled slots of a 20-row table and report
    under shuffled entries.  Returns, per case, (res row, next id, sorted keys, sorted values)."""
    rng = np.random.default_rng(seed)
    n, V = len(call), call[0][1].size
    slot = rng.permutation(20)[:n]
    entry = rng.permutation(16)[:n]
    table = np.zeros((20, V), np.float32)
    for j, c in enumerate(call):
        table[slot[j]] = c[1]
    res, nxt, keys, vals = rows_probe(table, slot, entry, [c[2] for c in call], [c[3] for c in call], [c[4] for c in call])
    return [(res[entry[j]], int(nxt[entry[j]]), keys[j], vals[j]) for j in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("V", [512, 4095, 4096, 4097, 8193, 151936])
def test_rows_sampler_matches_oracle(rows_probe, V):
    cases = sc.cases(V)
    lg, T, top_p, want = sc.empty_nucleus_case(V)
    cases += [("empty-nucleus", lg, T, top_p, 0.5), ("empty-nucleus-c0", lg, T, top_p, 0.0)]
    for size, calls in ((1, groups(cases, [1], V)[:12]), (5, groups(cases, [5, 16], V + 1)), (16, groups(cases, [16], V + 2))):
        for ci, call in enumerate(calls):
            for (label, lg, T, top_p, coin), (res, nxt, keys, vals) in zip(call, run_call(rows_probe, call, V * 31 + ci)):
                tok, six, n0, last, sp, si = ob.sample_top_p(lg, T, top_p, coin, sorted_out=True)
                what = f"V {V} calls of {size}, call {ci}: {label} (n0 {n0}, last {last})"
                assert int(res[7]) == n0, f"{what}: device n0 {res[7]}"
                assert_bits_equal(keys[:n0], sp, f"{what}: sorted probabilities")
                assert np.array_equal(vals[:n0], si), f"{what}: sorted order differs at {np.nonzero(vals[:n0] != si)[0][:8]}"
                assert np.all(keys[n0:] == -1.0), f"{what}: rejected keys"
                assert (int(res[0]), res[1:7].tolist()) == (tok, six), f"{what}: device {res[0]} {res[1:7].tolist()}, oracle {tok} {six}"
                assert nxt == tok, f"{what}: next {nxt}"
                if label.startswith("empty"):
                    assert (tok, six) == (want, [0] * 6)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [512, 4097, 151936])
def test_rows_sampler_nonfinite_and_copies(rows_probe, probe, V):
    """Rows with NaN / +-inf logits (no defined reference answer) equal the single-row sampler; sixteen copies of one row with
    sixteen coins give each coin's single-row result."""
    rng = np.random.default_rng(V)
    base = (rng.standard_normal(V) * 2).astype(np.float32)
    odd = []
    for name, idx, val in (("nan", [3], np.nan), ("pinf", [V // 2], np.inf), ("ninf", [0, V - 1, 77], -np.inf),
                           ("ninf-most", list(range(0, V, 2)), -np.inf), ("all-nan", list(range(V)), np.nan)):
        lg = base.copy(); lg[idx] = val
        odd.append((name, lg, 0.7, 0.8, 0.5))
    normal = sc.cases(V)[:6]
    call = [normal[0], odd[0], normal[1], odd[1], odd[2], normal[2], odd[3], odd[4]]
    for (label, lg, T, top_p, coin), (res, nxt, keys, vals) in zip(call, run_call(rows_probe, call, V)):
        out, k1, v1 = probe(lg, T, top_p, coin)
        what = f"V {V} {label}"
        assert res[:9].tolist() == out.tolist(), f"{what}: {res[:9].tolist()} vs single row {out.tolist()}"
        assert nxt == int(out[0])
        assert_bits_equal(keys, k1, f"{what}: sorted keys"); assert np.array_equal(vals, v1), f"{what}: sorted values"
    lg = normal[0][1]
    coins = [0.0, float(sc.MAX_COIN)] + sc.coins(V, 14)
    call = [("copy", lg, 1.0, 0.95, c) for c in coins]
    for c, (res, nxt, _k, _v) in zip(coins, run_call(rows_probe, call, V + 5)):
        out, _, _ = probe(lg, 1.0, 0.95, c)
        assert res[:9].tolist() == out.tolist() and nxt == int(out[0]), f"V {V} coin {c}"


# ------------------------------------------------------------------------------------------------ 2. through the engine
class Session:
    """One session in a batch slot, sampled (temperature > 0, coins from its own xorshift stream) or greedy, and beside it the
    same session alone on its own multi-kernel engine."""

    def __init__(self, batch, slot, ref, prompt, penalty, T, top_p, S, prefill, seed):
        self.batch, self.slot, self.ref, self.penalty, self.T, self.top_p = batch, slot, ref, penalty, T, top_p
        self.prompt = np.asarray(prompt, np.uint32)
        self.ids = np.zeros(S + 1, np.uint32)
        self.ids[: len(prompt)] = self.prompt
        self.pos, self.state, self.coin = 0, seed, 0.0
        if prefill and len(prompt) > 1:
            n = len(prompt) - 1
            batch.prefill(slot, self.ids, 0, n)
            ref.prefill(self.ids, 0, n)
            self.pos = n

    def entry(self):
        c, self.state = ob.random_f32(self.state)
        self.coin = float(c)
        return self.slot, self.ids, self.pos, self.penalty, self.T, self.top_p, self.coin

    def advance(self, got, six, what):
        if self.T == 0:
            want = (self.ref.next_greedy(self.ids, self.pos, 0, self.penalty), [0] * 6)
        else:
            want = self.ref.next_sampled(self.ids, self.pos, self.penalty, self.T, self.top_p, self.coin)
        assert (got, six) == want, f"{what} slot {self.slot} T {self.T} pos {self.pos}: {got} {six} vs {want}"
        assert_bits_equal(self.batch.logits(self.slot), self.ref.logits(), f"{what} slot {self.slot} pos {self.pos}: logits")
        if self.pos + 1 >= len(self.prompt):
            self.ids[self.pos + 1] = got
        self.pos += 1

    def check_cache(self, what):
        k, v = slot_kv(self.batch, self.slot, self.pos)
        rk, rv = engine_kv(self.ref, self.pos)
        assert_bits_equal(k, rk, f"{what} slot {self.slot}: K rows 0..{self.pos - 1}")
        assert_bits_equal(v, rv, f"{what} slot {self.slot}: V rows 0..{self.pos - 1}")


def step(batch, sessions, what):
    e = list(zip(*[s.entry() for s in sessions]))
    got, six = batch.next_sampled(*e)
    for s, g, x in zip(sessions, got, six):
        s.advance(g, x, what)
    return got, six


def run_sessions(path, S, flags, prompts, prefilled, penalties, temps, top_ps, steps, what, seed=5, all_every_call=False):
    eng = E.Engine(path, S, flags=flags)
    batch = eng.batch(len(prompts))
    refs = [nostream(path, S, flags) for _ in prompts]
    sess = [Session(batch, i, refs[i], prompts[i], penalties[i], temps[i], top_ps[i], S, prefilled[i], 1000 + i)
            for i in range(len(prompts))]
    rng = np.random.default_rng(seed)
    done = {i: 0 for i in range(len(sess))}
    target = {i: len(prompts[i]) - 1 - sess[i].pos + steps for i in range(len(sess))}
    while any(done[i] < target[i] for i in done):
        live = [i for i in done if done[i] < target[i]]
        pick = live if all_every_call else ([i for i in live if rng.random() < 0.7] or live[:1])
        if not all_every_call:
            rng.shuffle(pick)
        step(batch, [sess[i] for i in pick], what)
        for i in pick:
            done[i] += 1
    for s in sess:
        s.check_cache(what)
    for r in refs:
        r.close()
    eng.close()


ID_CASES = [(n, q, g, x) for n in ("toy-nano", "toy-qwen3", "mini-qwen3", "toy-qwen2") for q, g in file_variants(n)
            for x in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs,exact", ID_CASES,
                         ids=[f"{c[0]}-{quant_id(c[1], c[2])}-{'exact' if c[3] else 'fast'}" for c in ID_CASES])
def test_batch_sampling_bit_identical_to_single_sessions(name, quant, gs, exact):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    run_sessions(path, 64, E.FLAG_EXACT if exact else 0, prompts_for(spec.vocab, (1, 7, 16, 23, 40)), [False, True, False, True, True],
                 [PEN, 1.0, PEN, 1.0, PEN], [0.7, 0.0, 1.0, 5.0, 0.7], [0.8, 1.0, 0.95, 0.8, 1.0], 14,
                 f"{name} {quant_id(quant, gs)} {'exact' if exact else 'fast'}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [16, 17])
@pytest.mark.parametrize("name,gs", [("v16k-nano", 128), ("v152k-qwen3", 64)])
def test_batch_sampling_real_vocabularies(name, gs, n):
    """16 sessions fill one pass; with 17 the second pass holds one sampled entry.  top-p 0.95 at T 1.0: long scans."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, Q80, gs)
    temps = [0.0 if i % 5 == 4 else 1.0 for i in range(n)]
    temps[-1] = 1.0
    run_sessions(path, 32, 0, prompts_for(spec.vocab, [3 + (i * 5) % 11 for i in range(n)]), [i % 2 == 0 for i in range(n)],
                 [PEN if i % 3 else 1.0 for i in range(n)], temps, [0.95] * n, 3, f"{name} n={n}", all_every_call=True)


# ------------------------------------------------------------------------------------------------ 3. against the reference
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", [("toy-nano", Q80, 64), ("mini-qwen3", Q80, 128), ("toy-qwen2", F32, 128),
                                           ("v152k-qwen3", Q80, 64)])
def test_exact_batch_sampling_equals_reference(name, quant, gs):
    """Three sampled sessions (penalty 1.1, T 0.7, top-p 0.8, one xorshift stream each) in one exact-mode batch: ids and logits
    equal the oracle's logits + sampler, and the unmodified strict reference's ids where it is built."""
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S, P, n, steps = 40, 4, 3, 30
    seeds = [39, 7, 123]
    prompts = [np.asarray([17 + i, 18, 19 + i, 20], np.uint32) for i in range(n)]
    eng = E.Engine(path, S, flags=E.FLAG_EXACT)
    batch = eng.batch(n)
    ids = [np.zeros(S + 1, np.uint32) for _ in range(n)]
    for i in range(n):
        ids[i][:P] = prompts[i]
        batch.prefill(i, ids[i], 0, P - 1)
    state = list(seeds)
    o = [ob.NanoOracle(path, S) for _ in range(n)]
    for i in range(n):
        for p in range(P - 1):
            o[i].forward(int(ids[i][p]), p)
    for pos in range(P - 1, P - 1 + steps):
        coins = []
        for i in range(n):
            c, state[i] = ob.random_f32(state[i]); coins.append(float(c))
        order = [(pos + k) % n for k in range(n)]
        got, six = batch.next_sampled(order, [ids[i] for i in order], [pos] * n, [1.1] * n, [0.7] * n, [0.8] * n, [coins[i] for i in order])
        for k, i in enumerate(order):
            raw = o[i].forward(int(ids[i][pos]), pos)
            seen = np.unique(ids[i][:pos])
            lg = raw.copy(); lg[seen] = (raw[seen] / np.float32(1.1)).astype(np.float32)
            assert_bits_equal(batch.logits(i), lg, f"{name} session {i} pos {pos}: logits vs the oracle")
            assert (got[k], six[k]) == tuple(ob.sample_top_p(lg, 0.7, 0.8, coins[i])[:2]), f"{name} session {i} pos {pos}"
            ids[i][pos + 1] = got[k]
    for x in o:
        x.close()
    eng.close()
    assert len(set(ids[0][P:P + steps].tolist())) > 5              # it really sampled
    if ob.ref_available("strict"):
        for i in range(n):
            ref = ob.RefEngine(path, S, "strict", penalty=1.1, temperature=0.7, top_p=0.8, top_k=20, seed=seeds[i])
            want = np.zeros(S + 1, np.uint32); want[:P] = prompts[i]
            for pos in range(P - 1 + steps):
                want[pos + 1] = ref.next(want, pos, 1 if pos < P - 1 else 0)
            assert ids[i][:P + steps].tolist() == want[:P + steps].tolist(), f"{name} session {i} vs the strict reference"


# ------------------------------------------------------------------------------------------------ 4. ties
@pytest.mark.gpu
def test_batch_sampling_ties_first_copies(tie_model):
    """Exactly tied classifier rows: a sampled entry's six ids are the winning class's first six copies."""
    path, cls_of, firsts = tie_model
    spec = mf.PRESETS["v152k-qwen3-untied"]
    S = 24
    first_set = set(firsts.tolist())
    prompts = [np.random.default_rng(3 + i).integers(0, spec.vocab, 6).astype(np.uint32) for i in range(3)]
    eng = E.Engine(path, S)
    batch = eng.batch(3)
    refs = [nostream(path, S) for _ in range(3)]
    sess = [Session(batch, i, refs[i], prompts[i], 1.0, 0.7, 0.8, S, i != 1, 50 + i) for i in range(3)]
    for _ in range(8):
        _got, six = step(batch, sess, "ties")
        for s, x in zip(sess, six):
            members = np.nonzero(cls_of == cls_of[x[0]])[0]
            assert x[0] in first_set
            if members.size >= 6:
                assert x == members[:6].tolist(), f"slot {s.slot}: six ids {x}, first copies {members[:6].tolist()}"
    for r in refs:
        r.close()
    eng.close()


# ------------------------------------------------------------------------------------------------ 5. isolation
@pytest.mark.gpu
@pytest.mark.parametrize("name,quant,gs", [("toy-nano", Q80, 64), ("v16k-nano", Q80, 128)])
def test_engine_sampling_untouched_by_batch_sampling(name, quant, gs):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    S = 32
    toks = mf.teacher_tokens(S, spec.vocab)

    def run(eng, batch):
        ids = np.zeros(S + 1, np.uint32); ids[:4] = toks[:4]
        other = prompts_for(spec.vocab, [S], 90)[0]
        out, logits, st = [], [], 39
        for pos in range(S - 1):
            c, st = ob.random_f32(st)
            tok, six = eng.next_sampled(ids, pos, PEN, 0.7, 0.8, float(c))
            if pos >= 3:
                ids[pos + 1] = tok
            out.append((tok, six)); logits.append(eng.logits())
            if batch is not None:
                batch.next_sampled([pos % 2], [other], [pos // 2], [PEN], [1.0], [0.95], [0.25])
        return out, np.stack(logits), engine_kv(eng, S - 1)

    alone = E.Engine(path, S)
    want = run(alone, None)
    alone.close()
    eng = E.Engine(path, S)
    got = run(eng, eng.batch(2))
    assert got[0] == want[0]
    assert_bits_equal(got[1], want[1], "the engine's logits")
    assert_bits_equal(got[2][0], want[2][0], "the engine's K rows"); assert_bits_equal(got[2][1], want[2][1], "the engine's V rows")
    eng.close()


# ------------------------------------------------------------------------------------------------ 6. refusals
@pytest.mark.gpu
def test_batch_sampling_refusals():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    S = 48
    eng = nostream(path, S)
    batch = eng.batch(3)
    toks = [mf.teacher_tokens(S + 1, spec.vocab, 50 + i) for i in range(3)]
    batch.prefill(0, toks[0], 0, 20)
    batch.prefill(1, toks[1], 0, 10)
    batch.next_sampled([0, 1], toks[:2], [20, 10], [PEN, PEN], [0.7, 0.0], [0.8, 0.8], [0.5, 0.5])

    def state():
        return [slot_kv(batch, s, S) for s in range(3)] + [batch.logits(s) for s in range(3)]
    before = state()
    bad = toks[0].copy(); bad[5] = spec.vocab
    bad_now = toks[0].copy(); bad_now[21] = spec.vocab
    ns = lambda sl, ids, pos, pen, T=None: batch.next_sampled(sl, ids, pos, pen, T or [0.7] * len(sl), [0.8] * len(sl), [0.5] * len(sl))  # noqa: E731
    cases = [
        (lambda: ns([], [], [], []), "no entries"),
        (lambda: ns([3], toks[:1], [21], [1.0]), "slot 3"),
        (lambda: ns([0, 0], toks[:2], [21, 11], [1.0, 1.0]), "twice"),
        (lambda: ns([0, 1], toks[:2], [21, S], [1.0, 1.0]), "past"),
        (lambda: ns([1, 0], [toks[1], bad_now], [11, 21], [1.0, 1.0]), "out of range"),
        (lambda: ns([1, 0], [toks[1], bad], [11, 21], [1.0, PEN]), "out of range"),
        (lambda: ns([0, 1], toks[:2], [21, 11], [PEN, PEN], [0.7, -0.5]), "temperature"),
        (lambda: ns([0, 1], toks[:2], [21, 11], [PEN, PEN], [float("nan"), 0.7]), "temperature"),
        (lambda: ns([0, 1], toks[:2], [21, 11], [PEN, PEN], [0.0, -np.inf]), "temperature"),
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
    # the seen sets are unchanged too: the next accepted call gives what a fresh engine gives
    ref = nostream(path, S)
    ref.prefill(toks[0], 0, 20)
    ref.next_sampled(toks[0], 20, PEN, 0.7, 0.8, 0.5)
    want = ref.next_sampled(toks[0], 21, PEN, 0.7, 0.8, 0.5)
    got, six = ns([0], toks[:1], [21], [PEN])
    assert (got[0], six[0]) == want
    assert_bits_equal(batch.logits(0), ref.logits(), "logits after the refusals")
    ref.close()
    eng.lora_load(mf.write_lora(spec))
    for fn in (lambda: ns([0], toks[:1], [22], [1.0]), lambda: ns([2], toks[2:], [0], [1.0], [0.0])):
        with pytest.raises(E.NB200Error, match="LoRA"):
            fn()
    eng.lora_enable(False)
    ns([0], toks[:1], [22], [1.0])
    eng.close()


# ------------------------------------------------------------------------------------------------ 7. launch counts
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 16, 17])
@pytest.mark.parametrize("mix", ["greedy", "sampled", "second-pass"])
def test_batch_sampling_launch_count(n, mix):
    """passes * (1 + 5L + 2) + sampled_passes * 3 (prepare, sort, pick); all greedy equals nb200_batch_next_greedy's count."""
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, Q80, 64)
    eng = E.Engine(path, 64)
    batch = eng.batch(17)
    M = batch.info()["chunk"]
    toks = [mf.teacher_tokens(64, spec.vocab, 60 + i) for i in range(n)]
    T = {"greedy": [0.0] * n, "sampled": [0.8] * n, "second-pass": [0.0] * (n - 1) + [0.8 if n > M else 0.0]}[mix]
    passes = -(-n // M)
    sampled_passes = len({i // M for i in range(n) if T[i] > 0})
    before = eng.launches
    batch.next_sampled(list(range(n)), toks, [3] * n, [1.0] * n, T, [0.9] * n, [0.5] * n)
    got = eng.launches - before
    assert got == passes * (1 + 5 * spec.n_layer + 2) + sampled_passes * 3, got
    if mix == "greedy":
        before = eng.launches
        batch.next_greedy(list(range(n)), toks, [4] * n, [1.0] * n)
        assert eng.launches - before == got
    eng.close()


# ------------------------------------------------------------------------------------------------ CPU: stack frames, spills
def test_sample_rows_kernels_have_no_stack_frame():
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", nb_build.ENGINE_SO],
                         capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    res = {}
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m and "k_sample" in m.group(1):
            res[m.group(1)] = lines[i + 1]
    rows = {f: r for f, r in res.items() if "k_sample_rows_" in f}
    assert len(rows) == 2 and len(res) == 4, sorted(res)
    for f, r in res.items():
        assert re.search(r"STACK:0\b", r) and re.search(r"LOCAL:0\b", r), f"{f}: {r.strip()}"
