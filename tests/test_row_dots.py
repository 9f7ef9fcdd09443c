"""Every fast-mode row dot of both decode paths, one row at a time, against float64 of the very codes it consumed.

tests/row_dot_probe.cu calls the real device functions: on the streaming side st_prep<QUANT, LPG> builds the operand region
and st_row_q80_lpg, st_rows_q80_warp, st_row_q4k and st_row_f32 read weight rows laid out as ring tiles; on the multi-kernel
side q80_load + q80_consume<RB, LPG, ORD>, rows_f32<RB> and rows_q4k<RB> read the engine's weight layout.

What is asserted:
  * st_row_q80_lpg (every lane geometry the kernel's search can pick) and q80_consume<..., true> equal the oracle's ordered
    group sum (nor_matvec_q80, infer.c:654-679) bit for bit: their comments promise the reference's order.
  * A row's value does not depend on where it sits: its slot in a block of RB rows, the block size, its place in the
    tile, and the lanes of the warp or team (all must hold the same bits).
  * Every other dot stays within an a-priori bound of the float64 value of the same codes and scales:
        |got - ref64| <= (m + 4) * 2^-24 * sum|terms| + 2^-149 * sum_t (1 + F_t)
    m is the number of fp32 terms in the row (Q80: 16-byte chunks, Q4K: 32-element groups, F32: 4-float steps), and every
    term passes through fewer than m + 4 roundings in any summation order (Q4K: two products and three adds inside a group
    term, then the sum).  sum|terms| adds the absolute values of the sub-products (a Q4K group term is four of them, which
    can cancel).  The second part covers underflow: a rounding in the subnormal range loses at most 2^-150, and a product of
    three factors whose first product underflows carries that loss times the remaining factor; F_t, the largest factor of
    sub-product t, bounds that for either order of the two multiplications.  The bound holds for any summation order, and
    a single missing or doubled term at these lengths is far outside it.  Inputs keep every product and partial sum finite.

Inputs are the quantiser edge vectors of test_gpu_ops.py tiled with normal groups, and weight rows built by hand: codes at
+-127 (also all matching the activation's signs), all-zero groups and zero scales, subnormal and very large group scales,
and rows whose exact dot cancels to about 0.  The row count leaves a partial last row block.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from nano_b200 import build as nb_build
from oracle import bindings as ob
from test_gpu_ops import o_q4k_quant, o_q80_quant, oracle, q4k_edge_vector, q80_edge_vector
from test_stream_prep_probe import q4k_reference, tiled

HERE = os.path.dirname(os.path.abspath(__file__))
gpu = pytest.mark.gpu
f32, f64 = np.float32, np.float64
U, TINY = 2.0 ** -24, 2.0 ** -149
R = 27                          # rows: 27 % 4 == 3 and 27 % 2 == 1, so the last block of 2 or 4 rows is partial
TERM_MAX = 1e4                  # largest term: products and sums stay finite, and huge activation groups do not dwarf the rest
W_MAX = 1e30                    # largest weight or weight scale


def compile_probe(out_dir):
    so = os.path.join(out_dir, "librowdot.so")
    subprocess.run([nb_build.NVCC, *nb_build.GENCODE, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-diag-suppress", "128",
                    "-I" + nb_build.CSRC, os.path.join(HERE, "row_dot_probe.cu"), "-o", so], check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    return so


def test_probe_compiles_for_sm90a(tmp_path):
    so = compile_probe(str(tmp_path))
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", so], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in out, out


@pytest.fixture(scope="module")
def probe():
    lib = C.CDLL(compile_probe(tempfile.mkdtemp(prefix="nb200_rowdot_")))
    u32, vp = C.c_uint32, C.c_void_p
    lib.probe_stream_dots.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, u32, u32, u32, u32, vp, u32, vp, u32, vp, u32, u32,
                                      vp, vp, u32, vp]
    lib.probe_mk_dots.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_uint64, vp, C.c_uint64, u32, u32, vp, u32, vp, vp]
    return lib


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def act_bytes(quant, n, gs):
    b = n * 4 if quant == 0x00 else ((n + 15) & ~15) + (n // gs) * 4 + 16 if quant == 0x80 else n + (n // 32) * 16
    return (b + 15) & ~15


def stream_dots(lib, quant, lpg, form, x, wmain, waux, rb=1, lg2=1, gteam=1, shift=0, tile_rows=0):
    """(row values, operand region) of one probe_stream_dots call"""
    x = np.ascontiguousarray(x, f32)
    n, gs = x.size, (lpg * 16 if quant == 0x80 else 1)
    wmain = np.ascontiguousarray(wmain).view(np.uint8).reshape(R, -1)
    waux = np.ascontiguousarray(waux).view(np.uint8).reshape(R, -1) if waux is not None else np.zeros((R, 0), np.uint8)
    out = np.full(R, np.nan, f32)
    act = np.zeros(act_bytes(quant, n, gs), np.uint8)
    mm = np.zeros(1, np.uint32)
    rc = lib.probe_stream_dots(quant, lpg, form, rb, lg2, gteam, shift, tile_rows, ptr(x), n, ptr(wmain), wmain.shape[1], ptr(waux),
                               waux.shape[1], R, ptr(out), ptr(act), act.size, ptr(mm))
    assert rc == 0, f"probe_stream_dots returned {rc}"
    assert mm[0] == 0, f"{mm[0]} rows differ between the lanes that hold them"
    return out, act


def mk_dots(lib, quant, lpg, ordered, rb, w, waux, n, act):
    w = np.ascontiguousarray(w)
    waux = np.ascontiguousarray(waux) if waux is not None else np.zeros(4, np.uint8)
    out = np.full(R, np.nan, f32)
    mm = np.zeros(1, np.uint32)
    rc = lib.probe_mk_dots(quant, lpg, int(ordered), rb, ptr(w), w.nbytes, ptr(waux), waux.nbytes, R, n, ptr(act), act.size, ptr(out), ptr(mm))
    assert rc == 0, f"probe_mk_dots returned {rc}"
    assert mm[0] == 0, f"{mm[0]} rows differ between the lanes that hold them"
    return out


def same_bits(vals, what):
    base = vals[0][1].view(np.uint32)
    for name, v in vals[1:]:
        bad = np.nonzero(v.view(np.uint32) != base)[0]
        assert bad.size == 0, f"{what}: rows {bad[:8]} differ between {vals[0][0]} and {name}: {vals[0][1][bad[:4]]} vs {v[bad[:4]]}"


def check_bound(got, ref, m, absterms, factor, what):
    """the a-priori bound of the module docstring, row by row; prints the worst share of it that a row uses"""
    got = np.asarray(got, f64)
    assert np.all(np.isfinite(got)), f"{what}: non-finite rows {np.nonzero(~np.isfinite(got))[0][:8]}"
    bound = (m + 4) * U * absterms.reshape(R, -1).sum(1) + TINY * (1.0 + factor.reshape(R, -1)).sum(1)
    share = np.abs(got - ref) / bound
    w = int(np.argmax(share))
    print(f"{what}: worst share of the bound {share[w]:.3g} (row {w}, |err| {abs(got[w] - ref[w]):.3g}, bound {bound[w]:.3g})")
    assert share[w] <= 1.0, f"{what}: row {w} is {share[w]:.3g} x the bound off: got {got[w]!r}, float64 {ref[w]!r}"
    return share.max()


# ---------------------------------------------------------------- Q80
def q80_weights(xq, xs, gs, seed):
    """R rows of codes [R, n] and group scales [R, G], one kind of edge per row (row % 8)"""
    n, G = xq.size, xq.size // gs
    rng = np.random.default_rng(seed)
    wq = rng.integers(-127, 128, (R, n)).astype(np.int8)
    ws = (np.abs(rng.standard_normal((R, G))) * 0.02 + 1e-4).astype(f64)
    for r in range(R):
        kind = r % 8
        if kind == 1:
            wq[r] = np.where(rng.random(n) < 0.5, 127, -127)                                  # codes at +-127
        elif kind == 2:
            wq[r] = np.where(xq >= 0, 127, -127)                                              # ... all adding up
        elif kind == 3:
            wq[r].reshape(G, gs)[::2] = 0; ws[r, 1::3] = 0.0                                  # zero groups, zero scales
        elif kind == 4:
            ws[r] = np.exp(rng.uniform(np.log(1.4e-45), np.log(1.1e-38), G))                 # subnormal scales
        elif kind == 5:
            ws[r] = 1e30 * rng.uniform(0.5, 1.0, G)                                           # very large scales
        elif kind == 7:
            pick = rng.integers(0, 4, G)
            g4 = wq[r].reshape(G, gs)
            g4[pick == 0] = 127; g4[pick == 1] = 0
            ws[r, pick == 2] = 3e-42; ws[r, pick == 3] = 1e25
    # |isum * ws * xs| <= TERM_MAX for any codes
    cap = np.minimum(TERM_MAX / (16129.0 * gs * np.maximum(xs.astype(f64), 1e-45)), W_MAX)
    ws = np.minimum(ws, cap).astype(f32)
    isum = q80_group_sums(wq, xq, gs)
    for r in range(6, R, 8):                                                                   # cancels to about 0
        t = isum[r] * ws[r].astype(f64) * xs.astype(f64)
        h = int(np.argmax(np.abs(isum[r] * xs.astype(f64)) * cap))      # the group that can carry the rest
        if isum[r, h] != 0 and xs[h] != 0:
            v = -(t.sum() - t[h]) / (isum[r, h] * f64(xs[h]))
            if abs(v) <= cap[h]:
                ws[r, h] = f32(v)
    return wq, ws


def q80_group_sums(wq, xq, k):
    """exact integer dots over consecutive runs of k elements: [R, n / k]"""
    return (wq.reshape(R, -1, k).astype(np.int64) * xq.reshape(-1, k).astype(np.int64)).sum(-1)


def q80_ordered(xq, xs, wq, ws, gs):
    """the oracle's ordered group sum (nor_matvec_q80)"""
    y = np.zeros(R, f32)
    oracle().nor_matvec_q80(y.ctypes.data_as(ob.f32p), xq.ctypes.data_as(ob.i8p), xs.ctypes.data_as(ob.f32p),
                            wq.ctypes.data_as(ob.i8p), ws.ctypes.data, xq.size, R, gs)
    return y


def q80_check_fast(got, xq, xs, wq, ws, gs, what):
    """bound over 16-byte chunks (the fast forms' terms: one lane's 16 codes x the two scales)"""
    ic = q80_group_sums(wq, xq, 16).astype(f64)
    wsc = np.repeat(ws.astype(f64), gs // 16, axis=1); xsc = np.repeat(xs.astype(f64), gs // 16)
    ref = (q80_group_sums(wq, xq, gs) * ws.astype(f64) * xs.astype(f64)).sum(1)
    terms = np.abs(ic * wsc * xsc)
    factor = np.maximum(np.maximum(np.abs(ic), np.abs(wsc)), np.abs(xsc)[None, :])
    return check_bound(got, ref, xq.size // 16, terms, factor, what)


def lpg_geometries(G, lpg):
    """every (lg2, gteam) the streaming kernel's geometry search can pick for a row of G groups (stream.cuh, kernel start)"""
    out = []
    c = lpg
    while c >= 1:
        if not (G * c > 32 and c > 1):
            out.append((c, min(G, 32 // c)))
        c //= 2
    return out


def split_act_q80(act, n, gs):
    p = (n + 15) & ~15
    return act[:n].view(np.int8).copy(), act[p: p + (n // gs) * 4].view(f32).copy()


# One group up to st_prep_max_n; n % 512 = 0, 64, 128, 256, 320, 384 (a row is whole groups of 64 or 128, so the shortest
# tail of a 512-byte step is one group); G % 32 != 0 past 32 groups (several team passes, the last one partial).
@gpu
@pytest.mark.parametrize("lpg,n", [(8, 128), (8, 384), (8, 640), (8, 3840), (8, 3968), (8, 4096), (8, 4224), (8, 7680), (8, 11520),
                                   (4, 64), (4, 576), (4, 3840), (4, 3904), (4, 3968), (4, 4096), (4, 7680), (4, 11520)])
def test_stream_q80_dots(probe, lpg, n):
    gs, G = lpg * 16, n // (lpg * 16)
    x = tiled(q80_edge_vector(gs), n, n + gs)
    hq, hs = o_q80_quant(x, gs)
    wq, ws = q80_weights(hq, hs, gs, n * 3 + lpg)
    runs = []
    for lg2, gteam in lpg_geometries(G, lpg):                         # shared tiles: the reference's ordered sum, bit for bit
        for tile_rows in (0, 5):
            got, act = stream_dots(probe, 0x80, lpg, 0, x, wq, ws, lg2=lg2, gteam=gteam, tile_rows=tile_rows)
            xq, xs = split_act_q80(act, n, gs)
            want = q80_ordered(xq, xs, wq, ws, gs)
            bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
            assert bad.size == 0, (f"st_row_q80_lpg<{lpg}> lg2 {lg2} gteam {gteam}: rows {bad[:8]} differ from the ordered sum: "
                                   f"{got[bad[:4]]} vs {want[bad[:4]]}")
    for rb, shift, tile_rows in [(1, 0, 0), (2, 0, 0), (4, 0, 0), (4, 1, 7), (2, 1, 7), (4, 3, 6)]:   # owned tiles
        got, act = stream_dots(probe, 0x80, lpg, 1, x, wq, ws, rb=rb, shift=shift, tile_rows=tile_rows)
        runs.append((f"RB {rb} shift {shift} tile {tile_rows}", got))
    same_bits(runs, f"st_rows_q80_warp<{lpg}, RB> n {n}")
    xq, xs = split_act_q80(act, n, gs)
    q80_check_fast(runs[0][1], xq, xs, wq, ws, gs, f"st_rows_q80_warp<{lpg}, 1|2|4> n {n}")


def mk_act_q80(xq, xs, n, gs):
    a = np.zeros(act_bytes(0x80, n, gs), np.uint8)
    p = (n + 15) & ~15
    a[:n] = xq.view(np.uint8); a[p: p + xs.size * 4] = xs.view(np.uint8)
    return a


@gpu
@pytest.mark.parametrize("lpg", [2, 4, 8, 16])
@pytest.mark.parametrize("n", ["gs", "3gs", "2048+gs", 3840, 4096, 7680, 11520])
def test_multikernel_q80_dots(probe, lpg, n):
    gs = lpg * 16
    n = {"gs": gs, "3gs": 3 * gs, "2048+gs": 2048 + gs}.get(n, n)   # one group, three groups, a partial last 1024-byte step
    x = tiled(q80_edge_vector(gs), n, n + 7 * gs)
    xq, xs = o_q80_quant(x, gs)
    wq, ws = q80_weights(xq, xs, gs, n * 5 + lpg)
    act = mk_act_q80(xq, xs, n, gs)
    want = q80_ordered(xq, xs, wq, ws, gs)
    for rb in (1, 2, 4):
        got = mk_dots(probe, 0x80, lpg, True, rb, wq, ws, n, act)
        bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
        assert bad.size == 0, f"q80_consume<{rb}, {lpg}, true> n {n}: rows {bad[:8]} differ from the ordered sum: {got[bad[:4]]} vs {want[bad[:4]]}"
    runs = [(f"RB {rb}", mk_dots(probe, 0x80, lpg, False, rb, wq, ws, n, act)) for rb in (1, 2, 4)]
    same_bits(runs, f"q80_consume<RB, {lpg}, false> n {n}")
    q80_check_fast(runs[0][1], xq, xs, wq, ws, gs, f"q80_consume<1|2|4, {lpg}, false> n {n}")


# ---------------------------------------------------------------- Q4K
def q4k_weight_blocks(x, seed):
    """R rows of oracle Q4K blocks [R, n / 256, 160], one kind of edge per row (row % 8); row 6 (mod 8) cancels to about 0"""
    n = x.size
    rng = np.random.default_rng(seed)
    amax = np.maximum(np.abs(x.astype(f64)).reshape(-1, 256).max(1), 1e-30)
    lim = np.repeat(np.minimum(TERM_MAX / (128.0 * amax), W_MAX), 256)     # a group's sub-products stay below TERM_MAX
    W = rng.standard_normal((R, n))
    for r in range(R):
        kind = r % 8
        if kind == 1:
            W[r] = np.resize(np.repeat([0.75, -1.25, 0.0, 2.0], 32), n)                       # constant groups: codes 0 / 15
        elif kind == 2:
            W[r] = -np.abs(W[r]) - 0.5                                                         # all negative: large biases
        elif kind == 3:
            W[r].reshape(-1, 32)[::2] = 0.0                                                    # zero groups
        elif kind == 4:
            W[r] *= 1e-41                                                                      # subnormal group scales
        elif kind == 5:
            W[r] *= 1e30                                                                       # very large group scales
        elif kind == 7:
            W[r] *= np.repeat(10.0 ** rng.integers(-39, 25, n // 32), 32)
    W = np.clip(W, -lim, lim).astype(f32)
    blocks = np.zeros(R * (n // 256) * 160, np.uint8)
    oracle().nor_q4k_quantize_rows(blocks.ctypes.data_as(ob.u8p), W.ctypes.data_as(ob.f32p), R, n)
    return blocks.reshape(R, n // 256, 160)


def q4k_terms(blocks, xc, sq, bq):
    """sub-products [R, G, 4] (sp sq spq, sp bq spp, sq bp sqq, 32 bp bq) and their largest factors, in float64"""
    R_, nb = blocks.shape[:2]
    n = nb * 256
    wc, sp, bp = zip(*(q4k_reference(blocks[r].reshape(-1), n) for r in range(R_)))
    wc = np.stack(wc).astype(np.int64).reshape(R_, -1, 32); sp = np.stack(sp).astype(f64); bp = np.stack(bp).astype(f64)
    xc = xc.astype(np.int64).reshape(-1, 32); sq = sq.astype(f64); bq = bq.astype(f64)
    spq = (wc * xc).sum(-1).astype(f64); spp = wc.sum(-1).astype(f64); sqq = xc.sum(-1).astype(f64)
    subs = np.stack([sp * sq * spq, sp * bq * spp, sq * bp * sqq, 32.0 * bp * bq], -1)
    factor = np.stack([np.maximum(np.maximum(np.abs(sp), np.abs(sq)), spq), np.maximum(np.maximum(np.abs(sp), np.abs(bq)), spp),
                       np.maximum(np.maximum(np.abs(sq), np.abs(bp)), np.broadcast_to(sqq, sp.shape)),
                       np.maximum(np.maximum(32.0, np.abs(bp)), np.abs(bq))], -1)
    return subs, factor


def q4k_cancel(blocks, xc, sq, bq):
    """row 6 (mod 8): the last block's super-scale chosen so that the row's exact dot is about 0 (it is linear in it)"""
    for r in range(6, R, 8):
        one = blocks[r: r + 1].copy()
        one[0, -1, 12:16] = np.frombuffer(f32(1.0).tobytes(), np.uint8)
        s = q4k_terms(one, xc, sq, bq)[0][0]
        pv = (s[-8:, 0] - s[-8:, 1]).sum()                               # the last block's sp-terms at ss = 1 (sp = s6 exactly)
        rest = (s[:-8, 0] - s[:-8, 1] - s[:-8, 2] + s[:-8, 3]).sum() + (s[-8:, 3] - s[-8:, 2]).sum()
        if pv != 0 and np.isfinite(rest / pv) and abs(rest / pv) < 1e30:
            blocks[r, -1, 12:16] = np.frombuffer(f32(-rest / pv).tobytes(), np.uint8)
    return blocks


def q4k_act_from_region(act, n):
    codes = np.empty(n, np.uint8)
    codes[0::2] = act[: n // 2]; codes[1::2] = act[n // 2: n]
    rec = act[n: n + (n // 32) * 16].view(f32).reshape(-1, 4)
    return codes, rec[:, 0].copy(), rec[:, 1].copy()


def q4k_check(got, blocks, xc, sq, bq, what):
    subs, factor = q4k_terms(blocks, xc, sq, bq)
    ref = (subs[..., 0] - subs[..., 1] - subs[..., 2] + subs[..., 3]).sum(1)
    return check_bound(got, ref, xc.size // 32, np.abs(subs), factor, what)


def q4k_planes(blocks):
    """(nibble plane [R, n / 2], side records [R, n / 256 * 20]) as the engine holds a Q4K matrix"""
    return blocks[:, :, 32:160].reshape(R, -1).copy(), blocks[:, :, 12:32].reshape(R, -1).copy()


@gpu
@pytest.mark.parametrize("n", [256, 512, 1280, 3840, 4096, 7680])
def test_stream_q4k_dots(probe, n):
    x = tiled(q4k_edge_vector(), n, n + 1)
    hc, hsq, hbq = q4k_reference(o_q4k_quant(x), n)
    blocks = q4k_cancel(q4k_weight_blocks(x, n), hc, hsq, hbq)
    main, side = q4k_planes(blocks)
    runs = []
    for tile_rows in (0, 5):
        got, act = stream_dots(probe, 0x42, 8, 2, x, main, side, tile_rows=tile_rows)
        runs.append((f"tile {tile_rows}", got))
    same_bits(runs, f"st_row_q4k n {n}")
    xc, sq, bq = q4k_act_from_region(act, n)
    q4k_check(runs[0][1], blocks, xc, sq, bq, f"st_row_q4k n {n}")


@gpu
@pytest.mark.parametrize("n", [256, 512, 1280, 3840, 4096, 7680, 9728])
def test_multikernel_q4k_dots(probe, n):
    x = tiled(q4k_edge_vector(), n, n + 2)
    xc, sq, bq = q4k_reference(o_q4k_quant(x), n)
    blocks = q4k_cancel(q4k_weight_blocks(x, n + 1), xc, sq, bq)
    main, side = q4k_planes(blocks)
    act = np.zeros(act_bytes(0x42, n, 1), np.uint8)
    act[: n // 2] = xc[0::2]; act[n // 2: n] = xc[1::2]
    rec = np.zeros((n // 32, 4), f32)
    rec[:, 0] = sq; rec[:, 1] = bq; rec[:, 2] = xc.reshape(-1, 32).sum(1)
    act[n: n + rec.nbytes] = rec.view(np.uint8).reshape(-1)
    runs = [(f"RB {rb}", mk_dots(probe, 0x42, 8, False, rb, main, side, n, act)) for rb in (1, 2, 4)]
    same_bits(runs, f"rows_q4k<RB> n {n}")
    q4k_check(runs[0][1], blocks, xc, sq, bq, f"rows_q4k<1|2|4> n {n}")


# ---------------------------------------------------------------- F32
def f32_vector(n, seed):
    """normal values with tiny, subnormal, zero and large stretches"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n)
    k = n // 8
    x[:k] *= 1e-30; x[k: 2 * k] *= 1e-42; x[2 * k: 2 * k + 8] = 0.0; x[3 * k: 4 * k] *= 1e20
    return x.astype(f32)


def f32_weights(x, seed):
    n = x.size
    rng = np.random.default_rng(seed)
    W = rng.standard_normal((R, n))
    for r in range(R):
        kind = r % 8
        if kind == 1:
            W[r] = np.where(rng.random(n) < 0.5, 1.0, -1.0) * 3e4
        elif kind == 3:
            W[r, ::3] = 0.0
        elif kind == 4:
            W[r] *= 1e-40
        elif kind == 5:
            W[r] *= 1e25
        elif kind == 7:
            W[r] *= 10.0 ** rng.integers(-40, 30, n)
    lim = np.minimum(TERM_MAX / np.maximum(np.abs(x.astype(f64)), 1e-45), W_MAX)
    W = np.clip(W, -lim, lim).astype(f32)
    h = int(np.argmax(np.abs(x)))
    for r in range(6, R, 8):                                                                   # cancels to about 0
        c = (W[r].astype(f64) * x).sum() - f64(W[r, h]) * x[h]
        W[r, h] = f32(-c / f64(x[h]))
    return W


def f32_check(got, x, W, what):
    p = W.astype(f64) * x.astype(f64)
    return check_bound(got, p.sum(1), x.size // 4, np.abs(p), np.zeros_like(p), what)


F32_N = [208, 4000, 3840, 3968, 4096, 7680, 11520]


@gpu
@pytest.mark.parametrize("n", F32_N)
def test_stream_f32_dots(probe, n):
    x = f32_vector(n, n)
    W = f32_weights(x, n + 3)
    runs = []
    for tile_rows in (0, 3):
        got, act = stream_dots(probe, 0x00, 8, 3, x, W, None, tile_rows=tile_rows)
        runs.append((f"tile {tile_rows}", got))
    assert np.array_equal(act[: n * 4].view(np.uint32), x.view(np.uint32)), "operand region"
    same_bits(runs, f"st_row_f32 n {n}")
    f32_check(runs[0][1], x, W, f"st_row_f32 n {n}")


@gpu
@pytest.mark.parametrize("n", F32_N)
def test_multikernel_f32_dots(probe, n):
    x = f32_vector(n, n + 5)
    W = f32_weights(x, n + 7)
    act = np.zeros(act_bytes(0x00, n, 1), np.uint8)
    act[: n * 4] = x.view(np.uint8)
    runs = [(f"RB {rb}", mk_dots(probe, 0x00, 8, False, rb, W, None, n, act)) for rb in (1, 2, 4)]
    same_bits(runs, f"rows_f32<RB> n {n}")
    f32_check(runs[0][1], x, W, f"rows_f32<1|2|4> n {n}")
