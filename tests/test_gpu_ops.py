"""GPU parity tests, op level (through the C-ABI nb200_op_* entry points).

Bar: bit-exact for integer/byte work (activation codes, Q80/Q4K matvec results, which are fp32 combines of
exact integer dots in the reference's order); fp32 tree reductions within 1e-6 relative of the oracle in fast
mode and bit-exact in exact mode.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN, assert_bits_equal
from nano_b200 import engine as E, modelfile as mf
from oracle import bindings as ob

pytestmark = pytest.mark.gpu
O = None


def oracle():
    global O
    if O is None:
        O = ob.NanoOracle.lib()
    return O


def o_rmsnorm(x, g):
    out = np.empty_like(x)
    oracle().nor_rmsnorm(out.ctypes.data_as(ob.f32p), x.ctypes.data_as(ob.f32p), g.ctypes.data_as(ob.f32p), x.size)
    return out


def o_q80_quant(x, gs):
    q = np.zeros(x.size, np.int8); s = np.zeros(x.size // gs, np.float32)
    oracle().nor_q80_quantize(q.ctypes.data_as(ob.i8p), s.ctypes.data_as(ob.f32p), x.ctypes.data_as(ob.f32p), x.size, gs)
    return q, s


def o_q80_matvec(x, wq, ws, n, d, gs):
    q, s = o_q80_quant(x, gs)
    y = np.zeros(d, np.float32)
    oracle().nor_matvec_q80(y.ctypes.data_as(ob.f32p), q.ctypes.data_as(ob.i8p), s.ctypes.data_as(ob.f32p),
                            wq.ctypes.data_as(ob.i8p), ws.ctypes.data, n, d, gs)
    return y


def o_q4k_quant(x):
    b = np.zeros((x.size // 256) * 160, np.uint8)
    oracle().nor_q4k_quantize_rows(b.ctypes.data_as(ob.u8p), x.ctypes.data_as(ob.f32p), 1, x.size)
    return b


def edgey(rng, n):
    x = rng.standard_normal(n, dtype=np.float32)
    x[: min(32, n)] = 0.0                                      # all-zero group
    if n >= 96:
        x[32:64] = np.abs(x[32:64]) + np.float32(0.1)          # all-positive
        x[64:96] = -np.abs(x[64:96]) - np.float32(0.1)         # all-negative
    x[n // 2] = np.float32(3.5)                                # likely group max -> code 127 / ties nearby
    return x


@pytest.mark.parametrize("n", [32, 48, 768, 1024, 2560])
def test_rmsnorm_fast_and_exact(n):
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n, dtype=np.float32); g = (1 + 0.02 * rng.standard_normal(n, dtype=np.float32)).astype(np.float32)
    want = o_rmsnorm(x, g)
    got = E.op_rmsnorm(x, g, exact=0)
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max() + 1e-7
    assert_bits_equal(E.op_rmsnorm(x, g, exact=1), want, "exact rmsnorm")


@pytest.mark.parametrize("gs", [32, 64, 128, 256])
@pytest.mark.parametrize("n", [256, 768, 3072])
def test_q80_quantize_bit_exact(n, gs):
    x = edgey(np.random.default_rng(n + gs), n)
    q, s = E.op_q80_quantize(x, gs)
    wq, ws = o_q80_quant(x, gs)
    assert_bits_equal(s, ws, "scales"); assert_bits_equal(q, wq, "codes")


def test_q80_quantize_half_ties():
    """x/scale landing exactly on .5 must round away from zero (C round(), tensor.c:42)."""
    gs = 128
    x = np.zeros(gs, np.float32)
    x[0] = 127.0                       # scale = 1.0 exactly
    x[1:9] = [0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.5, -126.5]
    q, s = E.op_q80_quantize(x, gs)
    assert s[0] == 1.0
    assert q[1:9].tolist() == [1, 2, 3, -1, -2, -3, 127, -127]
    wq, _ = o_q80_quant(x, gs)
    assert_bits_equal(q, wq, "codes")


def q80_edge_vector(gs):
    """One group per edge case: a scale reciprocal that overflows (amax just below ~3.74e-37) or just does not, subnormal
    amax, signed zeros only, a single nonzero element, a negative maximum, exact .5 ties at scales other than 1, values
    5e-5 and 2e-3 from a tie, amax near FLT_MAX, and normal groups in between (mixed tiny and normal groups in one vector)."""
    rng = np.random.default_rng(gs)
    f = np.float32
    groups = []

    def grp(amax, sign=1.0):
        g = (rng.uniform(-1, 1, gs).astype(np.float32) * f(amax)).astype(np.float32)
        g[rng.integers(gs)] = f(sign) * f(amax)
        return g
    for amax in (3.6e-37, 3.7e-37, 3.73e-37, 3.75e-37, 3.8e-37, 1e-36, 1.17549435e-38):   # around the rinv overflow, FLT_MIN
        groups += [grp(amax), rng.standard_normal(gs).astype(np.float32)]
    for amax in (1e-40, 1.4e-45 * 5, 1.4e-45):                                              # subnormal amax
        groups.append(grp(amax))
    z = np.zeros(gs, np.float32); z[1::2] = -0.0
    groups.append(z)                                                                        # +-0 only
    one = np.zeros(gs, np.float32); one[gs // 3] = f(-2.5e-3)
    groups.append(one)                                                                      # a single nonzero element
    groups.append(grp(7.25, -1.0))                                                          # negative maximum
    for sc in (f(0.375), f(3.0517578125e-05), f(96.0)):                                     # exact ties at scale sc
        t = np.zeros(gs, np.float32)
        t[0] = f(127) * sc
        k = np.arange(1, gs) % 126
        t[1:] = ((k + f(0.5)) * sc * np.where(np.arange(1, gs) % 2, 1, -1)).astype(np.float32)
        groups.append(t)
        # x / scale 5e-5 from a tie (inside the fast path's 1e-3 fallback window) and 2e-3 from one (just outside it)
        nt = t.copy()
        off = np.array([5e-5, -5e-5, 2e-3, -2e-3], np.float32)[np.arange(1, gs) % 4]
        nt[1:] = ((k + f(0.5) + off) * sc * np.where(np.arange(1, gs) % 2, 1, -1)).astype(np.float32)
        groups.append(nt)
    groups += [grp(3.4e38), grp(3.3e38, -1.0), grp(1.7e38), grp(9e37)]                       # amax near FLT_MAX, above 2^126
    return np.concatenate(groups).astype(np.float32)


@pytest.mark.parametrize("gs", [32, 64, 128, 256])
def test_q80_quantize_edges_bit_exact(gs):
    """Codes and scales bit-identical to tensor.c:21-46 on groups at the edges of the float range.  With amax < ~3.74e-37
    the scale amax/127 is below 1/FLT_MAX and its reciprocal overflows: the fast path must fall back to the division."""
    x = q80_edge_vector(gs)
    q, s = E.op_q80_quantize(x, gs)
    wq, ws = o_q80_quant(x, gs)
    assert_bits_equal(s, ws, "scales")
    bad = np.nonzero(q != wq)[0]
    assert bad.size == 0, f"{bad.size} codes differ; first at {bad[:4]} (group {bad[0] // gs}): {q[bad[:4]]} vs {wq[bad[:4]]}"


def q4k_edge_vector():
    """Constant blocks (positive, negative, zero), tiny and huge blocks, all-negative and all-positive blocks, one
    nonzero element, and a block that mixes the extremes group by group."""
    rng = np.random.default_rng(11)
    f = np.float32
    blocks = [np.full(256, f(0.75)), np.full(256, f(-1.25)), np.zeros(256, np.float32),
              rng.standard_normal(256).astype(np.float32) * f(1e-38), rng.standard_normal(256).astype(np.float32) * f(1e-42),
              rng.standard_normal(256).astype(np.float32) * f(1e36), rng.uniform(-1.5e38, 1.5e38, 256).astype(np.float32),
              -np.abs(rng.standard_normal(256)).astype(np.float32) - f(0.5), np.abs(rng.standard_normal(256)).astype(np.float32) + f(0.5)]
    one = np.zeros(256, np.float32); one[77] = f(-3.0)
    blocks.append(one)
    mix = rng.standard_normal(256).astype(np.float32)
    mix[0:32] *= f(1e-39); mix[32:64] *= f(1e30); mix[64:96] = f(2.0); mix[96:128] = -np.abs(mix[96:128])
    blocks.append(mix)
    return np.concatenate(blocks).astype(np.float32)


def test_q4k_quantize_edges_bit_exact():
    x = q4k_edge_vector()
    assert_bits_equal(E.op_q4k_quantize(x), o_q4k_quant(x), "q4k activation blocks")
    want = np.zeros((x.size // 256) * 160, np.uint8)
    oracle().nor_q4k_quantize_rows(want.ctypes.data_as(ob.u8p), x.ctypes.data_as(ob.f32p), 1, x.size)
    assert_bits_equal(E.op_q4k_quantize_blocks(x), want, "q4k tensor blocks")


@pytest.mark.parametrize("n,d,gs", [(256, 7, 64), (256, 33, 32), (768, 64, 128), (1024, 1000, 128), (1024, 130, 64),
                                    (3072, 257, 128), (2048, 96, 256), (2560, 50, 128), (9728, 40, 128)])
def test_q80_matvec_bit_exact(n, d, gs):
    rng = np.random.default_rng(n * 7 + d)
    x = edgey(rng, n)
    wq, ws = mf.quantize_q80(rng.standard_normal((d, n), dtype=np.float32) * np.float32(0.02), gs)
    got = E.op_q80_matvec(x, wq, ws, n, d, gs)
    assert_bits_equal(got, o_q80_matvec(x, wq, ws, n, d, gs), "q80 matvec")


@pytest.mark.parametrize("n", [256, 1024, 3072])
def test_q4k_quantize_bit_exact(n):
    x = edgey(np.random.default_rng(n), n)
    assert_bits_equal(E.op_q4k_quantize(x), o_q4k_quant(x), "q4k activation blocks")


@pytest.mark.parametrize("n,d", [(256, 5), (1024, 64), (2048, 130), (3072, 257), (768, 8)])
def test_q4k_matvec_bit_exact(n, d):
    rng = np.random.default_rng(n + d)
    x = edgey(rng, n)
    W = (rng.standard_normal((d, n), dtype=np.float32) * np.float32(0.05)).astype(np.float32)
    wb = mf.quantize_q4k_blocks(W).reshape(-1)
    xb = o_q4k_quant(x)
    want = np.zeros(d, np.float32)
    oracle().nor_matvec_q4k(want.ctypes.data_as(ob.f32p), xb.ctypes.data_as(ob.u8p), wb.ctypes.data_as(ob.u8p), 0, d, n)
    assert_bits_equal(E.op_q4k_matvec(x, wb, n, d), want, "q4k matvec")


@pytest.mark.parametrize("lines,n", [(1, 256), (7, 768), (300, 1024), (70000, 256)])
def test_q4k_quantize_whole_tensor_bit_exact(lines, n):
    """quantize_tensor_q4k_in_situ (tensor.c:281-310): every block of every line, incl. > one 64 Ki-block chunk."""
    x = edgey(np.random.default_rng(lines + n), lines * n)
    got = E.op_q4k_quantize_blocks(x)
    want = np.zeros(got.size, np.uint8)
    oracle().nor_q4k_quantize_rows(want.ctypes.data_as(ob.u8p), x.ctypes.data_as(ob.f32p), lines, n)
    assert_bits_equal(got, want, "q4k tensor blocks")
    if lines * n <= 1 << 16:
        assert_bits_equal(got.reshape(-1, 160), mf.quantize_q4k_blocks(x.reshape(lines, n)).reshape(-1, 160), "vs the NumPy writer")


@pytest.mark.parametrize("n,d", [(256, 5), (1024, 64), (2048, 130), (3072, 257), (768, 8), (2560, 33)])
def test_q4k_matvec_prequantised_blocks_bit_exact(n, d):
    """matmul_q4k (tensor.c:438-471) with x given as blocks, as the reference's own callers pass it."""
    rng = np.random.default_rng(n * 3 + d)
    x = edgey(rng, n)
    W = (rng.standard_normal((d, n), dtype=np.float32) * np.float32(0.05)).astype(np.float32)
    wb = mf.quantize_q4k_blocks(W).reshape(-1)
    xb = o_q4k_quant(x)
    want = np.zeros(d, np.float32)
    oracle().nor_matvec_q4k(want.ctypes.data_as(ob.f32p), xb.ctypes.data_as(ob.u8p), wb.ctypes.data_as(ob.u8p), 0, d, n)
    assert_bits_equal(E.op_q4k_matvec_blocks(xb, wb, n, d), want, "q4k matvec on blocks")


def test_q4k_reference_kat():
    """infer/tools/export_q4k.c:394-450 recipe; outputs committed from the unmodified reference."""
    k = np.load(os.path.join(GOLDEN, "q4k_kat.npz"))
    assert_bits_equal(E.op_q4k_quantize(k["x"]), k["x_tensor"][44:], "activation")
    assert_bits_equal(E.op_q4k_matvec(k["x"], k["w_tensor"][44:], 768, 8), k["y"], "matmul_q4k")
    assert_bits_equal(E.op_q4k_quantize_blocks(k["W"]), k["w_tensor"][44:], "weight tensor")
    assert_bits_equal(E.op_q4k_matvec_blocks(k["x_tensor"][44:], k["w_tensor"][44:], 768, 8), k["y"], "matmul_q4k on blocks")


@pytest.mark.parametrize("n,d", [(16, 32), (32, 80), (768, 100), (2048, 768)])
def test_f32_matvec(n, d):
    rng = np.random.default_rng(n + d)
    x = rng.standard_normal(n, dtype=np.float32); W = rng.standard_normal((d, n), dtype=np.float32) * np.float32(0.02)
    want = np.zeros(d, np.float32)
    oracle().nor_matvec_f32(want.ctypes.data_as(ob.f32p), x.ctypes.data_as(ob.f32p), W.ctypes.data, n, d)
    got = E.op_f32_matvec(x, W, n, d, exact=0)
    assert np.abs(got - want).max() <= 2e-6 * np.abs(W).max() * np.abs(x).max() * n ** 0.5 + 1e-7
    assert_bits_equal(E.op_f32_matvec(x, W, n, d, exact=1), want, "exact f32 matvec")
