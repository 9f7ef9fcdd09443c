"""Bit-level check of the streaming kernel's activation prologue (st_prep, nano_b200/csrc/stream.cuh).

The prologue's Q80 codes and scales and its Q4K blocks live only in shared memory, and logits cannot show a wrong code in
a group whose scale is ~1e-39.  tests/stream_prep_probe.cu runs st_prep<QUANT, LPG> alone, for <0x80, 8>, <0x80, 4>,
<0x00, 8> and <0x42, 8>, on vectors given as exchange words (every word already carries the awaited epoch) or in shared
memory, and returns its operand region.  Without a gain: Q80 codes and scales equal tensor.c:21-46 (the oracle) bit for
bit, Q4K codes and group records equal the oracle's blocks, F32 values pass through unchanged; with a gain the F32
output is within a few ulp of a float64 rmsnorm.  Lengths run from one group to st_prep_max_n, so both poll batches and
the later batches' re-read are covered, and the Q80 / Q4K inputs are the quantiser edge vectors of test_gpu_ops.py.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from nano_b200 import build as nb_build
from oracle import bindings as ob
from test_gpu_ops import o_q4k_quant, o_q80_quant, q4k_edge_vector, q80_edge_vector

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def probe():
    d = tempfile.mkdtemp(prefix="nb200_probe_")
    so = os.path.join(d, "libprobe.so")
    subprocess.run([nb_build.NVCC, *nb_build.GENCODE, "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                    "-I" + nb_build.CSRC, os.path.join(HERE, "stream_prep_probe.cu"), "-o", so], check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    lib = C.CDLL(so)
    lib.probe_prep.argtypes = [C.c_int, C.c_int, C.c_int, ob.f32p, ob.f32p, C.c_uint32, ob.u8p, C.c_uint32]

    def run(quant, lpg, shared, x, gain=None):
        x = np.ascontiguousarray(x, np.float32)
        gs = lpg * 16 if quant == 0x80 else 1
        nbytes = {0x00: x.size * 4, 0x80: ((x.size + 15) & ~15) + (x.size // gs) * 4 + 16, 0x42: x.size + (x.size // 32) * 16}[quant]
        out = np.zeros((nbytes + 15) & ~15, np.uint8)
        g = None if gain is None else np.ascontiguousarray(gain, np.float32)
        rc = lib.probe_prep(quant, lpg, int(shared), x.ctypes.data_as(ob.f32p), None if g is None else g.ctypes.data_as(ob.f32p),
                            x.size, out.ctypes.data_as(ob.u8p), out.size)
        assert rc == 0, f"probe_prep returned {rc}"
        return out
    return run


def tiled(edge, n, seed):
    """`edge` interleaved with normal groups of the same size, repeated to n elements (edge groups land in every batch)."""
    rng = np.random.default_rng(seed)
    return np.resize(np.concatenate([edge, rng.standard_normal(edge.size).astype(np.float32)]), n).astype(np.float32)


@pytest.mark.parametrize("shared", [0, 1], ids=["exchange", "shared"])
@pytest.mark.parametrize("lpg,n", [(8, 128), (8, 1920), (8, 3840), (8, 3968), (8, 7808), (8, 11520),
                                   (4, 64), (4, 3904), (4, 7680), (4, 11520)])
def test_q80_codes_and_scales(probe, lpg, n, shared):
    gs = lpg * 16
    x = tiled(q80_edge_vector(gs), n, n + gs)
    out = probe(0x80, lpg, shared, x)
    q = out[:n].view(np.int8)
    s = out[(n + 15) & ~15: ((n + 15) & ~15) + (n // gs) * 4].view(np.float32)
    wq, ws = o_q80_quant(x, gs)
    assert np.array_equal(s.view(np.uint32), ws.view(np.uint32)), f"scales differ in groups {np.nonzero(s.view(np.uint32) != ws.view(np.uint32))[0][:8]}"
    bad = np.nonzero(q != wq)[0]
    assert bad.size == 0, f"{bad.size} codes differ; first at {bad[:4]} (group {bad[0] // gs}, amax {np.abs(x[bad[0] // gs * gs:][:gs]).max():.3e}): {q[bad[:4]]} vs {wq[bad[:4]]}"


def q4k_reference(blocks, n):
    """codes [n], group scale and bias [n / 32] of the oracle's blocks (tensor.c:113-141, 253-278)"""
    b = blocks.reshape(-1, 160)
    nib = b[:, 32:160]
    codes = np.empty((b.shape[0], 256), np.uint8)
    codes[:, 0::2] = nib & 0x0F; codes[:, 1::2] = nib >> 4
    ss = b[:, 12:16].copy().view(np.float32)[:, 0]; sb = b[:, 16:20].copy().view(np.float32)[:, 0]
    q = b[:, 20:32].astype(np.uint32)
    s6 = np.concatenate([q[:, 0:4] & 0x3F, (((q[:, 0:4] >> 6) << 4) | (q[:, 8:12] & 0x0F)) & 0x3F], axis=1)
    b6 = np.concatenate([q[:, 4:8] & 0x3F, (((q[:, 4:8] >> 6) << 4) | (q[:, 8:12] >> 4)) & 0x3F], axis=1)
    gsc = (s6.astype(np.float32) * ss[:, None]).astype(np.float32)
    gbi = (b6.astype(np.float32) * sb[:, None]).astype(np.float32)
    return codes.reshape(n), gsc.reshape(-1), gbi.reshape(-1)


@pytest.mark.parametrize("shared", [0, 1], ids=["exchange", "shared"])
@pytest.mark.parametrize("n", [256, 3840, 4096, 7680])
def test_q4k_codes_and_group_records(probe, n, shared):
    x = tiled(q4k_edge_vector(), n, n)
    out = probe(0x42, 8, shared, x)
    codes = np.empty(n, np.uint8)
    codes[0::2] = out[: n // 2]; codes[1::2] = out[n // 2: n]          # even / odd elements, one byte each
    rec = out[n: n + (n // 32) * 16].view(np.float32).reshape(-1, 4)  # {group scale, group bias, sum of codes, 0}
    wc, wsc, wbi = q4k_reference(o_q4k_quant(x), n)
    assert np.array_equal(codes, wc), f"codes differ at {np.nonzero(codes != wc)[0][:8]}"
    assert np.array_equal(rec[:, 0].view(np.uint32), wsc.view(np.uint32)), "group scales"
    assert np.array_equal(rec[:, 1].view(np.uint32), wbi.view(np.uint32)), "group biases"
    assert np.array_equal(rec[:, 2], wc.reshape(-1, 32).sum(axis=1).astype(np.float32)), "code sums"


@pytest.mark.parametrize("shared", [0, 1], ids=["exchange", "shared"])
@pytest.mark.parametrize("n", [208, 3840, 4000, 11520])
def test_f32_passthrough_and_rmsnorm(probe, n, shared):
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n).astype(np.float32)
    assert np.array_equal(probe(0x00, 8, shared, x)[: n * 4].view(np.uint32), x.view(np.uint32)), "values without a gain"
    g = (1 + 0.1 * rng.standard_normal(n)).astype(np.float32)
    got = probe(0x00, 8, shared, x, g)[: n * 4].view(np.float32)
    x64 = x.astype(np.float64)
    want = g.astype(np.float64) * x64 / np.sqrt(np.mean(x64 * x64) + 1e-5)
    ulps = np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    assert ulps.max() <= 8, f"rmsnorm: {ulps.max():.1f} ulp at {int(np.argmax(ulps))}"
