"""CPU tests of the host-side framing helpers of the reference API that our shim re-implements (tensor.h:153-163):
dequantize, parse_quantized_tensors, bytes_num_of_q4k_tensor, make_q4k_tensor, dequantize_tensor_q4k, pack_q4k_tensor,
unpack_q4k_tensor -- called on the SAME host buffers as the unmodified reference (oracle/_ref strict build) and compared bit for
bit.  The inputs are produced by the reference's own CPU quantisers, so no GPU is involved (VERDICT r1 rows a16 / a17)."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import assert_bits_equal
from nano_b200 import build as nb_build
from oracle import bindings as ob

REF_SO = os.path.join(ob.REF_DIR, "libnano_ref_strict.so")
pytestmark = pytest.mark.skipif(not (os.path.exists(REF_SO) and os.path.exists(nb_build.SHIM_SO) and os.path.exists(ob.REFHOST_SO)),
                                reason="needs oracle/_ref (reference build) and the shim libraries")

f32p, u32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)


class Q80(C.Structure):                # tensor.h:87-90
    _fields_ = [("q", C.c_void_p), ("s", C.c_void_p)]


def _proto(L):
    L.dequantize.argtypes = [C.POINTER(Q80), f32p, C.c_int, C.c_uint32]
    L.parse_quantized_tensors.restype = C.c_void_p
    L.parse_quantized_tensors.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_uint32]
    L.bytes_num_of_q4k_tensor.restype = C.c_uint64
    L.bytes_num_of_q4k_tensor.argtypes = [C.c_void_p]
    L.make_q4k_tensor.restype = C.c_void_p
    L.make_q4k_tensor.argtypes = [C.c_uint32, u32p]
    L.dequantize_tensor_q4k.argtypes = [C.c_void_p, f32p, u32p, u32p]
    L.pack_q4k_tensor.restype = C.c_void_p
    L.pack_q4k_tensor.argtypes = [C.c_void_p]
    L.unpack_q4k_tensor.restype = C.c_void_p
    L.unpack_q4k_tensor.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    return L


@pytest.fixture(scope="module")
def libs():
    C.CDLL(ob.REFHOST_SO, mode=C.RTLD_GLOBAL)            # the reference's tokenizer / utils / HAL objects the shim links against
    ref = _proto(C.CDLL(REF_SO, mode=C.RTLD_LOCAL))
    ref.quantize_tensor_q4k.restype = C.c_void_p
    ref.quantize_tensor_q4k.argtypes = [f32p, C.c_uint32, u32p]
    ref.quantize.argtypes = [C.POINTER(Q80), f32p, C.c_int, C.c_uint32]
    ours = _proto(C.CDLL(nb_build.SHIM_SO, mode=C.RTLD_LOCAL))
    return ref, ours


def _image(L, T):
    return np.frombuffer(C.string_at(T, L.bytes_num_of_q4k_tensor(T)), np.uint8).copy()


@pytest.mark.parametrize("shape", [[256], [3, 512], [2, 5, 768]])
def test_q4k_framing_helpers_match_the_reference(libs, shape):
    ref, ours = libs
    rng = np.random.default_rng(len(shape))
    t = (rng.standard_normal(shape, dtype=np.float32) * np.float32(0.3)).astype(np.float32)
    sh = (C.c_uint32 * len(shape))(*shape)
    T = ref.quantize_tensor_q4k(t.ctypes.data_as(f32p), len(shape), sh)          # the reference's CPU quantiser makes the input
    # size and raw image
    assert ours.bytes_num_of_q4k_tensor(T) == ref.bytes_num_of_q4k_tensor(T)
    # an empty tensor of the same shape has the same header fields and size (tensor.c:76-111)
    a, b = ref.make_q4k_tensor(len(shape), sh), ours.make_q4k_tensor(len(shape), sh)
    ia, ib = _image(ref, a), _image(ref, b)
    nhdr = 8 + 4 + 4 + 24 + 4                                                    # tensor.h:129-134: bytes, header, ndim, shape[6], num_blocks
    assert_bits_equal(ib[:nhdr], ia[:nhdr], "make_q4k_tensor header")
    assert ib.size == ia.size
    # dequantise the reference's tensor with both implementations
    n = int(np.prod(shape))
    out_r, out_o = np.zeros(n, np.float32), np.zeros(n, np.float32)
    nd_r, nd_o = C.c_uint32(0), C.c_uint32(0)
    sh_r, sh_o = (C.c_uint32 * 6)(), (C.c_uint32 * 6)()
    ref.dequantize_tensor_q4k(T, out_r.ctypes.data_as(f32p), C.byref(nd_r), sh_r)
    ours.dequantize_tensor_q4k(T, out_o.ctypes.data_as(f32p), C.byref(nd_o), sh_o)
    assert nd_o.value == nd_r.value == len(shape) and list(sh_o)[:len(shape)] == list(sh_r)[:len(shape)] == shape
    assert_bits_equal(out_o, out_r, "dequantize_tensor_q4k")
    # pack / unpack round trip (tensor.c: the packed form is the tensor image itself)
    pr, po = ref.pack_q4k_tensor(T), ours.pack_q4k_tensor(T)
    assert_bits_equal(_image(ref, po), _image(ref, pr), "pack_q4k_tensor")
    tot_r, tot_o = C.c_uint64(0), C.c_uint64(0)
    ur, uo = ref.unpack_q4k_tensor(pr, C.byref(tot_r)), ours.unpack_q4k_tensor(pr, C.byref(tot_o))
    assert tot_o.value == tot_r.value
    assert_bits_equal(_image(ref, uo), _image(ref, ur), "unpack_q4k_tensor")


@pytest.mark.parametrize("gs", [32, 64, 128])
def test_q80_parse_and_dequantize_match_the_reference(libs, gs):
    """parse_quantized_tensors walks a file-layout buffer of n tensors [int8 codes | fp32 scales] (tensor.c:49-62); dequantize tensor.c:12-17."""
    ref, ours = libs
    n_t, size_each = 3, 4 * gs * 5
    rng = np.random.default_rng(gs)
    x = rng.standard_normal((n_t, size_each), dtype=np.float32)
    buf = np.zeros(n_t * (size_each + 4 * (size_each // gs)), np.uint8)
    off = 0
    for i in range(n_t):                                                         # the reference's CPU quantiser fills the buffer in file layout
        q = Q80(buf.ctypes.data + off, buf.ctypes.data + off + size_each)
        ref.quantize(C.byref(q), x[i].ctypes.data_as(f32p), size_each, gs)
        off += size_each + 4 * (size_each // gs)
    pr, po = C.c_void_p(buf.ctypes.data), C.c_void_p(buf.ctypes.data)
    tr = ref.parse_quantized_tensors(C.byref(pr), n_t, size_each, gs)
    to = ours.parse_quantized_tensors(C.byref(po), n_t, size_each, gs)
    assert po.value == pr.value == buf.ctypes.data + buf.size                    # both advance the cursor past the n tensors
    ar = np.frombuffer(C.string_at(tr, n_t * 16), np.uint64)                     # Typed_Tensor = union of {q, s} pointers (16 bytes)
    ao = np.frombuffer(C.string_at(to, n_t * 16), np.uint64)
    assert_bits_equal(ao, ar, "parse_quantized_tensors")
    for i in range(n_t):
        q = Q80(int(ar[2 * i]), int(ar[2 * i + 1]))
        yr, yo = np.zeros(size_each, np.float32), np.zeros(size_each, np.float32)
        ref.dequantize(C.byref(q), yr.ctypes.data_as(f32p), size_each, gs)
        ours.dequantize(C.byref(q), yo.ctypes.data_as(f32p), size_each, gs)
        assert_bits_equal(yo, yr, f"dequantize tensor {i}")
        assert np.abs(yr - x[i]).max() < np.abs(x[i]).max() / 100.0              # and it is a dequantisation of what went in
