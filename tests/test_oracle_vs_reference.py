"""CPU tests: pin the oracle (oracle/nano_oracle.c) to the reference and to the committed goldens.

The reference has no test suite (SURVEY section 4); what pins behaviour is the embedded sort model
(infer/main_sort.c:6-3098, README.md:379) plus outputs of the unmodified strict reference, stored under tests/golden/
(SHA-256 digests in reference_outputs.json where the comparison is bit-exact; tests/golden/make_golden.py regenerates them).
"""
import json
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, assert_bits_equal
from nano_b200 import modelfile as mf
from oracle import bindings as ob

sys.path.insert(0, GOLDEN)
from make_golden import (LORA_CASES, STRICT_CASES, STRICT_SEQ, TOY_POSITIONS, q4k_writer_input,  # noqa: E402
                         q80_ops_inputs, sha)
sys.path.remove(GOLDEN)

REF_OUT = json.load(open(os.path.join(GOLDEN, "reference_outputs.json")))

TOY = [("toy-nano", mf.QUANT_F32, 128), ("toy-nano", mf.QUANT_Q80, 64), ("toy-nano", mf.QUANT_Q4K, 128),
       ("toy-qwen3", mf.QUANT_F32, 128), ("toy-qwen3", mf.QUANT_Q80, 64), ("toy-qwen3", mf.QUANT_Q4K, 128)]


def seq2seq_ids(eng, ids):
    """seq2seq of infer.c:1365-1402 restated over a forward(token,pos,causal=0) callable."""
    n = len(ids)
    for _ in range(eng.n_layer):
        for p in range(n):
            eng.forward(ids[p], p, 0)
    return [int(np.argmax(eng.forward(ids[p], p, 0))) for p in range(n)]


def test_sort_model_known_answers_oracle(sort_model):
    kat = json.load(open(os.path.join(GOLDEN, "sort6_kat.json")))
    assert kat["114515"] == "111455"          # README.md:379
    for src, want in kat.items():
        o = ob.NanoOracle(sort_model, 6)
        got = seq2seq_ids(o, [17 + int(c) for c in src])     # digits are ids 17..26 (tokenizer/nano_80.json)
        assert "".join(str(t - 17) for t in got) == want, (src, got)
        o.close()


def test_sort_model_fixture_is_the_embedded_one(sort_model):
    """the committed fixture is byte for byte the model embedded in the reference (its seq2seq answers are sort6_kat.json)"""
    assert sha(sort_model) == REF_OUT["sort6_model"]


@pytest.mark.parametrize("name,quant,gs", TOY)
def test_oracle_matches_golden_logits(name, quant, gs):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    gold = np.load(os.path.join(GOLDEN, "toy_logits.npz"))[f"{name}_{quant:02x}_{gs}"]
    o = ob.NanoOracle(path, 24)
    toks = mf.teacher_tokens(24, spec.vocab)
    rows = []
    for pos in range(24):
        lg = o.forward(toks[pos], pos)
        if pos in (0, 1, 7, 23):
            rows.append(lg)
    assert_bits_equal(np.stack(rows), gold, f"{name} {quant:#x}")
    o.close()


@pytest.mark.parametrize("name,quant,gs", STRICT_CASES)
def test_oracle_bit_identical_to_strict_reference(name, quant, gs):
    spec = mf.PRESETS[name]
    path = mf.cached_model(spec, quant, gs)
    want = REF_OUT["strict"][f"{name}_{quant:02x}_{gs}"]
    o = ob.NanoOracle(path, STRICT_SEQ)
    toks = mf.teacher_tokens(STRICT_SEQ, spec.vocab)
    for pos in range(STRICT_SEQ):
        assert sha(o.forward(toks[pos], pos)) == want["logits"][pos], f"{name} pos {pos}: logits differ from the strict reference"
    ok, ov = o.kv()
    assert sha(ok) == want["k_cache"], "k cache"
    assert sha(ov) == want["v_cache"], "v cache"
    o.close()


def test_oracle_greedy_with_penalty_matches_reference():
    spec = mf.PRESETS["toy-nano"]
    path = mf.cached_model(spec, mf.QUANT_Q80, 64)
    S, P = 24, 5
    o = ob.NanoOracle(path, S)
    ids_o = np.zeros(S + 1, np.uint32); ids_o[:P] = [9, 8, 7, 9, 8]
    for pos in range(S - 1):
        ids_o[pos + 1] = o.next_greedy(ids_o, pos, 1 if pos < P - 1 else 0, 1.3)
    assert ids_o.tolist() == REF_OUT["greedy_penalty_1.3_ids"]
    o.close()


def test_q4k_writer_matches_reference_quantiser():
    """nano_b200.modelfile.quantize_q4k_blocks (NumPy) == tensor.c:312 quantize_tensor_q4k, byte for byte."""
    w = q4k_writer_input()
    mine = mf.q4k_frame((37, 512), 37 * 2) + mf.quantize_q4k_blocks(w).tobytes()
    assert sha(mine) == REF_OUT["q4k_tensor"], "q4k tensor bytes"


def test_q4k_kat_oracle():
    """Recipe of infer/tools/export_q4k.c:394-450 (seed 39, d=8, n=768): committed reference outputs."""
    k = np.load(os.path.join(GOLDEN, "q4k_kat.npz"))
    L = ob.NanoOracle.lib()
    W, x = k["W"], k["x"]
    wb = np.zeros(8 * 3 * 160, np.uint8); xb = np.zeros(3 * 160, np.uint8)
    L.nor_q4k_quantize_rows(wb.ctypes.data_as(ob.u8p), W.ctypes.data_as(ob.f32p), 8, 768)
    L.nor_q4k_quantize_rows(xb.ctypes.data_as(ob.u8p), x.ctypes.data_as(ob.f32p), 1, 768)
    assert_bits_equal(wb, k["w_tensor"][44:], "weight blocks")
    assert_bits_equal(xb, k["x_tensor"][44:], "activation blocks")
    y = np.zeros(8, np.float32)
    L.nor_matvec_q4k(y.ctypes.data_as(ob.f32p), xb.ctypes.data_as(ob.u8p), wb.ctypes.data_as(ob.u8p), 0, 8, 768)
    assert_bits_equal(y, k["y"], "matmul_q4k")
    assert_bits_equal(mf.quantize_q4k_blocks(W.reshape(8, 768)).reshape(-1), k["w_tensor"][44:], "numpy writer")


def test_q80_ops_match_reference():
    O = ob.NanoOracle.lib()
    x, wq, ws, n, d, gs = q80_ops_inputs()
    q_o = np.zeros(n, np.int8); s_o = np.zeros(n // gs, np.float32)
    O.nor_q80_quantize(q_o.ctypes.data_as(ob.i8p), s_o.ctypes.data_as(ob.f32p), x.ctypes.data_as(ob.f32p), n, gs)
    want = REF_OUT["q80_ops"]
    assert sha(q_o) == want["codes"], "codes"
    assert sha(s_o) == want["scales"], "scales"
    y_o = np.zeros(d, np.float32)
    O.nor_matvec_q80(y_o.ctypes.data_as(ob.f32p), q_o.ctypes.data_as(ob.i8p), s_o.ctypes.data_as(ob.f32p),
                     wq.ctypes.data_as(ob.i8p), ws.ctypes.data, n, d, gs)
    assert sha(y_o) == want["matmul_quant"], "matmul_quant"


def test_expf_ref_equals_host_libm():
    """The exact-mode device expf (csrc/expf_ref.cuh) evaluated on the host == libm expf on sampled floats."""
    from nano_b200 import engine as E
    import struct
    fb = lambda f: struct.unpack("<I", struct.pack("<f", f))[0]
    L = ob.NanoOracle.lib()
    for lo, hi in ((0, fb(89.0)), (0x80000000, fb(-104.5))):
        b = np.arange(lo, hi, 997, dtype=np.uint32)
        x = b.view(np.float32)
        want = np.empty_like(x)
        L.nor_expf_array(want.ctypes.data_as(ob.f32p), x.ctypes.data_as(ob.f32p), x.size)
        assert_bits_equal(E.host_expf_ref(x), want, "expf")


def test_lora_golden_is_what_the_reference_computes():
    """Pins tests/golden/lora_logits.npz (the GPU LoRA tests' fixture) to the strict reference's digests with the same synthetic
    plug-in, checks that the plug-in writer's layout is the one parse_lora_file reads (infer.c:436-500), and that the plug-in
    changes the reference's logits (toy_logits.npz holds them without it)."""
    spec = mf.PRESETS["toy-nano"]
    lora = mf.write_lora(spec, 8, 16, seed=7)
    assert len(lora) == 256 + 4 * spec.n_layer * 8 * (4 * spec.n_embd + 2 * spec.n_embd + 2 * spec.kv_dim)
    gold = np.load(os.path.join(GOLDEN, "lora_logits.npz"))
    base = np.load(os.path.join(GOLDEN, "toy_logits.npz"))
    for quant, gs in LORA_CASES[:2]:
        key = f"toy-nano_{quant:02x}_{gs}"
        for i, pos in enumerate(TOY_POSITIONS):
            assert sha(gold[key][i]) == REF_OUT["lora"][key]["logits"][pos], f"lora golden {quant:#x} pos {pos}"
            assert np.abs(gold[key][i] - base[key][i]).max() > 1e-2, "the plug-in must change the logits"


@pytest.mark.skipif(not ob.ref_available("strict"), reason="needs the unmodified reference (oracle/_ref)")
@pytest.mark.parametrize("quant,gs", LORA_CASES)
def test_reference_harness_takes_the_plug_in_per_call(quant, gs):
    """RefEngine.forward(..., lora=): with the plug-in loaded, lora=True is what the reference computes with it and lora=False
    (what seq2seq passes) what it computes for the plain model -- both against the committed strict-reference digests."""
    if not ob.ref_has_forward_lora():
        pytest.skip("the reference harness in oracle/_ref predates orh_forward_lora (llm_forward without the plug-in)")
    spec = mf.PRESETS["toy-nano"]
    key = f"toy-nano_{quant:02x}_{gs}"
    path = mf.cached_model(spec, quant, gs)
    toks = mf.teacher_tokens(len(REF_OUT["lora"][key]["logits"]), spec.vocab)
    r = ob.RefEngine(path, len(toks), "strict"); r.load_lora(mf.write_lora(spec, 8, 16, seed=7))
    for pos, want in enumerate(REF_OUT["lora"][key]["logits"]):
        assert sha(r.forward(toks[pos], pos, lora=True)) == want, f"with the plug-in, pos {pos}"
    for pos, want in enumerate(REF_OUT["strict"][key]["logits"]):
        assert sha(r.forward(toks[pos], pos, lora=False)) == want, f"without the plug-in, pos {pos}"
    r.close()
