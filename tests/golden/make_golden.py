"""Regenerates the committed golden fixtures from the UNMODIFIED reference (strict build).

Run in the build container (needs /root/reference):   python tests/golden/make_golden.py

  sort6_model.bin      the reference's only in-tree fixture: the FP32 sort model embedded in
                       infer/main_sort.c:6-3098 (49,452 bytes), extracted through oracle/ref_harness.c
  sort6_kat.json       seq2seq answers of the reference on it (README.md:379 "114515 -> 111455" and four more)
  toy_logits.npz       teacher-forced logits of the strict reference on seeded synthetic toy files
                       (nano_b200/modelfile.py presets, seed 39) at a few positions, F32 / Q80 / Q4K
  lora_logits.npz      the same with a seeded synthetic LoRA plug-in (rank 8, alpha 16) attached to toy-nano
  q4k_kat.npz          Q4K op-level vectors following the recipe of infer/tools/export_q4k.c:394-450
                       (seed 39 xorshift, d=8, n=768): reference quantize_tensor_q4k bytes + matmul_q4k outputs
  reference_outputs.json  SHA-256 digests of what the strict reference computes for the bit-exact tests (teacher-forced
                       logits and KV caches, greedy ids with a repetition penalty, Q80 / Q4K op outputs, LoRA logits and KV
                       rows), so those tests compare against the reference without it:  python tests/golden/make_golden.py --digests
  export_nano.npz      the reference exporter (export.py) run on the seeded tiny GPT of nano_export_weights(): SHA-256 digests
                       of its F32 / Q80 / LoRA files, the model's RoPE tables and its PyTorch logits over 12 teacher-forced
                       positions:  python tests/golden/make_golden.py --export
  reference_noise_floor.json  max |fast build - strict build| of the reference's logits per quantised test file; the floors of
                       the stream-matrix files alone:  python tests/golden/make_golden.py --floors
"""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from nano_b200 import modelfile as mf            # noqa: E402
from oracle import bindings as ob               # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
TOY_CONFIGS = [("toy-nano", mf.QUANT_F32, 128), ("toy-nano", mf.QUANT_Q80, 64), ("toy-nano", mf.QUANT_Q4K, 128),
               ("toy-qwen3", mf.QUANT_F32, 128), ("toy-qwen3", mf.QUANT_Q80, 64), ("toy-qwen3", mf.QUANT_Q4K, 128)]
TOY_SEQ = 24
TOY_POSITIONS = [0, 1, 7, 23]


def xorshift_f32(n, seed=39):
    """utils.c:959-970 random_f32 stream."""
    M = 0xFFFFFFFFFFFFFFFF
    st = seed
    out = np.zeros(n, np.float32)
    for i in range(n):
        st ^= st >> 12; st ^= (st << 25) & M; st ^= st >> 27
        out[i] = np.float32((((st * 0x2545F4914F6CDD1D) & M) >> 32 >> 8) / 16777216.0)
    return out


def sha(a) -> str:
    """digest of the bytes of an array (or of a bytes object): equal digests <=> bit-identical outputs"""
    return hashlib.sha256(a if isinstance(a, bytes) else np.ascontiguousarray(a).tobytes()).hexdigest()


# shared with the tests that compare against these digests
STRICT_CASES = TOY_CONFIGS + [("toy-nano-odd", mf.QUANT_F32, 128), ("mini-qwen3", mf.QUANT_Q80, 128)]
STRICT_SEQ = 20
LORA_CASES = [(mf.QUANT_F32, 128), (mf.QUANT_Q80, 64), (mf.QUANT_Q4K, 128)]
LORA_KV_POSITIONS = [0, 5, TOY_SEQ - 1]


def q80_ops_inputs():
    rng = np.random.default_rng(3)
    n, d, gs = 512, 40, 64
    x = rng.standard_normal(n, dtype=np.float32)
    x[64:128] = 0.0
    wq, ws = mf.quantize_q80(rng.standard_normal((d, n), dtype=np.float32) * 0.02, gs)
    return x, wq, ws, n, d, gs


def q4k_writer_input():
    rng = np.random.default_rng(7)
    w = (rng.standard_normal((37, 512), dtype=np.float32) * np.float32(0.05)).astype(np.float32)
    w[3, :32] = 0.0                       # all-zero group
    w[5, 32:64] = np.abs(w[5, 32:64])     # all-positive group (bias 0)
    w[6, 64:96] = -np.abs(w[6, 64:96])    # all-negative group (FLT_TRUE_MIN max quirk)
    return w


# tiny Nano GPT of the exporter tests (reference model.py shapes: head_dim 32, GQA 4q / 2kv)
NANO_EXPORT_CONFIG = dict(block_size=32, vocab_size=160, n_layer=2, n_embd=128, n_head=4, n_kv_head=2, n_hidden=256)
NANO_EXPORT_SEQ = 12
NANO_EXPORT_LORA = (4, 8)       # rank, alpha


def nano_export_tokenizer():
    V = NANO_EXPORT_CONFIG["vocab_size"]
    return {"itos": [chr(0x4E00 + i) for i in range(V)], "vocab_size": V, "special_tokens": [chr(0x4E00), chr(0x4E01)]}


def nano_export_weights(seed: int = 5):
    """Seeded state dict of the tiny GPT in the reference's module naming (tied classifier), and a seeded LoRA state dict
    (`layers.<l>.attention.w{q,k,v,o}.lora_{a,b}.weight`).  float32 NumPy arrays."""
    c = NANO_EXPORT_CONFIG
    rng = np.random.default_rng(seed)
    E, F, V, hd = c["n_embd"], c["n_hidden"], c["vocab_size"], c["n_embd"] // c["n_head"]
    KD = c["n_kv_head"] * hd
    w = lambda *shape: (rng.standard_normal(shape, dtype=np.float32) * np.float32(0.06)).astype(np.float32)
    gain = lambda: (1 + 0.1 * rng.standard_normal(E, dtype=np.float32)).astype(np.float32)
    sd = {"tok_embeddings.weight": w(V, E)}
    for l in range(c["n_layer"]):
        p = f"layers.{l}."
        sd.update({p + "attention.wq.weight": w(E, E), p + "attention.wk.weight": w(KD, E), p + "attention.wv.weight": w(KD, E),
                   p + "attention.wo.weight": w(E, E), p + "feed_forward.w1.weight": w(F, E), p + "feed_forward.w2.weight": w(E, F),
                   p + "feed_forward.w3.weight": w(F, E), p + "attention_norm.weight": gain(), p + "ffn_norm.weight": gain()})
    sd["norm.weight"] = gain()
    sd["output.weight"] = sd["tok_embeddings.weight"]
    r = NANO_EXPORT_LORA[0]
    lora = {}
    for l in range(c["n_layer"]):
        for proj, (o, i) in (("wq", (E, E)), ("wk", (KD, E)), ("wv", (KD, E)), ("wo", (E, E))):
            lora[f"layers.{l}.attention.{proj}.lora_a.weight"] = w(r, i)
            lora[f"layers.{l}.attention.{proj}.lora_b.weight"] = w(o, r)
    return sd, lora


def export_digests(reference_root: str = os.path.dirname(ob.REFERENCE_SRC)):
    """export_nano.npz from the reference's own model.py / export.py (needs torch and the reference tree)."""
    import tempfile
    import torch
    sys.path.insert(0, reference_root)
    import model as ref_model                                       # the reference's model.py
    import export as ref_export                                     # the reference's export.py
    sys.path.remove(reference_root)
    sd, lora = nano_export_weights()
    m = ref_model.GPT(ref_model.ModelConfig(**NANO_EXPORT_CONFIG)).float().eval()
    missing, unexpected = m.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in sd.items()}, strict=False)
    assert not unexpected and all(k.endswith("attention.mask") for k in missing), (missing, unexpected)
    m.output.weight = m.tok_embeddings.weight                       # keep the classifier tied, as the reference builds it
    toks = mf.teacher_tokens(NANO_EXPORT_SEQ, NANO_EXPORT_CONFIG["vocab_size"])
    with torch.no_grad():
        logits = np.stack([m(torch.tensor([list(map(int, toks[: p + 1]))], dtype=torch.long))[0][0, -1].float().numpy()
                           for p in range(NANO_EXPORT_SEQ)])
    out = {"freqs_cos": m.freqs_cos.numpy().copy(), "freqs_sin": m.freqs_sin.numpy().copy(), "logits": logits}
    with tempfile.TemporaryDirectory() as td:
        f32, q80, lp = (os.path.join(td, n) for n in ("f32.bin", "q80.bin", "lora.bin"))
        ref_export.export_model(m, nano_export_tokenizer(), f32)
        ref_export.export_quantized(m, nano_export_tokenizer(), q80, group_size=64)
        r, a = NANO_EXPORT_LORA
        ref_export.export_lora({k: torch.from_numpy(v.copy()) for k, v in lora.items()}, {"lora_rank": r, "lora_alpha": a}, m.config, lp)
        for key, path in (("f32_sha256", f32), ("q80_sha256", q80), ("lora_sha256", lp)):
            out[key] = np.array(sha(open(path, "rb").read()))
    np.savez_compressed(os.path.join(HERE, "export_nano.npz"), **out)
    print("export digests written")


# the quantised files of tests/test_gpu_stream_matrix.py
MATRIX_FLOOR_CASES = ([(n, q, g) for n in ("kvm1-nano", "kvm4-qwen3-hd128", "kvm4-qwen3-hd64", "ffn3840-nano")
                       for q, g in ((mf.QUANT_Q80, 128), (mf.QUANT_Q80, 64), (mf.QUANT_Q4K, 128))] +
                      [("qwen3-4b-2l", mf.QUANT_Q80, 128), ("ffn3968-nano", mf.QUANT_Q80, 128), ("ffn3968-nano", mf.QUANT_Q80, 64),
                       ("ffn4096-nano", mf.QUANT_Q4K, 128), ("ffn4096-nano", mf.QUANT_Q80, 64), ("ffn7680-nano", mf.QUANT_Q4K, 128),
                       ("ffn7680-nano", mf.QUANT_Q80, 128), ("ffn11520-nano", mf.QUANT_Q80, 128), ("ffn11520-nano", mf.QUANT_Q80, 64),
                       ("ffn7936-nano", mf.QUANT_Q4K, 128), ("ffn7936-nano", mf.QUANT_Q80, 128), ("ffn11648-nano", mf.QUANT_Q80, 128)])


def noise_floors(cases, S=40):
    """Noise floor of the reference itself: max |logit(fast build) - logit(strict build)| of the SAME source on the SAME
    file (SURVEY finding 11), over S teacher-forced positions.  The fast-mode GPU tolerance is max(north-star tolerance,
    1.5 x this floor)."""
    floors = {}
    for name, quant, gs in cases:
        spec = mf.PRESETS[name]
        path = mf.cached_model(spec, quant, gs)
        a = ob.RefEngine(path, S, "strict")
        toks = mf.teacher_tokens(S, spec.vocab)
        strict = [a.forward(toks[p], p) for p in range(S)]
        worst = 0.0
        for fl in ("fast_v3", "fast_v4"):
            b = ob.RefEngine(path, S, fl)
            for p in range(S):
                worst = max(worst, float(np.abs(b.forward(toks[p], p) - strict[p]).max()))
            b.close()
        a.close()
        floors[f"{name}_{quant:02x}_{gs}"] = worst
        print(name, f"{quant:#x}", gs, worst)
    return floors


def reference_digests():
    """reference_outputs.json from the unmodified strict reference (oracle/_ref)."""
    ob.build()
    out = {"sort6_model": sha(ob.sort_model_bytes()), "strict": {}, "lora": {}}
    for name, quant, gs in STRICT_CASES:
        spec = mf.PRESETS[name]
        r = ob.RefEngine(mf.cached_model(spec, quant, gs), STRICT_SEQ, "strict")
        toks = mf.teacher_tokens(STRICT_SEQ, spec.vocab)
        logits = [sha(r.forward(toks[pos], pos)) for pos in range(STRICT_SEQ)]
        k, v = r.kv()
        out["strict"][f"{name}_{quant:02x}_{gs}"] = {"logits": logits, "k_cache": sha(k), "v_cache": sha(v)}
        r.close()

    S, P = 24, 5
    r = ob.RefEngine(mf.cached_model(mf.PRESETS["toy-nano"], mf.QUANT_Q80, 64), S, "strict", penalty=1.3)
    ids = np.zeros(S + 1, np.uint32); ids[:P] = [9, 8, 7, 9, 8]
    for pos in range(S - 1):
        ids[pos + 1] = r.next(ids, pos, 1 if pos < P - 1 else 0)
    out["greedy_penalty_1.3_ids"] = ids.tolist()
    r.close()

    L = ob.RefEngine.lib("strict")
    w = q4k_writer_input()
    T = L.quantize_tensor_q4k(w.ctypes.data_as(ob.f32p), 2, (C.c_uint32 * 2)(*w.shape))
    out["q4k_tensor"] = sha(np.ctypeslib.as_array(C.cast(T, ob.u8p), shape=(L.bytes_num_of_q4k_tensor(T),)))

    x, wq, ws, n, d, gs = q80_ops_inputs()
    q = np.zeros(n, np.int8); s = np.zeros(n // gs, np.float32)
    t = ob.Q80Tensor(q.ctypes.data_as(ob.i8p), s.ctypes.data_as(ob.f32p))
    L.quantize(C.byref(t), x.ctypes.data_as(ob.f32p), n, gs)
    tw = ob.Q80Tensor(wq.ctypes.data_as(ob.i8p), ws.ctypes.data_as(ob.f32p))
    y = np.zeros(d, np.float32)
    L.matmul_quant(y.ctypes.data_as(ob.f32p), C.byref(t), C.byref(tw), n, d, gs)
    out["q80_ops"] = {"codes": sha(q), "scales": sha(s), "matmul_quant": sha(y)}

    spec = mf.PRESETS["toy-nano"]
    lora = mf.write_lora(spec, 8, 16, seed=7)
    for quant, gs in LORA_CASES:
        r = ob.RefEngine(mf.cached_model(spec, quant, gs), TOY_SEQ, "strict"); r.load_lora(lora)
        toks = mf.teacher_tokens(TOY_SEQ, spec.vocab)
        logits = [sha(r.forward(toks[pos], pos)) for pos in range(TOY_SEQ)]
        k, v = r.kv()
        out["lora"][f"toy-nano_{quant:02x}_{gs}"] = {
            "logits": logits,
            "k_rows": [[sha(k[layer, pos]) for pos in LORA_KV_POSITIONS] for layer in range(spec.n_layer)],
            "v_rows": [[sha(v[layer, pos]) for pos in LORA_KV_POSITIONS] for layer in range(spec.n_layer)]}
        r.close()
    json.dump(out, open(os.path.join(HERE, "reference_outputs.json"), "w"), indent=1)
    print("reference digests written")


def main():
    ob.build()
    sm = ob.sort_model_bytes()
    open(os.path.join(HERE, "sort6_model.bin"), "wb").write(sm)
    ref = ob.RefEngine(sm, 6, penalty=0.0, temperature=0.0, top_p=0.0, top_k=1)
    kat = {s: ref.seq2seq(s, 6) for s in ["251212", "114515", "654321", "000000", "909090", "123321", "777111"]}
    json.dump(kat, open(os.path.join(HERE, "sort6_kat.json"), "w"), indent=1)
    print("sort KAT", kat)

    out = {}
    for name, quant, gs in TOY_CONFIGS:
        spec = mf.PRESETS[name]
        path = mf.cached_model(spec, quant, gs)
        r = ob.RefEngine(path, TOY_SEQ, "strict")
        toks = mf.teacher_tokens(TOY_SEQ, spec.vocab)
        rows = []
        for pos in range(TOY_SEQ):
            lg = r.forward(toks[pos], pos)
            if pos in TOY_POSITIONS:
                rows.append(lg)
        key = f"{name}_{quant:02x}_{gs}"
        out[key] = np.stack(rows)
        r.close()
        print(key, out[key].shape, float(np.abs(out[key]).max()))
    np.savez_compressed(os.path.join(HERE, "toy_logits.npz"), **out)

    # LoRA plug-in (infer.c:792-808, 898-903): strict-reference logits with a seeded synthetic plug-in attached
    lora_out = {}
    for quant, gs in [(mf.QUANT_F32, 128), (mf.QUANT_Q80, 64)]:
        spec = mf.PRESETS["toy-nano"]
        path = mf.cached_model(spec, quant, gs)
        r = ob.RefEngine(path, TOY_SEQ, "strict")
        r.load_lora(mf.write_lora(spec, 8, 16, seed=7))
        toks = mf.teacher_tokens(TOY_SEQ, spec.vocab)
        rows = [r.forward(toks[pos], pos) for pos in range(TOY_SEQ)]
        lora_out[f"toy-nano_{quant:02x}_{gs}"] = np.stack([rows[p] for p in TOY_POSITIONS])
        r.close()
    np.savez_compressed(os.path.join(HERE, "lora_logits.npz"), **lora_out)

    floors = noise_floors(TOY_CONFIGS + [("mini-qwen3", mf.QUANT_Q80, 128), ("mini-nano", mf.QUANT_Q80, 128), ("mini-nano", mf.QUANT_Q4K, 128)]
                          + MATRIX_FLOOR_CASES)
    json.dump(floors, open(os.path.join(HERE, "reference_noise_floor.json"), "w"), indent=1)
    print("floors", floors)

    # Q4K KAT
    L = ob.RefEngine.lib("strict")
    d, n = 8, 768
    rnd = xorshift_f32(d * n + n)
    W = (rnd[: d * n] - np.float32(0.5)).astype(np.float32)
    x = (rnd[d * n:] - np.float32(0.5)).astype(np.float32)
    shape_w = (C.c_uint32 * 2)(d, n)
    shape_x = (C.c_uint32 * 1)(n)
    TW = L.quantize_tensor_q4k(W.ctypes.data_as(ob.f32p), 2, shape_w)
    TX = L.quantize_tensor_q4k(x.ctypes.data_as(ob.f32p), 1, shape_x)
    nbw = L.bytes_num_of_q4k_tensor(TW); nbx = L.bytes_num_of_q4k_tensor(TX)
    wb = np.ctypeslib.as_array(C.cast(TW, ob.u8p), shape=(nbw,)).copy()
    xb = np.ctypeslib.as_array(C.cast(TX, ob.u8p), shape=(nbx,)).copy()
    y = np.zeros(d, np.float32)
    L.matmul_q4k(y.ctypes.data_as(ob.f32p), TX, TW, 0)
    np.savez_compressed(os.path.join(HERE, "q4k_kat.npz"), W=W, x=x, w_tensor=wb, x_tensor=xb, y=y)
    print("q4k kat y", y)
    reference_digests()
    export_digests()


if __name__ == "__main__":
    if "--digests" in sys.argv:
        reference_digests()
    elif "--export" in sys.argv:
        export_digests()
    elif "--floors" in sys.argv:           # add the stream-matrix floors to the committed ones
        ob.build()
        path = os.path.join(HERE, "reference_noise_floor.json")
        floors = json.load(open(path))
        floors.update(noise_floors(MATRIX_FLOOR_CASES))
        json.dump(floors, open(path, "w"), indent=1)
    else:
        main()
