"""A float64 restatement of the whole forward pass of an F32 model file, for the tight-tolerance tests.

The C oracle and the CUDA engine both compute in fp32; this computes the same function in float64 from the file's fp32
parameters, so |engine - ref64| can be compared with |oracle - ref64|: the CUDA result must be as close to the exact
answer as the reference-order fp32 computation is, within a small factor.  All teacher-forced positions are computed at
once (a prefill with a causal mask), which is what the token-by-token decode computes position by position.

Restated from the reference's forward pass (infer.c:713-1018): embedding, rmsnorm (eps 1e-5), Qwen3 per-head q/k rmsnorm,
RoPE on adjacent pairs (Nano, tables read from the file) or on half-split pairs (Qwen3, table built from theta 1e6),
causal GQA softmax attention scaled by 1/sqrt(head_dim), SwiGLU, the tied classifier.
"""
import ctypes
import ctypes.util

import numpy as np

from nano_b200 import modelfile as mf


def _libm():
    lib = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
    lib.powf.restype = ctypes.c_float
    lib.powf.argtypes = [ctypes.c_float, ctypes.c_float]
    return lib


def load_f32(path):
    """The parameters of an F32 model file as float64 arrays, and its ModelSpec."""
    raw = np.fromfile(path, dtype=np.uint8)
    hdr = raw[:256].view(np.uint32)
    block, V, L, E, H, KV, F, tied, head_dim = (int(v) for v in hdr[6:15])
    arch, quant = int(hdr[4]), int(hdr[15])
    assert quant == mf.QUANT_F32 and tied, "the float64 reference reads tied F32 files"
    spec = mf.ModelSpec("file", arch, block, V, L, E, H, KV, F, head_dim, tied)
    Q, K, hd = spec.q_dim, spec.kv_dim, spec.hd
    off = 256 + int(raw[256:260].view(np.uint32)[0])          # the tokenizer section starts with its own length
    fl = raw[off:].view(np.float32)
    cur = 0

    def take(*shape):
        nonlocal cur
        n = int(np.prod(shape))
        a = fl[cur: cur + n].astype(np.float64).reshape(shape)
        cur += n
        return a
    p = {"attn_norm": take(L, E), "ffn_norm": take(L, E), "final_norm": take(E), "emb": take(V, E),
         "wq": take(L, Q, E), "wk": take(L, K, E), "wv": take(L, K, E), "wo": take(L, E, Q),
         "w1": take(L, F, E), "w2": take(L, E, F), "w3": take(L, F, E)}
    if arch == mf.ARCH_QWEN3:
        p["q_norm"], p["k_norm"] = take(L, hd), take(L, hd)
        # the model's fp32 frequencies exactly as the engines build them (infer.c:189-204): 1.0f / powf(1e6f, (float)(2i) / hd)
        # with the C library's powf (NumPy's float32 power differs from it by an ulp on some frequencies, an error that grows
        # with the position); the angles pos * freq are fp32 products, their cos / sin are taken in float64
        powf = _libm().powf
        freq = np.array([np.float32(1.0) / np.float32(powf(1e6, float(np.float32(2 * i) / np.float32(hd))))
                         for i in range(hd // 2)], dtype=np.float32)
        ang = (np.arange(block, dtype=np.float32)[:, None] * freq[None, :]).astype(np.float32)
        p["cos"], p["sin"] = np.cos(ang.astype(np.float64)), np.sin(ang.astype(np.float64))
    else:
        p["cos"], p["sin"] = take(block, hd // 2), take(block, hd // 2)
    return spec, p


def _rmsnorm(x, g):
    return g * (x / np.sqrt(np.mean(x * x, axis=-1, keepdims=True) + 1e-5))


def _rope(h, cos, sin, halfsplit):
    """h: [S, heads, hd]; cos / sin: [S, hd / 2]"""
    c, s = cos[:, None, :], sin[:, None, :]
    out = np.empty_like(h)
    if halfsplit:
        half = h.shape[-1] // 2
        a, b = h[..., :half], h[..., half:]
        out[..., :half] = a * c - b * s
        out[..., half:] = b * c + a * s
    else:
        a, b = h[..., 0::2], h[..., 1::2]
        out[..., 0::2] = a * c - b * s
        out[..., 1::2] = a * s + b * c
    return out


def forward(spec, p, tokens):
    """Teacher-forced prefill of `tokens`: (logits [S, V], k rows [L, S, kv_dim] post-RoPE, v rows [L, S, kv_dim])."""
    S = len(tokens)
    H, KV, hd = spec.n_head, spec.n_kv_head, spec.hd
    kvm = H // KV
    qwen3 = spec.arch == mf.ARCH_QWEN3
    cos, sin = p["cos"][:S], p["sin"][:S]
    mask = np.triu(np.full((S, S), -np.inf), 1)
    x = p["emb"][np.asarray(tokens, dtype=np.int64)]
    ks, vs = [], []
    for l in range(spec.n_layer):
        xb = _rmsnorm(x, p["attn_norm"][l])
        q = (xb @ p["wq"][l].T).reshape(S, H, hd)
        k = (xb @ p["wk"][l].T).reshape(S, KV, hd)
        v = (xb @ p["wv"][l].T).reshape(S, KV, hd)
        if qwen3:
            q, k = _rmsnorm(q, p["q_norm"][l]), _rmsnorm(k, p["k_norm"][l])
        q, k = _rope(q, cos, sin, qwen3), _rope(k, cos, sin, qwen3)
        ks.append(k.reshape(S, KV * hd)); vs.append(v.reshape(S, KV * hd))
        o = np.empty((S, H, hd))
        for h in range(H):
            sc = (q[:, h, :] @ k[:, h // kvm, :].T) / np.sqrt(hd) + mask
            sc = np.exp(sc - sc.max(axis=1, keepdims=True))
            o[:, h, :] = (sc / sc.sum(axis=1, keepdims=True)) @ v[:, h // kvm, :]
        x = x + o.reshape(S, H * hd) @ p["wo"][l].T
        xb = _rmsnorm(x, p["ffn_norm"][l])
        h1, h3 = xb @ p["w1"][l].T, xb @ p["w3"][l].T
        x = x + (h1 / (1.0 + np.exp(-h1)) * h3) @ p["w2"][l].T
    logits = _rmsnorm(x, p["final_norm"]) @ p["emb"].T
    return logits, np.stack(ks), np.stack(vs)
