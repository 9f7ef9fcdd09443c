"""Writer for bd4sur/Nano model files (F32 / Q80 / Q4K) with seeded synthetic weights.

There are no real weights in the reference repo or in this environment (SURVEY finding 5), so every
parity/bench configuration runs on synthetic weights written in the reference's on-disk format:

* header + section order ........ infer/infer.c:220-320 (parse_model_file), :100-217 (memory_map_params)
* Nano tokenizer records ........ infer/infer.c:263-307, export.py:72-113
* Qwen tokenizer records ........ infer/tokenizer.c:14-48 (exactly 151,669 entries are read, infer.c:313)
* Q80 tensor = int8 codes then fp32 group scales, one tensor per layer ... infer/tensor.c:49-62,
  arithmetic of export.py:40-63 (round-half-even on w/scale)
* Q4K tensor = 44 B frame + 160 B blocks ... infer/tensor.c:83-110, block quantiser :144-242

The Q4K block quantiser here is a vectorised float32 NumPy restatement of tensor.c:144-242; tests check it
bit-for-bit against the reference's own `quantize_tensor_q4k` (tests/test_oracle_vs_reference.py).

This is format tooling (SURVEY §8 row f1), not part of the decode hot path.
"""
from __future__ import annotations

import dataclasses
import math
import os
import struct
from typing import Dict, Optional

import numpy as np

ARCH_NANO, ARCH_QWEN2, ARCH_QWEN3 = 0, 2, 3
QUANT_F32, QUANT_Q80, QUANT_Q4K = 0x00, 0x80, 0x42
QWEN_TOKENIZER_ENTRIES = 151669          # infer.c:313
FLT_TRUE_MIN = np.float32(1.401298464324817e-45)
FLT_MAX = np.float32(3.4028234663852886e38)


@dataclasses.dataclass(frozen=True)
class ModelSpec:
    name: str
    arch: int
    block_size: int
    vocab: int
    n_layer: int
    n_embd: int
    n_head: int
    n_kv_head: int
    n_hidden: int
    head_dim: int = 0          # only meaningful for arch 3 (infer.h:97)
    tied: int = 1

    @property
    def hd(self) -> int:
        return self.head_dim if self.arch == ARCH_QWEN3 else self.n_embd // self.n_head

    @property
    def q_dim(self) -> int:
        return self.hd * self.n_head if self.arch == ARCH_QWEN3 else self.n_embd

    @property
    def kv_dim(self) -> int:
        return self.hd * self.n_kv_head

    def n_weights(self) -> int:
        """Quantisable weights read once per token (layers + classifier), SURVEY §8(d) `W`."""
        E, F, Q, K = self.n_embd, self.n_hidden, self.q_dim, self.kv_dim
        per_layer = Q * E + 2 * K * E + E * Q + 3 * F * E
        return self.n_layer * per_layer + self.vocab * E

    def bytes_per_token(self, quant: int, gs: int, pos: float) -> float:
        """Algorithmic HBM bytes for one decoded token at position `pos` (SURVEY §8(d) formula B(p))."""
        bpw = {QUANT_F32: 4.0, QUANT_Q80: 1.0 + 4.0 / max(gs, 1), QUANT_Q4K: 148.0 / 256.0}[quant]
        L, E = self.n_layer, self.n_embd
        b = self.n_weights() * bpw + 4 * E * (2 * L + 1)
        if self.arch == ARCH_QWEN3:
            b += 8 * L * self.hd
        b += 8 * L * self.kv_dim * (pos + 1) + 8 * L * self.kv_dim + 4 * E
        return b


PRESETS: Dict[str, ModelSpec] = {
    # README.md:35-46 / config/model.json
    "nano-168m": ModelSpec("nano-168m", ARCH_NANO, 512, 16384, 24, 768, 16, 8, 2048),
    # tools/export_qwen.py:30-41
    "qwen3-0.6b": ModelSpec("qwen3-0.6b", ARCH_QWEN3, 40960, 151936, 28, 1024, 16, 8, 3072, 128),
    "qwen3-1.7b": ModelSpec("qwen3-1.7b", ARCH_QWEN3, 40960, 151936, 28, 2048, 16, 8, 6144, 128),
    "qwen3-4b": ModelSpec("qwen3-4b", ARCH_QWEN3, 40960, 151936, 36, 2560, 32, 8, 9728, 128),
    # small shapes for oracle-speed parity tests
    "toy-nano": ModelSpec("toy-nano", ARCH_NANO, 64, 512, 2, 256, 4, 2, 512),
    "toy-nano-odd": ModelSpec("toy-nano-odd", ARCH_NANO, 32, 96, 2, 32, 4, 2, 16),       # sort-model shape
    "toy-qwen3": ModelSpec("toy-qwen3", ARCH_QWEN3, 128, 2048, 2, 256, 4, 2, 512, 64),
    "mini-qwen3": ModelSpec("mini-qwen3", ARCH_QWEN3, 256, 4096, 4, 512, 8, 4, 1024, 128),
    "mini-nano": ModelSpec("mini-nano", ARCH_NANO, 256, 2048, 4, 768, 16, 8, 2048),
    # loader branches: untied Q80 classifier (infer.c:206-216) and the Qwen2 architecture (infer.c:175-179: biases parsed, never applied)
    "toy-nano-untied": ModelSpec("toy-nano-untied", ARCH_NANO, 64, 512, 2, 256, 4, 2, 512, 0, 0),
    "toy-qwen3-untied": ModelSpec("toy-qwen3-untied", ARCH_QWEN3, 128, 2048, 2, 256, 4, 2, 512, 64, 0),
    "toy-qwen2": ModelSpec("toy-qwen2", ARCH_QWEN2, 64, 512, 2, 256, 4, 2, 512),
    # long-context shapes (2 layers of the Nano-168M / Qwen3-0.6B layer shape): attention with many splits and segments
    "long-nano": ModelSpec("long-nano", ARCH_NANO, 4096, 2048, 2, 768, 16, 8, 2048),
    "long-qwen3": ModelSpec("long-qwen3", ARCH_QWEN3, 4096, 4096, 2, 1024, 16, 8, 3072, 128),
    # 2-layer shapes that select every instantiation of the streaming kernel and of the split-KV attention kernel
    # (KVM = n_head / n_kv_head in {1, 2, 4}) and every activation-prologue width class (tests/test_gpu_stream_matrix.py)
    "kvm1-nano": ModelSpec("kvm1-nano", ARCH_NANO, 2048, 2048, 2, 512, 8, 8, 1024),
    "kvm4-qwen3-hd128": ModelSpec("kvm4-qwen3-hd128", ARCH_QWEN3, 2048, 4096, 2, 1024, 16, 4, 2048, 128),
    "kvm4-qwen3-hd64": ModelSpec("kvm4-qwen3-hd64", ARCH_QWEN3, 2048, 4096, 2, 512, 8, 2, 1024, 64),
    "hd52-nano": ModelSpec("hd52-nano", ARCH_NANO, 2048, 1024, 2, 208, 4, 2, 520),          # hd % 16 != 0, partial prologue slots
    "qwen3-4b-2l": ModelSpec("qwen3-4b-2l", ARCH_QWEN3, 256, 4096, 2, 2560, 32, 8, 9728, 128),   # Qwen3-4B layer shape
    "ffn3840-nano": ModelSpec("ffn3840-nano", ARCH_NANO, 64, 512, 2, 256, 4, 2, 3840),      # one full poll batch
    "ffn3968-nano": ModelSpec("ffn3968-nano", ARCH_NANO, 64, 512, 2, 256, 4, 2, 3968),      # one slot into the second batch
    "ffn4096-nano": ModelSpec("ffn4096-nano", ARCH_NANO, 64, 512, 2, 256, 4, 2, 4096),      # Q4K: second warp slot
    "ffn7680-nano": ModelSpec("ffn7680-nano", ARCH_NANO, 64, 512, 2, 256, 4, 2, 7680),      # Q4K: st_prep_max_n
    "ffn7936-nano": ModelSpec("ffn7936-nano", ARCH_NANO, 64, 512, 2, 256, 4, 2, 7936),      # Q4K: one block past it
    "ffn11520-nano": ModelSpec("ffn11520-nano", ARCH_NANO, 64, 512, 2, 256, 4, 2, 11520),   # Q80 / F32: st_prep_max_n
    "ffn11648-nano": ModelSpec("ffn11648-nano", ARCH_NANO, 64, 512, 2, 256, 4, 2, 11648),   # Q80 / F32: one group past it
}


# ------------------------------------------------------------------------------------------------
# quantisers
# ------------------------------------------------------------------------------------------------
def quantize_q80(w: np.ndarray, gs: int):
    """export.py:40-63: per-group symmetric int8, scale = max|w|/127, round-half-even."""
    flat = np.ascontiguousarray(w, dtype=np.float32).reshape(-1, gs)
    amax = np.abs(flat).max(axis=1)
    scale = (amax / np.float32(127.0)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.rint(flat / scale[:, None])
    q = np.nan_to_num(q, nan=0.0).astype(np.int8)
    return q.reshape(-1), scale


def _nearest_int(v: np.ndarray) -> np.ndarray:
    """tensor.c:4-9 (magic-constant round-half-even), bit-exact in float32."""
    t = (v.astype(np.float32) + np.float32(12582912.0)).astype(np.float32)
    return (t.view(np.int32) & 0x007FFFFF) - 0x00400000


def quantize_q4k_blocks(x: np.ndarray) -> np.ndarray:
    """Quantise rows of 256 floats into 160-byte Q4K blocks (tensor.c:144-242). x: [..., n], n % 256 == 0."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    assert x.shape[-1] % 256 == 0, "Q4K writer requires n % 256 == 0 (SURVEY Appendix B)"
    g = x.reshape(-1, 8, 32)
    nb = g.shape[0]
    lo = np.minimum(g.min(axis=2), FLT_MAX)
    hi = np.maximum(g.max(axis=2), FLT_TRUE_MIN)
    neg = lo <= 0
    s = np.where(neg, (hi - lo) / np.float32(15.0), hi / np.float32(15.0)).astype(np.float32)
    b = np.where(neg, -lo, np.float32(0.0)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = ((g + b[:, :, None]) / s[:, :, None]).astype(np.float32)
    ratio = np.where(s[:, :, None] == 0, np.float32(0.0), ratio)
    codes = (_nearest_int(ratio) & 0x0F).astype(np.uint8).reshape(nb, 256)
    codes[np.repeat(s == 0, 32, axis=1).reshape(nb, 256)] = 0
    nib = (codes[:, 0::2] & 0x0F) | (codes[:, 1::2] << 4)

    smax = np.maximum(s.max(axis=1), FLT_TRUE_MIN)
    bmax = np.maximum(b.max(axis=1), FLT_TRUE_MIN)
    ss = (smax / np.float32(63.0)).astype(np.float32)
    sb = (bmax / np.float32(63.0)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        s6 = np.where(ss[:, None] == 0, 0, _nearest_int(np.where(ss[:, None] == 0, 0, s / ss[:, None])) & 0x3F).astype(np.uint8)
        b6 = np.where(sb[:, None] == 0, 0, _nearest_int(np.where(sb[:, None] == 0, 0, b / sb[:, None])) & 0x3F).astype(np.uint8)

    out = np.zeros((nb, 160), dtype=np.uint8)
    out[:, 0:4] = np.frombuffer(struct.pack("<I", QUANT_Q4K), dtype=np.uint8)
    out[:, 4:8] = np.frombuffer(struct.pack("<I", 256), dtype=np.uint8)
    out[:, 12:16] = ss.view(np.uint8).reshape(nb, 4)
    out[:, 16:20] = sb.view(np.uint8).reshape(nb, 4)
    for k in range(4):
        out[:, 20 + k] = ((s6[:, 4 + k] & 0x30) << 2) | (s6[:, k] & 0x3F)
        out[:, 24 + k] = ((b6[:, 4 + k] & 0x30) << 2) | (b6[:, k] & 0x3F)
        out[:, 28 + k] = ((b6[:, 4 + k] & 0x0F) << 4) | (s6[:, 4 + k] & 0x0F)
    out[:, 32:160] = nib
    return out


def q4k_frame(shape, nblocks: int) -> bytes:
    """44-byte tensor frame (tensor.c:83-110)."""
    dims = list(shape) + [0] * (6 - len(shape))
    total = 44 + nblocks * 160
    return struct.pack("<QII6II", total, QUANT_Q4K, len(shape), *dims, nblocks)


# ------------------------------------------------------------------------------------------------
# tokenizer sections
# ------------------------------------------------------------------------------------------------
def _nano_tokenizer_section(vocab: int) -> bytes:
    """All-single-codepoint vocabulary (ids 0..V-1 -> U+4E00+i; ids 17..26 -> '0'..'9' like nano_80.json)."""
    rec = np.zeros((vocab, 3), dtype=np.uint32)
    rec[:, 0] = 1                               # {len=1, is_special=0, 0, 0}
    rec[:, 1] = np.arange(vocab, dtype=np.uint32)
    rec[:, 2] = 0x4E00 + np.arange(vocab, dtype=np.uint32)
    for d in range(10):
        if 17 + d < vocab:
            rec[17 + d, 2] = ord("0") + d
    body = rec.tobytes()
    return struct.pack("<II", 8 + len(body), vocab) + body


def nano_tokenizer_section_from_config(tokenizer_config: dict) -> bytes:
    """The Nano tokenizer section of a real export (export.py:72-113): `itos` (list of token strings), `special_tokens`."""
    vocab, special = tokenizer_config["itos"], set(tokenizer_config.get("special_tokens", []))
    parts = []
    for i, t in enumerate(vocab):
        parts.append(struct.pack("<BBBBI", len(t), 1 if t in special else 0, 255, 255, i) + struct.pack("<%dI" % len(t), *[ord(c) for c in t]))
    body = b"".join(parts)
    return struct.pack("<II", 8 + len(body), int(tokenizer_config["vocab_size"])) + body


def _qwen_tokenizer_section(vocab: int) -> bytes:
    n = max(vocab, QWEN_TOKENIZER_ENTRIES)
    parts = []
    for i in range(n):
        s = b"t%d" % i
        parts.append(struct.pack("<fI", -float(i), len(s)) + s)
    body = b"".join(parts)
    pad = (-(8 + len(body))) % 16
    body += b"\0" * pad
    return struct.pack("<II", 8 + len(body), 16) + body


# ------------------------------------------------------------------------------------------------
# writer
# ------------------------------------------------------------------------------------------------
def _rope_table(block: int, hd: int, theta: float = 10000.0):
    """model.py:88-94 precompute_freqs_cis in float32."""
    idx = np.arange(0, hd, 2, dtype=np.float32)[: hd // 2]
    freqs = (np.float32(1.0) / np.power(np.float32(theta), idx / np.float32(hd))).astype(np.float32)
    ang = np.outer(np.arange(block, dtype=np.float32), freqs).astype(np.float32)
    return np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)


def write_model(path: str, spec: ModelSpec, quant: int, gs: int = 128, seed: int = 39,
                cls_gain: float = 1.0, fast: bool = False) -> dict:
    """Write a synthetic model file. Weights ~ N(0, 0.02^2) (wo, w3: 0.02/sqrt(2L)), norm gains 1+N(0,0.02^2),
    tied classifier (SURVEY §8(d)). Returns {'path','bytes','spec','quant','gs'}.
    `cls_gain` scales the embedding/classifier rows (bigger top-1 margins for greedy tests)."""
    rng = np.random.default_rng(seed)
    L, E, F, V = spec.n_layer, spec.n_embd, spec.n_hidden, spec.vocab
    Q, K, hd = spec.q_dim, spec.kv_dim, spec.hd
    if quant == QUANT_Q80:
        assert E % gs == 0 and Q % gs == 0 and F % gs == 0, "group size must divide E, q_dim and F"
    if quant == QUANT_Q4K:
        assert E % 256 == 0 and Q % 256 == 0 and F % 256 == 0, "Q4K needs n % 256 == 0"

    hdr = np.zeros(64, dtype=np.uint32)
    hdr[0], hdr[1] = 0x42443453, 0x55524C4D
    hdr[2], hdr[3] = 2025, 12
    hdr[4] = spec.arch
    hdr[6:15] = [spec.block_size, V, L, E, spec.n_head, spec.n_kv_head, F, spec.tied, spec.head_dim]
    hdr[15], hdr[16] = quant, gs if quant == QUANT_Q80 else 0

    def normal(n, std):
        return (rng.standard_normal(n, dtype=np.float32) * np.float32(std)).astype(np.float32)

    def synth_q80(d, n, sd):
        """fast=True (multi-GB bench files): draw int8 codes and group scales directly instead of quantising floats.
        Same byte layout and value range as a quantised N(0, sd^2) tensor (max-abs of a 128-group ~ 2.7 sd)."""
        q = rng.integers(-127, 128, size=d * n, dtype=np.int8)
        s = (np.float32(2.7 * sd / 127.0) * (np.float32(0.8) + np.float32(0.4) * rng.random(d * n // gs, dtype=np.float32))).astype(np.float32)
        return q, s
    assert not fast or quant == QUANT_Q80, "fast synthesis is implemented for Q80 files"

    std = 0.02
    std_o = 0.02 / math.sqrt(2 * L)
    tensors = [("wq", Q, E, std), ("wk", K, E, std), ("wv", K, E, std), ("wo", E, Q, std_o),
               ("w1", F, E, std), ("w2", E, F, std), ("w3", F, E, std_o)]

    with open(path, "wb") as f:
        f.write(hdr.tobytes())
        f.write(_nano_tokenizer_section(V) if spec.arch == ARCH_NANO else _qwen_tokenizer_section(V))
        f.write((np.float32(1.0) + normal(L * E, 0.02)).tobytes())
        f.write((np.float32(1.0) + normal(L * E, 0.02)).tobytes())
        f.write((np.float32(1.0) + normal(E, 0.02)).tobytes())

        emb = None if fast else normal(V * E, std * cls_gain).reshape(V, E)
        if fast:
            q, s = synth_q80(V, E, std * cls_gain)
            f.write(q.tobytes()); f.write(s.tobytes())
        elif quant == QUANT_F32:
            f.write(emb.tobytes())
        elif quant == QUANT_Q80:
            q, s = quantize_q80(emb, gs)
            f.write(q.tobytes()); f.write(s.tobytes())
        else:
            blk = quantize_q4k_blocks(emb)
            f.write(q4k_frame((V, E), blk.shape[0])); f.write(blk.tobytes())
        del emb

        for _name, d, n, sd in tensors:
            if quant == QUANT_Q4K:
                f.write(q4k_frame((L, d, n), L * d * (n // 256)))
            for _l in range(L):
                if fast:
                    q, s = synth_q80(d, n, sd)
                    f.write(q.tobytes()); f.write(s.tobytes())
                    continue
                w = normal(d * n, sd).reshape(d, n)
                if quant == QUANT_F32:
                    f.write(w.tobytes())
                elif quant == QUANT_Q80:
                    q, s = quantize_q80(w, gs)
                    f.write(q.tobytes()); f.write(s.tobytes())
                else:
                    f.write(quantize_q4k_blocks(w).tobytes())

        if spec.arch == ARCH_QWEN2:
            f.write(np.zeros(L * (Q + 2 * K), dtype=np.float32).tobytes())
        if spec.arch == ARCH_QWEN3:
            f.write((np.float32(1.0) + normal(L * hd, 0.02)).tobytes())
            f.write((np.float32(1.0) + normal(L * hd, 0.02)).tobytes())
        if spec.arch in (ARCH_NANO, ARCH_QWEN2):
            c, s = _rope_table(spec.block_size, hd)
            f.write(c.tobytes()); f.write(s.tobytes())
        # arch 3: the reference rebuilds its table (infer.c:189-204) and never reads one from the file;
        # Q4K arch-3 files end right after k_norm (tools/export_q4k.c:176-204). Nothing is written -- unless an untied
        # classifier follows: the reference steps over a table-sized gap first (infer.c:201-202).
        if not spec.tied:
            assert quant == QUANT_Q80, "untied classifier: Q80 only (infer.c:206-216; the F32 pointer is a reference bug, Q4K is always tied)"
            if spec.arch == ARCH_QWEN3:
                f.write(np.zeros(2 * spec.block_size * (hd // 2), dtype=np.float32).tobytes())
            q, s = quantize_q80(normal(V * E, std * cls_gain).reshape(V, E), gs)
            f.write(q.tobytes()); f.write(s.tobytes())
        size = f.tell()
    return {"path": path, "bytes": size, "spec": spec, "quant": quant, "gs": gs}


def write_model_from_weights(path: str, spec: ModelSpec, quant: int, gs: int, weights: Dict[str, np.ndarray],
                             tokenizer_section: Optional[bytes] = None, rope_tables: bool = True, version=(2026, 1),
                             rope: Optional[tuple] = None) -> dict:
    """Write a model file from GIVEN float32 weights (the export path: tools/export_qwen.py:442-636 for arch 3, export.py:228-475 for
    arch 0) in the same section order as `write_model`.  `weights`: attn_norm [L,E], ffn_norm [L,E], final_norm [E], emb [V,E],
    wq [L,Q,E], wk [L,K,E], wv [L,K,E], wo [L,E,Q], w1 [L,F,E], w2 [L,E,F], w3 [L,F,E]; arch 3 also q_norm [L,hd], k_norm [L,hd];
    an untied model also cls [V,E] (Q80 files only, infer.c:206-216).  `rope_tables`: arch 3 files of the reference exporter carry a
    (cos, sin) table the engine never reads (infer.c:189-204 rebuilds it); written by default so that the untied classifier, which
    the loader looks for behind a table-sized gap (infer.c:201-202), lands where the reference expects it.  `rope`: the (cos, sin)
    tables to write, [block_size, hd/2] each -- an exporter passes the checkpoint's own buffers (arch 0 engines READ this table,
    infer.c:181-187, and torch's pow / cos differ from NumPy's by an ulp here and there); default: `_rope_table`."""
    L, E, F, V = spec.n_layer, spec.n_embd, spec.n_hidden, spec.vocab
    Q, K, hd = spec.q_dim, spec.kv_dim, spec.hd
    shapes = {"attn_norm": (L, E), "ffn_norm": (L, E), "final_norm": (E,), "emb": (V, E), "wq": (L, Q, E), "wk": (L, K, E), "wv": (L, K, E),
              "wo": (L, E, Q), "w1": (L, F, E), "w2": (L, E, F), "w3": (L, F, E)}
    if spec.arch == ARCH_QWEN3:
        shapes.update({"q_norm": (L, hd), "k_norm": (L, hd)})
    if not spec.tied:
        shapes["cls"] = (V, E)
    w = {}
    for k, shp in shapes.items():
        a = np.ascontiguousarray(weights[k], dtype=np.float32)
        assert a.shape == shp, f"{k}: shape {a.shape}, expected {shp}"
        w[k] = a
    if quant == QUANT_Q80:
        assert E % gs == 0 and Q % gs == 0 and F % gs == 0, "group size must divide E, q_dim and F"
    if quant == QUANT_Q4K:
        assert E % 256 == 0 and Q % 256 == 0 and F % 256 == 0 and spec.tied, "Q4K needs n % 256 == 0 and a tied classifier"
    assert spec.tied or quant == QUANT_Q80, "untied classifier: Q80 files only"
    assert spec.arch != ARCH_QWEN2, "Qwen2 export (biases) is not provided"

    hdr = np.zeros(64, dtype=np.uint32)
    hdr[0], hdr[1] = 0x42443453, 0x55524C4D
    hdr[2], hdr[3] = version                     # the current exporters write 2026 / 1 (export.py:240-241); the engine does not look at it
    hdr[4], hdr[5] = spec.arch, 36               # model type, config length (export.py:255-256)
    hdr[6:15] = [spec.block_size, V, L, E, spec.n_head, spec.n_kv_head, F, spec.tied, spec.head_dim if spec.arch == ARCH_QWEN3 else spec.hd]
    hdr[15], hdr[16] = quant, gs if quant == QUANT_Q80 else 0

    def emit(f, a2d):
        if quant == QUANT_F32:
            f.write(a2d.tobytes())
        elif quant == QUANT_Q80:
            q, s = quantize_q80(a2d, gs)
            f.write(q.tobytes()); f.write(s.tobytes())
        else:
            f.write(quantize_q4k_blocks(a2d).tobytes())

    with open(path, "wb") as f:
        f.write(hdr.tobytes())
        f.write(tokenizer_section if tokenizer_section is not None else
                (_nano_tokenizer_section(V) if spec.arch == ARCH_NANO else _qwen_tokenizer_section(V)))
        f.write(w["attn_norm"].tobytes()); f.write(w["ffn_norm"].tobytes()); f.write(w["final_norm"].tobytes())
        if quant == QUANT_Q4K:
            f.write(q4k_frame((V, E), V * (E // 256)))
        emit(f, w["emb"])
        for name, d, n in (("wq", Q, E), ("wk", K, E), ("wv", K, E), ("wo", E, Q), ("w1", F, E), ("w2", E, F), ("w3", F, E)):
            if quant == QUANT_Q4K:
                f.write(q4k_frame((L, d, n), L * d * (n // 256)))
            for l in range(L):
                emit(f, w[name][l])
        if spec.arch == ARCH_QWEN3:
            f.write(w["q_norm"].tobytes()); f.write(w["k_norm"].tobytes())
        if spec.arch == ARCH_NANO or (rope_tables and quant != QUANT_Q4K) or not spec.tied:
            c, sn = rope if rope is not None else _rope_table(spec.block_size, hd, 1000000.0 if spec.arch == ARCH_QWEN3 else 10000.0)
            c, sn = np.ascontiguousarray(c, np.float32), np.ascontiguousarray(sn, np.float32)
            assert c.shape == sn.shape == (spec.block_size, hd // 2), (c.shape, spec.block_size, hd)
            f.write(c.tobytes()); f.write(sn.tobytes())
        if not spec.tied:
            q, s = quantize_q80(w["cls"], gs)
            f.write(q.tobytes()); f.write(s.tobytes())
        size = f.tell()
    return {"path": path, "bytes": size, "spec": spec, "quant": quant, "gs": gs}


def write_lora(spec: ModelSpec, rank: int = 8, alpha: int = 16, seed: int = 7, std: float = 0.05) -> bytes:
    """A synthetic LoRA plug-in image in the reference's layout (infer.c:436-500): 256-byte header
    {magic0, magic1, major, minor, model_type, config_length, rank, alpha, n_layer, n_embd, n_head, n_kv_head, n_hidden,
    lora_config} then fp32 tensors wq_a (L,r,E), wq_b (L,E,r), wk_a (L,r,E), wk_b (L,kv,r), wv_a, wv_b, wo_a (L,r,E),
    wo_b (L,E,r).  Both factors are non-zero so that every branch contributes."""
    rng = np.random.default_rng(seed)
    L, E, K = spec.n_layer, spec.n_embd, spec.kv_dim
    hdr = np.zeros(64, dtype=np.uint32)
    hdr[0], hdr[1], hdr[2], hdr[3] = 0x42443453, 0x41524F4C, 2025, 12
    hdr[4], hdr[5] = spec.arch, 32
    hdr[6:14] = [rank, alpha, L, E, spec.n_head, spec.n_kv_head, spec.n_hidden, 0]
    parts = [hdr.tobytes()]
    for rows_b in (E, K, K, E):
        parts.append((rng.standard_normal(L * rank * E, dtype=np.float32) * np.float32(std)).tobytes())
        parts.append((rng.standard_normal(L * rows_b * rank, dtype=np.float32) * np.float32(std)).tobytes())
    return b"".join(parts)


def cached_model(spec: ModelSpec, quant: int, gs: int = 128, seed: int = 39, cache_dir: Optional[str] = None,
                 cls_gain: float = 1.0, fast: bool = False) -> str:
    """Write (once) into a cache directory and return the path."""
    cache_dir = cache_dir or os.environ.get("NB200_MODEL_CACHE", "/tmp/nb200_models")
    os.makedirs(cache_dir, exist_ok=True)
    qn = {QUANT_F32: "f32", QUANT_Q80: f"q80g{gs}", QUANT_Q4K: "q4k"}[quant]
    g = ("" if cls_gain == 1.0 else f"_cg{cls_gain:g}") + ("_fast" if fast else "")
    path = os.path.join(cache_dir, f"{spec.name}_{qn}_s{seed}{g}.bin")
    if not os.path.exists(path):
        tmp = path + f".tmp{os.getpid()}"
        write_model(tmp, spec, quant, gs, seed, cls_gain, fast)
        os.replace(tmp, path)
    return path


def teacher_tokens(n: int, vocab: int, seed: int = 39) -> np.ndarray:
    """xorshift* stream of utils.c:959-965 (random_u32), reduced mod min(V, 151669) (SURVEY App. E.4)."""
    mod = min(vocab, QWEN_TOKENIZER_ENTRIES)
    st = seed & 0xFFFFFFFFFFFFFFFF
    out = np.zeros(n, dtype=np.uint32)
    M = 0xFFFFFFFFFFFFFFFF
    for i in range(n):
        st ^= st >> 12
        st ^= (st << 25) & M
        st ^= st >> 27
        out[i] = (((st * 0x2545F4914F6CDD1D) & M) >> 32) % mod
    return out
