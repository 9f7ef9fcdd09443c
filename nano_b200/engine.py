"""ctypes binding of libnano_b200.so (include/nano_b200.h).

This is plumbing for tests and bench.py; the product is the C-ABI library itself.  The binding fails loudly
when the library is missing or when there is no CUDA device -- there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Tuple

import numpy as np

from . import build as _build

f32p = C.POINTER(C.c_float)
u32p = C.POINTER(C.c_uint32)
u8p = C.POINTER(C.c_uint8)
i8p = C.POINTER(C.c_int8)

FLAG_EXACT, FLAG_NO_GRAPH, FLAG_NO_PDL, FLAG_NO_STREAM = 0x1, 0x2, 0x4, 0x10
F_X, F_XBA, F_HB, F_Q, F_LOGITS, F_KROW, F_VROW, F_ACT_I8, F_ACT_SCALE = 0, 2, 4, 6, 9, 13, 14, 20, 21
MATVEC_EPILOGUES = ("store", "qkv", "resid", "swiglu", "cls")      # kernels.cuh `Epilogue`, in value order

EXPORTS = [
    "nb200_last_error", "nb200_device_count", "nb200_engine_create", "nb200_engine_destroy", "nb200_get_config",
    "nb200_forward", "nb200_read_logits", "nb200_next_greedy", "nb200_next_sampled", "nb200_decode_greedy", "nb200_prefill",
    "nb200_verify_greedy", "nb200_decode_lookup", "nb200_read_buffer",
    "nb200_write_x", "nb200_run_layer", "nb200_profile_tokens", "nb200_trace_token", "nb200_read_attn_trace", "nb200_kernel_launches", "nb200_launches_per_token", "nb200_weight_bytes",
    "nb200_op_rmsnorm", "nb200_op_q80_quantize", "nb200_op_q80_matvec", "nb200_op_f32_matvec",
    "nb200_op_q4k_quantize", "nb200_op_q4k_matvec",
    "nb200_op_q4k_quantize_blocks", "nb200_op_q4k_matvec_blocks",
    "nb200_lora_load", "nb200_lora_enable", "nb200_lora_unload",
    "nb200_engine_create_tp", "nb200_tp_export", "nb200_tp_attach_ipc", "nb200_tp_attach_local",
    "nb200_batch_create", "nb200_batch_destroy", "nb200_batch_prefill", "nb200_batch_next_greedy", "nb200_batch_next_sampled",
    "nb200_batch_verify_greedy", "nb200_batch_read_logits", "nb200_batch_read_kv", "nb200_batch_info",
]


class Config(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in (
        "arch", "quant", "group_size", "block_size", "vocab_size", "n_layer", "n_embd", "n_head", "n_kv_head",
        "n_hidden", "tied", "head_dim", "q_dim", "kv_dim", "max_seq_len", "tp_rank", "tp_size")] + [("reserved", C.c_uint32 * 7)]


class NB200Error(RuntimeError):
    pass


_lib = None


def lib():
    global _lib
    if _lib is None:
        path = os.environ.get("NB200_ENGINE_SO", _build.ENGINE_SO)     # developer hook: the fine-trace build (tools/gpu_trace.py)
        if not os.path.exists(path):
            raise NB200Error(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                             "(nano_b200 has no CPU fallback)")
        L = C.CDLL(path)
        L.nb200_last_error.restype = C.c_char_p
        L.nb200_engine_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_uint32]
        L.nb200_engine_create_tp.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_uint32,
                                             C.c_uint32, C.c_uint32]
        L.nb200_tp_export.argtypes = [C.c_void_p, C.c_void_p]
        L.nb200_tp_attach_ipc.argtypes = [C.c_void_p, C.c_void_p]
        L.nb200_tp_attach_local.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.nb200_engine_destroy.argtypes = [C.c_void_p]
        L.nb200_get_config.argtypes = [C.c_void_p, C.POINTER(Config)]
        L.nb200_forward.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.nb200_read_logits.argtypes = [C.c_void_p, f32p]
        L.nb200_next_greedy.argtypes = [C.c_void_p, u32p, C.c_uint32, C.c_int, C.c_float, u32p]
        L.nb200_next_sampled.argtypes = [C.c_void_p, u32p, C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_float, u32p, u32p]
        L.nb200_decode_greedy.argtypes = [C.c_void_p, u32p, C.c_uint32, C.c_uint32, C.c_float, f32p, f32p]
        L.nb200_prefill.argtypes = [C.c_void_p, u32p, C.c_uint32, C.c_uint32, f32p]
        L.nb200_verify_greedy.argtypes = [C.c_void_p, u32p, C.c_uint32, C.c_uint32, C.c_float, u32p, f32p]
        L.nb200_decode_lookup.argtypes = [C.c_void_p, u32p, C.c_uint32, C.c_uint32, C.c_float, C.c_uint32, C.c_uint32, u32p, f32p, f32p]
        L.nb200_read_buffer.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32]
        L.nb200_write_x.argtypes = [C.c_void_p, f32p, C.c_uint32]
        L.nb200_run_layer.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.nb200_profile_tokens.argtypes = [C.c_void_p, u32p, C.c_uint32, C.c_uint32, f32p, u32p]
        L.nb200_trace_token.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64), C.c_uint32, u32p]
        L.nb200_read_attn_trace.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.nb200_kernel_launches.restype = C.c_uint64
        L.nb200_kernel_launches.argtypes = [C.c_void_p]
        L.nb200_launches_per_token.restype = C.c_uint32
        L.nb200_launches_per_token.argtypes = [C.c_void_p]
        L.nb200_weight_bytes.restype = C.c_uint64
        L.nb200_weight_bytes.argtypes = [C.c_void_p]
        L.nb200_op_rmsnorm.argtypes = [f32p, f32p, f32p, C.c_uint32, C.c_uint32]
        L.nb200_op_q80_quantize.argtypes = [i8p, f32p, f32p, C.c_uint32, C.c_uint32]
        L.nb200_op_q80_matvec.argtypes = [f32p, f32p, i8p, f32p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.nb200_op_f32_matvec.argtypes = [f32p, f32p, f32p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.nb200_op_q4k_quantize.argtypes = [u8p, f32p, C.c_uint32]
        L.nb200_op_q4k_matvec.argtypes = [f32p, f32p, u8p, C.c_uint32, C.c_uint32]
        L.nb200_op_q4k_quantize_blocks.argtypes = [u8p, f32p, C.c_uint64]
        L.nb200_op_q4k_matvec_blocks.argtypes = [f32p, u8p, u8p, C.c_uint32, C.c_uint32]
        L.nb200_lora_load.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.nb200_lora_enable.argtypes = [C.c_void_p, C.c_int]
        L.nb200_lora_unload.argtypes = [C.c_void_p]
        L.nb200_batch_create.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p)]
        L.nb200_batch_destroy.argtypes = [C.c_void_p]
        L.nb200_batch_prefill.argtypes = [C.c_void_p, C.c_uint32, u32p, C.c_uint32, C.c_uint32, f32p]
        L.nb200_batch_next_greedy.argtypes = [C.c_void_p, C.c_uint32, u32p, C.POINTER(u32p), u32p, f32p, u32p, f32p]
        L.nb200_batch_next_sampled.argtypes = [C.c_void_p, C.c_uint32, u32p, C.POINTER(u32p), u32p, f32p, f32p, f32p, f32p, u32p, u32p,
                                               f32p]
        L.nb200_batch_verify_greedy.argtypes = [C.c_void_p, C.c_uint32, u32p, C.POINTER(u32p), u32p, u32p, f32p, u32p, f32p]
        L.nb200_batch_read_logits.argtypes = [C.c_void_p, C.c_uint32, f32p]
        L.nb200_batch_read_kv.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, f32p, C.c_uint32]
        L.nb200_batch_info.argtypes = [C.c_void_p, u32p]
        L.nb200_host_expf_ref.restype = C.c_float
        L.nb200_host_expf_ref.argtypes = [C.c_float]
        L.nb200_host_expf_ref_array.argtypes = [f32p, f32p, C.c_uint64]
        _lib = L
    return _lib


def _check(rc: int):
    if rc != 0:
        raise NB200Error(f"nb200 error {rc}: {lib().nb200_last_error().decode()}")


def device_count() -> int:
    return int(lib().nb200_device_count())


def _p(a: np.ndarray, t):
    return a.ctypes.data_as(t)


def _attention_kind(att: int):
    return {0: None, 1: "exact", 2: "generic", 3: f"fast<{att >> 8}>"}[att & 0xff]


class Engine:
    """One model resident in the HBM of one GPU."""

    def __init__(self, model, max_seq: int, device: int = 0, flags: int = 0, tp: Optional[Tuple[int, int]] = None):
        """tp=(rank, size) creates one rank of a tensor-parallel group; attach it (tp_attach_ipc / TpGroup) before use."""
        L = lib()
        if isinstance(model, (str, os.PathLike)):
            image = np.fromfile(model, dtype=np.uint8)
        else:
            image = np.frombuffer(bytes(model), dtype=np.uint8)
        self.h = C.c_void_p()
        self._batches = []
        if tp is None:
            _check(L.nb200_engine_create(C.byref(self.h), image.ctypes.data, image.size, max_seq, device, flags))
        else:
            _check(L.nb200_engine_create_tp(C.byref(self.h), image.ctypes.data, image.size, max_seq, device, flags,
                                            int(tp[0]), int(tp[1])))
        self._refresh()

    def _refresh(self):
        L = lib()
        cfg = Config()
        _check(L.nb200_get_config(self.h, C.byref(cfg)))
        self.cfg = cfg
        for n, _t in Config._fields_[:-1]:
            setattr(self, n, int(getattr(cfg, n)))
        self.vocab = self.vocab_size
        self.path = {4: "streaming kernel (persistent grid, per-CTA TMA ring over weights and KV, L2 grid barriers)",
                     1: "multi-kernel CUDA graph with PDL", 0: "multi-kernel direct launches"}[int(cfg.reserved[0]) & 0xff]
        # streaming kernel: CTAs of its grid (NB200_STREAM_WIDTH, or the fastest width timed at creation); None on the other paths
        self.stream_width = ((int(cfg.reserved[0]) >> 8) & 0xffff) or None
        # CTAs per thread-block cluster of the streaming kernel's launch; None on a plain launch and on the other paths
        self.stream_cluster = (int(cfg.reserved[0]) >> 24) or None
        # creation-time calibration of the two fast paths (large one-GPU Q80 engines): us per token of each, None when not measured
        self.calibration = ({"streaming_us_per_token": int(cfg.reserved[1]), "multikernel_us_per_token": int(cfg.reserved[2]),
                             "stream_width": self.stream_width, "stream_cluster": self.stream_cluster}
                            if int(cfg.reserved[1]) and int(cfg.reserved[2]) else None)

    def kernels(self) -> dict:
        """Kernels of the multi-kernel path this engine has launched or captured (include/nano_b200.h, reserved[3] / [4]):
        {"matvec": set of (epilogue, RB), "attention": "exact" | "generic" | "fast<KVM>" | None}.  Read afresh on every call:
        direct launches record a kernel on its first use, a captured graph at creation."""
        cfg = Config()
        _check(lib().nb200_get_config(self.h, C.byref(cfg)))
        mask, att = int(cfg.reserved[3]), int(cfg.reserved[4])
        mv = {(epi, rb) for i, epi in enumerate(MATVEC_EPILOGUES) for j, rb in enumerate((1, 2, 4)) if mask >> (3 * i + j) & 1}
        return {"matvec": mv, "attention": _attention_kind(att)}

    def prefill_info(self) -> dict:
        """Batched prefill (reserved[5] / [6]): {"chunk": positions per pass over the weights (0 before the first prefill),
        "attention": the attention kernel of the last prefill, named as in kernels()}."""
        cfg = Config()
        _check(lib().nb200_get_config(self.h, C.byref(cfg)))
        return {"chunk": int(cfg.reserved[5]), "attention": _attention_kind(int(cfg.reserved[6]))}

    # ---- LoRA plug-in ----
    def lora_load(self, image: bytes) -> None:
        buf = np.frombuffer(bytes(image), dtype=np.uint8)
        _check(lib().nb200_lora_load(self.h, buf.ctypes.data, buf.size))
        self._refresh()

    def lora_enable(self, on: bool) -> None:
        _check(lib().nb200_lora_enable(self.h, 1 if on else 0))
        self._refresh()

    def lora_unload(self) -> None:
        _check(lib().nb200_lora_unload(self.h))
        self._refresh()

    # ---- tensor parallel ----
    def tp_export(self) -> bytes:
        """64-byte CUDA IPC handle of this rank's exchange block (send it to the other ranks' processes)."""
        buf = C.create_string_buffer(64)
        _check(lib().nb200_tp_export(self.h, buf))
        return buf.raw

    def tp_attach_ipc(self, handles) -> None:
        """handles: the tp_size 64-byte handles in rank order (this rank's own entry is ignored)."""
        blob = b"".join(bytes(h) for h in handles)
        assert len(blob) == 64 * self.tp_size
        _check(lib().nb200_tp_attach_ipc(self.h, blob))
        self._refresh()

    def logits_slice(self) -> Tuple[int, int]:
        """[lo, hi) of the logits this rank computes (the whole vector on one GPU)."""
        per = self.vocab // self.tp_size
        return self.tp_rank * per, (self.tp_rank + 1) * per

    def batch(self, n_slots: int) -> "Batch":
        """A batch of n_slots independent sessions decoded together over this engine's weights (nb200_batch_*)."""
        b = Batch(self, n_slots)
        self._batches.append(b)
        return b

    def close(self):
        if getattr(self, "h", None):
            for b in list(getattr(self, "_batches", [])):      # a batch must go before its engine
                b.close()
            lib().nb200_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, token: int, pos: int, causal: int = 1) -> np.ndarray:
        _check(lib().nb200_forward(self.h, int(token), int(pos), int(causal)))
        return self.logits()

    def forward_nolog(self, token: int, pos: int, causal: int = 1) -> None:
        _check(lib().nb200_forward(self.h, int(token), int(pos), int(causal)))

    def logits(self) -> np.ndarray:
        out = np.empty(self.vocab, dtype=np.float32)
        _check(lib().nb200_read_logits(self.h, _p(out, f32p)))
        return out

    def next_greedy(self, ids: np.ndarray, pos: int, prefilling: int, penalty: float = 1.0) -> int:
        nxt = C.c_uint32(0)
        _check(lib().nb200_next_greedy(self.h, _p(ids, u32p), pos, prefilling, penalty, C.byref(nxt)))
        return int(nxt.value)

    def next_sampled(self, ids: np.ndarray, pos: int, penalty: float, temperature: float, top_p: float, coin: float):
        """generate_next_token with temperature > 0, sampled on the device; returns (token, six most probable ids)."""
        nxt = C.c_uint32(0); top6 = (C.c_uint32 * 6)()
        _check(lib().nb200_next_sampled(self.h, _p(ids, u32p), pos, penalty, temperature, top_p, coin, C.byref(nxt), top6))
        return int(nxt.value), list(top6)

    def decode_greedy(self, ids: np.ndarray, n_prompt: int, n_total: int, penalty: float = 1.0) -> Tuple[float, float]:
        """Device-resident loop; fills ids[n_prompt:n_total] in place. Returns (prefill_ms, decode_ms)."""
        assert ids.dtype == np.uint32 and ids.size >= n_total
        a, b = C.c_float(0), C.c_float(0)
        _check(lib().nb200_decode_greedy(self.h, _p(ids, u32p), n_prompt, n_total, penalty, C.byref(a), C.byref(b)))
        return float(a.value), float(b.value)

    def prefill(self, ids: np.ndarray, pos0: int, n: int) -> float:
        """Batched prompt prefill of ids[pos0:pos0+n] at positions pos0.. (K/V rows only; continue with forward / next_greedy /
        next_sampled at pos0+n).  Returns the device time in ms."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        assert ids.size >= pos0 + n
        ms = C.c_float(0)
        _check(lib().nb200_prefill(self.h, _p(ids, u32p), int(pos0), int(n), C.byref(ms)))
        return float(ms.value)

    def verify_greedy(self, ids: np.ndarray, pos: int, n: int, penalty: float = 1.0) -> int:
        """Speculative verification of the n-1 drafted ids ids[pos+1:pos+n] in one pass: returns the number a accepted and writes
        the greedy id at pos+a into ids[pos+a+1] in place (ids: uint32, at least pos+n+1 entries).  The device time of the pass
        is left in self.verify_ms."""
        assert ids.dtype == np.uint32 and ids.flags.c_contiguous and ids.size >= pos + n + 1
        acc, ms = C.c_uint32(0), C.c_float(0)
        _check(lib().nb200_verify_greedy(self.h, _p(ids, u32p), int(pos), int(n), penalty, C.byref(acc), C.byref(ms)))
        self.verify_ms = float(ms.value)
        return int(acc.value)

    def decode_lookup(self, ids: np.ndarray, n_prompt: int, n_total: int, penalty: float = 1.0, ngram_max: int = 3,
                      draft_max: Optional[int] = None):
        """decode_greedy with drafts looked up in the context and verified (nb200_decode_lookup): fills ids[n_prompt:n_total] in
        place with decode_greedy's ids.  draft_max None: the chunk size - 1.  Returns ([verify passes, steps without a draft,
        drafted ids, accepted ids], prefill_ms, decode_ms)."""
        assert ids.dtype == np.uint32 and ids.flags.c_contiguous and ids.size >= n_total
        stats = np.zeros(4, np.uint32)
        a, b = C.c_float(0), C.c_float(0)
        _check(lib().nb200_decode_lookup(self.h, _p(ids, u32p), int(n_prompt), int(n_total), penalty, int(ngram_max),
                                         0xffffffff if draft_max is None else int(draft_max), _p(stats, u32p), C.byref(a), C.byref(b)))
        return stats.tolist(), float(a.value), float(b.value)

    def read(self, field: int, count: int, layer: int = 0, pos: int = 0, dtype=np.float32) -> np.ndarray:
        out = np.zeros(count, dtype=dtype)
        _check(lib().nb200_read_buffer(self.h, field, layer, pos, out.ctypes.data, count))
        return out

    def write_x(self, x: np.ndarray) -> None:
        x = np.ascontiguousarray(x, dtype=np.float32)
        _check(lib().nb200_write_x(self.h, _p(x, f32p), x.size))

    def run_layer(self, layer: int, pos: int, causal: int = 1) -> None:
        _check(lib().nb200_run_layer(self.h, layer, pos, causal))

    def profile_tokens(self, ids: np.ndarray, start: int, n: int):
        """Per-kernel-class (ms, launches): embed, qkv, attention, o, w13, w2, classifier."""
        ms = np.zeros(7, np.float32); cnt = np.zeros(7, np.uint32)
        _check(lib().nb200_profile_tokens(self.h, _p(ids, u32p), start, n, _p(ms, f32p), _p(cnt, u32p)))
        return ms, cnt

    def trace_token(self, token: int, pos: int) -> np.ndarray:
        """clock64() stamps (SM cycles) of CTA 0 after every grid barrier of one token (persistent kernel only)."""
        cap = 1024 + 256
        buf = np.zeros(cap, np.uint64); n = C.c_uint32(0)
        _check(lib().nb200_trace_token(self.h, token, pos, buf.ctypes.data_as(C.POINTER(C.c_uint64)), cap, C.byref(n)))
        return buf[: n.value]

    def attn_trace(self) -> np.ndarray:
        """%globaltimer stamps (ns) of layer L/2's attention kernel in the last token (engine created with NB200_ATTN_DBG=1)."""
        buf = np.zeros(32, np.uint64)
        _check(lib().nb200_read_attn_trace(self.h, buf.ctypes.data_as(C.POINTER(C.c_uint64))))
        return buf

    @property
    def launches(self) -> int:
        return int(lib().nb200_kernel_launches(self.h))

    @property
    def launches_per_token(self) -> int:
        return int(lib().nb200_launches_per_token(self.h))

    @property
    def weight_bytes(self) -> int:
        return int(lib().nb200_weight_bytes(self.h))


class Batch:
    """Up to n_slots sessions sharing one engine's weights; each slot has its own K / V cache, seen set and logits
    (include/nano_b200.h, nb200_batch_*).  Create it with Engine.batch; Engine.close closes it first."""

    def __init__(self, engine: Engine, n_slots: int):
        self.engine = engine
        self.h = C.c_void_p()
        _check(lib().nb200_batch_create(engine.h, int(n_slots), C.byref(self.h)))
        self.device_ms = 0.0        # device time of the last next_greedy / next_sampled / verify_greedy

    def info(self) -> dict:
        """{"chunk": positions per pass M, "slots": n_slots, "attention": the attention kernel, named as Engine.kernels()}"""
        out = np.zeros(4, np.uint32)
        _check(lib().nb200_batch_info(self.h, _p(out, u32p)))
        return {"chunk": int(out[0]), "slots": int(out[1]), "attention": _attention_kind(int(out[2]))}

    def prefill(self, slot: int, ids: np.ndarray, pos0: int, n: int) -> float:
        """Engine.prefill into one slot's cache; returns the device time in ms."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        assert ids.size >= pos0 + n
        ms = C.c_float(0)
        _check(lib().nb200_batch_prefill(self.h, int(slot), _p(ids, u32p), int(pos0), int(n), C.byref(ms)))
        return float(ms.value)

    def next_greedy(self, slots, ids, pos, penalties) -> list:
        """Entry i is Engine.next_greedy(ids[i], pos[i], 0, penalties[i]) in slot slots[i]; returns the next ids."""
        n = len(slots)
        assert len(ids) == len(pos) == len(penalties) == n
        arrs = [np.ascontiguousarray(a, dtype=np.uint32) for a in ids]
        ptrs = (u32p * n)(*[_p(a, u32p) for a in arrs])
        s = np.asarray(slots, np.uint32); p = np.asarray(pos, np.uint32); pen = np.asarray(penalties, np.float32)
        out = np.zeros(n, np.uint32)
        ms = C.c_float(0)
        _check(lib().nb200_batch_next_greedy(self.h, n, _p(s, u32p), ptrs, _p(p, u32p), _p(pen, f32p), _p(out, u32p), C.byref(ms)))
        self.device_ms = float(ms.value)
        return out.tolist()

    def next_sampled(self, slots, ids, pos, penalties, temperatures, top_ps, coins):
        """Entry i is Engine.next_sampled(ids[i], pos[i], penalties[i], temperatures[i], top_ps[i], coins[i]) in slot slots[i],
        or next_greedy's entry where temperatures[i] == 0 (its six ids are zeros); returns (next ids, six ids per entry)."""
        n = len(slots)
        assert len(ids) == len(pos) == len(penalties) == len(temperatures) == len(top_ps) == len(coins) == n
        arrs = [np.ascontiguousarray(a, dtype=np.uint32) for a in ids]
        ptrs = (u32p * n)(*[_p(a, u32p) for a in arrs])
        s = np.asarray(slots, np.uint32); p = np.asarray(pos, np.uint32)
        pen, T, tp, c = (np.asarray(v, np.float32) for v in (penalties, temperatures, top_ps, coins))
        out = np.zeros(n, np.uint32); six = np.zeros((n, 6), np.uint32)
        ms = C.c_float(0)
        _check(lib().nb200_batch_next_sampled(self.h, n, _p(s, u32p), ptrs, _p(p, u32p), _p(pen, f32p), _p(T, f32p), _p(tp, f32p),
                                              _p(c, f32p), _p(out, u32p), _p(six, u32p), C.byref(ms)))
        self.device_ms = float(ms.value)
        return out.tolist(), six.tolist()

    def verify_greedy(self, slots, ids, pos, n_pos, penalties) -> list:
        """Entry i is Engine.verify_greedy(ids[i], pos[i], n_pos[i], penalties[i]) in slot slots[i]: returns the accepted counts
        and writes each entry's greedy id at pos+a into ids[i][pos+a+1] in place (ids[i]: uint32, at least pos+n_pos+1
        entries).  The device time of the call is left in self.device_ms."""
        n = len(slots)
        assert len(ids) == len(pos) == len(n_pos) == len(penalties) == n
        for a, p, k in zip(ids, pos, n_pos):
            assert a.dtype == np.uint32 and a.flags.c_contiguous and a.size >= p + k + 1
        ptrs = (u32p * n)(*[_p(a, u32p) for a in ids])
        s = np.asarray(slots, np.uint32); p = np.asarray(pos, np.uint32); k = np.asarray(n_pos, np.uint32)
        pen = np.asarray(penalties, np.float32)
        acc = np.zeros(n, np.uint32)
        ms = C.c_float(0)
        _check(lib().nb200_batch_verify_greedy(self.h, n, _p(s, u32p), ptrs, _p(p, u32p), _p(k, u32p), _p(pen, f32p), _p(acc, u32p),
                                               C.byref(ms)))
        self.device_ms = float(ms.value)
        return acc.tolist()

    def logits(self, slot: int) -> np.ndarray:
        out = np.empty(self.engine.vocab, dtype=np.float32)
        _check(lib().nb200_batch_read_logits(self.h, int(slot), _p(out, f32p)))
        return out

    def read(self, field: int, count: int, slot: int, layer: int = 0, pos: int = 0) -> np.ndarray:
        """A K (F_KROW) or V (F_VROW) cache row of a slot, as Engine.read gives the engine's."""
        out = np.zeros(count, dtype=np.float32)
        _check(lib().nb200_batch_read_kv(self.h, int(slot), int(field), int(layer), int(pos), _p(out, f32p), int(count)))
        return out

    def close(self):
        if getattr(self, "h", None):
            lib().nb200_batch_destroy(self.h)
            self.h = None
            if self in self.engine._batches:
                self.engine._batches.remove(self)

    def __del__(self):
        try:
            if getattr(self, "h", None) and getattr(self.engine, "h", None):
                self.close()
        except Exception:
            pass


class TpGroup:
    """All ranks of a tensor-parallel group inside ONE process (one engine per visible GPU, one host thread per rank
    for the blocking calls).  Multi-process hosts (one rank per process, e.g. under torchrun) use Engine(tp=...) with
    tp_export / tp_attach_ipc instead -- see bench.py."""

    def __init__(self, model, max_seq: int, size: int, flags: int = 0, devices=None):
        if isinstance(model, (str, os.PathLike)):
            model = np.fromfile(model, dtype=np.uint8).tobytes()
        devices = list(devices) if devices is not None else list(range(size))
        self.ranks = [Engine(model, max_seq, device=devices[r], flags=flags, tp=(r, size)) for r in range(size)]
        arr = (C.c_void_p * size)(*[e.h for e in self.ranks])
        for e in self.ranks:
            _check(lib().nb200_tp_attach_local(e.h, arr))
            e._refresh()
        self.size = size
        self.vocab = self.ranks[0].vocab

    def _all(self, fn):
        import threading
        out = [None] * self.size; err = [None] * self.size

        def run(r):
            try:
                out[r] = fn(self.ranks[r], r)
            except BaseException as ex:      # noqa: BLE001 - re-raised below
                err[r] = ex
        ts = [threading.Thread(target=run, args=(r,)) for r in range(self.size)]
        for t in ts: t.start()
        for t in ts: t.join()
        for ex in err:
            if ex is not None: raise ex
        return out

    def forward(self, token: int, pos: int, causal: int = 1) -> np.ndarray:
        parts = self._all(lambda e, r: e.forward(token, pos, causal))
        full = np.empty(self.vocab, np.float32)
        for e, p in zip(self.ranks, parts):
            lo, hi = e.logits_slice(); full[lo:hi] = p[lo:hi]
        return full

    def next_greedy(self, ids: np.ndarray, pos: int, prefilling: int, penalty: float = 1.0) -> int:
        got = self._all(lambda e, r: e.next_greedy(ids, pos, prefilling, penalty))
        assert len(set(got)) == 1, f"ranks disagree: {got}"
        return got[0]

    def decode_greedy(self, ids: np.ndarray, n_prompt: int, n_total: int, penalty: float = 1.0):
        copies = [ids.copy() for _ in range(self.size)]
        times = self._all(lambda e, r: e.decode_greedy(copies[r], n_prompt, n_total, penalty))
        for c in copies[1:]:
            assert np.array_equal(c[:n_total], copies[0][:n_total]), "ranks disagree on the decoded ids"
        ids[:n_total] = copies[0][:n_total]
        return max(t[0] for t in times), max(t[1] for t in times)

    def close(self):
        for e in self.ranks: e.close()


# ---- op-level wrappers (host arrays in/out) ----
def op_rmsnorm(x, gain, exact=0):
    x = np.ascontiguousarray(x, np.float32); gain = np.ascontiguousarray(gain, np.float32)
    out = np.empty_like(x)
    _check(lib().nb200_op_rmsnorm(_p(out, f32p), _p(x, f32p), _p(gain, f32p), x.size, exact))
    return out


def op_q80_quantize(x, gs):
    x = np.ascontiguousarray(x, np.float32)
    codes = np.empty(x.size, np.int8); scales = np.empty(x.size // gs, np.float32)
    _check(lib().nb200_op_q80_quantize(_p(codes, i8p), _p(scales, f32p), _p(x, f32p), x.size, gs))
    return codes, scales


def op_q80_matvec(x, w_codes, w_scales, n, d, gs):
    x = np.ascontiguousarray(x, np.float32); w_codes = np.ascontiguousarray(w_codes, np.int8)
    w_scales = np.ascontiguousarray(w_scales, np.float32)
    out = np.empty(d, np.float32)
    _check(lib().nb200_op_q80_matvec(_p(out, f32p), _p(x, f32p), _p(w_codes, i8p), _p(w_scales, f32p), n, d, gs))
    return out


def op_f32_matvec(x, w, n, d, exact=0):
    x = np.ascontiguousarray(x, np.float32); w = np.ascontiguousarray(w, np.float32)
    out = np.empty(d, np.float32)
    _check(lib().nb200_op_f32_matvec(_p(out, f32p), _p(x, f32p), _p(w, f32p), n, d, exact))
    return out


def op_q4k_quantize(x):
    x = np.ascontiguousarray(x, np.float32)
    blocks = np.zeros((x.size // 256) * 160, np.uint8)
    _check(lib().nb200_op_q4k_quantize(_p(blocks, u8p), _p(x, f32p), x.size))
    return blocks


def op_q4k_matvec(x, w_blocks, n, d):
    x = np.ascontiguousarray(x, np.float32); w_blocks = np.ascontiguousarray(w_blocks, np.uint8)
    out = np.empty(d, np.float32)
    _check(lib().nb200_op_q4k_matvec(_p(out, f32p), _p(x, f32p), _p(w_blocks, u8p), n, d))
    return out


def op_q4k_quantize_blocks(x):
    """Whole tensor (size % 256 == 0) -> reference 160-byte blocks (quantize_tensor_q4k_in_situ)."""
    x = np.ascontiguousarray(x, np.float32).reshape(-1)
    blocks = np.zeros((x.size // 256) * 160, np.uint8)
    _check(lib().nb200_op_q4k_quantize_blocks(_p(blocks, u8p), _p(x, f32p), x.size // 256))
    return blocks


def op_q4k_matvec_blocks(x_blocks, w_blocks, n, d):
    """matmul_q4k with both operands already in the reference block layout."""
    x_blocks = np.ascontiguousarray(x_blocks, np.uint8); w_blocks = np.ascontiguousarray(w_blocks, np.uint8)
    out = np.empty(d, np.float32)
    _check(lib().nb200_op_q4k_matvec_blocks(_p(out, f32p), _p(x_blocks, u8p), _p(w_blocks, u8p), n, d))
    return out


def host_expf_ref(x: np.ndarray) -> np.ndarray:
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(x)
    lib().nb200_host_expf_ref_array(_p(out, f32p), _p(x, f32p), x.size)
    return out
