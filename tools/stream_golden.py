"""Bit-exact fixture of the streaming decode kernel: digests of its logits and K/V rows on seeded 2-layer models.

The cases cover the O and W2 phases (the two matvecs whose operand is not normalised) on shared and on warp-owned tiles
(NB200_OWNED_ROWS=2 forces the latter), Q80 with groups of 64 and 128, and Q4K.  Each case runs `S` teacher-forced
positions on the streaming kernel and records a sha256 digest of every position's logits and of the K / V rows of every
layer at a few positions.  tests/test_gpu_stream_golden.py replays the cases and compares digests.

Regenerate (on a GPU, from a commit whose streaming kernel is known good):
    python tools/stream_golden.py            # writes tests/golden/stream_digests.json
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from nano_b200 import engine as E, modelfile as mf  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "stream_digests.json")
Q80, Q4K = mf.QUANT_Q80, mf.QUANT_Q4K

# (case id, preset, quant, group size, extra NB200_* settings, positions).  long-nano / long-qwen3 have the layer shapes of
# Nano-168M and Qwen3-0.6B; 96 positions take the attention range past one split (hd 48: 80 rows per item) so the O phase
# also reads merged outputs.  ffn3968-nano puts W2 groups in the second poll batch of a warp; ffn7680-nano puts W2 Q4K
# blocks in the second warp slot.
CASES = [
    ("long-nano-q80g128", "long-nano", Q80, 128, {}, 96),
    ("long-nano-q80g64", "long-nano", Q80, 64, {}, 96),
    ("long-nano-q80g128-owned", "long-nano", Q80, 128, {"NB200_OWNED_ROWS": "2"}, 96),
    ("long-nano-q80g64-owned", "long-nano", Q80, 64, {"NB200_OWNED_ROWS": "2"}, 96),
    ("ffn3968-nano-q80g128", "ffn3968-nano", Q80, 128, {}, 40),
    ("ffn3968-nano-q80g64-owned", "ffn3968-nano", Q80, 64, {"NB200_OWNED_ROWS": "2"}, 40),
    ("long-qwen3-q4k", "long-qwen3", Q4K, 128, {}, 96),
    ("long-qwen3-q4k-owned", "long-qwen3", Q4K, 128, {"NB200_OWNED_ROWS": "2"}, 96),
    ("ffn7680-nano-q4k", "ffn7680-nano", Q4K, 128, {}, 40),
]


def _digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()[:32]


def run_case(case):
    """Digests of one case, plus the path the engine ran (the NB200_* settings apply while the engine is created)."""
    cid, preset, quant, gs, extra, S = case
    spec = mf.PRESETS[preset]
    path = mf.cached_model(spec, quant, gs)
    saved = {k: os.environ.get(k) for k in ["NB200_STREAM", *extra]}
    os.environ["NB200_STREAM"] = "1"
    os.environ.update(extra)
    try:
        eng = E.Engine(path, S)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    try:
        toks = mf.teacher_tokens(S, spec.vocab)
        logits = [_digest(eng.forward(toks[p], p)) for p in range(S)]
        kv = {}
        for pos in (0, 1, S // 2, S - 1):
            for l in range(spec.n_layer):
                kv[f"{l}/{pos}"] = [_digest(eng.read(E.F_KROW, spec.kv_dim, l, pos)), _digest(eng.read(E.F_VROW, spec.kv_dim, l, pos))]
        return {"path": eng.path, "logits": logits, "kv": kv}
    finally:
        eng.close()


def main():
    out = {}
    for case in CASES:
        r = run_case(case)
        if not r["path"].startswith("streaming"):
            raise SystemExit(f"{case[0]}: expected the streaming kernel, engine runs {r['path']}")
        out[case[0]] = {"logits": r["logits"], "kv": r["kv"]}
        print(case[0], "ok", r["logits"][-1])
    with open(FIXTURE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", FIXTURE)


if __name__ == "__main__":
    main()
