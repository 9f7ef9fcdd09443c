"""Prompt prefill: nb200_prefill against the token-at-a-time prompt segment of nb200_decode_greedy.

    python tools/prefill_bench.py [--workloads nano-168m-q80,qwen3-0.6b-q80,qwen3-0.6b-q4k]

For each workload of bench.py (same model files, same max_seq_len) and prompt lengths 16, 128 and 496 (Nano-168M) or 2047:
  token_ms    the prompt segment (prefill_ms) of decode_greedy on the default engine, median of 3 after 1 warm-up;
  prefill_ms  nb200_prefill's device_ms on the same engine, median of 5 after 2 warm-ups;
  pos/s of each and the speed-up;
  equal       the prefilled K/V rows of every layer equal, bit for bit, those of a FLAG_NO_STREAM engine that ran the prompt
              position by position with nb200_forward.
Prints one JSON line with the card's name and power limit (read-only nvidia-smi query).  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from nano_b200 import engine as E, modelfile as mf  # noqa: E402

LENGTHS = {"nano-168m-q80": (16, 128, 496), "qwen3-0.6b-q80": (16, 128, 2047), "qwen3-0.6b-q4k": (16, 128, 2047)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.splitlines()[0]
        name, pl = (s.strip() for s in out.split(","))
        return name, float(pl)
    except Exception:          # noqa: BLE001 - the card is reported as unknown rather than failing the measurement
        return "unknown", None


def rows(eng, kv_dim, n):
    k = np.stack([[eng.read(E.F_KROW, kv_dim, l, p) for p in range(n)] for l in range(eng.n_layer)])
    v = np.stack([[eng.read(E.F_VROW, kv_dim, l, p) for p in range(n)] for l in range(eng.n_layer)])
    return k, v


def same_bits(a, b):
    return a.shape == b.shape and bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))


def measure(workload):
    preset, _quant, _gs, seq = bench.WORKLOADS[workload]
    spec = mf.PRESETS[preset]
    path = bench.model_path(workload)
    lengths = LENGTHS[workload]
    toks = mf.teacher_tokens(seq + 1, spec.vocab)
    eng = E.Engine(path, seq)
    out = []
    for n in lengths:
        ids = np.zeros(seq + 2, np.uint32); ids[:n + 1] = toks[:n + 1]
        tok = []
        for rep in range(4):
            a = ids.copy()
            pre_ms, _ = eng.decode_greedy(a, n + 1, n + 1)        # the prompt segment runs positions 0 .. n-1
            if rep:
                tok.append(pre_ms)
        pf = []
        for rep in range(7):
            ms = eng.prefill(ids, 0, n)
            if rep >= 2:
                pf.append(ms)
        out.append({"workload": workload, "prompt": n, "path": eng.path.split(" (")[0],
                    "token_ms": float(np.median(tok)), "prefill_ms": float(np.median(pf)), "chunk": eng.prefill_info()["chunk"]})
        out[-1]["_rows"] = rows(eng, spec.kv_dim, n)
    eng.close()
    ref = E.Engine(path, seq, flags=E.FLAG_NO_STREAM)
    done = 0
    for r in out:
        n = r["prompt"]
        for p in range(done, n):
            ref.forward_nolog(int(toks[p]), p)
        done = n
        k, v = rows(ref, spec.kv_dim, n)
        gk, gv = r.pop("_rows")
        r["equal"] = same_bits(gk, k) and same_bits(gv, v)
        r["token_pos_per_s"] = round(n / (r["token_ms"] / 1e3), 1)
        r["prefill_pos_per_s"] = round(n / (r["prefill_ms"] / 1e3), 1)
        r["speedup"] = round(r["token_ms"] / r["prefill_ms"], 2)
    ref.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(LENGTHS))
    args = ap.parse_args()
    name, pl = card()
    res = []
    for w in args.workloads.split(","):
        res += measure(w)
    print(json.dumps({"card": name, "power_limit_w": pl, "rows": res}))


if __name__ == "__main__":
    main()
