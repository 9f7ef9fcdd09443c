"""Batched multi-session decode: nb200_batch_next_greedy against the engine's single-session nb200_decode_greedy.

    python tools/batch_bench.py [--workloads nano-168m-q80,qwen3-0.6b-q80,qwen3-0.6b-q4k] [--sessions 1,2,4,8,16] [--upto N]

For each workload of bench.py (same model file, same max_seq_len) and each number of sessions B:
  B sessions in one batch on the default engine, each with its own 16-token prompt (nb200_batch_prefill of positions 0..14),
  then greedy steps of all B sessions together (penalty 1.0) until every session holds `upto` ids (512 for Nano-168M, 2048
  for Qwen3-0.6B, or --upto);
  agg_tok_s      B * steps / the summed device_ms (CUDA events) of the steps;
  per_session    agg_tok_s / B;
  vs_single      agg_tok_s / single_tok_s, where single_tok_s is nb200_decode_greedy's decode rate for one session of the same
                 length on the same engine's default path (median of 3 after 1 warm-up).
Session 0's ids are checked against the single-session ids of a FLAG_NO_STREAM engine (same prompt, same length): `equal`.
Prints one JSON line with the card's name and power limit (read-only nvidia-smi query).  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from nano_b200 import engine as E, modelfile as mf  # noqa: E402
from prefill_bench import card  # noqa: E402

UPTO = {"nano-168m-q80": 512, "qwen3-0.6b-q80": 2048, "qwen3-0.6b-q4k": 2048}
PROMPT = 16


def single_rate(eng, prompt, upto):
    rates = []
    for rep in range(4):
        ids = np.zeros(upto + 1, np.uint32); ids[:PROMPT] = prompt
        _pre, dec_ms = eng.decode_greedy(ids, PROMPT, upto)
        if rep:
            rates.append((upto - PROMPT) / (dec_ms / 1e3))
    return float(np.median(rates))


def measure(workload, sessions, upto):
    preset, _quant, _gs, seq = bench.WORKLOADS[workload]
    spec = mf.PRESETS[preset]
    path = bench.model_path(workload)
    upto = min(upto or UPTO[workload], seq)
    prompts = [mf.teacher_tokens(PROMPT, spec.vocab, 100 + i)[:PROMPT] for i in range(max(sessions))]
    eng = E.Engine(path, seq)
    single = single_rate(eng, prompts[0], upto)
    ref = E.Engine(path, seq, flags=E.FLAG_NO_STREAM)
    ids = np.zeros(upto + 1, np.uint32); ids[:PROMPT] = prompts[0]
    ref.decode_greedy(ids, PROMPT, upto)
    want = ids[:upto].copy()
    ref.close()
    out = []
    for B in sessions:
        batch = eng.batch(B)
        ids = [np.zeros(upto + 1, np.uint32) for _ in range(B)]
        for i in range(B):
            ids[i][:PROMPT] = prompts[i]
            batch.prefill(i, ids[i], 0, PROMPT - 1)
        ms = 0.0
        slots = list(range(B))
        for pos in range(PROMPT - 1, upto - 1):
            got = batch.next_greedy(slots, ids, [pos] * B, [1.0] * B)
            ms += batch.device_ms
            for i in range(B):
                ids[i][pos + 1] = got[i]
        steps = upto - PROMPT
        agg = B * steps / (ms / 1e3)
        out.append({"workload": workload, "sessions": B, "upto": upto, "chunk": batch.info()["chunk"],
                    "agg_tok_s": round(agg, 1), "per_session_tok_s": round(agg / B, 1), "single_tok_s": round(single, 1),
                    "single_path": eng.path.split(" (")[0], "vs_single": round(agg / single, 2),
                    "equal": bool(np.array_equal(ids[0][:upto], want))})
        batch.close()
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(UPTO))
    ap.add_argument("--sessions", default="1,2,4,8,16")
    ap.add_argument("--upto", type=int, default=0, help="ids per session at the end (default: 512 Nano-168M, 2048 Qwen3-0.6B)")
    args = ap.parse_args()
    name, pl = card()
    sessions = [int(s) for s in args.sessions.split(",")]
    res = []
    for w in args.workloads.split(","):
        res += measure(w, sessions, args.upto)
    print(json.dumps({"card": name, "power_limit_w": pl, "rows": res}))


if __name__ == "__main__":
    main()
