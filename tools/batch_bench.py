"""Batched multi-session decode: nb200_batch_next_greedy against the engine's single-session nb200_decode_greedy.

    python tools/batch_bench.py [--workloads nano-168m-q80,qwen3-0.6b-q80,qwen3-0.6b-q4k] [--sessions 1,2,4,8,16] [--upto N]
                                [--temperature T --top-p P]

For each workload of bench.py (same model file, same max_seq_len) and each number of sessions B:
  B sessions in one batch on the default engine, each with its own 16-token prompt (nb200_batch_prefill of positions 0..14),
  then greedy steps of all B sessions together (penalty 1.0) until every session holds `upto` ids (512 for Nano-168M, 2048
  for Qwen3-0.6B, or --upto);
  agg_tok_s      B * steps / the summed device_ms (CUDA events) of the steps;
  per_session    agg_tok_s / B;
  vs_single      agg_tok_s / single_tok_s, where single_tok_s is nb200_decode_greedy's decode rate for one session of the same
                 length on the same engine's default path (median of 3 after 1 warm-up).
Session 0's ids are checked against the single-session ids of a FLAG_NO_STREAM engine (same prompt, same length): `equal`.
With --temperature T --top-p P (T > 0) every session also runs the same schedule through nb200_batch_next_sampled, its coins
drawn from its own xorshift stream (oracle.bindings.random_f32, seed 1000 + session):
  sampled_agg_tok_s   B * steps / the summed device_ms of the sampled steps;
  sample_ms           the mean over positions of (sampled device_ms - greedy device_ms): what sampling adds to a call;
  single_sampled_tok_s  Engine.next_sampled's rate for one session (host clock around the calls, each of which ends in a
                      synchronise);
and `equal` becomes: session 0's sampled ids equal a FLAG_NO_STREAM engine's next_sampled ids with the same coins.
Prints one JSON line with the card's name and power limit (read-only nvidia-smi query).  Writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from nano_b200 import engine as E, modelfile as mf  # noqa: E402
from oracle import bindings as ob  # noqa: E402
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


def coin_stream(session, n):
    st, out = 1000 + session, []
    for _ in range(n):
        c, st = ob.random_f32(st)
        out.append(float(c))
    return out


def single_sampled(eng, prompt, upto, T, top_p, coins):
    """One session through Engine.next_sampled from position PROMPT - 1 (prompt prefilled): (ids, tok/s on the host clock)."""
    ids = np.zeros(upto + 1, np.uint32); ids[:PROMPT] = prompt
    eng.prefill(ids, 0, PROMPT - 1)
    t0 = time.perf_counter()
    for k, pos in enumerate(range(PROMPT - 1, upto - 1)):
        ids[pos + 1] = eng.next_sampled(ids, pos, 1.0, T, top_p, coins[k])[0]
    return ids[:upto].copy(), (upto - PROMPT) / (time.perf_counter() - t0)


def measure(workload, sessions, upto, T=0.0, top_p=1.0):
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
    steps = upto - PROMPT
    if T > 0:
        coins = [coin_stream(i, steps) for i in range(max(sessions))]
        want, _ = single_sampled(ref, prompts[0], upto, T, top_p, coins[0])
        single_sampled(eng, prompts[0], upto, T, top_p, coins[0])         # warm-up
        _, single_s = single_sampled(eng, prompts[0], upto, T, top_p, coins[0])
    ref.close()
    out = []
    for B in sessions:
        batch = eng.batch(B)
        ids = [np.zeros(upto + 1, np.uint32) for _ in range(B)]
        for i in range(B):
            ids[i][:PROMPT] = prompts[i]
            batch.prefill(i, ids[i], 0, PROMPT - 1)
        greedy_ms = []
        slots = list(range(B))
        for pos in range(PROMPT - 1, upto - 1):
            got = batch.next_greedy(slots, ids, [pos] * B, [1.0] * B)
            greedy_ms.append(batch.device_ms)
            for i in range(B):
                ids[i][pos + 1] = got[i]
        agg = B * steps / (sum(greedy_ms) / 1e3)
        row = {"workload": workload, "sessions": B, "upto": upto, "chunk": batch.info()["chunk"],
               "agg_tok_s": round(agg, 1), "per_session_tok_s": round(agg / B, 1), "single_tok_s": round(single, 1),
               "single_path": eng.path.split(" (")[0], "vs_single": round(agg / single, 2),
               "equal": bool(np.array_equal(ids[0][:upto], want))}
        batch.close()
        if T > 0:
            batch = eng.batch(B)
            ids = [np.zeros(upto + 1, np.uint32) for _ in range(B)]
            for i in range(B):
                ids[i][:PROMPT] = prompts[i]
                batch.prefill(i, ids[i], 0, PROMPT - 1)
            sampled_ms = []
            for k, pos in enumerate(range(PROMPT - 1, upto - 1)):
                got, _six = batch.next_sampled(slots, ids, [pos] * B, [1.0] * B, [T] * B, [top_p] * B, [coins[i][k] for i in range(B)])
                sampled_ms.append(batch.device_ms)
                for i in range(B):
                    ids[i][pos + 1] = got[i]
            sagg = B * steps / (sum(sampled_ms) / 1e3)
            row.update({"temperature": T, "top_p": top_p, "sampled_agg_tok_s": round(sagg, 1),
                        "sample_ms": round(float(np.mean(np.subtract(sampled_ms, greedy_ms))), 4),
                        "single_sampled_tok_s": round(single_s, 1), "equal": bool(np.array_equal(ids[0][:upto], want))})
            batch.close()
        out.append(row)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(UPTO))
    ap.add_argument("--sessions", default="1,2,4,8,16")
    ap.add_argument("--upto", type=int, default=0, help="ids per session at the end (default: 512 Nano-168M, 2048 Qwen3-0.6B)")
    ap.add_argument("--temperature", type=float, default=0.0, help="> 0: also measure nb200_batch_next_sampled")
    ap.add_argument("--top-p", type=float, default=1.0)
    args = ap.parse_args()
    name, pl = card()
    sessions = [int(s) for s in args.sessions.split(",")]
    res = []
    for w in args.workloads.split(","):
        res += measure(w, sessions, args.upto, args.temperature, args.top_p)
    print(json.dumps({"card": name, "power_limit_w": pl, "rows": res}))


if __name__ == "__main__":
    main()
