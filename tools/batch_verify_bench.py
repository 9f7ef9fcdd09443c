"""Batched speculative greedy decoding: nb200_batch_verify_greedy against nb200_batch_next_greedy at the same number of sessions.

    python tools/batch_verify_bench.py [--workloads nano-168m-q80,qwen3-0.6b-q80,qwen3-0.6b-q4k] [--sessions 1,2,4,8]
                                       [--rates 0,0.1,0.25,0.5] [--upto N]

For each workload of bench.py (same model file, same max_seq_len) and each number of sessions B:
  B sessions in one batch on the default engine, each with its own 16-token prompt (nb200_batch_prefill of positions 0..14);
  every session's reference continuation is its greedy ids on a FLAG_NO_STREAM engine (nb200_decode_greedy).
  verify: calls of nb200_batch_verify_greedy until every session holds `upto` ids (512 for Nano-168M, 2048 for Qwen3-0.6B, or
      --upto).  In each call every live session drafts k = 16 // B - 1 ids (at least 0) from its reference continuation, each
      draft replaced by a random other id with probability `rate` (as tools/lookup_bench.py (b)), so a call fills B * (k + 1)
      <= 16 rows, one pass;
      tok_s            ids produced by all sessions / the summed device_ms (CUDA events) of the calls;
      mean_ids_per_entry  ids produced / entries verified (a + 1 per entry);
      equal            session 0's ids equal its reference (the NO_STREAM engine's);
  greedy_tok_s: nb200_batch_next_greedy over the same sessions and lengths (penalty 1.0), B * steps / summed device_ms.
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


def start(eng, B, prompts, length):
    batch = eng.batch(B)
    ids = [np.zeros(length, np.uint32) for _ in range(B)]
    for i in range(B):
        ids[i][:PROMPT] = prompts[i]
        batch.prefill(i, ids[i], 0, PROMPT - 1)
    return batch, ids


def greedy_rate(eng, B, prompts, upto):
    batch, ids = start(eng, B, prompts, upto + 1)
    ms = 0.0
    for pos in range(PROMPT - 1, upto - 1):
        got = batch.next_greedy(list(range(B)), ids, [pos] * B, [1.0] * B)
        ms += batch.device_ms
        for i in range(B):
            ids[i][pos + 1] = got[i]
    batch.close()
    return B * (upto - PROMPT) / (ms / 1e3)


def verify_run(eng, B, prompts, refs, upto, rate, vocab, M, seed=5):
    rng = np.random.default_rng(seed)
    k = max(M // B - 1, 0)
    batch, ids = start(eng, B, prompts, upto + M + 1)
    pos = [PROMPT - 1] * B
    ms, entries = 0.0, 0
    while True:
        live = [i for i in range(B) if pos[i] + 1 < upto]
        if not live:
            break
        n_pos = []
        for i in live:
            m = min(k + 1, upto - 1 - pos[i])
            d = refs[i][pos[i] + 1: pos[i] + m].copy()
            bad = rng.random(d.size) < rate
            d[bad] = (d[bad] + 1 + rng.integers(0, vocab - 1, int(bad.sum()))) % vocab
            ids[i][pos[i] + 1: pos[i] + m] = d
            n_pos.append(m)
        acc = batch.verify_greedy(live, [ids[i] for i in live], [pos[i] for i in live], n_pos, [1.0] * len(live))
        ms += batch.device_ms
        entries += len(live)
        for i, a in zip(live, acc):
            pos[i] += a + 1
    batch.close()
    produced = sum(p - (PROMPT - 1) for p in pos)
    return {"rate": rate, "drafts_per_entry": k, "tok_s": round(produced / (ms / 1e3), 1),
            "mean_ids_per_entry": round(produced / entries, 2), "equal": bool(np.array_equal(ids[0][:upto], refs[0][:upto]))}


def measure(workload, sessions, rates, upto):
    preset, _quant, _gs, seq = bench.WORKLOADS[workload]
    spec = mf.PRESETS[preset]
    path = bench.model_path(workload)
    upto = min(upto or UPTO[workload], seq)
    prompts = [mf.teacher_tokens(PROMPT, spec.vocab, 100 + i)[:PROMPT] for i in range(max(sessions))]
    ref = E.Engine(path, seq, flags=E.FLAG_NO_STREAM)
    refs = []
    for p in prompts:
        ids = np.zeros(upto + 1, np.uint32); ids[:PROMPT] = p
        ref.decode_greedy(ids, PROMPT, upto)
        refs.append(ids[:upto].copy())
    ref.close()
    eng = E.Engine(path, seq)
    probe = eng.batch(1)
    M = probe.info()["chunk"]
    probe.close()
    greedy_rate(eng, 1, prompts, min(upto, PROMPT + 32))          # warm-up of both calls' kernels
    verify_run(eng, 1, prompts, refs, min(upto, PROMPT + 32), 0.0, spec.vocab, M)
    out = []
    for B in sessions:
        g = greedy_rate(eng, B, prompts, upto)
        for r in rates:
            row = {"workload": workload, "sessions": B, "upto": upto, "chunk": M, "greedy_tok_s": round(g, 1)}
            row.update(verify_run(eng, B, prompts, refs, upto, r, spec.vocab, M))
            row["vs_greedy"] = round(row["tok_s"] / g, 2)
            out.append(row)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(UPTO))
    ap.add_argument("--sessions", default="1,2,4,8")
    ap.add_argument("--rates", default="0,0.1,0.25,0.5")
    ap.add_argument("--upto", type=int, default=0, help="ids per session at the end (default: 512 Nano-168M, 2048 Qwen3-0.6B)")
    args = ap.parse_args()
    name, pl = card()
    sessions = [int(s) for s in args.sessions.split(",")]
    rates = [float(r) for r in args.rates.split(",")]
    res = []
    for w in args.workloads.split(","):
        res += measure(w, sessions, rates, args.upto)
    print(json.dumps({"card": name, "power_limit_w": pl, "rows": res}))


if __name__ == "__main__":
    main()
