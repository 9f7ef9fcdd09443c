"""Speculative greedy decoding: nb200_verify_greedy and nb200_decode_lookup against the engine's plain greedy paths.

    python tools/lookup_bench.py [--workloads nano-168m-q80,qwen3-0.6b-q80,qwen3-0.6b-q4k] [--b-upto 512]

For each workload of bench.py (same model file, same max_seq_len), with its 16-token prompt:
  (a) verify_ms[n]    device time (CUDA events) of one nb200_verify_greedy pass of n = 1, 2, 4, 8, 16 positions at the middle of
                      the bench length (median of 5 after 1 warm-up), next to the time of one token of the default path and of
                      the multi-kernel path (NB200_FLAG_NO_STREAM): nb200_decode_greedy's decode device_ms over the bench length
                      divided by its tokens (median of 3 after 1 warm-up);
  (b) controlled acceptance: decoding from the prompt to --b-upto ids with verify passes of n = 8 and 16 positions whose n-1
      drafts are the reference continuation (the NO_STREAM engine's greedy ids) with each id replaced by a random one with
      probability `rate`; tok_s = ids produced / summed verify device_ms, mean_ids_per_pass = ids produced / passes; ids are
      checked against the reference (`equal`); break_even: the mean ids per pass at which tok_s reaches the default path's
      rate (linear interpolation between the measured rates; None if no measured rate reaches it);
  (c) nb200_decode_lookup (ngram_max 3, draft_max M-1) on bench.py's workload (prompt 16, greedy to 512 / 2048), its
      stats and tok_s = decoded ids / decode device_ms (this segment includes the host's drafting between passes), next to
      nb200_decode_greedy on the default path; `equal`: its ids equal the NO_STREAM engine's nb200_decode_greedy ids.
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
RATES = (0.0, 0.1, 0.25, 0.5, 1.0)


def greedy(eng, prompt, upto, reps=4):
    """(ids, ms per decoded token: median over reps - 1 runs after a warm-up)."""
    ms = []
    for rep in range(reps):
        ids = np.zeros(upto + 1, np.uint32); ids[:PROMPT] = prompt
        _pre, dec_ms = eng.decode_greedy(ids, PROMPT, upto)
        if rep:
            ms.append(dec_ms / (upto - PROMPT))
    return ids[:upto].copy(), float(np.median(ms))


def verify_times(eng, ref_ids, pos):
    eng.prefill(ref_ids, 0, pos)
    out = {}
    for n in (1, 2, 4, 8, 16):
        t = []
        for rep in range(6):
            ids = ref_ids.copy()
            eng.verify_greedy(ids, pos, n)
            if rep:
                t.append(eng.verify_ms)
        out[n] = round(float(np.median(t)), 4)
    return out


def controlled(eng, ref_ids, upto, n, rate, vocab, seed=5):
    rng = np.random.default_rng(seed)
    ids = np.zeros(upto + n + 1, np.uint32); ids[:PROMPT] = ref_ids[:PROMPT]
    eng.prefill(ids, 0, PROMPT - 1)
    pos, passes, ms = PROMPT - 1, 0, 0.0
    while pos + 1 < upto:
        m = min(n, upto - 1 - pos)
        d = ref_ids[pos + 1: pos + m].copy()
        bad = rng.random(d.size) < rate
        d[bad] = (d[bad] + 1 + rng.integers(0, vocab - 1, int(bad.sum()))) % vocab
        ids[pos + 1: pos + m] = d
        a = eng.verify_greedy(ids, pos, m)
        ms += eng.verify_ms
        passes += 1
        pos += a + 1
    produced = pos - (PROMPT - 1)
    return {"n": n, "rate": rate, "tok_s": round(produced / (ms / 1e3), 1), "mean_ids_per_pass": round(produced / passes, 2),
            "equal": bool(np.array_equal(ids[:upto], ref_ids[:upto]))}


def break_even(rows, target):
    pts = sorted((r["mean_ids_per_pass"], r["tok_s"]) for r in rows)
    for (x0, y0), (x1, y1) in zip(pts, pts[1:]):
        if y0 < target <= y1 and y1 > y0:
            return round(x0 + (target - y0) * (x1 - x0) / (y1 - y0), 2)
    return None


def measure(workload, b_upto):
    preset, _quant, _gs, seq = bench.WORKLOADS[workload]
    spec = mf.PRESETS[preset]
    path = bench.model_path(workload)
    upto = min(UPTO[workload], seq)
    prompt = mf.teacher_tokens(PROMPT, spec.vocab)[:PROMPT]
    eng = E.Engine(path, seq)
    ref = E.Engine(path, seq, flags=E.FLAG_NO_STREAM)
    ref_ids, mk_ms = greedy(ref, prompt, upto)
    def_ids, def_ms = greedy(eng, prompt, upto)
    row = {"workload": workload, "upto": upto, "path": eng.path.split(" (")[0],
           "token_ms_default": round(def_ms, 4), "token_ms_multikernel": round(mk_ms, 4)}
    # (a)
    row["verify_ms"] = verify_times(eng, np.concatenate([ref_ids, np.zeros(17, np.uint32)]), upto // 2)
    # (b)
    bu = min(b_upto, upto)
    ctl = [controlled(eng, ref_ids, bu, n, r, spec.vocab) for n in (8, 16) for r in RATES]
    row["controlled"] = ctl
    row["controlled_upto"] = bu
    row["break_even_ids_per_pass"] = {n: break_even([c for c in ctl if c["n"] == n], 1e3 / def_ms) for n in (8, 16)}
    # (c)
    runs = []
    for rep in range(3):
        ids = np.zeros(upto + 1, np.uint32); ids[:PROMPT] = prompt
        stats, _pre, dec_ms = eng.decode_lookup(ids, PROMPT, upto, 1.0, 3)
        if rep:
            runs.append(dec_ms)
    row["lookup"] = {"tok_s": round((upto - PROMPT) / (float(np.median(runs)) / 1e3), 1), "stats": stats,
                     "mean_ids_per_pass": round(stats[3] / stats[0] + 1, 2) if stats[0] else None,
                     "equal": bool(np.array_equal(ids[:upto], ref_ids))}
    row["greedy_default_tok_s"] = round(1e3 / def_ms, 1)
    row["greedy_default_equal_ids"] = bool(np.array_equal(def_ids, ref_ids))
    ref.close(); eng.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(UPTO))
    ap.add_argument("--b-upto", type=int, default=512, help="ids at the end of each controlled-acceptance run (b)")
    args = ap.parse_args()
    name, pl = card()
    res = [measure(w, args.b_upto) for w in args.workloads.split(",")]
    print(json.dumps({"card": name, "power_limit_w": pl, "rows": res}))


if __name__ == "__main__":
    main()
