"""Decode rate of the streaming kernel against its grid width (NB200_STREAM_WIDTH), on bench.py's workloads.

    python tools/width_bench.py [--workloads nano-168m-q80,qwen3-0.6b-q80,qwen3-0.6b-q4k] [--repeats 3] [--widths W,W,..]
                                [--no-trace]

For each workload one engine per width is created: the widths the model allows among num_sms, 7/8 .. 3/8 and 1/3 of it,
and the narrowest it allows.  Then bench.py's step -- the 16-token prompt, then greedy decode to seq -- runs on each engine
in turn, `--repeats` times, widths alternated.  Every width must decode the same ids.  Printed per width: the median decode
rate, the spread (max - min over the repeats) and the us per token.  Then tools/gpu_trace.py's per-phase cycle medians of
CTA 0 at num_sms and at the fastest width, so a change of rate can be put on the exchange / skew or on the row work.  The
card's name and power limit are printed first.
"""
import argparse
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from nano_b200 import engine as E, modelfile as mf  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        return f"nvidia-smi unavailable ({ex})"


def engine_at(path, seq, width):
    """(engine on `width` CTAs, None) or (None, the error: it names the widths the model allows)."""
    os.environ["NB200_STREAM"] = "1"
    os.environ["NB200_STREAM_WIDTH"] = str(width)
    try:
        return E.Engine(path, seq), None
    except E.NB200Error as ex:
        return None, str(ex)
    finally:
        os.environ.pop("NB200_STREAM_WIDTH", None)
        os.environ.pop("NB200_STREAM", None)


def sweep(workload, repeats, ns, widths=None):
    preset, _quant, _gs, seq = bench.WORKLOADS[workload]
    spec = mf.PRESETS[preset]
    path = bench.model_path(workload)
    n_dec = seq - bench.PROMPT
    _none, err = engine_at(path, seq, 0)
    m = re.search(r"runs on (\d+)\.\.(\d+) CTAs", err or "")
    if not m:
        raise SystemExit(f"{workload}: no width range in {err!r}")
    wmin = int(m.group(1))
    cands = widths or (ns, *(ns * k // 8 for k in range(7, 2, -1)), ns // 3, wmin)
    cands = sorted({w for w in cands if wmin <= w <= ns}, reverse=True)
    engines = {}
    for w in cands:
        eng, err = engine_at(path, seq, w)
        if eng is None:
            raise SystemExit(f"{workload}: width {w}: {err}")
        assert eng.stream_width == w, (eng.stream_width, w)
        engines[w] = eng
    rates = {w: [] for w in engines}
    ref_ids = None
    for rep in range(repeats + 1):                     # round 0 warms every engine up
        for w, eng in sorted(engines.items(), reverse=True):
            ids = bench.prompt_ids(spec, seq)
            _pre, dec_ms = eng.decode_greedy(ids, bench.PROMPT, seq)
            if ref_ids is None:
                ref_ids = ids.copy()
            assert np.array_equal(ids, ref_ids), f"{workload}: ids at width {w} differ from width {max(engines)}"
            if rep:
                rates[w].append(n_dec / (dec_ms * 1e-3))
    print(f"\n{workload} (seq {seq}, {n_dec} decoded tokens per run, {repeats} runs per width, alternated; ids identical at every width)")
    print(f"  {'width':>5} {'tok/s median':>13} {'spread':>8} {'us/token':>9}")
    for w in sorted(rates, reverse=True):
        r = rates[w]
        print(f"  {w:5d} {np.median(r):13.1f} {max(r) - min(r):8.1f} {1e6 / np.median(r):9.1f}    runs {[round(x, 1) for x in r]}")
    for eng in engines.values():
        eng.close()
    return max(rates, key=lambda w: np.median(rates[w]))


def trace(workload, width):
    preset, quant, _gs, seq = bench.WORKLOADS[workload]
    qname = {mf.QUANT_Q80: "q80", mf.QUANT_Q4K: "q4k", mf.QUANT_F32: "f32"}[quant]
    env = dict(os.environ, NB200_STREAM="1", NB200_STREAM_WIDTH=str(width))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gpu_trace.py"), preset, str(seq), qname],
                         env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in out.stdout.splitlines() if "per-layer phase medians" in ln or ln.lstrip().startswith("layer0")]
    print(f"  gpu_trace.py at width {width}:" + ("" if lines else f" failed: {out.stderr.strip()[-400:]}"))
    for ln in lines:
        print("    " + ln.strip())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="nano-168m-q80,qwen3-0.6b-q80,qwen3-0.6b-q4k")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--widths", default="", help="comma-separated widths instead of the default list")
    ap.add_argument("--no-trace", action="store_true")
    a = ap.parse_args()
    if E.device_count() < 1:
        raise SystemExit("width_bench.py needs a CUDA device")
    import torch
    ns = torch.cuda.get_device_properties(0).multi_processor_count
    print("card:", card(), f"| {ns} SMs")
    for wl in a.workloads.split(","):
        best = sweep(wl, a.repeats, ns, [int(w) for w in a.widths.split(",") if w])
        if not a.no_trace:
            for w in sorted({ns, best}, reverse=True):
                trace(wl, w)


if __name__ == "__main__":
    main()
