"""Inputs for the temperature / top-p sampler tests (test_sampler_oracle.py on the CPU, test_gpu_sampler.py on the GPU).

Each case is (label, logits [V] float32, temperature, top_p, coin).  The families:
* normal logits, sigma 0.5 / 2 / 8 at temperatures 0.05 / 0.7 / 1 / 5, offsets 0 and +-80: n0 from 1 to all of V;
* ties: all logits equal (n0 = V, the stop near 0.8 V, beyond the first 4096-entry chunk) and logits on a 0.25 grid;
* a peaked distribution: the stop is at sorted index 0 whatever the coin;
* stops exactly at sorted index 4095, 4096 and 8191 (top_p = the float32 prefix sum just before it), the chunk edges of the
  device scan;
* scans that never stop: top_p = 1 (cutoff 0: underflowed zeros are candidates) and top_p above the total;
* coins 0, 0.5, the largest random_f32 value (2^24 - 1) / 2^24, and a coin with fl(coin * cum) equal to a partial CDF sum.
The n0 = 0 case (top_p below 1 / V over a near-flat distribution) is `empty_nucleus_case`; the reference has no defined
result there, so only the engine's rule is tested.
"""
import numpy as np

from oracle import bindings as ob

CHUNK = 4096                                    # kSampChunk, nano_b200/csrc/sample.cu
MAX_COIN = np.float32((2 ** 24 - 1) / 2 ** 24)  # the largest random_f32 value (utils.c:968-970)


def coins(seed=39, n=1):
    st, out = seed, []
    for _ in range(n):
        c, st = ob.random_f32(st)
        out.append(float(c))
    return out


def exact_cdf_coin(logits, T, top_p):
    """A coin with fl(coin * cum) == the CDF sum at some k < last, so the strict `r < cdf` decides the pick; or None."""
    _, _, n0, last, sp, _ = ob.sample_top_p(logits, T, top_p, 0.0, sorted_out=True)
    if n0 == 0 or last < 1:
        return None
    cdf = np.add.accumulate(sp[: last + 1], dtype=np.float32)          # sequential float32 sums, as the scans add them
    cum = cdf[last]
    for k in sorted({last // 2, last - 1, 0, last // 3}):
        target = cdf[k]
        c = np.float32(target / cum)
        for _ in range(64):
            r = np.float32(c * cum)
            if r == target and 0 <= c < 1:
                return float(c)
            c = np.nextafter(c, np.float32(2) if r < target else np.float32(-1), dtype=np.float32)
    return None


def chunk_edge_top_p(logits, T, j):
    """top_p that makes the top-p scan stop exactly at sorted index j (cum[j - 1] > top_p is false, cum[j] > top_p is true)."""
    _, _, n0, _, sp, _ = ob.sample_top_p(logits, T, 1.0, 0.0, sorted_out=True)     # top_p 1: cutoff 0, every index a candidate
    if n0 <= j:
        return None
    cum = np.add.accumulate(sp[: j + 1], dtype=np.float32)      # the sorted prefix does not depend on the cutoff
    top_p = float(cum[j - 1])
    _, _, n0, last = ob.sample_top_p(logits, T, top_p, 0.0)
    return top_p if last == j and n0 > j + 1 else None


def cases(V, seed=0):
    rng = np.random.default_rng(V * 7 + seed)
    base_coins = [0.0, 0.5, float(MAX_COIN)] + coins(V, 2)
    out = []
    k = 0
    for sigma in (0.5, 2.0, 8.0):
        for T in (0.05, 0.7, 1.0, 5.0):
            off = (0.0, 80.0, -80.0)[k % 3]
            k += 1
            lg = (rng.standard_normal(V) * sigma + off).astype(np.float32)
            for c in base_coins:
                out.append((f"normal-s{sigma:g}-T{T:g}-o{off:g}-c{c:.3f}", lg, T, 0.8, c))
            c = exact_cdf_coin(lg, T, 0.8)
            if c is not None:
                out.append((f"normal-s{sigma:g}-T{T:g}-exactcoin", lg, T, 0.8, c))
    flat = np.full(V, 1.25, np.float32)
    for c in base_coins:
        out.append((f"equal-c{c:.3f}", flat, 0.7, 0.8, c))
    c = exact_cdf_coin(flat, 0.7, 0.8)
    if c is not None:
        out.append(("equal-exactcoin", flat, 0.7, 0.8, c))
    quarter = (np.round(rng.standard_normal(V) * 4) / 4).astype(np.float32)
    for top_p in (0.8, 0.95):
        for c in base_coins[:3]:
            out.append((f"quarter-p{top_p}-c{c:.3f}", quarter, 1.0, top_p, c))
        c = exact_cdf_coin(quarter, 1.0, top_p)
        if c is not None:
            out.append((f"quarter-p{top_p}-exactcoin", quarter, 1.0, top_p, c))
    peaked = (rng.standard_normal(V) * 0.5).astype(np.float32)
    peaked[V // 3] = 40.0
    for c in base_coins:
        out.append((f"peaked-c{c:.3f}", peaked, 1.0, 0.8, c))
    near_flat = (rng.standard_normal(V) * 0.05).astype(np.float32)
    for j in (CHUNK - 1, CHUNK, 2 * CHUNK - 1):
        for name, lg in (("nearflat", near_flat), ("equal", flat), ("quarter", quarter)):
            top_p = chunk_edge_top_p(lg, 1.0, j)
            if top_p is None:
                continue
            for c in (0.0, 0.5, float(MAX_COIN)):
                out.append((f"stop{j}-{name}-c{c:.3f}", lg, 1.0, top_p, c))
    wide = (rng.standard_normal(V) * 8).astype(np.float32)
    for top_p in (1.0, 1.5):
        for name, lg, T in (("wide", wide, 0.05), ("nearflat", near_flat, 1.0)):
            for c in (0.0, 0.5, float(MAX_COIN)):
                out.append((f"nostop-p{top_p}-{name}-c{c:.3f}", lg, T, top_p, c))
    return out


def empty_nucleus_case(V):
    """top_p = 0 over a near-flat distribution: cutoff 1 / (V - 1) is above every probability (n0 = 0).  Two indices share the
    largest logit, so the first-max rule is visible."""
    lg = np.zeros(V, np.float32)
    bump = np.float32(0.25 / V)
    lg[V // 2 + 3] = bump
    lg[V - 1] = bump
    return lg, 1.0, 0.0, V // 2 + 3
