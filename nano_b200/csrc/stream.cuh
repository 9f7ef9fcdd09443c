// stream.cuh -- the grid-wide persistent decode kernel (fast mode, one GPU): every SM keeps HBM streaming across
// phase, layer and token boundaries, and no phase boundary costs a fence or a barrier.
//
// One CTA per SM (cooperative launch).  Warp 15 of every CTA is a PRODUCER: it walks the static per-token schedule
//   for l in layers: QKV tiles | K/V tiles of this CTA's attention item | O tiles | W1|W3 tiles | W2 tiles ; classifier tiles
// and issues cp.async.bulk (TMA bulk copies, mbarrier complete_tx) into a shared-memory ring, as far ahead as the ring
// allows -- it never waits for a phase to end.  Weights come from a per-CTA, tile-ordered copy of the model (built once
// at load: a tile = [rows x (row bytes + 16)] [rows x aux] in exactly the order the CTA consumes it, so a tile is ONE
// bulk copy); K/V tiles come straight from the head-major KV cache.
//
// Activations between phases (x, q/k/v of the position, attention output, SwiGLU output) travel through small
// L2-resident vectors of 64-bit words {fp32 value, 32-bit epoch}: a producing warp publishes a finished element with
// ONE 8-byte store, a consuming CTA polls the words it needs until they carry the epoch of the exchange it is waiting
// for.  Value and epoch arrive together (single-copy atomic), so there is no fence, no counter and no grid barrier on
// the per-phase path (a release fence or a counter barrier costs several times a store -> poll hand-off: tools/micro/
// lat_bench.cu, bar_bench.cu).  Vectors that every CTA reads are written to kStRep replicas (different L2 slices, so
// that all SMs reading one hot copy at once do not queue on one slice: tools/micro/exchange_bench.cu).
//   Why a word is never overwritten before its readers are done: a CTA reads an entire vector before it produces
//   anything of the next exchange, so "all of exchange k has arrived" implies every producer of exchange k has finished
//   reading exchange k-1; the writer of a later exchange into the same buffer has (transitively) seen all of k.
// One true grid barrier per token (release/acquire, at the classifier) orders the plain stores -- KV-cache rows, logits,
// ids, repetition-penalty flags -- against the next token's reads (TMA reads of the cache included).
//
// Arithmetic (fast mode only; the bit-exact mode never runs this kernel): exact integer group dots; the fp32 combine of a
// quantised row (infer.c:668-674, tensor.c:425-430) in the reference's order on shared tiles and as one partial per lane
// + a warp tree on warp-owned tiles; tree reductions for rmsnorm / attention, expf and the division by sqrt(head_dim) as
// the reference.  Reference: llm_forward infer/infer.c:971-1018, transformer_block_forward :713-966.
#pragma once
#include "kernels.cuh"
#include "stream_args.h"

namespace nb {

// ---------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// A spin that cannot hang the GPU: after ~2 s the kernel records a code and traps (the host sees a launch failure).
// The spins themselves are inline.  A call to an out-of-line function makes its caller save every live register to the
// stack (local memory) around the call, and with the consumers' state at the 128-register cap that put spill stores and
// reloads on the hot path of every phase.  The give-up is out of line but never returns, so its call sites save nothing.
[[noreturn]] static __device__ __noinline__ void st_give_up(uint32_t *err, uint32_t code) {
    if (err) *err = code;
    __threadfence_system();
    __trap();
}
// A polling warp must not monopolise the SM's MIO pipe (mbarrier, shared-memory and shuffle instructions share it): measured with
// the producer busy-polling a full ring, a 5-step warp shuffle reduction in a consumer warp took ~1000 cycles instead of ~150.
// `sleep_ns` > 0: back off between polls (the producer runs ahead of the consumers and is never latency-critical).
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity, uint32_t *err, uint32_t code, uint32_t sleep_ns = 20) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (sleep_ns) __nanosleep(sleep_ns);
        if (clock64() - t0 > 4000000000ll) st_give_up(err, code);
    }
}
// threadIdx.x through an opaque read, in the consumers' device functions: the compiler cannot hoist what is derived from it
// (lane offsets, slot indices) out of the layer loop, where it would stay live across every phase (128-register cap)
__device__ __forceinline__ uint32_t st_tid() { uint32_t t; asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t)); return t; }
// barrier among the 15 consumer warps only (the producer warp never takes part)
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, %0;" ::"n"(kConsThreads) : "memory"); }

// ---------------------------------------------------------------- exchange words {value, epoch}
__device__ __forceinline__ void xw_ld2(const unsigned long long *p, unsigned long long &a, unsigned long long &b) {
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ unsigned long long xw_ld1(const unsigned long long *p) {
    unsigned long long a;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(a) : "l"(p) : "memory");
    return a;
}
__device__ __forceinline__ void xw_st(unsigned long long *p, float v, uint32_t epoch) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(((unsigned long long)epoch << 32) | __float_as_uint(v)) : "memory");
}
constexpr uint32_t kXwAny = 0xffffffffu;        // timing experiments only (NB200_ABLATE & 16): accept any epoch
__device__ __forceinline__ bool xw_ok(unsigned long long w, uint32_t need) { return (uint32_t)(w >> 32) == need || need == kXwAny; }
__device__ __forceinline__ float xw_val(unsigned long long w) { return __uint_as_float((uint32_t)w); }
// 4 consecutive words (32-byte aligned) -> float4 once all of them carry `need`
// a failed poll of a spin: the clock is read every 256th time only (the loop stays loads and compares), give up after ~2 s
__device__ __forceinline__ void xw_spin_guard(uint32_t it, long long &t0, uint32_t *err, uint32_t code) {
    if ((it & 255u) == 0) {
        if (t0 == 0) t0 = clock64();
        else if (clock64() - t0 > 4000000000ll) st_give_up(err, code);
    }
}
__device__ __forceinline__ float4 xw_poll4(const unsigned long long *p, uint32_t need, uint32_t *err) {
    unsigned long long a, b, c, d;
    long long t0 = 0;
    for (uint32_t it = 1;; it++) {
        xw_ld2(p, a, b); xw_ld2(p + 2, c, d);
        if (xw_ok(a, need) && xw_ok(b, need) && xw_ok(c, need) && xw_ok(d, need)) break;
        xw_spin_guard(it, t0, err, 0x50u);
    }
    return make_float4(xw_val(a), xw_val(b), xw_val(c), xw_val(d));
}
__device__ __forceinline__ float xw_poll1(const unsigned long long *p, uint32_t need, uint32_t *err) {
    unsigned long long a = xw_ld1(p);
    if (!xw_ok(a, need)) {
        const long long t0 = clock64();
        do {
            a = xw_ld1(p);
            if (clock64() - t0 > 4000000000ll) st_give_up(err, 0x51u);
        } while (!xw_ok(a, need));
    }
    return xw_val(a);
}
// one element into every replica of a vector, the stores spread over the `ts` lanes of a team (tl = lane within the team)
__device__ __forceinline__ void xw_publish(unsigned long long *base, uint32_t rs, uint32_t idx, float v, uint32_t epoch, uint32_t tl, uint32_t ts) {
    for (uint32_t r = tl; r < (uint32_t)kStRep; r += ts) xw_st(base + (size_t)r * rs + idx, v, epoch);
}

// ---------------------------------------------------------------- schedule helpers shared by producer and consumers
// split of the attention range over CTAs: as few (kv head, split) items as keep an item under ~chunk_target rows
__device__ __forceinline__ void st_attn_plan(uint32_t range, uint32_t nsplit_max, uint32_t chunk_target, uint32_t &nsplit, uint32_t &chunk) {
    uint32_t ns = (range + chunk_target - 1) / chunk_target;
    if (ns < 1) ns = 1;
    if (ns > nsplit_max) ns = nsplit_max;
    uint32_t c = (range + ns - 1) / ns;
    c = (c + 7u) & ~7u;
    chunk = c;
    nsplit = (range + c - 1) / c;
}

struct StRing {
    uint64_t *full, *empty;
    volatile uint32_t *tile_id;   // [nstages] running index of the tile that owns the stage (written by the producer before the copy).
                                  // Warp-owned tiles are consumed out of step, and mbarrier parity is only unambiguous one phase
                                  // apart: a consumer first waits for ITS tile to own the stage, then for the bytes.
    unsigned char *buf;
    uint32_t nstages, stage_bytes;
};
__device__ __forceinline__ void mbar_arrive_n(uint64_t *bar, uint32_t n) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(n) : "memory");
}
struct StCursor { uint32_t s, par; };     // stage and parity of the next tile (producer: empty parity; consumer: full parity)
__device__ __forceinline__ void st_advance(StCursor &c, uint32_t nstages) { if (++c.s == nstages) { c.s = 0; c.par ^= 1u; } }
struct StOwn { uint32_t row0[5], rows[5]; };      // the rows this CTA owns of every phase kind (shared memory; computed once)
// the consumers' token state (shared memory, identical in every CTA; thread 0 advances it at the end of a token)
struct StStep { uint32_t step, pos, tok, range, nsplit, chunk, causal, n_prompt, advance; float pen; };
// How the 32 lanes of a warp share the rows of a tile, per phase kind (computed once per launch, kept in shared memory:
// run-time integer divisions cost ~150 cycles each and sat on every phase's critical path).
// Q80: a row of G groups is owned by a team of gteam * lg2 lanes (lg2 lanes split the 16-byte chunks of one group);
// rw = rows per warp pass.  F32 / Q4K: one warp per row.
struct StGeo {
    uint8_t lg2[5], gteam[5], ts[5], rw[5], mode[5];      // mode: 0 single rows, 1 pair (w1, w3) on adjacent teams, 2 pair done by one team
    uint8_t team[5][32], tl[5][32];                       // per lane: team index within the warp, lane index within the team
    uint8_t gl[5][32], ul[5][32];                         // per lane: group within the team pass, lane within the group
};

// ---------------------------------------------------------------- producer (warp 15, lane 0)
__device__ __forceinline__ void st_issue_kind(const StreamArgs &g, const StRing &r, StCursor &c, uint32_t &issued, const StKind &k, const uint8_t *base, uint32_t rows) {
    const uint8_t *src = base + k.off;
    for (uint32_t done = 0; done < rows; done += k.tile_rows) {
        const uint32_t tr = min(k.tile_rows, rows - done);
        const uint32_t bytes = (tr * (k.row_stride + k.aux_stride) + 15u) & ~15u;
        mbar_wait(&r.empty[c.s], c.par, g.err, 0x10u, 200);
        r.tile_id[c.s] = issued++;
        mbar_expect_tx(&r.full[c.s], bytes);
        bulk_g2s(r.buf + (size_t)c.s * r.stage_bytes, src, bytes, &r.full[c.s]);
        st_advance(c, r.nstages);
        src += k.tile_stride;
    }
}

static __device__ void st_producer(const StreamArgs &g, const StRing &r, const StOwn &own, uint32_t cta, volatile uint32_t *progress,
                                   uint32_t pos0, uint32_t causal, uint32_t advance) {
    const Dims &d = g.d;
    StCursor c{0u, 1u};                       // parity 1 passes at once on a stage's first use
    uint32_t issued = 0;                      // running tile index
    const uint8_t *base = g.stream + (uint64_t)cta * g.cta_stride;
    const size_t kvl = (size_t)d.KV * d.max_seq * d.hd;
    for (uint32_t step = 0; step < g.n_steps; step++) {
        const uint32_t pos = pos0 + (advance ? step : 0u);
        const uint32_t range = causal ? pos + 1u : d.max_seq;
        uint32_t nsplit, chunk;
        st_attn_plan(range, g.nsplit_max, g.chunk_target, nsplit, chunk);
        for (uint32_t l = 0; l < d.L; l++) {
            const uint8_t *lb = base + (uint64_t)l * g.layer_stride;
            st_issue_kind(g, r, c, issued, g.kind[SK_QKV], lb, own.rows[SK_QKV]);
            if (cta < d.KV * nsplit) {
                const uint32_t kvh = cta / nsplit, sp = cta % nsplit;
                const uint32_t t0 = min(range, sp * chunk), t1 = min(range, t0 + chunk);
                const float *kb = g.kc + l * kvl + (size_t)kvh * d.max_seq * d.hd;
                const float *vb = g.vc + l * kvl + (size_t)kvh * d.max_seq * d.hd;
                for (uint32_t t = t0; t < t1; t += g.kv_tile_rows) {
                    const uint32_t tr = min(g.kv_tile_rows, t1 - t), bytes = tr * d.hd * 4u;
                    // The previous token's row was written with plain stores during this launch: it may be fetched once this
                    // CTA's consumers have passed that token's grid barrier (older rows: at least one barrier or launch ago).
                    if (step > 0 && pos > 0 && pos - 1u >= t && pos - 1u < t + tr) {
                        if (*progress < step) {
                            const long long c0 = clock64();
                            while (*progress < step) { __nanosleep(200); if (clock64() - c0 > 4000000000ll) st_give_up(g.err, 0x11u); }
                        }
                        asm volatile("fence.proxy.async.global;" ::: "memory");     // generic-proxy stores of this launch -> async-proxy (TMA) read
                    }
                    mbar_wait(&r.empty[c.s], c.par, g.err, 0x12u, 200);
                    r.tile_id[c.s] = issued++;
                    mbar_expect_tx(&r.full[c.s], 2u * bytes);
                    unsigned char *dst = r.buf + (size_t)c.s * r.stage_bytes;
                    bulk_g2s(dst, kb + (size_t)t * d.hd, bytes, &r.full[c.s]);
                    bulk_g2s(dst + (size_t)g.kv_tile_rows * d.hd * 4u, vb + (size_t)t * d.hd, bytes, &r.full[c.s]);
                    st_advance(c, r.nstages);
                }
            }
            st_issue_kind(g, r, c, issued, g.kind[SK_O], lb, own.rows[SK_O]);
            st_issue_kind(g, r, c, issued, g.kind[SK_W13], lb, own.rows[SK_W13]);
            st_issue_kind(g, r, c, issued, g.kind[SK_W2], lb, own.rows[SK_W2]);
        }
        st_issue_kind(g, r, c, issued, g.kind[SK_CLS], base + g.cls_off, own.rows[SK_CLS]);
    }
}

// ---------------------------------------------------------------- activation prologue (consumer threads)
// Source vector (exchange words of epoch `need`, or the embedding row in shared memory) -> (rmsnorm) -> activation
// operand of the matvec in shared memory, straight from registers:
//   Q80 (tensor.c:21-46): one quantisation group per lane team, 4 elements per lane; F32: normalised floats;
//   Q4K (tensor.c:144-242): one 256-element block per warp, 8 elements per lane.
// act layouts as in kernels.cuh (act_region_bytes).  KMAX warp slots per warp stay in registers between the
// sum-of-squares pass and the quantise pass (host checks n <= st_prep_max_n).
// fine-grained stamps inside a phase: compiled in only with -DNB200_FINE_TRACE (each costs ~200 cycles on the stamped path: a
// divergent clock read + generic store in front of the next warp-synchronous instruction -- they distort what they measure)
#ifdef NB200_FINE_TRACE
#define ST_DBG(k) do { if (dbg && threadIdx.x == 0) dbg[k] = clock64(); } while (0)
#else
#define ST_DBG(k) do { } while (0)
#endif
constexpr int kStPollB = 2;          // Q80 / F32 warp slots whose exchange words are polled together
static_assert(kStKmax % kStPollB == 0, "stream kernel: poll batches cover the warp slots");
template <int QUANT, int LPG>
__device__ __forceinline__ void st_prep(const StreamArgs &g, const unsigned long long *xsrc, const float *ssrc, uint32_t need, const float *__restrict__ gain,
                                        uint32_t n, unsigned char *act, float *red, unsigned long long *dbg) {
    const int lane = st_tid() & 31, warp = st_tid() >> 5;
    ST_DBG(0);
    if (gain) {      // the gain is applied after the sum of squares: start pulling its lines into L1 while the source is awaited
        for (uint32_t i = st_tid() * 32u; i < n; i += kConsThreads * 32u) asm volatile("prefetch.global.L1 [%0];" ::"l"(gain + i));
    }
    auto nrm = [&](float4 v, float4 gn, float inv) -> float4 {      // infer.c:611: weight * (ss * x)
        return make_float4(__fmul_rn(gn.x, __fmul_rn(inv, v.x)), __fmul_rn(gn.y, __fmul_rn(inv, v.y)),
                           __fmul_rn(gn.z, __fmul_rn(inv, v.z)), __fmul_rn(gn.w, __fmul_rn(inv, v.w)));
    };
    auto sq = [](float4 v, float ss) -> float { return fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, ss)))); };
    auto inverse = [&](float ss) -> float {                         // infer.c:601-609, tree sum in a fixed order
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
        cbar();
        float tot = 0.0f;
#pragma unroll
        for (int w = 0; w < kConsWarps; w++) tot += red[w];
        tot = __fdiv_rn(tot, (float)n);
        tot = __fadd_rn(tot, 1e-5f);
        return __fdiv_rn(1.0f, __fsqrt_rn(tot));
    };
    if constexpr (QUANT == 0x42) {
        uint32_t *xe = reinterpret_cast<uint32_t *>(act);
        uint32_t *xo = reinterpret_cast<uint32_t *>(act + n / 2);
        float4 *gp = reinterpret_cast<float4 *>(act + n);
        const uint32_t NB = n / 256u;
        float4 v[kStKmaxQ4K][2];
        float ss = 0.0f;
#pragma unroll
        for (int j = 0; j < kStKmaxQ4K; j++) {
            const uint32_t b = warp + kConsWarps * j, base = b * 256u + lane * 8u;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                v[j][h] = make_float4(0, 0, 0, 0);
                if (b < NB) {
                    v[j][h] = ssrc ? *reinterpret_cast<const float4 *>(ssrc + base + 4 * h) : xw_poll4(xsrc + base + 4 * h, need, g.err);
                    ss = sq(v[j][h], ss);
                }
            }
        }
        ST_DBG(1);
        float inv = 1.0f;
        if (gain) inv = inverse(ss);
        ST_DBG(2);
#pragma unroll
        for (int j = 0; j < kStKmaxQ4K; j++) {
            const uint32_t b = warp + kConsWarps * j;
            if (b < NB) {                                            // warp-uniform
                float4 a0 = v[j][0], a1 = v[j][1];
                if (gain) {
                    const float4 *gp4 = reinterpret_cast<const float4 *>(gain + b * 256u + lane * 8u);
                    a0 = nrm(a0, __ldg(gp4), inv); a1 = nrm(a1, __ldg(gp4 + 1), inv);
                }
                const float vv[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                uint32_t c[8]; int csum, s6, b6; float sc, sbias;
                q4k_quantize_block(vv, c, csum, sc, sbias, s6, b6);
                xe[b * 32 + lane] = c[0] | (c[2] << 8) | (c[4] << 16) | (c[6] << 24);
                xo[b * 32 + lane] = c[1] | (c[3] << 8) | (c[5] << 16) | (c[7] << 24);
                if ((lane & 3) == 0) gp[b * 8 + (lane >> 2)] = make_float4(__fmul_rn((float)s6, sc), __fmul_rn((float)b6, sbias), (float)csum, 0.0f);
            }
        }
    } else {
        // Q80: a group (gs elements) is held by LG = gs/4 lanes, 4 elements (one float4) per lane, GW = 32/LG groups per warp slot
        // (measured: one group per warp with 4 elements per lane has the shorter dependent chain; 8 per lane was ~600 cycles slower).
        // F32: no grouping semantics, 128-element slots.
        constexpr uint32_t gs = (QUANT == 0x80) ? LPG * 16u : 128u;
        constexpr uint32_t LG = gs / 4u;                                 // lanes per group (16 or 32)
        constexpr uint32_t GW = 32u / LG;                                // groups per warp slot
        static_assert(LG == 16 || LG == 32, "stream kernel: Q80 group size 64 or 128");
        const uint32_t G = (n + gs - 1u) / gs;                           // F32: n % 4 == 0 only, the last slot may be partial
        const uint32_t sub = lane / LG, li = lane % LG;
        auto slot_i = [&](int j) -> uint32_t { return ((warp + kConsWarps * j) * GW + sub) * gs + li * 4u; };
        // a slot's 4 values (0 past n) once they are known to have arrived: shared source, or exchange words already polled
        auto reread = [&](int j) -> float4 {
            const uint32_t i = slot_i(j);
            float4 a = make_float4(0, 0, 0, 0);
            if (i < n) {
                if (ssrc) a = *reinterpret_cast<const float4 *>(ssrc + i);
                else {
                    unsigned long long w0, w1, w2, w3;
                    xw_ld2(xsrc + i, w0, w1); xw_ld2(xsrc + i + 2, w2, w3);
                    a = make_float4(xw_val(w0), xw_val(w1), xw_val(w2), xw_val(w3));
                }
            }
            return a;
        };
        // The slots are read in batches of kStPollB: every load of a batch is in flight before its first epoch is looked at,
        // and a batch that is not complete is polled again whole.  Every n <= 15 * kStPollB * 128 (all phases of Nano and
        // Qwen3-0.6B) is one batch, i.e. one round trip.  Only the first batch stays in registers until the quantise pass;
        // later batches are read again there (their words cannot change before this CTA has published its next exchange).
        // Holding all six slots took 48 staging + 24 value registers and spilled to local memory on every phase.
        float4 v[kStPollB];
        float ss = 0.0f;
#pragma unroll
        for (int j0 = 0; j0 < kStKmax; j0 += kStPollB) {
            float4 vb[kStPollB];
            if (ssrc) {
#pragma unroll
                for (int b = 0; b < kStPollB; b++) vb[b] = reread(j0 + b);
            } else {
                unsigned long long w[kStPollB][4];
                long long t0 = 0;
                for (uint32_t it = 1;; it++) {
                    bool ok = true;
#pragma unroll
                    for (int b = 0; b < kStPollB; b++) {
                        // defined on every path (a slot past n reads as 0.0f): a register written only under a predicate
                        // stays live around the layer loop, as the compiler cannot see that it is never read unwritten
                        w[b][0] = w[b][1] = w[b][2] = w[b][3] = 0ull;
                        const uint32_t i = slot_i(j0 + b);
                        if (i < n) { xw_ld2(xsrc + i, w[b][0], w[b][1]); xw_ld2(xsrc + i + 2, w[b][2], w[b][3]); }
                    }
#pragma unroll
                    for (int b = 0; b < kStPollB; b++) {
                        if (slot_i(j0 + b) < n) ok = ok && xw_ok(w[b][0], need) && xw_ok(w[b][1], need) && xw_ok(w[b][2], need) && xw_ok(w[b][3], need);
                    }
                    if (ok) break;
                    xw_spin_guard(it, t0, g.err, 0x50u);
                }
#pragma unroll
                for (int b = 0; b < kStPollB; b++) vb[b] = make_float4(xw_val(w[b][0]), xw_val(w[b][1]), xw_val(w[b][2]), xw_val(w[b][3]));
            }
#pragma unroll
            for (int b = 0; b < kStPollB; b++) {
                ss = sq(vb[b], ss);                                   // slot order, as one pass over all slots
                if (j0 == 0) v[b] = vb[b];
            }
        }
        ST_DBG(1);
        float inv = 1.0f;
        if (gain && !(g.ablate & 8u)) inv = inverse(ss);
        ST_DBG(2);
#pragma unroll
        for (int j = 0; j < kStKmax; j++) {
            const uint32_t g0 = (warp + kConsWarps * j) * GW;
            if (g0 < G) {                                            // warp-uniform
                const uint32_t gi = g0 + sub, i = gi * gs + li * 4u;
                const bool on = i < n;
                float4 a = (j < kStPollB) ? v[j] : reread(j);
                if (gain && on) a = nrm(a, __ldg(reinterpret_cast<const float4 *>(gain + i)), inv);
                if constexpr (QUANT == 0x00) {
                    if (on) *reinterpret_cast<float4 *>(act + (size_t)i * 4u) = a;
                } else {
                    int8_t *codes = reinterpret_cast<int8_t *>(act);
                    float *scales = reinterpret_cast<float *>(act + ((n + 15u) & ~15u));
                    // tensor.c:21-46.  amax over the group with one REDUX (the values are non-negative: uint order == float order);
                    // the exact scale amax/127 is off the codes' critical path; codes come from q = v * (127/amax) rounded with the
                    // magic-number add, and any q within 1e-3 of a .5 boundary goes through the exact division + round().
                    const float av[4] = {a.x, a.y, a.z, a.w};
                    float amax = fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w)));
                    const uint32_t gmask = (LG == 32u) ? 0xffffffffu : (0xffffu << (16u * sub));
                    amax = __uint_as_float(__reduce_max_sync(gmask, __float_as_uint(amax)));
                    const float sc = __fdiv_rn(amax, 127.0f);
                    const float rinv = __fdividef(127.0f, amax);
                    if (on) {
                        uint32_t pk = 0;
                        if (sc != 0.0f && !(g.ablate & 1u)) {
                            int cq[4]; bool tie = rinv == 0.0f;
#pragma unroll
                            for (int u = 0; u < 4; u++) {
                                const float q = av[u] * rinv, aq = fabsf(q);
                                const float rr = aq + 12582912.0f;                 // 1.5 * 2^23: the integer nearest to aq sits in the mantissa
                                const float cf = rr - 12582912.0f;
                                const int c = __float_as_int(rr) - 0x4b400000;
                                // rinv = inf (amax < ~3.74e-37) makes this NaN and rinv = 0 (__fdividef, amax > 2^126) makes
                                // every code 0: both take the exact path
                                tie = tie || !(fabsf(aq - cf) <= 0.499f);
                                cq[u] = q < 0.0f ? -c : c;
                            }
                            pk = ((uint32_t)cq[0] & 0xffu) | (((uint32_t)cq[1] & 0xffu) << 8) | (((uint32_t)cq[2] & 0xffu) << 16) | (((uint32_t)cq[3] & 0xffu) << 24);
                            if (tie) {                                           // rare: some q within 1e-3 of a tie -> the exact division + round()
                                pk = 0;                                          // (inline, one division site per slot: q80_code_slow is a call)
#pragma unroll 1
                                for (uint32_t u = 0; u < 4u; u++) {
                                    const float x = u == 0u ? a.x : u == 1u ? a.y : u == 2u ? a.z : a.w;
                                    pk |= ((uint32_t)(int)roundf(__fdiv_rn(x, sc)) & 0xffu) << (8u * u);
                                }
                            }
                        }
                        *reinterpret_cast<uint32_t *>(codes + i) = pk;
                        if (li == 0) scales[gi] = sc;
                    }
                }
            }
        }
    }
    ST_DBG(3);
    cbar();
    ST_DBG(4);
}

// ---------------------------------------------------------------- row dots on a shared-memory tile
// Q80, matmul_quant infer.c:654-679.  A row of G = n/gs groups is owned by a team of gteam * LG2 lanes: LG2 lanes share
// the 16-byte chunks of one group (chunk order rotated by the group index: the lanes of a quarter-warp hit different
// banks), an xor-shuffle over those LG2 lanes leaves the exact integer group sum in each of them, and the fp32 terms are
// summed in group order (the reference's left-to-right sum) by every lane of the team, so the row value ends up in all of
// the team's lanes.  Rows longer than gteam groups take several passes (LG2 = 1 then).
template <int LPG>
__device__ __forceinline__ float st_row_q80_lpg(const unsigned char *wrow, const float *srow, uint32_t n, const unsigned char *act,
                                                uint32_t lg2, uint32_t gteam, uint32_t gl, uint32_t u, uint32_t team_base, unsigned long long *dbg = nullptr) {
    constexpr uint32_t gs = LPG * 16;
    ST_DBG(10);
    const float *xs = reinterpret_cast<const float *>(act + ((n + 15u) & ~15u));
    const uint32_t G = n / gs;
    float val = 0.0f;
    for (uint32_t g0 = 0; g0 < G; g0 += gteam) {               // warp-uniform
        const uint32_t gi = g0 + gl;
        const uint32_t gc = gi < G ? gi : G - 1u;
        const unsigned char *wp = wrow + (size_t)gc * gs, *xp = act + (size_t)gc * gs;
        int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
        for (uint32_t c = u; c < (uint32_t)LPG; c += lg2) {
            const uint32_t off = ((c + gl * lg2) % LPG) * 16u;
            const int4 w = *reinterpret_cast<const int4 *>(wp + off), xq = *reinterpret_cast<const int4 *>(xp + off);
            a0 = __dp4a(w.x, xq.x, a0); a1 = __dp4a(w.y, xq.y, a1); a2 = __dp4a(w.z, xq.z, a2); a3 = __dp4a(w.w, xq.w, a3);
        }
        int isum = (a0 + a1) + (a2 + a3);
        for (uint32_t o = 1; o < lg2; o <<= 1) isum += __shfl_xor_sync(0xffffffffu, isum, o);
        ST_DBG(11);
        const float term = __fmul_rn(__fmul_rn((float)isum, srow[gc]), xs[gc]);
        ST_DBG(12);
        const uint32_t cnt = min(gteam, G - g0);
        for (uint32_t j0 = 0; j0 < cnt; j0 += 8u) {           // the shuffles of a batch are issued before the ordered adds
            float t8[8];
#pragma unroll
            for (int j = 0; j < 8; j++) t8[j] = __shfl_sync(0xffffffffu, term, team_base + ((j0 + j) * lg2 & 31u));
#pragma unroll
            for (int j = 0; j < 8; j++) if (j0 + j < cnt) val = __fadd_rn(val, t8[j]);
        }
        ST_DBG(13);
    }
    return val;
}
// Throughput form for warp-owned tiles: a whole warp owns RB rows, lanes split K in 16-byte chunks (512 bytes per step,
// conflict-free).  Nothing crosses lanes inside the loop: every lane keeps one fp32 partial per row
// (exact integer sum of its 16 codes x the two group scales), the steps are independent of each other so the loads of
// several steps are in flight at once, and one xor-butterfly per row at the end leaves the value in every lane.
// (Fast mode: the fp32 summation order differs from matmul_quant infer.c:654-679; the bit-exact mode never runs this kernel.)
template <int LPG, int RB>
__device__ __forceinline__ void st_rows_q80_warp(const unsigned char *wrow, uint32_t row_stride, const unsigned char *srow, uint32_t aux_stride,
                                                 uint32_t n, const unsigned char *act, float (&val)[RB]) {
    constexpr uint32_t gs = LPG * 16;
    const int lane = st_tid() & 31;
    const float *xs = reinterpret_cast<const float *>(act + ((n + 15u) & ~15u));
    float acc[RB];
#pragma unroll
    for (int r2 = 0; r2 < RB; r2++) acc[r2] = 0.0f;
    auto step = [&](uint32_t k) {
        const int4 xq = *reinterpret_cast<const int4 *>(act + k);
        const uint32_t gi = k / gs;
        const float xsc = xs[gi];
#pragma unroll
        for (int r2 = 0; r2 < RB; r2++) {
            const int4 w = *reinterpret_cast<const int4 *>(wrow + (size_t)r2 * row_stride + k);
            const float ws = reinterpret_cast<const float *>(srow + (size_t)r2 * aux_stride)[gi];
            const int s0 = __dp4a(w.y, xq.y, __dp4a(w.x, xq.x, 0)), s1 = __dp4a(w.w, xq.w, __dp4a(w.z, xq.z, 0));
            acc[r2] = fmaf((float)(s0 + s1), ws * xsc, acc[r2]);
        }
    };
    uint32_t k = lane * 16u;
    const uint32_t full = n & ~511u;
#pragma unroll 2
    for (; k < full; k += 512u) step(k);
    if (k < n) step(k);
#pragma unroll
    for (int r2 = 0; r2 < RB; r2++) val[r2] = warp_sum(acc[r2]);
}
// F32: matmul infer.c:637-651, fast mode (one warp per row: lane-split FMA + tree)
__device__ __forceinline__ float st_row_f32(const unsigned char *wrow, uint32_t n, const unsigned char *act) {
    const int lane = st_tid() & 31;
    const float *x = reinterpret_cast<const float *>(act);
    float acc = 0.0f;
#pragma unroll 2
    for (uint32_t k = lane * 4u; k < n; k += 128u) {
        const float4 w = *reinterpret_cast<const float4 *>(wrow + (size_t)k * 4u), xv = *reinterpret_cast<const float4 *>(x + k);
        acc = fmaf(w.x, xv.x, acc); acc = fmaf(w.y, xv.y, acc); acc = fmaf(w.z, xv.z, acc); acc = fmaf(w.w, xv.w, acc);
    }
    return warp_sum(acc);
}
// Q4K: matmul_q4k / dot_two_blocks_q4k tensor.c:359-471 (one warp per row; one lane = one 32-element group per step; side: 20-byte records)
__device__ __forceinline__ float st_row_q4k(const unsigned char *wrow, const unsigned char *side, uint32_t n, const unsigned char *act) {
    const int lane = st_tid() & 31;
    const uint32_t *xe = reinterpret_cast<const uint32_t *>(act);
    const uint32_t *xo = reinterpret_cast<const uint32_t *>(act + n / 2);
    const float4 *gp = reinterpret_cast<const float4 *>(act + n);
    const uint32_t rowbytes = n / 2u;
    float val = 0.0f;
    for (uint32_t k0 = 0; k0 < rowbytes; k0 += 512u) {
        const uint32_t k = k0 + lane * 16u;
        const bool on = k < rowbytes;
        const uint32_t grp = k / 16u, blk = grp >> 3, gi = grp & 7u, j = gi & 3u;
        float term = 0.0f;
        if (on) {
            const int4 w = *reinterpret_cast<const int4 *>(wrow + k);
            const uint32_t *rec = reinterpret_cast<const uint32_t *>(side + (size_t)blk * 20u);
            const float ssc = __uint_as_float(rec[0]), sbi = __uint_as_float(rec[1]);
            const uint32_t bs = (rec[2] >> (8 * j)) & 0xff, bb = (rec[3] >> (8 * j)) & 0xff, bh = (rec[4] >> (8 * j)) & 0xff;
            const uint32_t s6 = (gi < 4) ? (bs & 0x3f) : ((((bs >> 6) << 4) | (bh & 0x0f)) & 0x3f);
            const uint32_t b6 = (gi < 4) ? (bb & 0x3f) : ((((bb >> 6) << 4) | (bh >> 4)) & 0x3f);
            const float sp = __fmul_rn((float)s6, ssc), bp = __fmul_rn((float)b6, sbi);
            const int4 e4 = *reinterpret_cast<const int4 *>(xe + grp * 4), o4 = *reinterpret_cast<const int4 *>(xo + grp * 4);
            const float4 q = gp[grp];
            const int wv[4] = {w.x, w.y, w.z, w.w}, ev[4] = {e4.x, e4.y, e4.z, e4.w}, ov[4] = {o4.x, o4.y, o4.z, o4.w};
            int spq = 0, spp = 0;
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const int lo = wv[t] & 0x0f0f0f0f, hi = (wv[t] >> 4) & 0x0f0f0f0f;
                spq = __dp4a(lo, ev[t], spq); spq = __dp4a(hi, ov[t], spq);
                spp = __dp4a(lo, 0x01010101, spp); spp = __dp4a(hi, 0x01010101, spp);
            }
            term = __fmul_rn(__fmul_rn(sp, q.x), (float)spq);                       // tensor.c:425-428, left to right
            term = __fsub_rn(term, __fmul_rn(__fmul_rn(sp, q.y), (float)spp));
            term = __fsub_rn(term, __fmul_rn(__fmul_rn(q.x, bp), q.z));
            term = __fadd_rn(term, __fmul_rn(__fmul_rn(32.0f, bp), q.y));
        }
        val = __fadd_rn(val, term);             // lane-local partial (fast mode: the order of the fp32 sum differs from tensor.c:425-471)
    }
    return warp_sum(val);
}

// ---------------------------------------------------------------- one matvec phase: tiles from the ring -> epilogue
// The epilogue is selected at run time so that the kernel holds ONE copy of the row loops.
// Every finished element is published at once (st.relaxed {value, epoch}); nothing else marks the end of a phase.
// Two ways to share the tiles of a phase among the 15 consumer warps:
//   shared tiles (few rows per CTA: latency matters): every warp works on every tile, rows spread over lane teams;
//   owned tiles  (many rows per CTA: throughput matters): tile j belongs to warp j % 15, which walks its rows alone
//                with full-warp K-split dots while the other warps do the same on their tiles.
template <int QUANT, int LPG>
__device__ __forceinline__ void st_consume(const StreamArgs &g, const StRing &r, StCursor &c, uint32_t &tcount, const StKind &k, uint32_t epi, uint32_t layer,
                                           uint32_t row0, uint32_t rows, uint32_t epoch, const unsigned char *act, uint32_t pos, float pen,
                                           float *xown, MatvecSmem &ms, const StGeo &geo, uint32_t kid, unsigned long long *dbg) {
    const Dims &d = g.d;
    const int lane = st_tid() & 31, warp = st_tid() >> 5;
    float bestv = -FLT_MAX; uint32_t besti = 0xffffffffu;
    // epilogue of one finished row (value in all `ts` lanes of its team; `ri` = index among the rows this CTA owns)
    auto emit = [&](uint32_t row, uint32_t ri, float v, float v3, bool pub, uint32_t tl, uint32_t ts) {
        if (epi == EPI_SWIGLU) {
            // rows (2i, 2i+1) = (w1 row i, w3 row i); infer.c:937-944
            if (pub) {
                const float sg = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-v)));
                xw_publish(g.xv[2], g.rs[2], row >> 1, __fmul_rn(__fmul_rn(v, sg), v3), epoch, tl, ts);
            }
        } else if (epi == EPI_RESID) {
            const float xn = __fadd_rn(xown[ri], v);                    // infer.c:906, :963
            __syncwarp();
            if (pub) {
                if (tl == 0) xown[ri] = xn;
                xw_publish(g.xv[0], g.rs[0], row, xn, epoch, tl, ts);
            }
        } else if (epi == EPI_QKV) {
            if (pub && tl == 0) {
                xw_st(g.xq + row, v, epoch);
                if (row >= d.q_dim + d.kv_dim) {                         // V rows also go to the cache for later positions
                    const uint32_t cc = row - d.q_dim - d.kv_dim, h = cc / d.hd, i = cc % d.hd;
                    g.vc[(size_t)layer * d.KV * d.max_seq * d.hd + ((size_t)h * d.max_seq + pos) * d.hd + i] = v;
                }
            }
        } else if (pub) {
            // classifier: infer.c:1156-1167 penalty (division, any sign), then first-max argmax :1026-1037 (rows ascend per lane)
            if (pen != 1.0f && __ldcg(g.seen + row)) v = __fdiv_rn(v, pen);
            if (tl == 0) g.logits[row] = v;
            if (v > bestv) { bestv = v; besti = row; }
        }
    };
    if (k.owned) {
        // ---- owned tiles ----
        StCursor cc = c;
        uint32_t j = 0;
        for (uint32_t done = 0; done < rows; done += k.tile_rows, j++) {
            if (j % kConsWarps == (uint32_t)warp) {
                const uint32_t tr = min(k.tile_rows, rows - done), want = tcount + j;
                if (r.tile_id[cc.s] != want) {
                    const long long t0 = clock64();
                    while (r.tile_id[cc.s] != want) { __nanosleep(20); if (clock64() - t0 > 4000000000ll) st_give_up(g.err, 0x28u); }
                }
                mbar_wait(&r.full[cc.s], cc.par, g.err, 0x29u);
                const unsigned char *tile = r.buf + (size_t)cc.s * r.stage_bytes;
                const unsigned char *aux = tile + (size_t)tr * k.row_stride;
                // rows in blocks of 4 / 2 / 1 (SwiGLU tiles hold whole (w1, w3) pairs: an even row count)
                // (unrolled over the block size: a run-time index into v would put it in local memory)
                auto out = [&](uint32_t rr, const auto &v, uint32_t cnt) {
                    constexpr uint32_t RB = sizeof(v) / sizeof(v[0]);
                    if (epi == EPI_SWIGLU) {
#pragma unroll
                        for (uint32_t u = 0; u + 1u < RB; u += 2u) if (u + 1u < cnt) emit(row0 + done + rr + u, done + rr + u, v[u], v[u + 1u], true, (uint32_t)lane, 32u);
                    } else {
#pragma unroll
                        for (uint32_t u = 0; u < RB; u++) if (u < cnt) emit(row0 + done + rr + u, done + rr + u, v[u], 0.0f, true, (uint32_t)lane, 32u);
                    }
                };
                uint32_t rr = 0;
                if constexpr (QUANT == 0x80) {
                    for (; rr + 4u <= tr; rr += 4u) {
                        float v[4];
                        st_rows_q80_warp<LPG, 4>(tile + (size_t)rr * k.row_stride, k.row_stride, aux + (size_t)rr * k.aux_stride, k.aux_stride, k.n, act, v);
                        out(rr, v, 4u);
                    }
                    if (rr + 2u <= tr) {
                        float v[2];
                        st_rows_q80_warp<LPG, 2>(tile + (size_t)rr * k.row_stride, k.row_stride, aux + (size_t)rr * k.aux_stride, k.aux_stride, k.n, act, v);
                        out(rr, v, 2u); rr += 2u;
                    }
                    if (rr < tr) {
                        float v[1];
                        st_rows_q80_warp<LPG, 1>(tile + (size_t)rr * k.row_stride, k.row_stride, aux + (size_t)rr * k.aux_stride, k.aux_stride, k.n, act, v);
                        out(rr, v, 1u);
                    }
                } else {
                    for (; rr < tr; rr += 2u) {
                        const bool two = rr + 1u < tr;
                        const uint32_t r1 = two ? rr + 1u : rr;
                        float v[2];
                        if constexpr (QUANT == 0x42) {
                            v[0] = st_row_q4k(tile + (size_t)rr * k.row_stride, aux + (size_t)rr * k.aux_stride, k.n, act);
                            v[1] = two ? st_row_q4k(tile + (size_t)r1 * k.row_stride, aux + (size_t)r1 * k.aux_stride, k.n, act) : 0.0f;
                        } else {
                            v[0] = st_row_f32(tile + (size_t)rr * k.row_stride, k.n, act);
                            v[1] = two ? st_row_f32(tile + (size_t)r1 * k.row_stride, k.n, act) : 0.0f;
                        }
                        out(rr, v, two ? 2u : 1u);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive_n(&r.empty[cc.s], kConsWarps);      // the only consumer of this stage
            }
            st_advance(cc, r.nstages);
        }
        c = cc; tcount += j;
    } else {
        // ---- shared tiles: lanes per row team and rows per warp pass from the table computed at kernel start ----
        const uint32_t TS = geo.ts[kid], RW = geo.rw[kid], mode = geo.mode[kid], lg2 = geo.lg2[kid], gteam = geo.gteam[kid];
        const uint32_t team = geo.team[kid][lane], tl = geo.tl[kid][lane], team_base = team * TS, gl = geo.gl[kid][lane], ul = geo.ul[kid][lane];
        const bool lane_on = (uint32_t)lane < RW * TS;
        for (uint32_t done = 0; done < rows; done += k.tile_rows) {
            const uint32_t tr = min(k.tile_rows, rows - done);
            ST_DBG(5);
            mbar_wait(&r.full[c.s], c.par, g.err, 0x20u + epi);
            ST_DBG(6);
            const unsigned char *tile = r.buf + (size_t)c.s * r.stage_bytes;
            const unsigned char *aux = tile + (size_t)tr * k.row_stride;
            // rows of a warp pass: mode 0 one row per team; mode 1 the teams 2t, 2t+1 do the two rows of a pair; mode 2 a team does both
            const uint32_t step_rows = (mode == 2u) ? 2u * RW : RW;
            for (uint32_t rb = warp * step_rows; rb < tr; rb += kConsWarps * step_rows) {       // warp-uniform trip count
                const uint32_t rr = rb + (mode == 2u ? 2u * team : team);
                const bool valid = lane_on && rr < tr;
                const uint32_t rc = (rr < tr) ? rr : tr - 1u;
                auto one = [&](uint32_t r2) -> float {
                    const unsigned char *wrow = tile + (size_t)r2 * k.row_stride, *ax = aux + (size_t)r2 * k.aux_stride;
                    if constexpr (QUANT == 0x80) return st_row_q80_lpg<LPG>(wrow, reinterpret_cast<const float *>(ax), k.n, act, lg2, gteam, gl, ul, team_base, dbg);
                    else if constexpr (QUANT == 0x42) return st_row_q4k(wrow, ax, k.n, act);
                    else return st_row_f32(wrow, k.n, act);
                };
                float v = (g.ablate & 2u) ? 0.0f : one(rc), v3 = 0.0f;
                bool pub = valid;                                                 // does this team publish the element?
                if (mode == 2u && !(g.ablate & 2u)) v3 = one(min(rc + 1u, tr - 1u));
                else if (mode == 1u) { v3 = __shfl_sync(0xffffffffu, v, (lane + TS) & 31u); pub = valid && !(team & 1u); }
                ST_DBG(7);
                emit(row0 + done + rc, done + rc, v, v3, pub, tl, TS);
            }
            ST_DBG(8);
            __syncwarp();
            if (lane == 0) mbar_arrive(&r.empty[c.s]);
            st_advance(c, r.nstages);
            tcount++;
        }
    }
    ST_DBG(9);
    if (epi == EPI_CLS) {
#pragma unroll
        for (uint32_t o = 1u; o < 32u; o <<= 1) {                          // first max over the lanes of the warp
            const float ov = __shfl_xor_sync(0xffffffffu, bestv, o); const uint32_t oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (oi != 0xffffffffu && (besti == 0xffffffffu || ov > bestv || (ov == bestv && oi < besti))) { bestv = ov; besti = oi; }
        }
        if (lane == 0) { ms.best_v[warp] = bestv; ms.best_i[warp] = besti; }
    }
}

// ---------------------------------------------------------------- attention item (infer.c:814-879) on K/V tiles from the ring
// One CTA = one (kv head, split).  The item's rows are processed in segments of up to kStSegTiles ring tiles that are
// resident at the same time; per segment three passes with no cross-lane traffic in their inner loops:
//   scores : four lanes per cache row, all KVM query heads of the kv head (K row and q read in 16-byte chunks whose order
//            is rotated by the row index: conflict-free although rows are a multiple of 128 bytes apart)
//   softmax: warp m owns query head m: running max / sum over the segments (online softmax), p = exp(s - max) in place
//   P.V    : one thread per (head, pair of output dims), rows in order
// q (and the position's k) are normalised + RoPE'd in registers (norm_rope_apply) by one warp each; the position's own K / V
// rows (this step's QKV outputs) are written into their slots of the resident tile, so the passes treat all rows alike.
// A range held by one item is normalised and published at once; otherwise every item publishes its partial and the item
// of split 0 merges them in split order.
template <int KVM>
static __device__ void st_attention(const StreamArgs &g, const StRing &r, StCursor &c, uint32_t &tcount, uint32_t layer, uint32_t cta, uint32_t pos, uint32_t range,
                                    uint32_t nsplit, uint32_t chunk, uint32_t e_in, uint32_t e_out, float *sm, unsigned long long *dbg) {
    const Dims &d = g.d;
    if (cta >= d.KV * nsplit) return;
    ST_DBG(0);
    const uint32_t hd = d.hd, hd4 = hd / 4u, hd2 = hd / 2u;
    const uint32_t kvh = cta / nsplit, sp = cta % nsplit;
    const uint32_t t0 = min(range, sp * chunk), t1 = min(range, t0 + chunk);
    const size_t kvl = (size_t)d.KV * d.max_seq * hd;
    float *kbase = g.kc + layer * kvl + (size_t)kvh * d.max_seq * hd;
    const float *qn = g.qnorm ? g.qnorm + (size_t)layer * hd : nullptr, *kn = g.knorm ? g.knorm + (size_t)layer * hd : nullptr;
    const float *cr = g.rope_cos + (size_t)pos * (hd / 2), *ci = g.rope_sin + (size_t)pos * (hd / 2);
    uint32_t lpr = 1; while (lpr * 4 < hd) lpr <<= 1;
    const int lane = st_tid() & 31, warp = st_tid() >> 5;
    const uint32_t li = lane % lpr, col = li * 4;
    const bool colon = col < hd;
    const float dv = sqrtf((float)hd);
    const bool owns = pos >= t0 && pos < t1;
    const uint32_t kvr = g.kv_tile_rows, seg_max = (uint32_t)kStSegTiles * kvr;

    // shared-memory carve-up (floats)
    float *q_s = sm;                                   // [KVM][hd]   normalised + RoPE'd query heads
    float *S = q_s + KVM * hd;                         // [KVM][seg_max] scores, then probabilities
    float *st_scale = S + KVM * seg_max;               // [KVM] e^{m_old - m_new} of the current segment
    float *krow = st_scale + ((KVM + 3) & ~3);         // [hd] the position's k (post-RoPE), [hd] the position's v (16-byte aligned)
    float *outp = krow + 2 * hd;                       // [KVM][hd + 2]: acc, M, L

    // ---- this step's q / k / v: warp m < KVM prepares query head m, warp KVM the k row, warp KVM + 1 the v row ----
    if (warp < KVM + 2) {
        const RopeTab rt = rope_tab_load(cr, ci, d, col, colon);
        float4 gn = make_float4(0, 0, 0, 0), v4 = make_float4(0, 0, 0, 0);
        if (warp < KVM) {
            if (d.arch == 3u && colon) gn = __ldg(reinterpret_cast<const float4 *>(qn + col));
            if (colon) v4 = xw_poll4(g.xq + ((size_t)kvh * KVM + warp) * hd + col, e_in, g.err);
            v4 = norm_rope_apply(v4, gn, rt, d, lpr, col, colon);
            if (colon && (uint32_t)lane < lpr) *reinterpret_cast<float4 *>(q_s + warp * hd + col) = v4;
        } else if (owns) {
            if (warp == KVM) {
                if (d.arch == 3u && colon) gn = __ldg(reinterpret_cast<const float4 *>(kn + col));
                if (colon) v4 = xw_poll4(g.xq + d.q_dim + (size_t)kvh * hd + col, e_in, g.err);
                v4 = norm_rope_apply(v4, gn, rt, d, lpr, col, colon);
                if (colon && (uint32_t)lane < lpr) {
                    *reinterpret_cast<float4 *>(krow + col) = v4;
                    *reinterpret_cast<float4 *>(kbase + (size_t)pos * hd + col) = v4;             // K rows are cached post-RoPE
                }
            } else {
                if (colon) v4 = xw_poll4(g.xq + d.q_dim + d.kv_dim + (size_t)kvh * hd + col, e_in, g.err);
                if (colon && (uint32_t)lane < lpr) *reinterpret_cast<float4 *>(krow + hd + col) = v4;
            }
        }
    }
    // running state: warp m < KVM keeps (max, sum) of head m; thread j (and j + 480) keeps the accumulators of (head, dim pair) j
    float m_run = -FLT_MAX, l_run = 0.0f;
    float2 acc[2] = {make_float2(0.0f, 0.0f), make_float2(0.0f, 0.0f)};
    cbar();
    ST_DBG(1);

    for (uint32_t s0 = t0; s0 < t1; s0 += seg_max) {
        const uint32_t rows_seg = min(seg_max, t1 - s0), nt = (rows_seg + kvr - 1u) / kvr;
        unsigned long long stg = 0;                    // ring stage of resident tile i in byte i (two registers, not kStSegTiles)
        static_assert(kStSegTiles <= 8 && kStMaxStages <= 256, "stream kernel: stage indices packed in bytes");
#pragma unroll
        for (int i = 0; i < kStSegTiles; i++) {
            if ((uint32_t)i < nt) { mbar_wait(&r.full[c.s], c.par, g.err, 0x30u); stg |= (unsigned long long)c.s << (8 * i); st_advance(c, r.nstages); tcount++; }
        }
        auto stage_of = [&](uint32_t ti) -> uint32_t { return (uint32_t)(stg >> (8u * ti)) & 0xffu; };
        auto tile_k = [&](uint32_t ti) -> float * { return reinterpret_cast<float *>(r.buf + (size_t)stage_of(ti) * r.stage_bytes); };
        ST_DBG(2);
        if (owns && pos >= s0 && pos < s0 + rows_seg) {     // CTA-uniform: this step's k / v into their slots of the resident tile
            const uint32_t pr = pos - s0, ti = __umulhi(pr, g.kv_tile_magic), rr = pr - ti * kvr;
            float *kt = tile_k(ti);
            for (uint32_t i = st_tid(); i < hd; i += kConsThreads) {
                kt[(size_t)rr * hd + i] = krow[i];
                kt[(size_t)kvr * hd + (size_t)rr * hd + i] = krow[hd + i];
            }
            cbar();
        }
        ST_DBG(3);
        // ---- scores: task = (row, quarter of the dims), 4 adjacent lanes per row.  The K chunks of the row are loaded once and used for
        //      all KVM query heads (q chunks are broadcast reads); chunk order rotated by the row index: conflict-free although rows are
        //      a multiple of 128 bytes apart.  One round covers 120 rows. ----
        if (!(g.ablate & 4u)) {
            const uint32_t part = st_tid() & 3u;
            for (uint32_t idx = st_tid() >> 2; idx < ((rows_seg + 7u) & ~7u); idx += kConsThreads / 4u) {       // warp-uniform trip count (8 rows per warp)
                const bool on = idx < rows_seg;
                const uint32_t ic = on ? idx : 0u;
                const uint32_t ti = __umulhi(ic, g.kv_tile_magic), rr = ic - ti * kvr;
                const float *kr = tile_k(ti) + (size_t)rr * hd;
                const uint32_t rot = (hd4 & 3u) ? 0u : (4u * (ic & 7u)) % hd4;       // rotation keeps the 4 lanes' chunk sets disjoint only if hd % 16 == 0
                float a[KVM];
#pragma unroll
                for (int m = 0; m < KVM; m++) a[m] = 0.0f;
                constexpr int kUnroll = KVM >= 4 ? 2 : 4;      // KVM = 4: 4 chunks in flight held ~80 registers and spilled
#pragma unroll kUnroll
                for (uint32_t cc = part; cc < hd4; cc += 4u) {
                    uint32_t ch = cc + rot; if (ch >= hd4) ch -= hd4;
                    const float4 k4 = *reinterpret_cast<const float4 *>(kr + ch * 4u);
#pragma unroll
                    for (int m = 0; m < KVM; m++) {
                        const float4 q4 = *reinterpret_cast<const float4 *>(q_s + m * hd + ch * 4u);
                        a[m] = fmaf(k4.x, q4.x, fmaf(k4.y, q4.y, fmaf(k4.z, q4.z, fmaf(k4.w, q4.w, a[m]))));
                    }
                }
#pragma unroll
                for (int m = 0; m < KVM; m++) {
                    a[m] += __shfl_xor_sync(0xffffffffu, a[m], 1);
                    a[m] += __shfl_xor_sync(0xffffffffu, a[m], 2);
                    if (on && part == 0) S[m * seg_max + idx] = __fdiv_rn(a[m], dv);         // infer.c:858
                }
            }
        }
        cbar();
        ST_DBG(4);
        // ---- online softmax over the segment: warp m owns head m ----
        if (warp < KVM && !(g.ablate & 4u)) {
            float *Sm = S + warp * seg_max;
            float mx = -FLT_MAX;
            for (uint32_t i = lane; i < rows_seg; i += 32) mx = fmaxf(mx, Sm[i]);
            ST_DBG(12);
            mx = warp_max(mx);
            ST_DBG(13);
            const float mn = fmaxf(m_run, mx);
            const float sc_old = expf(m_run - mn);
            ST_DBG(14);
            float ls = 0.0f;
            for (uint32_t i = lane; i < rows_seg; i += 32) { const float pr = expf(Sm[i] - mn); Sm[i] = pr; ls += pr; }
            ST_DBG(15);
            ls = warp_sum(ls);
            l_run = fmaf(l_run, sc_old, ls);
            m_run = mn;
            if (lane == 0) st_scale[warp] = sc_old;
        }
        cbar();
        ST_DBG(5);
        // ---- P.V: thread j owns (head, dim pair) j; rows in order, four at a time (probabilities as one float4) ----
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const uint32_t j = st_tid() + u * kConsThreads;
            if (j < KVM * hd2 && !(g.ablate & 4u)) {
                const uint32_t m = j / hd2, dd = (j - m * hd2) * 2u;
                const float *Sm = S + m * seg_max;
                const float sc = st_scale[m];
                float2 a0 = make_float2(acc[u].x * sc, acc[u].y * sc), a1 = make_float2(0, 0), a2 = a1, a3 = a1;
                for (uint32_t ti = 0; ti < nt; ti++) {
                    const float *vt = tile_k(ti) + (size_t)kvr * hd + dd;
                    const uint32_t nr = min(kvr, rows_seg - ti * kvr);
                    const float *sp2 = Sm + ti * kvr;                   // kvr % 4 == 0: 16-byte aligned
                    uint32_t rr = 0;
                    for (; rr + 4u <= nr; rr += 4u) {
                        const float4 p4 = *reinterpret_cast<const float4 *>(sp2 + rr);
                        const float2 v0 = *reinterpret_cast<const float2 *>(vt + (size_t)rr * hd), v1 = *reinterpret_cast<const float2 *>(vt + (size_t)(rr + 1u) * hd);
                        const float2 v2 = *reinterpret_cast<const float2 *>(vt + (size_t)(rr + 2u) * hd), v3 = *reinterpret_cast<const float2 *>(vt + (size_t)(rr + 3u) * hd);
                        a0.x = fmaf(p4.x, v0.x, a0.x); a0.y = fmaf(p4.x, v0.y, a0.y); a1.x = fmaf(p4.y, v1.x, a1.x); a1.y = fmaf(p4.y, v1.y, a1.y);
                        a2.x = fmaf(p4.z, v2.x, a2.x); a2.y = fmaf(p4.z, v2.y, a2.y); a3.x = fmaf(p4.w, v3.x, a3.x); a3.y = fmaf(p4.w, v3.y, a3.y);
                    }
                    for (; rr < nr; rr++) {
                        const float pr = sp2[rr]; const float2 v0 = *reinterpret_cast<const float2 *>(vt + (size_t)rr * hd);
                        a0.x = fmaf(pr, v0.x, a0.x); a0.y = fmaf(pr, v0.y, a0.y);
                    }
                }
                acc[u] = make_float2((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y));
            }
        }
        cbar();
        ST_DBG(6);
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < kStSegTiles; i++) if ((uint32_t)i < nt) mbar_arrive(&r.empty[stage_of(i)]);
        }
    }
    ST_DBG(7);
    // ---- the item's partial: per head [acc[hd], M, L] ----
#pragma unroll
    for (int u = 0; u < 2; u++) {
        const uint32_t j = st_tid() + u * kConsThreads;
        if (j < KVM * hd2) { const uint32_t m = j / hd2, dd = (j - m * hd2) * 2u; outp[m * (hd + 2) + dd] = acc[u].x; outp[m * (hd + 2) + dd + 1u] = acc[u].y; }
    }
    if (warp < KVM && lane == 0) { outp[warp * (hd + 2) + hd] = m_run; outp[warp * (hd + 2) + hd + 1] = l_run; }
    const uint32_t pw = KVM * (hd + 2);                               // words of one partial
    cbar();
    ST_DBG(8);
    if (nsplit == 1) {          // the whole range in one item: normalise and publish
        for (uint32_t el = st_tid(); el < KVM * hd; el += kConsThreads) {
            const uint32_t m = el / hd, i = el - m * hd;
            const float ov = __fdiv_rn(outp[m * (hd + 2) + i], outp[m * (hd + 2) + hd + 1]);
#pragma unroll
            for (uint32_t rep = 0; rep < (uint32_t)kStRep; rep++) xw_st(g.xv[1] + (size_t)rep * g.rs[1] + ((size_t)kvh * KVM + m) * hd + i, ov, e_out);
        }
        return;
    }
    unsigned long long *part = g.xws + ((size_t)kvh * g.nsplit_max) * pw;
    if (sp != 0) {              // publish the partial; split 0 of the kv head merges
        for (uint32_t idx = st_tid(); idx < pw; idx += kConsThreads) xw_st(part + (size_t)sp * pw + idx, outp[idx], e_out);
        return;
    }
    ST_DBG(9);
    // ---- merge (split 0): own partial from shared memory, the others polled from the exchange words ----
    uint32_t region = st_attn_work_floats(KVM, hd, seg_max);
    if (g.nsplit_max * KVM * hd > region) region = g.nsplit_max * KVM * hd;
    float *wsc = sm + region;                            // [KVM][nsplit_max] weights e^{m_s - M}; before that: the maxima
    float *stat = wsc + KVM * g.nsplit_max;              // [KVM] L, then [KVM][nsplit_max] partial sums
    float own[4];                                        // this thread's slice of the own partial (pw <= 4 * 480 for hd <= 128, KVM <= 8)
#pragma unroll
    for (int u = 0; u < 4; u++) { const uint32_t idx = st_tid() + u * kConsThreads; own[u] = idx < pw ? outp[idx] : 0.0f; }
    cbar();                                              // outp / ws are about to be overwritten by the staging area
    float *macc = sm;                                    // [KVM][nsplit][hd]
    float *pl = stat + KVM;                              // [KVM][nsplit_max]
    auto place = [&](uint32_t s2, uint32_t idx, float v) {
        const uint32_t m = idx / (hd + 2), i = idx % (hd + 2);
        if (i < hd) macc[(m * nsplit + s2) * hd + i] = v;
        else if (i == hd) wsc[m * g.nsplit_max + s2] = v;
        else pl[m * g.nsplit_max + s2] = v;
    };
#pragma unroll
    for (int u = 0; u < 4; u++) { const uint32_t idx = st_tid() + u * kConsThreads; if (idx < pw) place(0, idx, own[u]); }
    for (uint32_t e0 = pw + st_tid(); e0 < nsplit * pw; e0 += 8u * kConsThreads) {       // eight loads in flight per thread before any epoch is checked
        unsigned long long w8[8];
#pragma unroll
        for (int u = 0; u < 8; u++) { const uint32_t e = e0 + u * kConsThreads; if (e < nsplit * pw) w8[u] = xw_ld1(part + e); }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const uint32_t e = e0 + u * kConsThreads;
            if (e < nsplit * pw) place(e / pw, e % pw, xw_ok(w8[u], e_out) ? xw_val(w8[u]) : xw_poll1(part + e, e_out, g.err));
        }
    }
    cbar();
    ST_DBG(10);
    if (warp < KVM) {
        float pm[2], pls[2];                             // nsplit_max <= 64: two slots per lane
#pragma unroll
        for (int q2 = 0; q2 < 2; q2++) {
            const uint32_t s2 = lane + 32 * q2;
            pm[q2] = (s2 < nsplit) ? wsc[warp * g.nsplit_max + s2] : -FLT_MAX;
            pls[q2] = (s2 < nsplit) ? pl[warp * g.nsplit_max + s2] : 0.0f;
        }
        const float M = warp_max(fmaxf(pm[0], pm[1]));
        float L = 0.0f;
        __syncwarp();
#pragma unroll
        for (int q2 = 0; q2 < 2; q2++) {
            const uint32_t s2 = lane + 32 * q2;
            if (s2 < nsplit) { const float w = expf(pm[q2] - M); wsc[warp * g.nsplit_max + s2] = w; L += pls[q2] * w; }
        }
        L = warp_sum(L);
        if (lane == 0) stat[warp] = L;
    }
    cbar();
    for (uint32_t el = st_tid(); el < KVM * hd; el += kConsThreads) {
        const uint32_t m = el / hd, i = el - m * hd;
        float o = 0.0f;
        for (uint32_t s2 = 0; s2 < nsplit; s2++) o = fmaf(macc[(m * nsplit + s2) * hd + i], wsc[m * g.nsplit_max + s2], o);
        const float ov = __fdiv_rn(o, stat[m]);
#pragma unroll
        for (uint32_t rep = 0; rep < (uint32_t)kStRep; rep++) xw_st(g.xv[1] + (size_t)rep * g.rs[1] + ((size_t)kvh * KVM + m) * hd + i, ov, e_out);
    }
    ST_DBG(11);
}

// ---------------------------------------------------------------- grid barrier, once per token (consumer warps; the producer keeps streaming)
__device__ __forceinline__ void st_grid_barrier(const StreamArgs &g, unsigned int &target_smem, volatile uint32_t *progress, uint32_t ncta) {
    cbar();
    if (st_tid() == 0) {
        const unsigned int target = target_smem + ncta;
        target_smem = target;
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(g.bar) : "memory");       // release: this CTA's plain stores of the token
        if (ld_acquire_u32(g.bar) < target) {
            const long long t0 = clock64();
            while (ld_acquire_u32(g.bar) < target) { if (clock64() - t0 > 4000000000ll) st_give_up(g.err, 0x40u); }
        }
        asm volatile("fence.proxy.async.global;" ::: "memory");      // the token's plain K/V stores are TMA-read by later tokens
        *progress = *progress + 1u;
    }
    cbar();
}

// ---------------------------------------------------------------- the kernel
template <int QUANT, int LPG, int KVM>
__global__ void __launch_bounds__(kThreads, 1) k_decode_stream(const __grid_constant__ StreamArgs gparam) {
    extern __shared__ __align__(128) unsigned char ssm[];
    // The argument block is read from shared memory: kernel parameters live in the constant bank, whose cache shares the
    // L1.5 with the instruction stream of this large kernel -- a parameter touched once per phase misses it every time.
    __shared__ __align__(16) StreamArgs sg;
    for (uint32_t i = threadIdx.x; i < sizeof(StreamArgs) / 4; i += kThreads) reinterpret_cast<uint32_t *>(&sg)[i] = reinterpret_cast<const uint32_t *>(&gparam)[i];
    __syncthreads();
    const StreamArgs &g = sg;
    __shared__ uint64_t full_bar[kStMaxStages], empty_bar[kStMaxStages];
    __shared__ volatile uint32_t stage_tile[kStMaxStages];
    __shared__ MatvecSmem ms;
    __shared__ StOwn own;
    __shared__ StGeo geo;
    __shared__ float xown[kStOwnMax];
    __shared__ volatile uint32_t s_progress;
    __shared__ unsigned int s_target;
    __shared__ StStep ss;
    const Dims &d = g.d;
    const uint32_t cta = blockIdx.x, ncta = gridDim.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    // Register budget: 512 threads x 1 CTA caps a thread at 128 registers, and whatever the consumers' layer loop keeps live
    // across a phase is paid for in every phase's peak (the prologue's staged words, the row loops' accumulators).  Values
    // that are loop-invariant or rarely used are therefore re-read from shared memory (sg, s_*) where they are needed.
    auto ring_of = [&]() { return StRing{full_bar, empty_bar, stage_tile, ssm + g.off_ring, g.nstages, g.stage_bytes}; };
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < g.nstages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsWarps); stage_tile[s] = 0xffffffffu; }
        s_progress = 0; s_target = 0;
        ss.step = 0; ss.pos = __ldcg(&g.st->pos);
        ss.causal = __ldcg(&g.st->is_causal); ss.n_prompt = __ldcg(&g.st->n_prompt); ss.advance = __ldcg(&g.st->advance);
        ss.pen = __ldcg(&g.st->penalty);
        ss.tok = __ldcg(&g.st->use_token) ? __ldcg(&g.st->token) : __ldcg(g.ids + ss.pos);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (threadIdx.x < 5) {          // the rows this CTA owns of every kind (64-bit divisions: once, not once per phase)
        const StKind &k = g.kind[threadIdx.x];
        const uint32_t u0 = (uint32_t)(((uint64_t)cta * k.units) / ncta), u1 = (uint32_t)(((uint64_t)(cta + 1) * k.units) / ncta);
        own.row0[threadIdx.x] = u0 * k.unit_rows; own.rows[threadIdx.x] = (u1 - u0) * k.unit_rows;
        // how a warp shares the rows of this kind: the candidate with the cheapest (passes x estimated chain latency)
        const uint32_t kid = threadIdx.x, rows = (u1 - u0) * k.unit_rows;
        uint32_t b_lg2 = 1, b_gt = 32, b_ts = 32, b_rw = 1, b_mode = (kid == SK_W13) ? 2u : 0u;
        if (QUANT == 0x80) {
            const uint32_t G = k.n / (LPG * 16u);
            uint32_t best = 0xffffffffu;
            for (uint32_t cand = LPG; cand >= 1u; cand >>= 1) {
                if (G * cand > 32u && cand > 1u) continue;
                const uint32_t gt = G < 32u / cand ? G : 32u / cand, t = gt * cand, rw = 32u / t;
                const uint32_t md = (kid == SK_W13) ? ((rw >= 2u && !(rw & 1u)) ? 1u : 2u) : 0u;
                const uint32_t per_pass = kConsWarps * (md == 2u ? 2u * rw : rw);
                const uint32_t tr = rows < k.tile_rows ? rows : k.tile_rows, ntl = tr ? (rows + k.tile_rows - 1u) / k.tile_rows : 0u;
                const uint32_t passes = ntl * ((tr + per_pass - 1u) / (per_pass ? per_pass : 1u));
                uint32_t lat = 300u + ((G + gt - 1u) / gt) * (80u * (LPG / cand) + 35u * (31u - __clz(cand)) + 120u + 5u * gt);
                if (md == 2u) lat *= 2u;
                const uint32_t cost = passes * lat;
                if (cost < best) { best = cost; b_lg2 = cand; b_gt = gt; b_ts = t; b_rw = rw; b_mode = md; }
            }
        }
        geo.lg2[kid] = (uint8_t)b_lg2; geo.gteam[kid] = (uint8_t)b_gt; geo.ts[kid] = (uint8_t)b_ts; geo.rw[kid] = (uint8_t)b_rw; geo.mode[kid] = (uint8_t)b_mode;
    }
    __syncthreads();
    if (threadIdx.x < 160) {
        const uint32_t kid = threadIdx.x >> 5, ln = threadIdx.x & 31u, ts = geo.ts[kid], rw = geo.rw[kid], lg2 = geo.lg2[kid];
        const uint32_t tm = ln / ts, tl = ln % ts;
        geo.team[kid][ln] = (uint8_t)(tm < rw ? tm : rw - 1u); geo.tl[kid][ln] = (uint8_t)tl;
        geo.gl[kid][ln] = (uint8_t)(tl / lg2); geo.ul[kid][ln] = (uint8_t)(tl % lg2);
    }
    __syncthreads();

    if (warp == kConsWarps) {
        if (lane == 0) st_producer(g, ring_of(), own, cta, &s_progress, ss.pos, ss.causal, ss.advance);
        return;
    }

    // the replica of a vector this CTA reads
    auto xv_rep = [&](int i) -> const unsigned long long * { return g.xv[i] + (size_t)(blockIdx.x % (uint32_t)kStRep) * g.rs[i]; };
    StCursor cur{0u, 0u};
    uint32_t tcount = 0;                                                // tiles consumed so far (the producer counts the same way)
    uint32_t act_flip = 0;                                              // consecutive phases alternate between the two operands
    // stamps (trace != nullptr: CTA 0 / thread 0, last step): [0..] after every phase; [1024..] inside layer L/2
    __shared__ uint32_t s_ti, s_tj;
    if (st_tid() == 0) { s_ti = 0; s_tj = 0; }
#define ST_TRACE() do { if (g.trace && cta == 0 && st_tid() == 0 && ss.step + 1 == g.n_steps && s_ti < 1000) g.trace[s_ti++] = clock64(); } while (0)
#define ST_STAMP() do { if (g.trace && cta == 0 && st_tid() == 0 && ss.step + 1 == g.n_steps && l == d.L / 2 && s_tj < 60) g.trace[1024 + s_tj++] = clock64(); } while (0)

    while (ss.step < g.n_steps) {
        ST_TRACE();
        if (st_tid() == 0) {       // read by the others after the barrier below
            ss.range = ss.causal ? ss.pos + 1u : d.max_seq;
            st_attn_plan(ss.range, g.nsplit_max, g.chunk_target, ss.nsplit, ss.chunk);
        }
        // embedding row (infer.c:987-988) into shared memory; the rows this CTA owns in the residual phases start from it
        {
            float *x_s = reinterpret_cast<float *>(ssm + g.off_xs);
            embed_row<kConsThreads>(g.emb_w, g.emb_aux, x_s, ss.tok, d);
            cbar();
            for (uint32_t i = st_tid(); i < own.rows[SK_O]; i += kConsThreads) xown[i] = x_s[own.row0[SK_O] + i];
        }
        // ---- layers 0..L-1: QKV | attention | O | W1,W3 | W2 ; pseudo-layer L: the classifier.  One call site per function. ----
#pragma unroll 1
        for (uint32_t l = 0; l <= d.L; l++) {
            ST_STAMP();
            // epochs of this token's exchanges: layer l publishes el + {1: q/k/v, 2: attention output, 3: x after O, 4: SwiGLU output, 5: x after W2}
            const uint32_t el = g.epoch_base + 5u * (ss.step * d.L + l);
#pragma unroll 1
            for (uint32_t ph = 0; ph < 4; ph++) {
                const bool cls = (l == d.L);
                const uint32_t kid = cls ? (uint32_t)SK_CLS : ph;
                const StKind &k = g.kind[kid];
                const unsigned long long *xsrc = xv_rep(0); const float *ssrc = nullptr; const float *gain = nullptr;
                uint32_t epi, need = el, eout = 0;                        // x after the previous layer's W2 carries epoch el(l-1) + 5 = el
                if (cls) { gain = g.g_final; epi = EPI_CLS; }
                else if (ph == SK_QKV) { if (l == 0) { xsrc = nullptr; ssrc = reinterpret_cast<const float *>(ssm + g.off_xs); } gain = g.g_attn + (size_t)l * d.E; epi = EPI_QKV; eout = el + 1u; }
                else if (ph == SK_O) { xsrc = xv_rep(1); need = el + 2u; epi = EPI_RESID; eout = el + 3u; }
                else if (ph == SK_W13) { need = el + 3u; gain = g.g_ffn + (size_t)l * d.E; epi = EPI_SWIGLU; eout = el + 4u; }
                else { xsrc = xv_rep(2); need = el + 4u; epi = EPI_RESID; eout = el + 5u; }
                unsigned long long *dbg = (g.trace && cta == 0 && ss.step + 1 == g.n_steps && l == d.L / 2) ? g.trace + 1100 + 16 * ph : nullptr;
                if (g.ablate & 16u) need = kXwAny;
                if (own.rows[kid]) {          // CTA-uniform: a CTA without rows of this kind neither reads the source nor publishes
                    act_flip ^= 1u;
                    unsigned char *act = ssm + (act_flip ? g.off_act2 : g.off_act);
                    st_prep<QUANT, LPG>(g, xsrc, ssrc, need, gain, k.n, act, ms.red, dbg);
                    ST_STAMP();
                    st_consume<QUANT, LPG>(g, ring_of(), cur, tcount, k, epi, l, own.row0[kid], own.rows[kid], eout, act, ss.pos, ss.pen, xown, ms, geo, kid, dbg);
                } else {
                    ST_STAMP();
                    const uint32_t t = st_tid();
                    if (cls && (t & 31u) == 0) { ms.best_v[t >> 5] = -FLT_MAX; ms.best_i[t >> 5] = 0xffffffffu; }
                }
                ST_STAMP();
                ST_TRACE();
                if (cls) break;
                if (ph == SK_QKV) {
                    st_attention<KVM>(g, ring_of(), cur, tcount, l, cta, ss.pos, ss.range, ss.nsplit, ss.chunk, (g.ablate & 16u) ? kXwAny : el + 1u, el + 2u, reinterpret_cast<float *>(ssm + g.off_attn), dbg ? g.trace + 1100 + 64 : nullptr);
                    ST_STAMP();
                    ST_TRACE();
                }
            }
        }
        cbar();
        if (st_tid() == 0) {
            float bv = ms.best_v[0]; uint32_t bi = ms.best_i[0];
            for (int w = 1; w < kConsWarps; w++)
                if (ms.best_i[w] != 0xffffffffu && (bi == 0xffffffffu || ms.best_v[w] > bv || (ms.best_v[w] == bv && ms.best_i[w] < bi))) { bv = ms.best_v[w]; bi = ms.best_i[w]; }
            g.cls_val[cta] = bv; g.cls_idx[cta] = bi;
        }
        st_grid_barrier(g, s_target, &s_progress, ncta);
        ST_TRACE();
        // ---- every CTA picks the token from the per-CTA partials (no second barrier) and advances its copy of the state ----
        {
            float bv = -FLT_MAX; uint32_t bi = 0xffffffffu;
            for (uint32_t c2 = st_tid(); c2 < ncta; c2 += kConsThreads) {
                const float v = __ldcg(g.cls_val + c2); const uint32_t i = __ldcg(g.cls_idx + c2);
                if (i != 0xffffffffu && (bi == 0xffffffffu || v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (oi != 0xffffffffu && (bi == 0xffffffffu || ov > bv || (ov == bv && oi < bi))) { bv = ov; bi = oi; }
            }
            const uint32_t t = st_tid();
            if ((t & 31u) == 0) { ms.best_v[t >> 5] = bv; ms.best_i[t >> 5] = bi; }
            cbar();
            if (st_tid() == 0) {
                bv = -FLT_MAX; bi = 0xffffffffu;
#pragma unroll 1
                for (int w = 0; w < kConsWarps; w++)
                    if (ms.best_i[w] != 0xffffffffu && (bi == 0xffffffffu || ms.best_v[w] > bv || (ms.best_v[w] == bv && ms.best_i[w] < bi))) { bv = ms.best_v[w]; bi = ms.best_i[w]; }
                if (bi == 0xffffffffu) bi = 0;       // all-NaN row: the reference's argmax returns index 0
                const uint32_t pos = ss.pos, tok = ss.tok;
                uint32_t nxt = bi;
                if (ss.advance) {
                    const bool forced = (pos + 1 < ss.n_prompt);     // infer.c:1250 is_prefilling
                    if (forced) nxt = __ldcg(g.ids + pos + 1);
                    if (cta == 0) {
                        g.seen[tok] = 1;                             // ids[0..pos] are "seen" for step pos+1
                        if (!forced) g.ids[pos + 1] = bi;
                        g.st->pos = pos + 1;
                        g.st->next_token = nxt;
                    }
                    ss.tok = nxt; ss.pos = pos + 1;
                } else if (cta == 0) {
                    g.st->next_token = bi;
                }
                ss.step = ss.step + 1u;
            }
            cbar();
        }
    }
#undef ST_TRACE
#undef ST_STAMP
}

}  // namespace nb
