// prefill.cuh -- batched prompt prefill (nb200_prefill): the causal forward pass of a chunk of up to kPrefillMax prompt
// positions per pass over the weights, K / V rows only (no classifier).
//
// Every kernel here runs the device functions of the multi-kernel token path (kernels.cuh) once per position of the chunk:
// the same activation prep at 512 threads, the same per-row dot products and epilogue arithmetic, the same attention CTA
// bodies.  A row's value does not depend on how many positions share the pass (nor on the row block: every row keeps its own
// accumulation order), so the K / V rows written are bit-identical to what nb200_forward writes position by position on the
// multi-kernel path of an engine with the same flags -- in exact mode, to the strict reference.
// What a chunk shares is the weight traffic: a Q80 weight tile is loaded into registers once and consumed against the
// activation codes of every position; F32 and Q4K row blocks are re-read per position, from L2 after the first.
//
// One chunk: k_prefill_embed, then per layer
//   QKV matvec (q, raw k, V rows) -> K-row pass (head-norm + RoPE -> K rows) -> attention -> O + residual
//   -> W1|W3 + SwiGLU -> W2 + residual.
// The K-row pass exists because position i of a chunk reads the K rows of positions pos0 .. pos0+i-1, which on the token
// path the attention kernels of those positions wrote.  It computes every row with the arithmetic of the attention kernel
// that follows (the lane-sliced norm_rope_apply of k_attention_fast, head_norm_rope for the generic and exact kernels), so
// the attention CTA that owns a row recomputes and stores the same bits again.
#pragma once
#include "kernels.cuh"

namespace nb {

constexpr int kPrefillMax = 16;     // positions per chunk at most (the engine picks M <= this from shared memory)
constexpr int kPrefillRB = 2;       // rows per warp of the prefill matvecs (even: SwiGLU pairs rows)

struct PrefillMvArgs {
    const void *w, *w_aux;                  // same layouts as MatvecArgs
    uint32_t rows, n;
    const float *src; uint32_t src_stride;  // position p's input vector: src + p * src_stride
    const float *gain;                      // rmsnorm gain or nullptr (plain quantise)
    float *out; uint32_t out_stride;        // QKV: q; RESID: x (in/out); SWIGLU: hb -- position p at out + p * out_stride
    float *out_k; uint32_t k_stride;        // QKV: raw k
    float *out_v;                           // QKV: V cache base of this layer [KV][max_seq][hd]
    uint32_t pos0, m;                       // the chunk: positions pos0 .. pos0+m-1
    uint32_t act_bytes;                     // one position's activation operand in shared memory (act_region_bytes)
    Dims d;
};

// the matvec epilogues (kernels.cuh) for one position of the chunk: lane 0 stores
template <int EPI, int RB>
__device__ __forceinline__ void prefill_store(const PrefillMvArgs &a, uint32_t p, uint32_t row0, const float (&val)[RB]) {
    if ((threadIdx.x & 31) != 0) return;
    float *out = a.out + (size_t)p * a.out_stride;
    if (EPI == EPI_SWIGLU) {
#pragma unroll
        for (int r = 0; r + 1 < RB; r += 2)
            if (row0 + r + 1 < a.rows) out[(row0 + r) >> 1] = swiglu(val[r], val[r + 1], a.d.exact != 0);
    } else {
#pragma unroll
        for (int r = 0; r < RB; r++) {
            const uint32_t row = row0 + r;
            if (row >= a.rows) break;
            if (EPI == EPI_RESID) out[row] = resid_add(__ldcg(out + row), val[r], nullptr, row);
            else qkv_store(a.d, row, val[r], out, a.out_k + (size_t)p * a.k_stride, a.out_v, a.pos0 + p);
        }
    }
}

// One Q80 row block against every position of the chunk: each weight tile is loaded once and q80_consume runs once per
// position, K ascending as in matvec_phase.  The next tile is requested before the current one is consumed: into registers,
// or (groups of 32, whose ordered sum needs more registers) towards L2 only, which keeps every variant free of spills.
template <int RB, int LPG, bool ORD>
__device__ __forceinline__ void prefill_rows_q80(const PrefillMvArgs &a, uint32_t row0, const unsigned char *act,
                                                 float (&val)[kPrefillMax][RB]) {
    constexpr bool kRegAhead = LPG > 2;
    const int8_t *W = static_cast<const int8_t *>(a.w);
    const float *S = static_cast<const float *>(a.w_aux);
    const int lane = threadIdx.x & 31;
    Q80Tile<RB> t;
    q80_load<RB, LPG>(t, W, S, row0, a.rows, a.n, 0);
    for (uint32_t k0 = 0; k0 < a.n; k0 += 1024) {
        Q80Tile<RB> nx;
        const bool more = k0 + 1024 < a.n;
        if (more) {
            if (kRegAhead) q80_load<RB, LPG>(nx, W, S, row0, a.rows, a.n, k0 + 1024);
            else {
#pragma unroll
                for (int r = 0; r < RB; r++) {
                    const int8_t *rw = W + (size_t)min(row0 + r, a.rows - 1) * a.n + k0 + 1024;
                    if (k0 + 1024 + lane * 32 < a.n) prefetch_l2(rw + lane * 32);     // 1 KB of the row: 32 B per lane
                }
            }
        }
#pragma unroll
        for (int p = 0; p < kPrefillMax; p++)
            if (p < (int)a.m) q80_consume<RB, LPG, ORD>(t, a.n, k0, act + (size_t)p * a.act_bytes, val[p]);
        if (more) {
            if (kRegAhead) t = nx;
            else q80_load<RB, LPG>(t, W, S, row0, a.rows, a.n, k0 + 1024);
        }
    }
}

// rmsnorm / quantise of every position's input into its own operand, then row blocks x positions; store(p, row0, val) finishes
// the RB rows from row0 of position p (k_prefill_matvec: prefill_store; the batch kernels of batch.cuh: their own stores).
// smem: m activation operands of act_bytes each | staging (2n floats, reused by every position's prep)
template <int QUANT, int RB, int LPG, class Store>
__device__ __forceinline__ void prefill_matvec_body(const PrefillMvArgs &a, unsigned char *act, float *red, Store &&store) {
    const bool exact = a.d.exact != 0;
    const uint32_t n = a.n;
    float *stage = reinterpret_cast<float *>(act + (size_t)a.m * a.act_bytes);
    for (uint32_t p = 0; p < a.m; p++) {
        unsigned char *ap = act + (size_t)p * a.act_bytes;
        const float *src = a.src + (size_t)p * a.src_stride;
        if (QUANT == 0x00) prep_f32<kThreads, false, 4>(src, a.gain, n, exact, reinterpret_cast<float *>(ap), stage, red);
        else if (QUANT == 0x80) prep_q80<kThreads, false, 4>(src, a.gain, n, LPG * 16, exact, ap, stage, red, nullptr, nullptr);
        else prep_q4k<kThreads, false, 4>(src, a.gain, n, exact, ap, stage, red, nullptr, nullptr);
    }
    const int warp = threadIdx.x >> 5;
    const uint32_t nblocks = (a.rows + RB - 1) / RB;
    for (uint32_t rb = blockIdx.x * kWarps + warp; rb < nblocks; rb += gridDim.x * kWarps) {
        const uint32_t row0 = rb * RB;
        if (QUANT == 0x80) {
            float val[kPrefillMax][RB];
#pragma unroll
            for (int p = 0; p < kPrefillMax; p++)
#pragma unroll
                for (int r = 0; r < RB; r++) val[p][r] = 0.0f;
            if (exact) prefill_rows_q80<RB, LPG, true>(a, row0, act, val);       // the reference's ordered group sum
            else {
                prefill_rows_q80<RB, LPG, false>(a, row0, act, val);             // one partial per lane, then the warp tree
#pragma unroll
                for (int p = 0; p < kPrefillMax; p++)
#pragma unroll
                    for (int r = 0; r < RB; r++) val[p][r] = warp_sum(val[p][r]);
            }
#pragma unroll
            for (int p = 0; p < kPrefillMax; p++)
                if (p < (int)a.m) store((uint32_t)p, row0, val[p]);
        } else {
            for (uint32_t p = 0; p < a.m; p++) {
                float val[RB];
                const unsigned char *ap = act + (size_t)p * a.act_bytes;
                if (QUANT == 0x00) rows_f32<RB>(static_cast<const float *>(a.w), row0, a.rows, n, ap, val);
                else rows_q4k<RB>(static_cast<const uint8_t *>(a.w), static_cast<const uint8_t *>(a.w_aux), row0, a.rows, n, ap, val);
                store(p, row0, val);
            }
        }
    }
}

template <int QUANT, int EPI, int RB, int LPG>
__global__ void __launch_bounds__(kThreads, 1) k_prefill_matvec(const PrefillMvArgs a) {
    extern __shared__ __align__(16) unsigned char act[];
    __shared__ float red[32];
    pdl_launch_dependents();
    prefetch_row_blocks<QUANT, RB>(a.w, a.rows, a.n, blockIdx.x, gridDim.x, 4);
    pdl_wait();
    prefill_matvec_body<QUANT, RB, LPG>(a, act, red, [&](uint32_t p, uint32_t row0, const float (&val)[RB]) { prefill_store<EPI, RB>(a, p, row0, val); });
}

// exact-mode F32 over the chunk (k_matvec_f32_exact's arithmetic): every position's operand, then unit(p, u, x) for unit u of
// every position p, one thread per unit (a row, or a w1 / w3 row pair for EPI_SWIGLU)
template <int EPI, class Unit>
__device__ __forceinline__ void prefill_f32_exact_body(const PrefillMvArgs &a, unsigned char *act, float *red, Unit &&unit) {
    const uint32_t n = a.n;
    float *stage = reinterpret_cast<float *>(act + (size_t)a.m * a.act_bytes);
    for (uint32_t p = 0; p < a.m; p++)
        prep_f32<kThreads>(a.src + (size_t)p * a.src_stride, a.gain, n, true, reinterpret_cast<float *>(act + (size_t)p * a.act_bytes), stage, red);
    const uint32_t nunits = (EPI == EPI_SWIGLU) ? a.rows / 2 : a.rows;
    for (uint32_t u = blockIdx.x * kThreads + threadIdx.x; u < nunits; u += gridDim.x * kThreads)
        for (uint32_t p = 0; p < a.m; p++) unit(p, u, reinterpret_cast<const float *>(act + (size_t)p * a.act_bytes));
}

// exact-mode F32 (k_matvec_f32_exact over the chunk): f32_exact_unit per position
template <int EPI>
__global__ void __launch_bounds__(kThreads, 1) k_prefill_matvec_f32_exact(const PrefillMvArgs a) {
    extern __shared__ __align__(16) unsigned char act[];
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    prefill_f32_exact_body<EPI>(a, act, red, [&](uint32_t p, uint32_t u, const float *x) {
        f32_exact_unit<EPI>(static_cast<const float *>(a.w), a.n, u, x, a.d, a.out + (size_t)p * a.out_stride,
                            a.out_k + (size_t)p * a.k_stride, a.out_v, a.pos0 + p, nullptr);
    });
}

// the embedding rows of the chunk's ids (embed_row, as k_embed), one CTA per position
struct PrefillEmbedArgs { const void *w, *w_aux; float *x; const uint32_t *ids; Dims d; };
NB_K __global__ void __launch_bounds__(256) k_prefill_embed(const PrefillEmbedArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    embed_row<256>(a.w, a.w_aux, a.x + (size_t)blockIdx.x * a.d.E, a.ids[blockIdx.x], a.d);
}

// K-row pass: head-norm (Qwen3) + RoPE of every position's raw k, stored as its K row.  One warp per (kv head, position).
// fast = 1: the arithmetic and lane slicing attn_stream_partial applies to the row of its own position (k_attention_fast);
// fast = 0: head_norm_rope over a staged row, as k_attention and k_attention_exact do.
struct PrefillKrowArgs {
    const float *kraw;                      // [m][kv_dim]
    float *kc;                              // K cache base of this layer [KV][max_seq][hd]
    const float *knorm, *rope_cos, *rope_sin;
    uint32_t pos0, fast;
    Dims d;
};
// One K row (one warp, lane = threadIdx.x & 31): kr is the raw k of the kv head, dst its cache row, cr / ci the RoPE row of its
// position, h a staging row in shared memory (fast = 0).  The body of k_prefill_krow and of the batch's k_vbatch_krow (batch.cuh).
__device__ __forceinline__ void krow_store(const float *kr, float *dst, const float *knorm, const float *cr, const float *ci,
                                           uint32_t fast, const Dims &d, float *h, int lane) {
    const uint32_t hd = d.hd;
    if (fast) {
        uint32_t lpr = 1; while (lpr * 4 < hd) lpr <<= 1;
        const uint32_t sub = lane / lpr, col = (lane % lpr) * 4;
        const bool colon = col < hd;
        float4 kk0 = make_float4(0, 0, 0, 0), gk = make_float4(0, 0, 0, 0);
        if (colon) {
            kk0 = __ldcg(reinterpret_cast<const float4 *>(kr + col));
            if (d.arch == 3u) gk = *reinterpret_cast<const float4 *>(knorm + col);
        }
        const RopeTab rt = rope_tab_load(cr, ci, d, col, colon);
        const float4 kk = norm_rope_apply(kk0, gk, rt, d, lpr, col, colon);     // every lane group of the warp (shuffles)
        if (sub == 0 && colon) *reinterpret_cast<float4 *>(dst + col) = kk;
    } else {
        for (uint32_t i = lane; i < hd; i += 32) h[i] = __ldcg(kr + i);
        __syncwarp();
        head_norm_rope(h, knorm, cr, ci, d, d.exact != 0);
        for (uint32_t i = lane; i < hd; i += 32) dst[i] = h[i];
    }
}

NB_K __global__ void __launch_bounds__(32) k_prefill_krow(const PrefillKrowArgs a) {
    __shared__ __align__(16) float h[512];
    pdl_launch_dependents();
    pdl_wait();
    const Dims &d = a.d;
    const uint32_t hd = d.hd, g = blockIdx.x, p = blockIdx.y, pos = a.pos0 + p;
    const int lane = threadIdx.x & 31;
    const float *kr = a.kraw + (size_t)p * d.kv_dim + (size_t)g * hd;
    const float *cr = a.rope_cos + (size_t)pos * (hd / 2), *ci = a.rope_sin + (size_t)pos * (hd / 2);
    float *dst = a.kc + ((size_t)g * d.max_seq + pos) * hd;
    krow_store(kr, dst, a.knorm, cr, ci, a.fast, d, h, lane);
}

// Attention of every position of the chunk: blockIdx.z = position p, which attends to rows [0, pos0 + p] through the token
// path's own CTA body with its q / raw k / output rows and its own split workspaces and tickets.
struct PrefillAttnArgs {
    AttnArgs at;            // position 0 of the chunk (st unused)
    AttnExactArgs ex;       // exact mode: position 0 of the chunk, att = [m][H][max_seq]
    uint32_t pos0;
};
__device__ __forceinline__ AttnArgs prefill_attn_at(const PrefillAttnArgs &pa, uint32_t p) {
    AttnArgs a = pa.at;
    const Dims &d = a.d;
    const size_t slots = (size_t)d.H * a.nsplit_max;
    a.q += (size_t)p * d.q_dim; a.kraw += (size_t)p * d.kv_dim; a.xba += (size_t)p * d.q_dim;
    a.ws_m += p * slots; a.ws_l += p * slots; a.ws_acc += p * slots * d.hd; a.ticket += (size_t)p * d.KV;
    return a;
}
template <int KVM>
__global__ void __launch_bounds__(kThreads, 1) k_prefill_attention_fast(const PrefillAttnArgs pa) {
    extern __shared__ __align__(16) float sm[];
    __shared__ uint32_t is_last;
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t p = blockIdx.z, pos = pa.pos0 + p, range = pos + 1;
    const AttnArgs a = prefill_attn_at(pa, p);
    uint32_t chunk, nsplit;
    attn_split_plan(range, a.nsplit_max, a.chunk_cap, chunk, nsplit);
    if (blockIdx.x >= nsplit) return;
    attn_item<KVM, kThreads, false>(a, blockIdx.y, blockIdx.x, pos, range, chunk, nsplit, sm, is_last);
}

// the generic and exact bodies are written for kAttnThreads threads
NB_K __global__ void __launch_bounds__(kAttnThreads, 1) k_prefill_attention(const PrefillAttnArgs pa) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float red[32];
    __shared__ uint32_t is_last;
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t p = blockIdx.z, pos = pa.pos0 + p;
    attn_generic_cta(prefill_attn_at(pa, p), blockIdx.y, blockIdx.x, pos, pos + 1, sm, red, is_last);
}

__device__ __forceinline__ AttnExactArgs prefill_exact_at(const PrefillAttnArgs &pa, uint32_t p) {
    AttnExactArgs a = pa.ex;
    const Dims &d = a.d;
    a.q += (size_t)p * d.q_dim; a.kraw += (size_t)p * d.kv_dim; a.xba += (size_t)p * d.q_dim;
    a.att += (size_t)p * d.H * d.max_seq;
    return a;
}
NB_K __global__ void __launch_bounds__(kAttnThreads) k_prefill_attention_exact(const PrefillAttnArgs pa) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t p = blockIdx.y, pos = pa.pos0 + p;
    attn_exact_cta(prefill_exact_at(pa, p), blockIdx.x, pos, pos + 1, sm, red);
}

}  // namespace nb
