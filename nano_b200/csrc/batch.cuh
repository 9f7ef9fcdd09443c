// batch.cuh -- batched multi-session decode (nb200_batch_next_greedy): one decode step of up to kPrefillMax independent
// sessions ("slots") per pass over the weights.
//
// A pass is prefill's chunk (prefill.cuh) with one position per session instead of consecutive positions of one prompt:
// entry p of the pass consumes ids[p] at position pos[p] of slot slot[p], whose K / V cache, seen set and logits row are its
// own.  Every kernel runs the multi-kernel token path's device functions once per entry, through prefill's matvec bodies
// (prefill_matvec_body, prefill_f32_exact_body) and the token path's attention CTA bodies, so a slot's K / V rows, logits and
// next id are bit-identical to what nb200_next_greedy gives on the multi-kernel path of an engine with the same flags.
//
// One pass: k_prefill_embed, then per layer
//   QKV matvec (q, raw k, V row of each entry's slot and position) -> attention -> O + residual -> W1|W3 + SwiGLU -> W2 + residual
// then the classifier (final rmsnorm, the slot's repetition penalty, logits row) and one argmax CTA per entry.
// The residual / SwiGLU matvecs do not depend on the position and are prefill's own kernels.  There is no K-row pass: the
// entries of a pass belong to different slots, so no entry reads a row another entry writes, and within an entry the
// attention CTA that owns row pos writes it before reading it, as on the token path.
#pragma once
#include "prefill.cuh"

namespace nb {

// one pass of nb200_batch_next_greedy, passed by value (warp-uniform reads from the parameter bank): entry p runs at position
// pos[p] of slot slot[p] with penalty pen[p] (the ids it consumes are on the device, for k_prefill_embed)
struct BatchPass {
    uint32_t slot[kPrefillMax], pos[kPrefillMax];
    float pen[kPrefillMax];
};

struct BatchMvArgs {
    PrefillMvArgs mv;           // the matrix, the entries' input rows and (QKV) their q / raw k rows; pos0 unused
    BatchPass bp;
    float *vc;                  // QKV: V cache of this layer in slot 0; slot s starts slot_elems floats further
    size_t slot_elems;          // floats of one slot's K (or V) cache, [L][KV][max_seq][hd]
    float *logits;              // CLS: [n_slots][V]
    const uint8_t *seen;        // CLS: [n_slots][V], 1 where the id occurred before the slot's position
};

// the token path's EPI_QKV (qkv_store) and EPI_CLS (penalty by division where seen, logits row) epilogues, for entry p: lane 0 stores
template <int EPI, int RB>
__device__ __forceinline__ void batch_store(const BatchMvArgs &b, uint32_t p, uint32_t row0, const float (&val)[RB]) {
    if ((threadIdx.x & 31) != 0) return;
    const PrefillMvArgs &a = b.mv;
    const uint32_t slot = b.bp.slot[p];
    if (EPI == EPI_CLS) {
        const float pen = b.bp.pen[p];
        float *lg = b.logits + (size_t)slot * a.d.V;
        const uint8_t *seen = b.seen + (size_t)slot * a.d.V;
#pragma unroll
        for (int r = 0; r < RB; r++) {
            const uint32_t row = row0 + r;
            if (row >= a.rows) break;
            float v = val[r];
            if (pen != 1.0f && seen[row]) v = __fdiv_rn(v, pen);      // infer.c:1156-1167, as matvec_phase's EPI_CLS
            lg[row] = v;
        }
    } else {
        float *vc = b.vc + (size_t)slot * b.slot_elems;
        const uint32_t pos = b.bp.pos[p];
#pragma unroll
        for (int r = 0; r < RB; r++) {
            const uint32_t row = row0 + r;
            if (row >= a.rows) break;
            qkv_store(a.d, row, val[r], a.out + (size_t)p * a.out_stride, a.out_k + (size_t)p * a.k_stride, vc, pos);
        }
    }
}

// QKV (EPI_QKV) and classifier (EPI_CLS) matvecs of a pass
template <int QUANT, int EPI, int RB, int LPG>
__global__ void __launch_bounds__(kThreads, 1) k_batch_matvec(const BatchMvArgs b) {
    extern __shared__ __align__(16) unsigned char act[];
    __shared__ float red[32];
    pdl_launch_dependents();
    prefetch_row_blocks<QUANT, RB>(b.mv.w, b.mv.rows, b.mv.n, blockIdx.x, gridDim.x, 4);
    pdl_wait();
    prefill_matvec_body<QUANT, RB, LPG>(b.mv, act, red, [&](uint32_t p, uint32_t row0, const float (&val)[RB]) { batch_store<EPI, RB>(b, p, row0, val); });
}

// exact-mode F32: f32_exact_unit per entry; the classifier stores the row and divides it where seen, as k_cls_finalize does
template <int EPI>
__global__ void __launch_bounds__(kThreads, 1) k_batch_matvec_f32_exact(const BatchMvArgs b) {
    extern __shared__ __align__(16) unsigned char act[];
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    const PrefillMvArgs &a = b.mv;
    prefill_f32_exact_body<EPI>(a, act, red, [&](uint32_t p, uint32_t u, const float *x) {
        const uint32_t slot = b.bp.slot[p];
        const float *W = static_cast<const float *>(a.w);
        if (EPI == EPI_CLS) {
            float *lg = b.logits + (size_t)slot * a.d.V;
            f32_exact_unit<EPI_STORE>(W, a.n, u, x, a.d, lg, nullptr, nullptr, 0, nullptr);
            const float pen = b.bp.pen[p];
            if (pen != 1.0f && b.seen[(size_t)slot * a.d.V + u]) lg[u] = __fdiv_rn(lg[u], pen);
        } else {
            f32_exact_unit<EPI_QKV>(W, a.n, u, x, a.d, a.out + (size_t)p * a.out_stride, a.out_k + (size_t)p * a.k_stride,
                                    b.vc + (size_t)slot * b.slot_elems, b.bp.pos[p], nullptr);
        }
    });
}

// Attention of every entry: blockIdx.z (exact: blockIdx.y) = entry p, which attends to rows [0, pos[p]] of its slot's cache
// through the token path's own CTA body, with its own q / raw k / output rows, split workspaces and tickets.
struct BatchAttnArgs {
    PrefillAttnArgs pa;         // the cache bases are slot 0's; pos0 unused
    BatchPass bp;
    size_t slot_elems;
};
__device__ __forceinline__ AttnArgs batch_attn_at(const BatchAttnArgs &b, uint32_t p) {
    AttnArgs a = prefill_attn_at(b.pa, p);
    const size_t off = (size_t)b.bp.slot[p] * b.slot_elems;
    a.kc += off; a.vc += off;
    return a;
}

template <int KVM>
__global__ void __launch_bounds__(kThreads, 1) k_batch_attention_fast(const BatchAttnArgs b) {
    extern __shared__ __align__(16) float sm[];
    __shared__ uint32_t is_last;
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t p = blockIdx.z, pos = b.bp.pos[p], range = pos + 1;
    uint32_t chunk, nsplit;
    attn_split_plan(range, b.pa.at.nsplit_max, b.pa.at.chunk_cap, chunk, nsplit);
    if (blockIdx.x >= nsplit) return;
    attn_item<KVM, kThreads, false>(batch_attn_at(b, p), blockIdx.y, blockIdx.x, pos, range, chunk, nsplit, sm, is_last);
}

NB_K __global__ void __launch_bounds__(kAttnThreads, 1) k_batch_attention(const BatchAttnArgs b) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float red[32];
    __shared__ uint32_t is_last;
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t p = blockIdx.z, pos = b.bp.pos[p];
    attn_generic_cta(batch_attn_at(b, p), blockIdx.y, blockIdx.x, pos, pos + 1, sm, red, is_last);
}

NB_K __global__ void __launch_bounds__(kAttnThreads) k_batch_attention_exact(const BatchAttnArgs b) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t p = blockIdx.y, pos = b.bp.pos[p];
    AttnExactArgs a = prefill_exact_at(b.pa, p);
    const size_t off = (size_t)b.bp.slot[p] * b.slot_elems;
    a.kc += off; a.vc += off;
    attn_exact_cta(a, blockIdx.x, pos, pos + 1, sm, red);
}

// First-max argmax of each entry's logits row, one CTA per entry: the token path's rule (k_cls_finalize, cls_finalize): the
// lowest index holding the largest value above -FLT_MAX, NaN never wins, and a row without such a value gives 0.
struct BatchArgmaxArgs { const float *logits; BatchPass bp; uint32_t *next; uint32_t V; };
NB_K __global__ void __launch_bounds__(1024) k_batch_argmax(const BatchArgmaxArgs a) {
    __shared__ float bvs[32];
    __shared__ uint32_t bis[32];
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t p = blockIdx.x;
    const float *lg = a.logits + (size_t)a.bp.slot[p] * a.V;
    float bv = -FLT_MAX; uint32_t bi = 0xffffffffu;
    for (uint32_t i = threadIdx.x; i < a.V; i += 1024) {
        const float v = lg[i];
        if (v > bv) { bv = v; bi = i; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { bvs[threadIdx.x >> 5] = bv; bis[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 32; w++) if (bvs[w] > bv || (bvs[w] == bv && bis[w] < bi)) { bv = bvs[w]; bi = bis[w]; }
        a.next[p] = (bi == 0xffffffffu) ? 0u : bi;      // all-NaN row: the reference's argmax returns index 0
    }
}

// Seen rows of a verify pass (nb200_verify_greedy), one CTA per row: row j is the engine's seen set (ids[0..pos)) plus the
// chunk's ids[0..j) (positions pos .. pos+j-1), so entry j of the pass's classifier penalises exactly what nb200_next_greedy at
// pos+j would.  The copy, then the marks.
struct VerifySeenArgs { uint8_t *rows; const uint8_t *seen; const uint32_t *ids; uint32_t V; };
NB_K __global__ void __launch_bounds__(1024) k_verify_seen(const VerifySeenArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t j = blockIdx.x;
    uint8_t *row = a.rows + (size_t)j * a.V;
    for (uint32_t i = threadIdx.x; i < a.V; i += 1024) row[i] = a.seen[i];
    __syncthreads();
    if (threadIdx.x < j) row[a.ids[threadIdx.x]] = 1;
}

}  // namespace nb
