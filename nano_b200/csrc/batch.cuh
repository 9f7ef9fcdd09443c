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
// attention CTA that owns row pos writes it before reading it, as on the token path.  (A verify pass, at the end of this file,
// has rows of one slot at consecutive positions and adds one.)
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

// ---------------- batched verification (nb200_batch_verify_greedy) ----------------
// A verify pass of a batch packs entries of 1 .. M rows: entry e runs the consumed id and its drafts at positions pos .. pos+n-1
// of its slot, rows r0 .. r0+n-1 of the pass.  The QKV matvec and the attention kernels above take a per-row (slot, position),
// so rows of one slot at consecutive positions need nothing new there; what is new is prefill's K-row pass with a per-row slot
// (a row reads the K rows of its entry's earlier rows), the seen rows, and saving / accepting the rows past the accepted ones on
// the device, so that a call of several passes never waits for the host.
// The verify pass's own kernels are named k_vbatch_*, apart from the decode pass's k_batch_* set.

// per entry of a pass (pass-local index e): its slot, first position, row count and first row
struct BatchVerifyEntries { uint32_t slot[kPrefillMax], pos[kPrefillMax], n[kPrefillMax], r0[kPrefillMax]; };

// K-row pass of a verify pass: krow_store (k_prefill_krow's body) for row r of the pass at (slot[r], pos[r]).  One warp per
// (kv head, row).
struct BatchKrowArgs {
    const float *kraw;                      // [R][kv_dim]
    float *kc;                              // K cache of this layer in slot 0; slot s starts slot_elems floats further
    size_t slot_elems;
    const float *knorm, *rope_cos, *rope_sin;
    BatchPass bp;                           // pen unused
    uint32_t fast;
    Dims d;
};
NB_K __global__ void __launch_bounds__(32) k_vbatch_krow(const BatchKrowArgs a) {
    __shared__ __align__(16) float h[512];
    pdl_launch_dependents();
    pdl_wait();
    const Dims &d = a.d;
    const uint32_t hd = d.hd, g = blockIdx.x, r = blockIdx.y, pos = a.bp.pos[r];
    float *kc = a.kc + (size_t)a.bp.slot[r] * a.slot_elems;
    krow_store(a.kraw + (size_t)r * d.kv_dim + (size_t)g * hd, kc + ((size_t)g * d.max_seq + pos) * hd, a.knorm,
               a.rope_cos + (size_t)pos * (hd / 2), a.rope_sin + (size_t)pos * (hd / 2), a.fast, d, h, threadIdx.x & 31);
}

// Seen rows of a verify pass, one CTA per row: row r is its slot's seen set (ids[0..pos), brought up to date by the host) plus
// the ids its entry's earlier rows consume (ids[first[r] .. r) of the pass), so the classifier of row r penalises exactly what
// nb200_next_greedy at pos[r] would.  Rows of entries at penalty 1 are not read by the classifier and are left alone.
struct BatchSeenArgs {
    uint8_t *rows;                          // [M][V]
    const uint8_t *seen;                    // the batch's seen sets [n_slots][V]
    const uint32_t *ids;                    // the ids the pass's rows consume
    BatchPass bp;
    uint32_t first[kPrefillMax];            // first row of row r's entry
    uint32_t V;
};
NB_K __global__ void __launch_bounds__(1024) k_vbatch_seen(const BatchSeenArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t r = blockIdx.x;
    if (a.bp.pen[r] == 1.0f) return;
    uint8_t *row = a.rows + (size_t)r * a.V;
    const uint8_t *src = a.seen + (size_t)a.bp.slot[r] * a.V;
    for (uint32_t i = threadIdx.x; i < a.V; i += 1024) row[i] = src[i];
    __syncthreads();
    if (threadIdx.x >= a.first[r] && threadIdx.x < r) row[a.ids[threadIdx.x]] = 1;
}

// Before a verify pass: the K and V rows its drafted rows will overwrite.  Row r (bit r of `drafted`: not the first row of its
// entry) at (slot[r], pos[r]) goes to save row r-1 (entries own disjoint rows, so M-1 save rows suffice), for every kv head of
// layer blockIdx.y.  Save layout [L][KV][M-1][hd].
struct BatchSaveArgs {
    const float *kc, *vc;                   // the batch's caches, slot 0
    float *ksave, *vsave;
    size_t slot_elems;
    BatchPass bp;
    uint32_t drafted, M;
    Dims d;
};
NB_K __global__ void __launch_bounds__(256) k_vbatch_save(const BatchSaveArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const Dims &d = a.d;
    const uint32_t r = blockIdx.x, l = blockIdx.y, hd = d.hd;
    if (!((a.drafted >> r) & 1u)) return;
    const size_t off = (size_t)a.bp.slot[r] * a.slot_elems + ((size_t)l * d.KV * d.max_seq + a.bp.pos[r]) * hd;
    const size_t sv = ((size_t)l * d.KV * (a.M - 1) + (r - 1)) * hd;
    for (uint32_t i = threadIdx.x; i < d.KV * hd; i += 256) {
        const uint32_t g = i / hd, c = i % hd;
        a.ksave[sv + (size_t)g * (a.M - 1) * hd + c] = a.kc[off + (size_t)g * d.max_seq * hd + c];
        a.vsave[sv + (size_t)g * (a.M - 1) * hd + c] = a.vc[off + (size_t)g * d.max_seq * hd + c];
    }
}

// After the argmax: per entry (blockIdx.x), a = the largest count whose greedy ids next[r0 .. r0+a) equal the drafts the next
// rows consumed, res[2e] = a and res[2e+1] = g_a; the slot's logits row becomes row r0+a of the pass, and the saved rows
// pos+a+1 .. pos+n-1 go back.  The copies are spread over blockIdx.y; every CTA of the entry finds the same a.
struct BatchAcceptArgs {
    const uint32_t *next, *ids;             // the pass's greedy ids and the ids its rows consumed
    const float *ws_logits;                 // [M][V] the pass's logits rows
    float *logits;                          // the batch's logits rows [n_slots][V]
    float *kc, *vc;
    const float *ksave, *vsave;
    size_t slot_elems;
    uint32_t *res;                          // [2 * entries of the pass]
    BatchVerifyEntries en;
    uint32_t M;
    Dims d;
};
NB_K __global__ void __launch_bounds__(1024) k_vbatch_accept(const BatchAcceptArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const Dims &d = a.d;
    const uint32_t e = blockIdx.x, r0 = a.en.r0[e], n = a.en.n[e], slot = a.en.slot[e], pos = a.en.pos[e], hd = d.hd;
    uint32_t acc = 0;
    while (acc + 1 < n && a.next[r0 + acc] == a.ids[r0 + acc + 1]) acc++;
    if (blockIdx.y == 0 && threadIdx.x == 0) { a.res[2 * e] = acc; a.res[2 * e + 1] = a.next[r0 + acc]; }
    const uint32_t tid = blockIdx.y * 1024 + threadIdx.x, stride = gridDim.y * 1024;
    const float *src = a.ws_logits + (size_t)(r0 + acc) * d.V;
    float *dst = a.logits + (size_t)slot * d.V;
    for (uint32_t i = tid; i < d.V; i += stride) dst[i] = src[i];
    // rows r0+acc+1 .. r0+n-1 (save rows r-1) back to positions pos+acc+1 .. pos+n-1, every layer and kv head
    const uint32_t rows = n - 1 - acc, per_row = d.L * d.KV * hd;
    for (uint32_t i = tid; i < rows * per_row; i += stride) {
        const uint32_t j = i / per_row, rest = i % per_row, lg = rest / hd, c = rest % hd;     // lg = layer * KV + kv head
        const size_t sv = ((size_t)lg * (a.M - 1) + (r0 + acc + j)) * hd + c;
        const size_t cv = (size_t)slot * a.slot_elems + ((size_t)lg * d.max_seq + pos + acc + 1 + j) * hd + c;
        a.kc[cv] = a.ksave[sv];
        a.vc[cv] = a.vsave[sv];
    }
}

}  // namespace nb
