// stream_args.h -- argument block and geometry helpers of the streaming decode kernel (stream.cuh), shared with the host
// code that builds the per-CTA weight streams (engine.cu).  No device code here.
#pragma once
#include "kernels.cuh"

namespace nb {

constexpr int kConsWarps = kWarps - 1;            // 15 consumer warps; warp 15 is the producer
constexpr int kConsThreads = kConsWarps * 32;
constexpr int kStMaxStages = 24;
constexpr int kStRep = 8;                         // replicas of every activation vector that ALL CTAs read (spread over L2 slices)
constexpr int kStOwnMax = 128;                    // residual rows one CTA can own (n_embd <= 128 * CTAs)
constexpr int kStCluster = 8;                     // CTAs per cluster of the cluster launch (the portable maximum): one kv head, at most 8 splits
enum { EPI_ATTN = 5 };
enum StKindId { SK_QKV = 0, SK_O = 1, SK_W13 = 2, SK_W2 = 3, SK_CLS = 4 };

struct StKind {               // geometry of one matvec phase kind (identical for every layer and every CTA)
    uint64_t off;             // byte offset of the kind's first tile inside a layer's slice of a CTA's stream (CLS: inside the stream)
    uint32_t units;           // row units of the fused matrix
    uint32_t unit_rows;       // rows per unit: 1, or 2 for W1|W3 (a SwiGLU pair never straddles CTAs or tiles)
    uint32_t tile_rows;       // rows per tile (multiple of unit_rows)
    uint32_t tile_stride;     // bytes between consecutive tiles in the stream
    uint32_t n;               // row length in elements
    uint32_t row_stride;      // bytes between rows inside a tile (row bytes + 16)
    uint32_t aux_stride;      // bytes between aux rows inside a tile (Q80: scales, Q4K: side records; 0 for F32)
    uint32_t owned;           // 1: throughput mode, every tile is consumed by ONE warp (tile j -> warp j % 15); 0: all warps share a tile
};

struct StreamArgs {
    const uint8_t *stream; uint64_t cta_stride, layer_stride, cls_off;
    StKind kind[5];
    uint32_t nstages, stage_bytes, kv_tile_rows, kv_tile_magic;      // magic = ceil(2^32 / kv_tile_rows): idx / kv_tile_rows == umulhi(idx, magic) for idx < 65536
    uint32_t off_ring, off_act, off_act2, off_xs, off_attn;     // byte offsets inside dynamic shared memory (two activation operands: consecutive phases alternate)
    uint32_t off_rx;                                  // cluster launch: split 0's merge staging (mbarrier, phase count, st_attn_rx_floats); 0 otherwise
    const float *g_attn, *g_ffn, *g_final;            // rmsnorm gains [L][E], [L][E], [E]
    const float *qnorm, *knorm, *rope_cos, *rope_sin;
    const void *emb_w, *emb_aux;
    float *logits, *kc, *vc;
    // activation exchange: 64-bit words {fp32 value, 32-bit epoch}.  xq: QKV outputs [q_dim + 2 kv_dim] (one copy: read per head);
    // xv[0] = x, xv[1] = attention output, xv[2] = SwiGLU output: kStRep replicas each, rs[i] words apart;
    // xws: split-KV partials [KV][nsplit_max][KVM * (hd + 2)]
    unsigned long long *xq, *xv[3], *xws;
    uint32_t rs[3];
    uint32_t epoch_base;                              // epochs handed out before this launch (host-maintained, monotonic)
    float *cls_val; uint32_t *cls_idx;                // per-CTA argmax partials
    DevState *st; uint32_t *ids; uint8_t *seen;
    unsigned int *bar;                                // grid barrier counter (zeroed by the host before every launch)
    uint32_t *err;                                    // set to a nonzero code before a spin gives up (and traps)
    uint32_t n_steps, nsplit_max, chunk_target;
    uint32_t ablate;                                  // timing experiments only (NB200_ABLATE, results are wrong): 1 no quantise math, 2 no row dots, 4 no attention math,
                                                      // 8 no sum of squares, 16 no waiting for epochs, 32 no publishing to replicas 1..7
    unsigned long long *trace;                        // optional: CTA 0 / thread 0 clock64() after every barrier of the LAST step
    Dims d;
};

// activation prologue: warp slots held in registers between the sum-of-squares pass and the quantise pass; the host
// checks n <= st_prep_max_n before choosing the streaming kernel
constexpr int kStKmax = 6, kStKmaxQ4K = 2;           // warp slots of 128 (Q80 / F32) or 256 (Q4K) elements
__host__ __device__ inline uint32_t st_prep_max_n(uint32_t quant, uint32_t gs) {
    (void)gs;
    return quant == 0x42u ? (uint32_t)kConsWarps * kStKmaxQ4K * 256u : (uint32_t)kConsWarps * kStKmax * 128u;
}
// quantisation groups (Q80, 64 elements at least) or blocks (Q4K) of an operand of at most st_prep_max_n elements
constexpr int kStGroupsMax = kConsWarps * kStKmax * 128 / 64;

// attention workspace of one CTA (floats): q [KVM][hd] | scores of a segment [KVM][seg rows] | per-head scale [KVM] |
// the position's k, v [2][hd] | the item's partial [KVM][hd + 2]; the merge of a multi-split head stages the partials of
// all splits in the same region, followed by the merge weights / partial sums [2][KVM][nsplit_max] and totals [KVM]
constexpr int kStSegTiles = 8;                    // ring tiles of K/V that an attention segment keeps resident
__host__ __device__ inline uint32_t st_attn_work_floats(uint32_t kvm, uint32_t hd, uint32_t seg_rows) {
    return kvm * hd + kvm * seg_rows + ((kvm + 3u) & ~3u) + 2u * hd + kvm * (hd + 2u) + 16u;
}
__host__ __device__ inline uint32_t st_attn_smem_floats(uint32_t kvm, uint32_t hd, uint32_t nsplit_max, uint32_t seg_rows) {
    uint32_t ws = st_attn_work_floats(kvm, hd, seg_rows);
    const uint32_t merge = nsplit_max * kvm * hd;
    if (merge > ws) ws = merge;
    return ws + 2u * kvm * nsplit_max + 2u * kvm + 16u;
}
// cluster launch: split 0's merge staging, a region of its own right behind the workspace st_attn_work_floats (which it does
// not overlay, unlike the plain launch's staging), floats after a 16-byte mbarrier + phase count:
// accumulators [KVM][kStCluster][hd], maxima / weights [KVM][nsplit_max], totals [KVM], partial sums [KVM][nsplit_max]
__host__ __device__ inline uint32_t st_attn_rx_floats(uint32_t kvm, uint32_t hd, uint32_t nsplit_max) {
    return kvm * (uint32_t)kStCluster * hd + 2u * kvm * nsplit_max + kvm;
}

}  // namespace nb
