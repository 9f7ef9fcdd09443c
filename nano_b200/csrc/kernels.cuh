// kernels.cuh -- sm_90a device code of the batch-1 decode engine.
//
// Everything on the per-token path of the reference (infer/infer.c:584-1018, infer/tensor.c) is here:
//   activation prep ....... rmsnorm (infer.c:601) + Q80 quantize (tensor.c:21) / Q4K quantize (tensor.c:144)
//   matvec ................ matmul (infer.c:637), matmul_quant (infer.c:654), matmul_q4k (tensor.c:438)
//   attention ............. q/k head-norm + RoPE (infer.c:814-835), GQA attention (infer.c:841-879)
//   epilogues ............. KV-cache store, residual add (infer.c:906,963), SwiGLU (infer.c:937),
//                           repetition penalty + argmax (infer.c:1156-1171, 1026-1037)
//
// Numerics contract (DESIGN.md "Numerics"):
//   * integer work (Q80 / Q4K group dots, activation codes) is exact;
//   * exact mode (and the nb200_op_* operator entry points): every fp32 combine that follows an integer dot is
//     evaluated in the reference's order with __fmul_rn/__fadd_rn (no FMA contraction), so a quantised matvec is
//     bit-identical to the strict reference given the same activation vector; rmsnorm, attention and the F32 matvec
//     use the reference's sequential order;
//   * fast mode: the integer group dots are still exact, their fp32 terms are summed as one partial per lane plus a
//     warp tree (Q80), and rmsnorm / attention / F32 matvec use parallel trees -- the deviation from the strict
//     reference stays under the reference's own -ffast-math build noise (tests/golden/reference_noise_floor.json).
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include <type_traits>

#include "expf_ref.cuh"

// Non-template kernels get internal linkage in translation units that only want the device helpers (stream.cu).
#ifndef NB_K
#define NB_K
#endif

namespace nb {

constexpr int kThreads = 512;            // matvec CTA: 16 warps
constexpr int kWarps = kThreads / 32;
constexpr int kAttnThreads = 256;
constexpr int kAttnWarps = kAttnThreads / 32;
constexpr float kTrueMin = 1.401298464324817e-45f;   // FLT_TRUE_MIN (tensor.c:159 quirk)

struct Dims {
    uint32_t arch, quant, gs;
    uint32_t block_size, V, L, E, H, KV, F, hd, q_dim, kv_dim, max_seq, kv_mul;
    uint32_t exact;
};

// Per-step state that lives in HBM so one captured graph serves every position.
struct DevState {
    uint32_t pos;          // position of the token being consumed (ids[pos])
    uint32_t is_causal;    // 0 => seq2seq mode, attend all max_seq rows (infer.c:849)
    uint32_t n_prompt;     // device loop: positions < n_prompt-1 are teacher-forced
    uint32_t advance;      // 1 => the classifier's last CTA appends the token and bumps pos
    float penalty;         // repetition penalty (1.0 => identity)
    uint32_t next_token;   // result of the step
    uint32_t cls_ticket;   // last-CTA election for the argmax
    uint32_t token;        // API mode: the token to consume (use_token = 1); device loop reads ids[pos]
    uint32_t use_token;
    uint32_t pad[3];
};

// ------------------------------------------------------------------------------------------------
// Tensor parallelism over NVLink peer memory (SURVEY 8e; there is no reference code for this, the reference is one CPU).
// Every rank owns a row slice of each matrix (whole kv-head groups for QKV/attention) and keeps the FULL activation
// vectors x / xba / hb in an "exchange block" that its peers can write.  Each element of those vectors is a 64-bit word
// {fp32 value, 32-bit epoch}: a producing kernel's epilogue pushes every finished element into every rank's copy with ONE
// 8-byte store (single-copy atomic, so the value and its epoch arrive together -- no fence, no flag, no ticket), and the
// consuming kernel's activation prologue spins per element until the epoch it expects has arrived.  Nothing is ever read
// remotely.  The epoch of exchange k of token t is t*nph + k, so a buffer reused by a later exchange can never be
// mistaken for the earlier one.  Row dots are computed exactly as on one GPU and every rank prepares the same full
// vector, so results are bit-identical to the single-GPU engine.
//   Why a buffer is never overwritten before its readers are done (no double buffering): a rank can only start the
//   exchange that rewrites x / xba / hb after it has consumed, from EVERY rank, the elements of a later exchange whose
//   producing kernels run (in stream order) after the kernels that read the old contents.
// ------------------------------------------------------------------------------------------------
constexpr int kTpMax = 8;
struct TpHdr {                     // first 256 bytes of the exchange block
    unsigned long long cls_v[kTpMax];   // per-rank argmax partials {value bits, epoch} / {index, epoch} (written by peers)
    unsigned long long cls_i[kTpMax];
    uint32_t epoch_base;           // exchanges completed by earlier tokens (local; bumped by the classifier's last CTA)
    uint32_t timeout;              // set when a spin gave up (peer died): results are garbage, the host reports an error
};
constexpr uint32_t kTpHdrBytes = 256;
struct TpArgs {
    uint32_t size, rank;           // size <= 1: single GPU, everything below ignored
    uint32_t wait_ph, signal_ph;   // 1-based exchange ids within a token (0 = none); epoch = epoch_base + id
    uint32_t nph;                  // exchanges per token
    uint32_t row_base;             // global index of local output row 0
    uint32_t out_off;              // byte offset of the output vector (64-bit elements) inside the exchange block
    uint32_t pad;
    unsigned char *peer[kTpMax];   // exchange block of every rank (peer[rank] = own)
};
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long *p) {
    unsigned long long v; asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ TpHdr *tp_hdr(const TpArgs &tp, uint32_t r) { return reinterpret_cast<TpHdr *>(tp.peer[r]); }
__device__ __forceinline__ unsigned long long tp_pack(uint32_t bits, uint32_t epoch) { return ((unsigned long long)epoch << 32) | bits; }
// spin until the 64-bit element carries an epoch >= need; gives up after ~4 s so a dead peer cannot hang the GPU
__device__ __forceinline__ uint32_t tp_spin_load(const TpArgs &tp, const unsigned long long *p, uint32_t need) {
    unsigned long long w = ld_relaxed_sys_u64(p);
    if ((int32_t)((uint32_t)(w >> 32) - need) < 0) {
        const long long t0 = clock64();
        do {
            w = ld_relaxed_sys_u64(p);
            if (clock64() - t0 > 8000000000ll) { tp_hdr(tp, tp.rank)->timeout = 1; break; }
        } while ((int32_t)((uint32_t)(w >> 32) - need) < 0);
    }
    return (uint32_t)w;
}
// push one finished element (with its epoch) into every rank's copy of the output vector
__device__ __forceinline__ void tp_store(const TpArgs &tp, uint32_t idx, float v, uint32_t epoch) {
    const unsigned long long w = tp_pack(__float_as_uint(v), epoch);
    for (uint32_t p = 0; p < tp.size; p++) st_relaxed_sys_u64(reinterpret_cast<unsigned long long *>(tp.peer[p] + tp.out_off) + idx, w);
}
__device__ __forceinline__ uint32_t tp_epoch(const TpArgs &tp, uint32_t ph) { return __ldcg(&tp_hdr(tp, tp.rank)->epoch_base) + ph; }

enum Epilogue { EPI_STORE = 0, EPI_QKV = 1, EPI_RESID = 2, EPI_SWIGLU = 3, EPI_CLS = 4 };

struct MatvecArgs {
    // weights (device layout, see engine.cu "HBM layout")
    const void *w;          // Q80: int8 [rows][n]; F32: float [rows][n]; Q4K: nibble plane [rows][n/2]
    const void *w_aux;      // Q80: float scales [rows][n/gs]; Q4K: side records [rows][n/256][20 B]
    uint32_t rows, n;
    // activation source
    const float *src;       // fp32 vector of length n
    const float *gain;      // rmsnorm gain or nullptr (plain quantise)
    // outputs
    float *out;             // STORE/SWIGLU/CLS: vector; RESID: x (in/out)
    float *out_k, *out_v;   // QKV: raw k scratch [kv_dim]; V cache base of this layer [KV][max_seq][hd]
    const DevState *st;
    DevState *st_rw;        // CLS only
    // CLS extras
    const uint8_t *seen;    // [V] 1 if id occurred at positions < pos
    uint8_t *seen_rw;
    float *cls_val; uint32_t *cls_idx;   // per-CTA partial argmax
    uint32_t *ids;          // device copy of output_ids
    // debug dump of the prepared activation (written by CTA 0 when non-null)
    int8_t *dump_codes; float *dump_scales;
    // persistent kernel: step state already in registers (saves an L2 round trip per phase)
    uint32_t state_known, pos_val; float pen_val;
    unsigned long long *dbg;     // optional: CTA 0 / thread 0 clock64() stamps inside the phase (tools/gpu_trace.py)
    Dims d;
    TpArgs tp;                   // tensor-parallel exchange (k_matvec<..., TP=true> only)
    const float *lora_add;       // RESID only: LoRA branch of the O projection, added to the matvec result BEFORE the residual (infer.c:898-908)
};
#define NB_STAMP(ptr, k) do { if ((ptr) && blockIdx.x == 0 && threadIdx.x == 0) (ptr)[k] = clock64(); } while (0)

// ------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int4 ldg_stream16(const void *p) {
    int4 v;
    asm("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
        : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
template <int NT>
__device__ __forceinline__ float block_sum(float v, float *red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < NT / 32) ? red[lane] : 0.0f;
    t = warp_sum(t);
    __syncthreads();
    return t;
}
template <int NT>
__device__ __forceinline__ float block_max(float v, float *red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_max(v);
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < NT / 32) ? red[lane] : -FLT_MAX;
    t = warp_max(t);
    __syncthreads();
    return t;
}
// tensor.c:4-9, exact in fp32
__device__ __forceinline__ int nearest_int_magic(float f) {
    float t = __fadd_rn(f, 12582912.f);
    return (__float_as_int(t) & 0x007fffff) - 0x00400000;
}
// programmatic dependent launch: let the next kernel start its weight prefetch, then wait for our inputs
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Stage the fp32 source vector into shared memory with L2 (.cg) loads: the vector was produced by other
// CTAs (another kernel, or another phase of the persistent kernel), so it must not come from L1 / the
// non-coherent path.
// LL (tensor parallel): src is a vector of {value, epoch} words; spin per element until exchange tp->wait_ph has landed.
// SB = loads in flight per thread: 1 keeps the register footprint of the persistent kernels, 4 (x float4) is what
// the stand-alone matvec kernels use.
template <int NT, bool LL = false, int SB = 1>
__device__ __forceinline__ void stage_vector(const float *src, const float *__restrict__ gain, int n, float *stage, const TpArgs *tp = nullptr) {
    float *gstage = stage + n;                       // the rmsnorm gain rides along (one L2 latency, not two)
    if (!LL && SB == 1) {
        for (int i = threadIdx.x; i < n; i += NT) {
            const float v = __ldcg(src + i);
            const float g = gain ? __ldg(gain + i) : 0.0f;
            stage[i] = v;
            if (gain) gstage[i] = g;
        }
        __syncthreads();
        return;
    }
    // Every load of a batch is issued before any result is used: a thread's share of a long vector (19 elements of
    // n = 9728 with 512 threads) costs a few L2 round trips instead of one per element.
    if (LL) {
        uint32_t need = 0;
        if (tp->wait_ph) need = tp_epoch(*tp, tp->wait_ph);
        const unsigned long long *e = reinterpret_cast<const unsigned long long *>(src);
        constexpr int B = 8;
        for (int i0 = threadIdx.x; i0 < n; i0 += NT * B) {
            unsigned long long w[B]; float g[B];
#pragma unroll
            for (int u = 0; u < B; u++) {
                const int i = i0 + u * NT;
                if (i < n) { w[u] = ld_relaxed_sys_u64(e + i); g[u] = gain ? __ldg(gain + i) : 0.0f; }
            }
#pragma unroll
            for (int u = 0; u < B; u++) {
                const int i = i0 + u * NT;
                if (i < n) {
                    uint32_t bits = (uint32_t)w[u];
                    if (tp->wait_ph && (int32_t)((uint32_t)(w[u] >> 32) - need) < 0) bits = tp_spin_load(*tp, e + i, need);
                    stage[i] = __uint_as_float(bits);
                    if (gain) gstage[i] = g[u];
                }
            }
        }
    } else {
        constexpr int B = 4;                         // x 4 floats per load
        const bool vec = ((n & 3) == 0) && (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(gain)) & 15) == 0);
        const int n4 = vec ? (n >> 2) : 0;
        const float4 *s4 = reinterpret_cast<const float4 *>(src);
        const float4 *g4 = reinterpret_cast<const float4 *>(gain);
        for (int i0 = threadIdx.x; i0 < n4; i0 += NT * B) {
            float4 v[B], g[B];
#pragma unroll
            for (int u = 0; u < B; u++) {
                const int i = i0 + u * NT;
                if (i < n4) { v[u] = __ldcg(s4 + i); if (gain) g[u] = __ldg(g4 + i); }
            }
#pragma unroll
            for (int u = 0; u < B; u++) {
                const int i = i0 + u * NT;
                if (i < n4) { reinterpret_cast<float4 *>(stage)[i] = v[u]; if (gain) reinterpret_cast<float4 *>(gstage)[i] = g[u]; }
            }
        }
        for (int i = (n4 << 2) + threadIdx.x; i < n; i += NT) {      // unaligned / n % 4 != 0 callers (op-level entry points only)
            stage[i] = __ldcg(src + i);
            if (gain) gstage[i] = __ldg(gain + i);
        }
    }
    __syncthreads();
}

// infer.c:601-614 over the staged vector.  fast: tree sum; exact: the reference's sequential sum (thread 0).
template <int NT>
__device__ __forceinline__ float rms_inverse(const float *stage, int n, bool exact, float *red) {
    float ss;
    if (!exact) {
        float acc = 0.0f;
        for (int i = threadIdx.x; i < n; i += NT) { const float v = stage[i]; acc = fmaf(v, v, acc); }
        ss = block_sum<NT>(acc, red);
    } else {
        if (threadIdx.x == 0) {
            float acc = 0.0f;
            for (int i = 0; i < n; i++) acc = __fadd_rn(acc, __fmul_rn(stage[i], stage[i]));
            red[0] = acc;
        }
        __syncthreads();
        ss = red[0];
        __syncthreads();
    }
    ss = __fdiv_rn(ss, (float)n);
    ss = __fadd_rn(ss, 1e-5f);
    return __fdiv_rn(1.0f, __fsqrt_rn(ss));
}

__device__ __forceinline__ float act_value(const float *stage, int n, bool has_gain, float inv, int i) {
    const float v = stage[i];
    return has_gain ? __fmul_rn(stage[n + i], __fmul_rn(inv, v)) : v;
}

// ------------------------------------------------------------------------------------------------
// Activation preparation into shared memory (each CTA redoes it: <= 39 KB of L2 reads, no grid sync)
// smem layouts (followed by fp32 staging copies of the source and of the rmsnorm gain, n floats each):
//   F32 : float v[n]
//   Q80 : int8 codes[n] | pad16 | float scales[n/gs]
//   Q4K : u32 xe[n/8] (even elements) | u32 xo[n/8] (odd elements) | float4 {sq,bq,sum_q,0}[n/32]
// ------------------------------------------------------------------------------------------------
__host__ __device__ inline uint32_t act_region_bytes(uint32_t quant, uint32_t n, uint32_t gs) {
    uint32_t b;
    if (quant == 0x00u) b = n * 4u;
    else if (quant == 0x80u) b = ((n + 15u) & ~15u) + (n / gs) * 4u + 16u;
    else b = n + (n / 32u) * 16u;
    return (b + 15u) & ~15u;
}
__host__ __device__ inline uint32_t act_smem_bytes(uint32_t quant, uint32_t n, uint32_t gs) {
    return act_region_bytes(quant, n, gs) + 2u * n * 4u;      // + staging copies of the source and the gain
}

template <int NT, bool LL = false, int SB = 1>
__device__ void prep_f32(const float *src, const float *__restrict__ gain, int n, bool exact, float *act, float *stage, float *red,
                         const TpArgs *tp = nullptr) {
    stage_vector<NT, LL, SB>(src, gain, n, stage, tp);
    float inv = 1.0f;
    if (gain) inv = rms_inverse<NT>(stage, n, exact, red);
    for (int i = threadIdx.x; i < n; i += NT) act[i] = act_value(stage, n, gain != nullptr, inv, i);
    __syncthreads();
}

// (int8) round(x / scale) of tensor.c:40-42, bit-exact with a fast path: q = x * (1/scale) is within ~4e-5 of the
// correctly rounded quotient for |q| <= 127, so unless q sits within 1e-3 of a .5 boundary the rounded integer is
// unambiguous; the rare boundary case takes the IEEE division + roundf path.
static __device__ __noinline__ int q80_code_slow(float v, float sc) { return (int)roundf(__fdiv_rn(v, sc)); }   // rare: kept out of line
__device__ __forceinline__ int q80_code(float v, float sc, float rinv) {
    const float q = v * rinv;
    const float a = fabsf(q), fl = floorf(a), frac = a - fl;
    if (fabsf(frac - 0.5f) < 1e-3f) return q80_code_slow(v, sc);
    const int c = (int)fl + (frac > 0.5f ? 1 : 0);
    return q < 0.0f ? -c : c;
}

// tensor.c:21-46 (division and round-half-away exactly as the strict reference; zero group -> 0)
template <int NT, bool LL = false, int SB = 1>
__device__ void prep_q80(const float *src, const float *__restrict__ gain, int n, int gs, bool exact,
                         unsigned char *act, float *stage, float *red, int8_t *dump_codes, float *dump_scales,
                         unsigned long long *dbg = nullptr, const TpArgs *tp = nullptr) {
    int8_t *codes = reinterpret_cast<int8_t *>(act);
    float *scales = reinterpret_cast<float *>(act + ((n + 15) & ~15));
    stage_vector<NT, LL, SB>(src, gain, n, stage, tp);
    NB_STAMP(dbg, 2);
    float inv = 1.0f;
    if (gain) inv = rms_inverse<NT>(stage, n, exact, red);
    NB_STAMP(dbg, 3);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int G = n / gs, epl = gs / 32;      // elements per lane (gs in {32,64,128,256})
    for (int g = warp; g < G; g += NT / 32) {
        float v[8];
        float amax = 0.0f;
        const int base = g * gs + lane * epl;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (j < epl) { v[j] = act_value(stage, n, gain != nullptr, inv, base + j); amax = fmaxf(amax, fabsf(v[j])); }
        }
        amax = warp_max(amax);
        const float sc = __fdiv_rn(amax, 127.0f);
        const float rinv = __frcp_rn(sc);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (j < epl) codes[base + j] = (int8_t)((sc == 0.0f) ? 0 : q80_code(v[j], sc, rinv));
        }
        if (lane == 0) scales[g] = sc;
    }
    __syncthreads();
    if (dump_codes && blockIdx.x == 0) {
        for (int i = threadIdx.x; i < n; i += NT) dump_codes[i] = codes[i];
        for (int i = threadIdx.x; i < G; i += NT) dump_scales[i] = scales[i];
    }
}

// quantize_one_block_q4k_in_situ (tensor.c:144-242) by one warp: lane l holds elements 8l..8l+7 of the 256-element block
// (group g = lanes 4g..4g+3).  Returns the 4-bit codes of the lane's elements, the group's code sum and 6-bit
// scale/bias codes (replicated in the 4 lanes of the group) and the block's two fp32 super-scales (all lanes).
__device__ __forceinline__ void q4k_quantize_block(const float (&v)[8], uint32_t (&c)[8], int &csum, float &ss, float &sbias, int &s6, int &b6) {
    float lo = FLT_MAX, hi = kTrueMin;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (v[j] > hi) hi = v[j];
        if (v[j] < lo) lo = v[j];
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    }
    const float s = (lo <= 0.0f) ? __fdiv_rn(__fsub_rn(hi, lo), 15.0f) : __fdiv_rn(hi, 15.0f);
    const float bias = (lo <= 0.0f) ? -lo : 0.0f;
    csum = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        c[j] = (s == 0.0f) ? 0u : (uint32_t)(nearest_int_magic(__fdiv_rn(__fadd_rn(v[j], bias), s)) & 0x0f);
        csum += (int)c[j];
    }
    csum += __shfl_xor_sync(0xffffffffu, csum, 1);
    csum += __shfl_xor_sync(0xffffffffu, csum, 2);
    float smax = fmaxf(kTrueMin, s), bmax = fmaxf(kTrueMin, bias);
#pragma unroll
    for (int o = 4; o <= 16; o <<= 1) {
        smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, o));
        bmax = fmaxf(bmax, __shfl_xor_sync(0xffffffffu, bmax, o));
    }
    ss = __fdiv_rn(smax, 63.0f); sbias = __fdiv_rn(bmax, 63.0f);
    s6 = (ss == 0.0f) ? 0 : (nearest_int_magic(__fdiv_rn(s, ss)) & 0x3f);
    b6 = (sbias == 0.0f) ? 0 : (nearest_int_magic(__fdiv_rn(bias, sbias)) & 0x3f);
}

// tensor.c:144-242 on 256-element blocks (n % 256 == 0); one warp per block, 8 elements per lane.
// dump (optional, CTA 0): codes[n] as bytes, then per group {s6,b6} and per block {ss,sbias} in dump_scales:
//   dump_scales[0..n/256)      = ss
//   dump_scales[n/256..2n/256) = sbias
//   dump_codes[n .. n + n/32)  = s6, dump_codes[n + n/32 .. n + 2n/32) = b6
template <int NT, bool LL = false, int SB = 1>
__device__ void prep_q4k(const float *src, const float *__restrict__ gain, int n, bool exact,
                         unsigned char *act, float *stage, float *red, int8_t *dump_codes, float *dump_scales, const TpArgs *tp = nullptr) {
    uint32_t *xe = reinterpret_cast<uint32_t *>(act);
    uint32_t *xo = reinterpret_cast<uint32_t *>(act + n / 2);
    float4 *gp = reinterpret_cast<float4 *>(act + n);
    stage_vector<NT, LL, SB>(src, gain, n, stage, tp);
    float inv = 1.0f;
    if (gain) inv = rms_inverse<NT>(stage, n, exact, red);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int NB = n / 256;
    const bool dump = dump_codes && blockIdx.x == 0;
    for (int b = warp; b < NB; b += NT / 32) {
        float v[8];
        const int base = b * 256 + lane * 8;
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = act_value(stage, n, gain != nullptr, inv, base + j);
        uint32_t c[8];
        int csum, s6, b6;
        float ss, sbias;
        q4k_quantize_block(v, c, csum, ss, sbias, s6, b6);
        xe[b * 32 + lane] = c[0] | (c[2] << 8) | (c[4] << 16) | (c[6] << 24);
        xo[b * 32 + lane] = c[1] | (c[3] << 8) | (c[5] << 16) | (c[7] << 24);
        if ((lane & 3) == 0)
            gp[b * 8 + (lane >> 2)] = make_float4(__fmul_rn((float)s6, ss), __fmul_rn((float)b6, sbias), (float)csum, 0.0f);
        if (dump) {
#pragma unroll
            for (int j = 0; j < 8; j++) dump_codes[base + j] = (int8_t)c[j];
            if ((lane & 3) == 0) {
                dump_codes[n + b * 8 + (lane >> 2)] = (int8_t)s6;
                dump_codes[n + n / 32 + b * 8 + (lane >> 2)] = (int8_t)b6;
            }
            if (lane == 0) { dump_scales[b] = ss; dump_scales[NB + b] = sbias; }
        }
    }
    __syncthreads();
}

// quantize_tensor_q4k_in_situ (tensor.c:281-310) for whole tensors whose last dimension is a multiple of 256: every
// 256-element block is independent, one warp per block, output in the reference's 160-byte block layout
// {u32 tag=0x42, u32 len=256, u32 meta=0, f32 s_scale, f32 s_bias, u8 sb[12], u8 value[128]} (tensor.h:96-114).
NB_K __global__ void __launch_bounds__(256) k_q4k_quantize_blocks(const float *__restrict__ x, unsigned long long nblocks, uint8_t *__restrict__ blocks) {
    const int lane = threadIdx.x & 31;
    const unsigned long long w0 = (unsigned long long)blockIdx.x * 8 + (threadIdx.x >> 5), nw = (unsigned long long)gridDim.x * 8;
    for (unsigned long long b = w0; b < nblocks; b += nw) {
        float v[8];
        const float4 *src = reinterpret_cast<const float4 *>(x + b * 256 + lane * 8);
        const float4 a0 = __ldg(src), a1 = __ldg(src + 1);
        v[0] = a0.x; v[1] = a0.y; v[2] = a0.z; v[3] = a0.w; v[4] = a1.x; v[5] = a1.y; v[6] = a1.z; v[7] = a1.w;
        uint32_t c[8];
        int csum, s6, b6;
        float ss, sbias;
        q4k_quantize_block(v, c, csum, ss, sbias, s6, b6);
        uint32_t *blk = reinterpret_cast<uint32_t *>(blocks + b * 160);
        blk[8 + lane] = (c[0] | (c[1] << 4)) | ((c[2] | (c[3] << 4)) << 8) | ((c[4] | (c[5] << 4)) << 16) | ((c[6] | (c[7] << 4)) << 24);
        uint32_t sb0 = 0, sb1 = 0, sb2 = 0;       // tensor.c:198-241 packing of the eight 6-bit scale / bias codes
#pragma unroll
        for (int g = 0; g < 4; g++) {
            const uint32_t sl = (uint32_t)__shfl_sync(0xffffffffu, s6, 4 * g), sh = (uint32_t)__shfl_sync(0xffffffffu, s6, 4 * (g + 4));
            const uint32_t bl = (uint32_t)__shfl_sync(0xffffffffu, b6, 4 * g), bh = (uint32_t)__shfl_sync(0xffffffffu, b6, 4 * (g + 4));
            sb0 |= ((((sh & 0x30u) << 2) | (sl & 0x3fu)) & 0xffu) << (8 * g);
            sb1 |= ((((bh & 0x30u) << 2) | (bl & 0x3fu)) & 0xffu) << (8 * g);
            sb2 |= ((((bh & 0x0fu) << 4) | (sh & 0x0fu)) & 0xffu) << (8 * g);
        }
        if (lane == 0) {
            blk[0] = 0x42u; blk[1] = 256u; blk[2] = 0u; blk[3] = __float_as_uint(ss); blk[4] = __float_as_uint(sbias);
            blk[5] = sb0; blk[6] = sb1; blk[7] = sb2;
        }
    }
}

// matmul_q4k (tensor.c:438-471) on the reference's own block layout for BOTH operands (x already quantised by the caller):
// one warp per row, lane = (block of the 4-block step, group); dot_two_blocks_q4k's integer sums with dp4a, its 4-term
// fp32 expression left to right, groups then blocks accumulated in the reference's order.
NB_K __global__ void __launch_bounds__(256) k_q4k_matvec_blocks(const uint8_t *__restrict__ wblocks, const uint8_t *__restrict__ xblocks,
                                                           uint32_t rows, uint32_t bpr, float *__restrict__ out) {
    const int lane = threadIdx.x & 31, gi = lane & 7, j = gi & 3;
    const uint32_t row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    float acc = 0.0f;
    for (uint32_t b0 = 0; b0 < bpr; b0 += 4) {
        const uint32_t b = b0 + (lane >> 3);
        const bool on = b < bpr;
        float term = 0.0f;
        if (on) {
            const uint8_t *wb = wblocks + ((size_t)row * bpr + b) * 160, *xb = xblocks + (size_t)b * 160;
            const uint32_t *wr = reinterpret_cast<const uint32_t *>(wb), *xr = reinterpret_cast<const uint32_t *>(xb);
            auto group_sb = [&](const uint32_t *rec, float &s, float &bb) {       // get_group_scale_and_bias, tensor.c:113-141
                const uint32_t bs = (rec[5] >> (8 * j)) & 0xff, bi = (rec[6] >> (8 * j)) & 0xff, bh = (rec[7] >> (8 * j)) & 0xff;
                const uint32_t s6 = (gi < 4) ? (bs & 0x3f) : ((((bs >> 6) << 4) | (bh & 0x0f)) & 0x3f);
                const uint32_t b6 = (gi < 4) ? (bi & 0x3f) : ((((bi >> 6) << 4) | (bh >> 4)) & 0x3f);
                s = __fmul_rn((float)s6, __uint_as_float(rec[3])); bb = __fmul_rn((float)b6, __uint_as_float(rec[4]));
            };
            float sp, bp, sq, bq;
            group_sb(wr, sp, bp); group_sb(xr, sq, bq);
            int spq = 0, spp = 0, sqq = 0;
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const int wv = (int)wr[8 + gi * 4 + t], xv = (int)xr[8 + gi * 4 + t];
                const int wl = wv & 0x0f0f0f0f, wh = (wv >> 4) & 0x0f0f0f0f, xl = xv & 0x0f0f0f0f, xh = (xv >> 4) & 0x0f0f0f0f;
                spq = __dp4a(wl, xl, spq); spq = __dp4a(wh, xh, spq);
                spp = __dp4a(wl, 0x01010101, spp); spp = __dp4a(wh, 0x01010101, spp);
                sqq = __dp4a(xl, 0x01010101, sqq); sqq = __dp4a(xh, 0x01010101, sqq);
            }
            term = __fmul_rn(__fmul_rn(sp, sq), (float)spq);                      // tensor.c:425-428, left to right
            term = __fsub_rn(term, __fmul_rn(__fmul_rn(sp, bq), (float)spp));
            term = __fsub_rn(term, __fmul_rn(__fmul_rn(sq, bp), (float)sqq));
            term = __fadd_rn(term, __fmul_rn(__fmul_rn(32.0f, bp), bq));
        }
        float dot = 0.0f;
        const int lead = lane & ~7;
#pragma unroll
        for (int g = 0; g < 8; g++) dot = __fadd_rn(dot, __shfl_sync(0xffffffffu, term, lead + g));
#pragma unroll
        for (int bb = 0; bb < 4; bb++) {
            const float t = __shfl_sync(0xffffffffu, dot, bb * 8);
            if (b0 + bb < bpr) acc = __fadd_rn(acc, t);
        }
    }
    if (lane == 0) out[row] = acc;
}

// ------------------------------------------------------------------------------------------------
// Row-block dot products.  A warp owns RB consecutive rows; lanes split K in 16-byte chunks
// (one 512-byte step per warp-wide load).  All variants return the row values replicated in
// every lane.
// ------------------------------------------------------------------------------------------------

// matmul_quant, infer.c:654-679.  LPG = lanes per quantisation group = gs/16.
// A tile is the weight codes + scales of one macro-step (2 x 512 bytes) of RB rows, held in registers so that
// it can be requested from HBM/L2 BEFORE the activation prologue (weights never depend on activations).
template <int RB>
struct Q80Tile { int4 w[2][RB]; float ws[2][RB]; };

template <int RB, int LPG>
__device__ __forceinline__ void q80_load(Q80Tile<RB> &t, const int8_t *__restrict__ W, const float *__restrict__ S, uint32_t row0,
                                         uint32_t rows, uint32_t n, uint32_t k0) {
    constexpr uint32_t gs = LPG * 16;
    const int lane = threadIdx.x & 31;
    const uint32_t G = n / gs;
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const uint32_t k = k0 + s * 512 + lane * 16;
        const bool on = k < n;
#pragma unroll
        for (int r = 0; r < RB; r++) {
            const uint32_t row = min(row0 + r, rows - 1);
            t.w[s][r] = on ? ldg_stream16(W + (size_t)row * n + k) : make_int4(0, 0, 0, 0);
            t.ws[s][r] = on ? __ldg(S + (size_t)row * G + k / gs) : 0.0f;
        }
    }
}

// ORD = true: the reference's left-to-right fp32 sum over groups, value replicated in every lane (exact mode, and the row-block
// helpers below).  ORD = false (fast mode): every lane keeps one fp32 partial per row -- nothing crosses lanes inside the K loop --
// and the caller finishes with one warp_sum per row.
template <int RB, int LPG, bool ORD = true>
__device__ __forceinline__ void q80_consume(const Q80Tile<RB> &t, uint32_t n, uint32_t k0, const unsigned char *act, float *val) {
    constexpr uint32_t gs = LPG * 16;
    constexpr int GPS = 32 / LPG;   // groups covered by one 512-byte step
    const int lane = threadIdx.x & 31;
    const int8_t *codes = reinterpret_cast<const int8_t *>(act);
    const float *xs = reinterpret_cast<const float *>(act + ((n + 15) & ~15));
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const uint32_t kbase = k0 + s * 512;
        if (kbase >= n) break;
        const uint32_t k = kbase + lane * 16;
        const bool on = k < n;
        const int4 xq = on ? *reinterpret_cast<const int4 *>(codes + k) : make_int4(0, 0, 0, 0);
        const float xsc = on ? xs[k / gs] : 0.0f;
#pragma unroll
        for (int r = 0; r < RB; r++) {
            int isum = __dp4a(t.w[s][r].x, xq.x, 0);
            isum = __dp4a(t.w[s][r].y, xq.y, isum);
            isum = __dp4a(t.w[s][r].z, xq.z, isum);
            isum = __dp4a(t.w[s][r].w, xq.w, isum);
            if (!ORD) { val[r] = fmaf((float)isum, t.ws[s][r] * xsc, val[r]); continue; }
#pragma unroll
            for (int o = 1; o < LPG; o <<= 1) isum += __shfl_xor_sync(0xffffffffu, isum, o);
            const float term = __fmul_rn(__fmul_rn((float)isum, t.ws[s][r]), xsc);
#pragma unroll
            for (int g = 0; g < GPS; g++) {
                const float v = __shfl_sync(0xffffffffu, term, g * LPG);
                if (kbase + g * gs < n) val[r] = __fadd_rn(val[r], v);
            }
        }
    }
}

template <int RB, int LPG>
__device__ __forceinline__ void rows_q80(const int8_t *__restrict__ W, const float *__restrict__ S, uint32_t row0,
                                         uint32_t rows, uint32_t n, const unsigned char *act, float *val, const Q80Tile<RB> *pre) {
#pragma unroll
    for (int r = 0; r < RB; r++) val[r] = 0.0f;
    for (uint32_t k0 = 0; k0 < n; k0 += 1024) {
        Q80Tile<RB> t;
        if (k0 == 0 && pre) t = *pre;
        else q80_load<RB, LPG>(t, W, S, row0, rows, n, k0);
        q80_consume<RB, LPG>(t, n, k0, act, val);
    }
}

// matmul, infer.c:637-651 (fast mode: lane-split FMA + tree; exact mode uses k_matvec_f32_exact)
template <int RB>
__device__ __forceinline__ void rows_f32(const float *__restrict__ W, uint32_t row0, uint32_t rows, uint32_t n,
                                         const unsigned char *act, float *val) {
    const int lane = threadIdx.x & 31;
    const float *x = reinterpret_cast<const float *>(act);
    float acc[RB];
#pragma unroll
    for (int r = 0; r < RB; r++) acc[r] = 0.0f;
    for (uint32_t k0 = 0; k0 < n; k0 += 256) {
        int4 w[2][RB];
        float4 xv[2];
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const uint32_t k = k0 + s * 128 + lane * 4;
            const bool on = k < n;
#pragma unroll
            for (int r = 0; r < RB; r++) {
                const uint32_t row = min(row0 + r, rows - 1);
                w[s][r] = on ? ldg_stream16(W + (size_t)row * n + k) : make_int4(0, 0, 0, 0);
            }
            xv[s] = on ? *reinterpret_cast<const float4 *>(x + k) : make_float4(0, 0, 0, 0);
        }
#pragma unroll
        for (int s = 0; s < 2; s++)
#pragma unroll
            for (int r = 0; r < RB; r++) {
                acc[r] = fmaf(__int_as_float(w[s][r].x), xv[s].x, acc[r]);
                acc[r] = fmaf(__int_as_float(w[s][r].y), xv[s].y, acc[r]);
                acc[r] = fmaf(__int_as_float(w[s][r].z), xv[s].z, acc[r]);
                acc[r] = fmaf(__int_as_float(w[s][r].w), xv[s].w, acc[r]);
            }
    }
#pragma unroll
    for (int r = 0; r < RB; r++) val[r] = warp_sum(acc[r]);
}

// matmul_q4k / dot_two_blocks_q4k, tensor.c:359-471.  One lane owns one 32-element group per step
// (16 bytes of nibbles); 8 lanes = one 256-element block.  side: 20-byte records {ss, sbias, sb[12]}.
template <int RB>
__device__ __forceinline__ void rows_q4k(const uint8_t *__restrict__ W, const uint8_t *__restrict__ side, uint32_t row0,
                                         uint32_t rows, uint32_t n, const unsigned char *act, float *val) {
    const int lane = threadIdx.x & 31;
    const uint32_t *xe = reinterpret_cast<const uint32_t *>(act);
    const uint32_t *xo = reinterpret_cast<const uint32_t *>(act + n / 2);
    const float4 *gp = reinterpret_cast<const float4 *>(act + n);
    const uint32_t rowbytes = n / 2, bpr = n / 256;
#pragma unroll
    for (int r = 0; r < RB; r++) val[r] = 0.0f;
    for (uint32_t k0 = 0; k0 < rowbytes; k0 += 512) {
        const uint32_t k = k0 + lane * 16;            // byte offset in the nibble row
        const bool on = k < rowbytes;
        const uint32_t grp = k / 16;                  // group index within the row
        const uint32_t blk = grp >> 3, gi = grp & 7, j = gi & 3;
        int4 w[RB];
        uint32_t sb0[RB], sb1[RB], sb2[RB];
        float ssc[RB], sbi[RB];
#pragma unroll
        for (int r = 0; r < RB; r++) {
            const uint32_t row = min(row0 + r, rows - 1);
            w[r] = on ? ldg_stream16(W + (size_t)row * rowbytes + k) : make_int4(0, 0, 0, 0);
            const uint32_t *rec = reinterpret_cast<const uint32_t *>(side + ((size_t)row * bpr + (on ? blk : 0)) * 20);
            ssc[r] = __uint_as_float(__ldg(rec + 0));
            sbi[r] = __uint_as_float(__ldg(rec + 1));
            sb0[r] = __ldg(rec + 2); sb1[r] = __ldg(rec + 3); sb2[r] = __ldg(rec + 4);
        }
        int4 e4 = make_int4(0, 0, 0, 0), o4 = make_int4(0, 0, 0, 0);
        float4 q = make_float4(0, 0, 0, 0);
        if (on) {
            e4 = *reinterpret_cast<const int4 *>(xe + grp * 4);
            o4 = *reinterpret_cast<const int4 *>(xo + grp * 4);
            q = gp[grp];
        }
#pragma unroll
        for (int r = 0; r < RB; r++) {
            const uint32_t bs = (sb0[r] >> (8 * j)) & 0xff, bb = (sb1[r] >> (8 * j)) & 0xff, bh = (sb2[r] >> (8 * j)) & 0xff;
            const uint32_t s6 = (gi < 4) ? (bs & 0x3f) : ((((bs >> 6) << 4) | (bh & 0x0f)) & 0x3f);
            const uint32_t b6 = (gi < 4) ? (bb & 0x3f) : ((((bb >> 6) << 4) | (bh >> 4)) & 0x3f);
            const float sp = __fmul_rn((float)s6, ssc[r]), bp = __fmul_rn((float)b6, sbi[r]);
            int spq = 0, spp = 0;
            const int wv[4] = {w[r].x, w[r].y, w[r].z, w[r].w};
            const int ev[4] = {e4.x, e4.y, e4.z, e4.w};
            const int ov[4] = {o4.x, o4.y, o4.z, o4.w};
#pragma unroll
            for (int t = 0; t < 4; t++) {
                const int lo = wv[t] & 0x0f0f0f0f, hi = (wv[t] >> 4) & 0x0f0f0f0f;
                spq = __dp4a(lo, ev[t], spq); spq = __dp4a(hi, ov[t], spq);
                spp = __dp4a(lo, 0x01010101, spp); spp = __dp4a(hi, 0x01010101, spp);
            }
            // tensor.c:425-428, left to right
            float term = __fmul_rn(__fmul_rn(sp, q.x), (float)spq);
            term = __fsub_rn(term, __fmul_rn(__fmul_rn(sp, q.y), (float)spp));
            term = __fsub_rn(term, __fmul_rn(__fmul_rn(q.x, bp), q.z));
            term = __fadd_rn(term, __fmul_rn(__fmul_rn(32.0f, bp), q.y));
            // per-block sequential sum over its 8 groups (lanes 8b..8b+7), then blocks in order
            float dot = 0.0f;
            const int lead = lane & ~7;
#pragma unroll
            for (int g = 0; g < 8; g++) dot = __fadd_rn(dot, __shfl_sync(0xffffffffu, term, lead + g));
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const float t = __shfl_sync(0xffffffffu, dot, b * 8);
                if (k0 + b * 128 < rowbytes) val[r] = __fadd_rn(val[r], t);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// One fused matvec phase = activation prep -> row blocks -> epilogue, executed by `ncta` cooperating CTAs
// (a whole kernel grid in the multi-kernel path, or the persistent grid of k_decode_mega).
// ------------------------------------------------------------------------------------------------
struct MatvecSmem {
    float red[32];
    float best_v[kWarps];
    uint32_t best_i[kWarps];
    uint32_t flag;
};

// Weights never depend on activations: pull a warp's first row blocks of a matrix towards L2 ahead of time
// (before the PDL wait / before a grid barrier), so the HBM latency hides behind the wait.
template <int QUANT, int RB>
__device__ __forceinline__ void prefetch_row_blocks(const void *w, uint32_t rows, uint32_t n, uint32_t cta, uint32_t ncta, uint32_t max_iters,
                                                    const void *aux = nullptr, uint32_t aux_row_bytes = 0, const float *gain = nullptr) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t nblocks = (rows + RB - 1) / RB;
    const uint32_t gwarp = cta * kWarps + warp, nwarps = ncta * kWarps;
    const uint32_t rowbytes = (QUANT == 0x00) ? n * 4u : (QUANT == 0x80) ? n : n / 2u;
    const uint32_t blkbytes = RB * rowbytes;
    uint32_t it = 0;
    for (uint32_t rb = gwarp; rb < nblocks && it < max_iters; rb += nwarps, it++) {
        const char *base = static_cast<const char *>(w) + (size_t)rb * blkbytes;
        for (uint32_t off = lane * 128u; off < blkbytes; off += 32u * 128u) prefetch_l2(base + off);
        if (aux) {
            const char *ab = static_cast<const char *>(aux) + (size_t)rb * RB * aux_row_bytes;
            for (uint32_t off = lane * 128u; off < RB * aux_row_bytes; off += 32u * 128u) prefetch_l2(ab + off);
        }
    }
    if (gain && warp == 0) for (uint32_t off = (cta * 32u + lane) * 32u; off < n; off += ncta * 32u * 32u) prefetch_l2(gain + off);
}

// D (Q80 only) = weight tiles a warp keeps in flight along K: tile d+D of a row block is requested as soon as tile d has
// been consumed, and the first D tiles are requested before the activation prologue.
template <int QUANT, int EPI, int RB, int LPG, bool TP = false, int D = 1, int SB = 1>
__device__ __forceinline__ void matvec_phase(const MatvecArgs &a, uint32_t cta, uint32_t ncta, unsigned char *act, MatvecSmem &ms) {
    const Dims &d = a.d;
    // tensor parallel: local row r is element rbase + r of the (replicated) output vector; QKV outputs stay local
    const uint32_t rbase = (TP && EPI != EPI_QKV) ? a.tp.row_base : 0u;
    const unsigned long long *out_ll = reinterpret_cast<const unsigned long long *>(a.out);     // TP: x is {value, epoch} words
    const bool exact = d.exact != 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t nblocks = (a.rows + RB - 1) / RB;
    const uint32_t gwarp = cta * kWarps + warp, nwarps = ncta * kWarps;
    float *stage = reinterpret_cast<float *>(act + act_region_bytes(QUANT, a.n, (QUANT == 0x80) ? LPG * 16 : 1));

    NB_STAMP(a.dbg, 0);
    // request this warp's first weight tile (and the residual it will add to) before the activation prologue
    Q80Tile<RB> pre[D];
    float xres[RB];
    const bool has_first = gwarp < nblocks;
    if (QUANT == 0x80 && has_first) {
#pragma unroll
        for (int dd = 0; dd < D; dd++)
            if (dd == 0 || dd * 1024u < a.n)
                q80_load<RB, LPG>(pre[dd], static_cast<const int8_t *>(a.w), static_cast<const float *>(a.w_aux), gwarp * RB, a.rows, a.n, dd * 1024u);
    }
    if (EPI == EPI_RESID && has_first) {
#pragma unroll
        for (int r = 0; r < RB; r++) {
            const uint32_t xi = rbase + min(gwarp * RB + r, a.rows - 1);
            xres[r] = TP ? __uint_as_float((uint32_t)__ldcg(out_ll + xi)) : __ldcg(a.out + xi);       // own rows: written by this rank
        }
    }

    if (QUANT == 0x00) prep_f32<kThreads, TP, SB>(a.src, a.gain, a.n, exact, reinterpret_cast<float *>(act), stage, ms.red, &a.tp);
    else if (QUANT == 0x80) { NB_STAMP(a.dbg, 1); prep_q80<kThreads, TP, SB>(a.src, a.gain, a.n, LPG * 16, exact, act, stage, ms.red, cta == 0 ? a.dump_codes : nullptr, a.dump_scales, a.dbg, &a.tp); }
    else prep_q4k<kThreads, TP, SB>(a.src, a.gain, a.n, exact, act, stage, ms.red, cta == 0 ? a.dump_codes : nullptr, a.dump_scales, &a.tp);
    uint32_t out_epoch = 0;
    if (TP && a.tp.signal_ph) out_epoch = tp_epoch(a.tp, a.tp.signal_ph);

    NB_STAMP(a.dbg, 4);
    const uint32_t pos = a.state_known ? a.pos_val : (a.st ? __ldcg(&a.st->pos) : 0);
    float bestv = -FLT_MAX; uint32_t besti = 0xffffffffu;
    float pen = 1.0f;
    if (EPI == EPI_CLS) pen = a.state_known ? a.pen_val : __ldcg(&a.st->penalty);

    // One row block = dot products + epilogue.  `first` is a compile-time tag: the first block of a warp consumes the
    // tile (and residual) requested before the prologue straight from registers.  (A run-time `&pre : nullptr` select
    // forces the tile through local memory, and local memory misses to L2 after every barrier's L1 invalidation.)
    auto do_block = [&](const uint32_t rb, auto first_tag) {
        constexpr bool kFirst = decltype(first_tag)::value;
        const uint32_t row0 = rb * RB;
        float val[RB];
        if (QUANT == 0x00) rows_f32<RB>(static_cast<const float *>(a.w), row0, a.rows, a.n, act, val);
        else if (QUANT == 0x80) {
#pragma unroll
            for (int r = 0; r < RB; r++) val[r] = 0.0f;
            Q80Tile<RB> t[D];
#pragma unroll
            for (int dd = 0; dd < D; dd++) {
                if (kFirst) t[dd] = pre[dd];
                else if (dd == 0 || dd * 1024u < a.n)
                    q80_load<RB, LPG>(t[dd], static_cast<const int8_t *>(a.w), static_cast<const float *>(a.w_aux), row0, a.rows, a.n, dd * 1024u);
            }
            auto kloop = [&](auto ord_tag) {
                constexpr bool kOrd = decltype(ord_tag)::value;
                for (uint32_t k0 = 0; k0 < a.n; k0 += D * 1024u) {
#pragma unroll
                    for (int dd = 0; dd < D; dd++) {
                        const uint32_t k = k0 + dd * 1024u;
                        if (dd == 0 || k < a.n) {
                            q80_consume<RB, LPG, kOrd>(t[dd], a.n, k, act, val);       // K ascending: the reference's group order
                            if (k + D * 1024u < a.n)
                                q80_load<RB, LPG>(t[dd], static_cast<const int8_t *>(a.w), static_cast<const float *>(a.w_aux), row0, a.rows, a.n, k + D * 1024u);
                        }
                    }
                }
            };
            if (exact) kloop(std::true_type{});
            else {
                kloop(std::false_type{});
#pragma unroll
                for (int r = 0; r < RB; r++) val[r] = warp_sum(val[r]);
            }
        } else rows_q4k<RB>(static_cast<const uint8_t *>(a.w), static_cast<const uint8_t *>(a.w_aux), row0, a.rows, a.n, act, val);

        if (EPI == EPI_SWIGLU) {
            // rows (2i, 2i+1) = (w1 row i, w3 row i); infer.c:937-944
#pragma unroll
            for (int r = 0; r + 1 < RB; r += 2) {
                const uint32_t row = row0 + r;
                if (lane == 0 && row + 1 < a.rows) {
                    const float v1 = val[r], v3 = val[r + 1];
                    const float sg = __fdiv_rn(1.0f, __fadd_rn(1.0f, exact ? expf_ref(-v1) : expf(-v1)));
                    const float hv = __fmul_rn(__fmul_rn(v1, sg), v3);
                    if (TP) tp_store(a.tp, rbase + (row >> 1), hv, out_epoch); else a.out[row >> 1] = hv;
                }
            }
        } else {
#pragma unroll
            for (int r = 0; r < RB; r++) {
                const uint32_t row = row0 + r;
                if (row >= a.rows) break;
                float v = val[r];
                if (EPI == EPI_STORE) { if (lane == 0) { if (TP) tp_store(a.tp, rbase + row, v, out_epoch); else a.out[row] = v; } }
                else if (EPI == EPI_RESID) {
                    if (lane == 0) {
                        const float xo = kFirst ? xres[r] : (TP ? __uint_as_float((uint32_t)__ldcg(out_ll + rbase + row)) : __ldcg(a.out + rbase + row));
                        if (a.lora_add) v = __fadd_rn(v, __ldcg(a.lora_add + rbase + row));       // accum(xb2, o1) precedes x += xb2
                        const float xn = __fadd_rn(xo, v);
                        if (TP) tp_store(a.tp, rbase + row, xn, out_epoch); else a.out[row] = xn;
                    }
                }
                else if (EPI == EPI_QKV) {
                    if (lane == 0) {
                        if (row < d.q_dim) a.out[row] = v;
                        else if (row < d.q_dim + d.kv_dim) a.out_k[row - d.q_dim] = v;
                        else {
                            const uint32_t c = row - d.q_dim - d.kv_dim, h = c / d.hd, i = c % d.hd;
                            a.out_v[((size_t)h * d.max_seq + pos) * d.hd + i] = v;
                        }
                    }
                } else if (EPI == EPI_CLS) {
                    // infer.c:1156-1167 penalty (division, any sign), then first-max argmax :1026-1037
                    if (pen != 1.0f && __ldcg(a.seen + rbase + row)) v = __fdiv_rn(v, pen);      // x / 1.0f == x: skip the lookup
                    if (lane == 0) a.out[rbase + row] = v;
                    if (v > bestv) { bestv = v; besti = rbase + row; }
                }
            }
        }
    };
    if (has_first) {
        if (QUANT == 0x80) do_block(gwarp, std::true_type{}); else do_block(gwarp, std::false_type{});
        for (uint32_t rb = gwarp + nwarps; rb < nblocks; rb += nwarps) do_block(rb, std::false_type{});
    }

    NB_STAMP(a.dbg, 5);
    if (EPI == EPI_CLS) {
        // rows were visited in ascending order per warp, so (bestv,besti) already holds the warp's first max
        if (lane == 0) { ms.best_v[warp] = bestv; ms.best_i[warp] = besti; }
        __syncthreads();
        if (threadIdx.x == 0) {
            float bv = ms.best_v[0]; uint32_t bi = ms.best_i[0];
            for (int w = 1; w < kWarps; w++)
                if (ms.best_v[w] > bv || (ms.best_v[w] == bv && ms.best_i[w] < bi)) { bv = ms.best_v[w]; bi = ms.best_i[w]; }
            a.cls_val[cta] = bv; a.cls_idx[cta] = bi;
        }
        __syncthreads();
    }
}

// Final argmax over the per-CTA partials + state update, by ONE full CTA.  Returns (in every thread) the token
// that the next step will consume (device loop) or the sampled token (API mode).
template <bool TP = false>
__device__ __forceinline__ uint32_t cls_finalize(const MatvecArgs &a, uint32_t ncta, MatvecSmem &ms) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float bv = -FLT_MAX; uint32_t bi = 0xffffffffu;
    for (uint32_t c = threadIdx.x; c < ncta; c += kThreads) {      // parallel fetch: a serial loop of L2 round trips costs ~40 us
        const float v = __ldcg(a.cls_val + c); const uint32_t i = __ldcg(a.cls_idx + c);
        if (i != 0xffffffffu && (v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi != 0xffffffffu && (ov > bv || (ov == bv && oi < bi))) { bv = ov; bi = oi; }
    }
    __syncthreads();
    if (lane == 0) { ms.best_v[warp] = bv; ms.best_i[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        bv = -FLT_MAX; bi = 0xffffffffu;
        for (int w = 0; w < kWarps; w++)
            if (ms.best_i[w] != 0xffffffffu && (ms.best_v[w] > bv || (ms.best_v[w] == bv && ms.best_i[w] < bi))) { bv = ms.best_v[w]; bi = ms.best_i[w]; }
        if (TP) {
            // all-gather of the per-rank (value, index) pairs through peer memory, then the same ordered pick on every rank
            const TpArgs &tp = a.tp;
            TpHdr *h = tp_hdr(tp, tp.rank);
            const uint32_t epoch = __ldcg(&h->epoch_base) + tp.nph;
            for (uint32_t p = 0; p < tp.size; p++) {
                st_relaxed_sys_u64(&tp_hdr(tp, p)->cls_v[tp.rank], tp_pack(__float_as_uint(bv), epoch));
                st_relaxed_sys_u64(&tp_hdr(tp, p)->cls_i[tp.rank], tp_pack(bi, epoch));
            }
            bv = -FLT_MAX; bi = 0xffffffffu;
            for (uint32_t r = 0; r < tp.size; r++) {
                const float v = __uint_as_float(tp_spin_load(tp, &h->cls_v[r], epoch)); const uint32_t i = tp_spin_load(tp, &h->cls_i[r], epoch);
                if (i != 0xffffffffu && (v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
            }
            h->epoch_base = epoch;
        }
        if (bi == 0xffffffffu) bi = 0;     // all-NaN row: the reference's argmax returns index 0
        DevState *st = a.st_rw;
        st->cls_ticket = 0;
        const uint32_t p = __ldcg(&st->pos);
        uint32_t nxt = bi;
        if (__ldcg(&st->advance)) {
            const uint32_t tok_in = __ldcg(a.ids + p);
            a.seen_rw[tok_in] = 1;                                  // ids[0..p] are "seen" for step p+1
            const bool forced = (p + 1 < __ldcg(&st->n_prompt));   // infer.c:1250 is_prefilling
            if (!forced) a.ids[p + 1] = bi; else nxt = __ldcg(a.ids + p + 1);
            st->pos = p + 1;
        }
        st->next_token = nxt;
        ms.flag = nxt;
    }
    __syncthreads();
    return ms.flag;
}

template <int QUANT, int EPI, int RB, int LPG, bool TP = false>
__global__ void __launch_bounds__(kThreads, 1) k_matvec(const MatvecArgs a) {
    constexpr int D = (QUANT != 0x80) ? 1 : (RB == 1) ? 4 : (RB == 2) ? 2 : 1;     // ~4 KB of weights in flight per warp
    extern __shared__ __align__(16) unsigned char act[];
    __shared__ MatvecSmem ms;
    pdl_launch_dependents();
    prefetch_row_blocks<QUANT, RB>(a.w, a.rows, a.n, blockIdx.x, gridDim.x, 4);
    pdl_wait();
    matvec_phase<QUANT, EPI, RB, LPG, TP, D, 4>(a, blockIdx.x, gridDim.x, act, ms);

    if (EPI == EPI_CLS) {
        if (threadIdx.x == 0) {
            __threadfence();
            const uint32_t t = atomicAdd(&a.st_rw->cls_ticket, 1u);
            ms.flag = (t == gridDim.x - 1) ? 1u : 0u;
        }
        __syncthreads();
        const bool last = ms.flag != 0;
        __syncthreads();
        if (last) { __threadfence(); cls_finalize<TP>(a, gridDim.x, ms); }
    }
}

// exact-mode F32 matvec: one thread per row, the reference's left-to-right sum (infer.c:645-649)
template <int EPI>
__global__ void __launch_bounds__(256) k_matvec_f32_exact(const MatvecArgs a) {
    extern __shared__ __align__(16) unsigned char act[];
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    prep_f32<256>(a.src, a.gain, a.n, true, reinterpret_cast<float *>(act), reinterpret_cast<float *>(act) + a.n, red);   // smem: 3n floats
    const float *x = reinterpret_cast<const float *>(act);
    const float *W = static_cast<const float *>(a.w);
    const Dims &d = a.d;
    const uint32_t pos = a.st ? a.st->pos : 0;
    const uint32_t nunits = (EPI == EPI_SWIGLU) ? a.rows / 2 : a.rows;
    for (uint32_t u = blockIdx.x * 256 + threadIdx.x; u < nunits; u += gridDim.x * 256) {
        const int per = (EPI == EPI_SWIGLU) ? 2 : 1;
        float res[2] = {0.0f, 0.0f};
        for (int p = 0; p < per; p++) {
            const float *wr = W + (size_t)(u * per + p) * a.n;
            float acc = 0.0f;
            for (uint32_t j = 0; j < a.n; j++) acc = __fadd_rn(acc, __fmul_rn(wr[j], x[j]));
            res[p] = acc;
        }
        const uint32_t row = u;
        if (EPI == EPI_SWIGLU) {
            const float sg = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf_ref(-res[0])));
            a.out[row] = __fmul_rn(__fmul_rn(res[0], sg), res[1]);
        } else if (EPI == EPI_STORE) a.out[row] = res[0];
        else if (EPI == EPI_RESID) a.out[row] = __fadd_rn(a.out[row], a.lora_add ? __fadd_rn(res[0], a.lora_add[row]) : res[0]);
        else if (EPI == EPI_QKV) {
            if (row < d.q_dim) a.out[row] = res[0];
            else if (row < d.q_dim + d.kv_dim) a.out_k[row - d.q_dim] = res[0];
            else {
                const uint32_t c = row - d.q_dim - d.kv_dim, h = c / d.hd, i = c % d.hd;
                a.out_v[((size_t)h * d.max_seq + pos) * d.hd + i] = res[0];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// LoRA branches (infer.c:792-808 q/k/v on the normalised fp32 activation, :898-903 o on the attention output):
//   t = A x          (rank dots of length n; fp32 `matmul`, infer.c:637-651)
//   y = (alpha/rank) (B t), then accum(base, y)      (`scale` :595, `accum` :589)
// Two small kernels per site; they run only when a plug-in is loaded (nb200_lora_load), on the multi-kernel path.
// ------------------------------------------------------------------------------------------------
struct LoraAArgs {
    const float *src; const float *gain;    // gain != nullptr: rmsnorm(src) * gain first (the q/k/v site reads xb)
    const float *A[3];                      // [rank][n] of this layer, one per branch
    uint32_t n, nmat, rank;
    float *t;                               // out [nmat][rank]
    uint32_t exact;
};
NB_K __global__ void __launch_bounds__(kThreads) k_lora_a(const LoraAArgs a) {
    extern __shared__ __align__(16) unsigned char act[];
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    float *x = reinterpret_cast<float *>(act);
    prep_f32<kThreads>(a.src, a.gain, (int)a.n, a.exact != 0, x, x + a.n, red);       // smem: 3n floats
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t u = blockIdx.x * kWarps + warp;
    if (u >= a.nmat * a.rank) return;
    const uint32_t m = u / a.rank, j = u - m * a.rank;
    const float *row = a.A[m] + (size_t)j * a.n;
    float val = 0.0f;
    if (a.exact) {
        if (lane == 0) for (uint32_t i = 0; i < a.n; i++) val = __fadd_rn(val, __fmul_rn(__ldg(row + i), x[i]));
    } else {
        for (uint32_t i = lane; i < a.n; i += 32) val = fmaf(__ldg(row + i), x[i], val);
        val = warp_sum(val);
    }
    if (lane == 0) a.t[u] = val;
}

struct LoraBArgs {
    const float *t;                         // [nmat][rank]
    const float *B[3]; uint32_t rows[3];    // [rows][rank] of this layer
    uint32_t nmat, rank;
    float scale;                            // (float)alpha / (float)rank
    float *dst[3];                          // accumulate targets (q, raw k, nullptr => V-cache row of `pos`) or the o1 buffer
    float *vcache;                          // V cache base of this layer [KV][max_seq][hd]
    uint32_t store;                         // 1: dst[0][i] = y (o site);  0: dst += y
    const DevState *st; Dims d;
};
NB_K __global__ void __launch_bounds__(256) k_lora_b(const LoraBArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    uint32_t i = blockIdx.x * 256 + threadIdx.x, m = 0;
    while (m < a.nmat && i >= a.rows[m]) { i -= a.rows[m]; m++; }
    if (m >= a.nmat) return;
    const float *row = a.B[m] + (size_t)i * a.rank, *t = a.t + m * a.rank;
    float val = 0.0f;
    for (uint32_t j = 0; j < a.rank; j++) val = __fadd_rn(val, __fmul_rn(__ldg(row + j), __ldcg(t + j)));      // matmul order, any mode
    val = __fmul_rn(val, a.scale);
    float *dst = a.dst[m];
    if (!dst) {
        const uint32_t pos = __ldcg(&a.st->pos), h = i / a.d.hd, e = i % a.d.hd;
        dst = a.vcache + ((size_t)h * a.d.max_seq + pos) * a.d.hd + e;
        i = 0;
    }
    dst[i] = a.store ? val : __fadd_rn(dst[i], val);
}

// ------------------------------------------------------------------------------------------------
// Embedding row fetch (infer.c:987-988 with the load-time dequantisation of :126-127 / :147-149)
// ------------------------------------------------------------------------------------------------
struct EmbedArgs {
    const void *w; const void *w_aux;   // same layouts as MatvecArgs (classifier/embedding table)
    float *x; const uint32_t *ids; const DevState *st; Dims d;
    uint32_t ll;                        // tensor parallel: x is a vector of {value, epoch} words (epoch unused for the local embedding)
};

NB_K __global__ void __launch_bounds__(256) k_embed(const EmbedArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const Dims &d = a.d;
    const uint32_t tok = a.st->use_token ? a.st->token : a.ids[a.st->pos];
    const uint32_t E = d.E;
    for (uint32_t i = threadIdx.x; i < E; i += 256) {
        float v;
        if (d.quant == 0x00u) v = static_cast<const float *>(a.w)[(size_t)tok * E + i];
        else if (d.quant == 0x80u) {
            const int8_t c = static_cast<const int8_t *>(a.w)[(size_t)tok * E + i];
            const float s = static_cast<const float *>(a.w_aux)[((size_t)tok * E + i) / d.gs];
            v = __fmul_rn((float)c, s);                                  // tensor.c:15-19
        } else {
            const uint32_t bpr = E / 256, blk = i >> 8, e = i & 255, g = e >> 5, j = g & 3;
            const uint8_t byte = static_cast<const uint8_t *>(a.w)[(size_t)tok * (E / 2) + (i >> 1)];
            const uint32_t c = (i & 1) ? (byte >> 4) : (byte & 0x0f);
            const uint32_t *rec = reinterpret_cast<const uint32_t *>(static_cast<const uint8_t *>(a.w_aux) + ((size_t)tok * bpr + blk) * 20);
            const float ss = __uint_as_float(rec[0]), sbi = __uint_as_float(rec[1]);
            const uint32_t bs = (rec[2] >> (8 * j)) & 0xff, bb = (rec[3] >> (8 * j)) & 0xff, bh = (rec[4] >> (8 * j)) & 0xff;
            const uint32_t s6 = (g < 4) ? (bs & 0x3f) : ((((bs >> 6) << 4) | (bh & 0x0f)) & 0x3f);
            const uint32_t b6 = (g < 4) ? (bb & 0x3f) : ((((bb >> 6) << 4) | (bh >> 4)) & 0x3f);
            v = __fsub_rn(__fmul_rn((float)c, __fmul_rn((float)s6, ss)), __fmul_rn((float)b6, sbi));   // tensor.c:274
        }
        if (a.ll) reinterpret_cast<unsigned long long *>(a.x)[i] = tp_pack(__float_as_uint(v), 0); else a.x[i] = v;
    }
}

// ------------------------------------------------------------------------------------------------
// Attention (infer.c:814-879): q/k head-norm + RoPE, split-KV partial softmax, last-CTA combine.
// KV cache layout: [L][KV][max_seq][hd] fp32 (head-major: one split reads one contiguous stream).
// ------------------------------------------------------------------------------------------------
struct AttnArgs {
    const float *q;          // raw q [q_dim]
    const float *kraw;       // raw k of this position [kv_dim]
    float *kc, *vc;          // cache bases of this layer [KV][max_seq][hd]
    const float *qnorm, *knorm;   // Qwen3 gains [hd] of this layer (nullptr otherwise)
    const float *rope_cos, *rope_sin;   // [block_size][hd/2]
    float *xba;              // out [q_dim]
    float *ws_m, *ws_l, *ws_acc;  // partials [H][nsplit_max], [H][nsplit_max], [H][nsplit_max][hd]
    uint32_t *ticket;        // [KV]
    const DevState *st;
    uint32_t nsplit_max, chunk_cap;
    Dims d;
    TpArgs tp;               // tensor parallel: xba is pushed to every rank (k_attention_fast<KVM, true>)
    unsigned long long *dbg; // optional %globaltimer stamps of kv head 0 (tools/gpu_attn_trace.py): [0..9] split 0, [16..21] merging CTA
};
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define AG_STAMP(cond, k) do { if (a.dbg && (cond) && threadIdx.x == 0) a.dbg[k] = gtime(); } while (0)

// one head vector: optional rmsnorm (Qwen3) + rope; in/out in shared memory; called by one warp
__device__ __forceinline__ void head_norm_rope(float *h, const float *__restrict__ gain, const float *__restrict__ cr,
                                               const float *__restrict__ ci, const Dims &d, bool exact) {
    const int lane = threadIdx.x & 31;
    const uint32_t hd = d.hd;
    if (d.arch == 3u) {
        float inv;
        if (!exact) {
            float acc = 0.0f;
            for (uint32_t i = lane; i < hd; i += 32) acc = fmaf(h[i], h[i], acc);
            acc = warp_sum(acc);
            inv = acc;
        } else {
            float acc = 0.0f;
            for (uint32_t i = 0; i < hd; i++) acc = __fadd_rn(acc, __fmul_rn(h[i], h[i]));
            inv = acc;
        }
        inv = __fdiv_rn(inv, (float)hd);
        inv = __fadd_rn(inv, 1e-5f);
        inv = __fdiv_rn(1.0f, __fsqrt_rn(inv));
        __syncwarp();
        for (uint32_t i = lane; i < hd; i += 32) h[i] = __fmul_rn(gain[i], __fmul_rn(inv, h[i]));
        __syncwarp();
        const uint32_t half = hd / 2;                  // infer.c:692-706
        for (uint32_t i = lane; i < half; i += 32) {
            const float c = cr[i], s = ci[i], v0 = h[i], v1 = h[i + half];
            h[i] = __fsub_rn(__fmul_rn(v0, c), __fmul_rn(v1, s));
            h[i + half] = __fadd_rn(__fmul_rn(v1, c), __fmul_rn(v0, s));
        }
    } else {                                            // infer.c:681-690
        for (uint32_t i = 2 * lane; i < hd; i += 64) {
            const float c = cr[i / 2], s = ci[i / 2], v0 = h[i], v1 = h[i + 1];
            h[i] = __fsub_rn(__fmul_rn(v0, c), __fmul_rn(v1, s));
            h[i + 1] = __fadd_rn(__fmul_rn(v0, s), __fmul_rn(v1, c));
        }
    }
    __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// Streaming (online-softmax) attention partial for one (kv head, range of positions), hd <= 128.
//   * every lane group (lpr lanes = one cache row) keeps its own running (max, sum, acc) for the KVM query heads of
//     the kv head: no score buffer, no block-wide softmax; K and V rows of a batch are requested together before any
//     is consumed (memory-level parallelism);
//   * q (and the position's k) are normalised + RoPE'd in registers by every lane group: no staging, no barriers;
//   * slots are merged with xor-shuffles inside a warp, then across warps through shared memory.
// Result (un-normalised): outp[m*(hd+2) + i] = sum_t e^{s_t - M} v_t[i],  outp[.. + hd] = M,  outp[.. + hd+1] = sum_t e^{s_t - M}.
// ------------------------------------------------------------------------------------------------
// per-warp rows of the workspace are (hd + 4) floats apart so the float4 stores stay 16-byte aligned for any hd % 4 == 0
__host__ __device__ inline uint32_t attn_stream_ws_floats(uint32_t kvm, uint32_t hd, uint32_t nwarps) { return nwarps * kvm * (hd + 4u) + kvm * (hd + 2u) + 16u; }
__host__ __device__ inline uint32_t attn_fast_smem_floats(uint32_t kvm, uint32_t hd, uint32_t chunk_cap, uint32_t nsplit_max, uint32_t nwarps) {
    (void)chunk_cap;
    uint32_t ws = attn_stream_ws_floats(kvm, hd, nwarps);
    const uint32_t merge = nsplit_max * kvm * hd;          // the merge stages all partial accumulators of a kv head over the workspace
    if (merge > ws) ws = merge;
    return ws + kvm * nsplit_max + 2u * kvm + 16u;
}

// head-norm (Qwen3) + RoPE of the float4 slice a lane holds of one head vector (infer.c:814-835); lpr lanes = one vector.
// The same arithmetic with the position's RoPE entries (and the head-norm gain) already in registers, so their loads can be
// issued together with the q / K / V loads instead of after the norm's shuffles.
struct RopeTab { float4 c, sn; };      // arch 3: cos/sin of the lane's 4 pair indices; otherwise {c0, s0, c1, s1} in c
__device__ __forceinline__ RopeTab rope_tab_load(const float *__restrict__ cr, const float *__restrict__ ci, const Dims &d, uint32_t col, bool colon) {
    RopeTab t; t.c = make_float4(0, 0, 0, 0); t.sn = make_float4(0, 0, 0, 0);
    if (colon) {
        if (d.arch == 3u) {
            const uint32_t half = d.hd / 2, i0 = (col < half) ? col : col - half;
            t.c = *reinterpret_cast<const float4 *>(cr + i0); t.sn = *reinterpret_cast<const float4 *>(ci + i0);
        } else {
            t.c = make_float4(cr[col / 2], ci[col / 2], cr[col / 2 + 1], ci[col / 2 + 1]);
        }
    }
    return t;
}
__device__ __forceinline__ float4 norm_rope_apply(float4 v, float4 gn, const RopeTab &rt, const Dims &d, uint32_t lpr, uint32_t col, bool colon) {
    if (d.arch == 3u) {
        float ss = colon ? fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, v.w * v.w))) : 0.0f;
        for (uint32_t o = lpr >> 1; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        ss = __fdiv_rn(ss, (float)d.hd);
        ss = __fadd_rn(ss, 1e-5f);
        const float inv = __fdiv_rn(1.0f, __fsqrt_rn(ss));
        if (colon) {
            v.x = __fmul_rn(gn.x, __fmul_rn(inv, v.x)); v.y = __fmul_rn(gn.y, __fmul_rn(inv, v.y));
            v.z = __fmul_rn(gn.z, __fmul_rn(inv, v.z)); v.w = __fmul_rn(gn.w, __fmul_rn(inv, v.w));
        }
        const uint32_t half = d.hd / 2, hl = lpr >> 1;
        float4 o4;
        o4.x = __shfl_xor_sync(0xffffffffu, v.x, hl); o4.y = __shfl_xor_sync(0xffffffffu, v.y, hl);
        o4.z = __shfl_xor_sync(0xffffffffu, v.z, hl); o4.w = __shfl_xor_sync(0xffffffffu, v.w, hl);
        if (colon) {
            const float4 c = rt.c, sn = rt.sn;
            if (col < half) {
                v.x = __fsub_rn(__fmul_rn(v.x, c.x), __fmul_rn(o4.x, sn.x)); v.y = __fsub_rn(__fmul_rn(v.y, c.y), __fmul_rn(o4.y, sn.y));
                v.z = __fsub_rn(__fmul_rn(v.z, c.z), __fmul_rn(o4.z, sn.z)); v.w = __fsub_rn(__fmul_rn(v.w, c.w), __fmul_rn(o4.w, sn.w));
            } else {
                v.x = __fadd_rn(__fmul_rn(v.x, c.x), __fmul_rn(o4.x, sn.x)); v.y = __fadd_rn(__fmul_rn(v.y, c.y), __fmul_rn(o4.y, sn.y));
                v.z = __fadd_rn(__fmul_rn(v.z, c.z), __fmul_rn(o4.z, sn.z)); v.w = __fadd_rn(__fmul_rn(v.w, c.w), __fmul_rn(o4.w, sn.w));
            }
        }
    } else if (colon) {
        const float c0 = rt.c.x, s0 = rt.c.y, c1 = rt.c.z, s1 = rt.c.w;
        const float x = v.x, y = v.y, z = v.z, w = v.w;
        v.x = __fsub_rn(__fmul_rn(x, c0), __fmul_rn(y, s0)); v.y = __fadd_rn(__fmul_rn(x, s0), __fmul_rn(y, c0));
        v.z = __fsub_rn(__fmul_rn(z, c1), __fmul_rn(w, s1)); v.w = __fadd_rn(__fmul_rn(z, s1), __fmul_rn(w, c1));
    }
    return v;
}

template <int KVM, int NT, bool SRC_GLOBAL>
__device__ __forceinline__ void attn_stream_partial(const Dims &d, const float *q_src, const float *kraw_src, const float *vrow_src,
                                                    float *kbase, const float *vbase, const float *qn, const float *kn,
                                                    const float *cr, const float *ci, uint32_t pos, uint32_t t0, uint32_t len,
                                                    float *ws, float *outp, unsigned long long *dbg = nullptr) {
#define AT_STAMP(k) do { if (dbg && threadIdx.x == 0) dbg[k] = clock64(); } while (0)
    constexpr int NW = NT / 32;
    constexpr int U = 4;                          // cache rows (K and V) requested per lane group before any is consumed
    AT_STAMP(0);         // cache rows (K and V) requested per lane group before any is consumed
    const uint32_t hd = d.hd;
    uint32_t lpr = 1; while (lpr * 4 < hd) lpr <<= 1;
    const uint32_t rpw = 32 / lpr;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t sub = lane / lpr, li = lane % lpr, col = li * 4;
    const bool colon = col < hd;
    const float dv = sqrtf((float)hd);              // infer.c:858 divides by sqrt(head_dim); expf as the reference (the sums stay parallel in fast mode)

    // Everything that does not depend on other loads is requested first: q, the position's RoPE entries, the head-norm
    // gain, and the warp's first batch of cache rows.  (One memory round trip instead of three or four in sequence.)
    const uint32_t stride = NW * rpw;
    float4 qv[KVM];
#pragma unroll
    for (int m = 0; m < KVM; m++) {
        qv[m] = make_float4(0, 0, 0, 0);
        if (colon) qv[m] = SRC_GLOBAL ? __ldcg(reinterpret_cast<const float4 *>(q_src + m * hd + col)) : *reinterpret_cast<const float4 *>(q_src + m * hd + col);
    }
    const RopeTab rt = rope_tab_load(cr, ci, d, col, colon);
    float4 gq = make_float4(0, 0, 0, 0);
    if (d.arch == 3u && colon) gq = *reinterpret_cast<const float4 *>(qn + col);
    // the current position's raw k / v rows and the k gain (used by the one warp whose batch contains `pos`: the split
    // that holds it is on every kv head's critical path)
    float4 kk0 = make_float4(0, 0, 0, 0), vv0 = make_float4(0, 0, 0, 0), gk = make_float4(0, 0, 0, 0);
    if (colon && t0 + len > pos) {
        kk0 = SRC_GLOBAL ? __ldcg(reinterpret_cast<const float4 *>(kraw_src + col)) : *reinterpret_cast<const float4 *>(kraw_src + col);
        vv0 = SRC_GLOBAL ? __ldcg(reinterpret_cast<const float4 *>(vrow_src + col)) : *reinterpret_cast<const float4 *>(vrow_src + col);
        if (d.arch == 3u) gk = *reinterpret_cast<const float4 *>(kn + col);
    }
    float4 kr[U], vr[U];
    auto request_batch = [&](uint32_t tb0) {
#pragma unroll
        for (int u = 0; u < U; u++) {
            const uint32_t tl = tb0 + u * stride + sub, t = t0 + tl;
            kr[u] = make_float4(0, 0, 0, 0); vr[u] = make_float4(0, 0, 0, 0);
            if (tl < len && colon && t != pos) {
                kr[u] = __ldcg(reinterpret_cast<const float4 *>(kbase + (size_t)t * hd + col));
                vr[u] = __ldcg(reinterpret_cast<const float4 *>(vbase + (size_t)t * hd + col));
            }
        }
    };
    uint32_t tb0 = warp * rpw;
    if (tb0 < len) request_batch(tb0);
#pragma unroll
    for (int m = 0; m < KVM; m++) qv[m] = norm_rope_apply(qv[m], gq, rt, d, lpr, col, colon);
    float mx[KVM], ls[KVM]; float4 av[KVM];
#pragma unroll
    for (int m = 0; m < KVM; m++) { mx[m] = -FLT_MAX; ls[m] = 0.0f; av[m] = make_float4(0, 0, 0, 0); }
    AT_STAMP(1);

    while (tb0 < len) {
        // scores of the whole batch first (independent shuffle-reductions), then ONE rescale of the running state
        float scr[U][KVM];
        bool vld[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const uint32_t tl = tb0 + u * stride + sub, t = t0 + tl;
            vld[u] = tl < len;
            // the current position's row: k is normalised + roped here (and stored for later tokens), v comes from the step's own output
            if (__any_sync(0xffffffffu, vld[u] && t == pos)) {
                const bool mine = vld[u] && t == pos;
                const float4 kk = norm_rope_apply(kk0, gk, rt, d, lpr, col, colon);      // executed by the whole warp (shuffles); only `mine` keeps it
                if (mine && colon) {
                    kr[u] = kk;
                    *reinterpret_cast<float4 *>(kbase + (size_t)pos * hd + col) = kk;
                    vr[u] = vv0;
                }
            }
#pragma unroll
            for (int m = 0; m < KVM; m++) {
                float sdot = kr[u].x * qv[m].x;
                sdot = fmaf(kr[u].y, qv[m].y, sdot); sdot = fmaf(kr[u].z, qv[m].z, sdot); sdot = fmaf(kr[u].w, qv[m].w, sdot);
                for (uint32_t o = lpr >> 1; o > 0; o >>= 1) sdot += __shfl_xor_sync(0xffffffffu, sdot, o);
                scr[u][m] = vld[u] ? __fdiv_rn(sdot, dv) : -FLT_MAX;
            }
        }
#pragma unroll
        for (int m = 0; m < KVM; m++) {
            float bm = scr[0][m];
#pragma unroll
            for (int u = 1; u < U; u++) bm = fmaxf(bm, scr[u][m]);
            const float mn = fmaxf(mx[m], bm);
            const float a = expf(mx[m] - mn);
            float l2 = ls[m] * a;
            float4 a4 = make_float4(av[m].x * a, av[m].y * a, av[m].z * a, av[m].w * a);
#pragma unroll
            for (int u = 0; u < U; u++) {
                const float pr = vld[u] ? expf(scr[u][m] - mn) : 0.0f;
                l2 += pr;
                a4.x = fmaf(pr, vr[u].x, a4.x); a4.y = fmaf(pr, vr[u].y, a4.y); a4.z = fmaf(pr, vr[u].z, a4.z); a4.w = fmaf(pr, vr[u].w, a4.w);
            }
            ls[m] = l2; av[m] = a4; mx[m] = mn;
        }
        tb0 += stride * U;
        if (tb0 < len) request_batch(tb0);
    }
    AT_STAMP(2);
    // merge the row slots of a warp
    for (uint32_t off = lpr; off < 32; off <<= 1) {
#pragma unroll
        for (int m = 0; m < KVM; m++) {
            const float mo = __shfl_xor_sync(0xffffffffu, mx[m], off), lo = __shfl_xor_sync(0xffffffffu, ls[m], off);
            float4 ao;
            ao.x = __shfl_xor_sync(0xffffffffu, av[m].x, off); ao.y = __shfl_xor_sync(0xffffffffu, av[m].y, off);
            ao.z = __shfl_xor_sync(0xffffffffu, av[m].z, off); ao.w = __shfl_xor_sync(0xffffffffu, av[m].w, off);
            const float mn = fmaxf(mx[m], mo), a = expf(mx[m] - mn), bsc = expf(mo - mn);
            ls[m] = ls[m] * a + lo * bsc;
            av[m].x = av[m].x * a + ao.x * bsc; av[m].y = av[m].y * a + ao.y * bsc;
            av[m].z = av[m].z * a + ao.z * bsc; av[m].w = av[m].w * a + ao.w * bsc;
            mx[m] = mn;
        }
    }
    if (sub == 0) {
#pragma unroll
        for (int m = 0; m < KVM; m++) {
            float *wp = ws + ((size_t)warp * KVM + m) * (hd + 4);
            if (colon) *reinterpret_cast<float4 *>(wp + col) = av[m];
            if (li == 0) { wp[hd] = mx[m]; wp[hd + 1] = ls[m]; }
        }
    }
    AT_STAMP(3);
    __syncthreads();
    AT_STAMP(4);
    // per (warp, head) weight e^{m_w - M}, computed once (slot hd+2 of the row), then a plain weighted sum per element
    if (threadIdx.x < NW * KVM) {
        const uint32_t m = threadIdx.x % KVM;
        float M = -FLT_MAX;
        for (int w = 0; w < NW; w++) M = fmaxf(M, ws[((size_t)w * KVM + m) * (hd + 4) + hd]);
        float *wp = ws + (size_t)threadIdx.x * (hd + 4);          // threadIdx.x == w * KVM + m
        wp[hd + 2] = expf(wp[hd] - M);
        wp[hd + 3] = M;
    }
    __syncthreads();
    for (uint32_t idx = threadIdx.x; idx < KVM * (hd + 2); idx += NT) {
        const uint32_t m = idx / (hd + 2), i = idx % (hd + 2);
        float r = 0.0f;
        if (i == hd) r = ws[(size_t)m * (hd + 4) + hd + 3];
        else {
#pragma unroll 4
            for (int w = 0; w < NW; w++) {
                const float *wp = ws + ((size_t)w * KVM + m) * (hd + 4);
                r = fmaf(wp[i < hd ? i : hd + 1], wp[hd + 2], r);
            }
        }
        outp[idx] = r;
    }
    __syncthreads();
    AT_STAMP(5);
#undef AT_STAMP
}

// One (kv head, split) item of the grid-wide paths: partial -> HBM workspace; the last CTA of the kv head merges.
// smem (floats): streaming workspace | wsc[KVM*nsplit_max] | stat[2*KVM]
template <int KVM, int NT, bool TP = false>
__device__ __forceinline__ void attn_item(const AttnArgs &a, uint32_t g, uint32_t split, uint32_t pos, uint32_t range, uint32_t chunk,
                                          uint32_t nsplit, float *sm, uint32_t &is_last) {
    constexpr int NW = NT / 32;
    const Dims &d = a.d;
    const uint32_t hd = d.hd;
    const uint32_t t0 = split * chunk, t1 = min(range, t0 + chunk), len = t1 - t0;
    float *ws = sm;
    float *outp = ws + (size_t)NW * KVM * (hd + 4);
    uint32_t region = NW * KVM * (hd + 4) + KVM * (hd + 2);           // the merge's staging area may be larger (attn_fast_smem_floats)
    if (a.nsplit_max * KVM * hd > region) region = a.nsplit_max * KVM * hd;
    float *wsc = sm + region;
    float *stat = wsc + KVM * a.nsplit_max;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float *cr = a.rope_cos + (size_t)pos * (hd / 2), *ci = a.rope_sin + (size_t)pos * (hd / 2);
    float *kbase = a.kc + (size_t)g * d.max_seq * hd, *vbase = a.vc + (size_t)g * d.max_seq * hd;
    const bool tr = (g == 0 && split == 0);
    AG_STAMP(tr, 2);
    attn_stream_partial<KVM, NT, true>(d, a.q + (size_t)g * KVM * hd, a.kraw + (size_t)g * hd, vbase + (size_t)pos * hd, kbase, vbase,
                                       a.qnorm, a.knorm, cr, ci, pos, t0, len, ws, outp);
    AG_STAMP(tr, 3);
    for (uint32_t idx = threadIdx.x; idx < KVM * hd; idx += NT) {
        const uint32_t m = idx / hd, i = idx % hd;
        a.ws_acc[((size_t)(g * KVM + m) * a.nsplit_max + split) * hd + i] = outp[m * (hd + 2) + i];
    }
    if (threadIdx.x < KVM) {
        const size_t slot = (size_t)(g * KVM + threadIdx.x) * a.nsplit_max + split;
        a.ws_m[slot] = outp[threadIdx.x * (hd + 2) + hd]; a.ws_l[slot] = outp[threadIdx.x * (hd + 2) + hd + 1];
    }
    __syncthreads();
    AG_STAMP(tr, 4);
    if (threadIdx.x == 0) {
        __threadfence();
        const uint32_t t = atomicAdd(a.ticket + g, 1u);
        is_last = (t == nsplit - 1) ? 1u : 0u;
    }
    __syncthreads();
    AG_STAMP(tr, 5);
    if (!is_last) return;      // uniform across the CTA
    __threadfence();
    AG_STAMP(g == 0, 16);
    // ---- merge.  Every load of the partials is issued before any is consumed (one L2 round trip instead of one per
    // unrolled group): the accumulators go to shared memory `macc` (it reuses the streaming workspace), the per-split
    // maxima / sums to registers; then warp m computes exp(m_s - M) and L for its head, and all threads combine in the
    // fixed split order. ----
    float *macc = sm;                                   // [KVM][nsplit][hd]: per head the source is one contiguous run
    {
        const uint32_t run4 = nsplit * hd / 4;           // float4 per head
        constexpr int B = 4;
        for (uint32_t e0 = threadIdx.x; e0 < KVM * run4; e0 += NT * B) {
            float4 v[B];
#pragma unroll
            for (int u = 0; u < B; u++) {
                const uint32_t e = e0 + u * NT;
                if (e < KVM * run4) {
                    const uint32_t m = e / run4, j = e - m * run4;
                    v[u] = __ldcg(reinterpret_cast<const float4 *>(a.ws_acc + (size_t)(g * KVM + m) * a.nsplit_max * hd) + j);
                }
            }
#pragma unroll
            for (int u = 0; u < B; u++) { const uint32_t e = e0 + u * NT; if (e < KVM * run4) reinterpret_cast<float4 *>(macc)[e] = v[u]; }
        }
    }
    if (warp < KVM) {
        const size_t base = (size_t)(g * KVM + warp) * a.nsplit_max;
        float pm[2], pl[2];                              // nsplit_max <= 64: two slots per lane
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const uint32_t s2 = lane + 32 * k;
            pm[k] = (s2 < nsplit) ? __ldcg(a.ws_m + base + s2) : -FLT_MAX;
            pl[k] = (s2 < nsplit) ? __ldcg(a.ws_l + base + s2) : 0.0f;
        }
        const float M = warp_max(fmaxf(pm[0], pm[1]));
        float L = 0.0f;
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const uint32_t s2 = lane + 32 * k;
            if (s2 < nsplit) { const float w = expf(pm[k] - M); wsc[warp * a.nsplit_max + s2] = w; L += pl[k] * w; }
        }
        L = warp_sum(L);
        if (lane == 0) stat[2 * warp] = L;
    }
    __syncthreads();
    AG_STAMP(g == 0, 17);
    uint32_t out_epoch = 0;
    if (TP) out_epoch = tp_epoch(a.tp, a.tp.signal_ph);
    for (uint32_t idx = threadIdx.x; idx < KVM * hd; idx += NT) {
        const uint32_t m = idx / hd, i = idx % hd;
        float o = 0.0f;
#pragma unroll 4
        for (uint32_t s2 = 0; s2 < nsplit; s2++) o = fmaf(macc[(m * nsplit + s2) * hd + i], wsc[m * a.nsplit_max + s2], o);
        const float ov = __fdiv_rn(o, stat[2 * m]);
        if (TP) tp_store(a.tp, a.tp.row_base + (g * KVM + m) * hd + i, ov, out_epoch); else a.xba[(size_t)(g * KVM + m) * hd + i] = ov;
    }
    if (threadIdx.x == 0) a.ticket[g] = 0;
    AG_STAMP(g == 0, 18);
}

template <int KVM, bool TP = false>
__global__ void __launch_bounds__(kThreads) k_attention_fast(const AttnArgs a) {      // same CTA shape as the megakernel => same bits
    extern __shared__ __align__(16) float sm[];
    __shared__ uint32_t is_last;
    pdl_launch_dependents();
    AG_STAMP(blockIdx.x == 0 && blockIdx.y == 0, 0);
    pdl_wait();
    const Dims &d = a.d;
    const uint32_t pos = __ldcg(&a.st->pos);
    const uint32_t range = __ldcg(&a.st->is_causal) ? pos + 1 : d.max_seq;
    AG_STAMP(blockIdx.x == 0 && blockIdx.y == 0, 1);
    uint32_t chunk = (range + a.nsplit_max - 1) / a.nsplit_max;
    chunk = max(chunk, 32u);
    chunk = min((chunk + 7u) & ~7u, a.chunk_cap);
    const uint32_t nsplit = (range + chunk - 1) / chunk;
    if (blockIdx.x >= nsplit) return;
    attn_item<KVM, kThreads, TP>(a, blockIdx.y, blockIdx.x, pos, range, chunk, nsplit, sm, is_last);
}

NB_K __global__ void __launch_bounds__(kAttnThreads) k_attention(const AttnArgs a) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float red[32];
    __shared__ uint32_t is_last;
    pdl_launch_dependents();
    pdl_wait();

    const Dims &d = a.d;
    const bool exact = d.exact != 0;
    const uint32_t hd = d.hd, kvm = d.kv_mul;
    const uint32_t g = blockIdx.y, split = blockIdx.x;
    const uint32_t pos = a.st->pos;
    const uint32_t range = a.st->is_causal ? pos + 1 : d.max_seq;
    uint32_t chunk = (range + a.nsplit_max - 1) / a.nsplit_max;
    chunk = max(chunk, 32u);
    chunk = min((chunk + 7u) & ~7u, a.chunk_cap);
    const uint32_t nsplit = (range + chunk - 1) / chunk;
    if (split >= nsplit) return;
    const uint32_t t0 = split * chunk, t1 = min(range, t0 + chunk), len = t1 - t0;
    const bool owner = (pos >= t0 && pos < t1);

    // smem carve-up
    float *qs = sm;                          // [kvm][hd]
    float *krow = qs + kvm * hd;             // [hd]
    float *sc = krow + hd;                   // [chunk_cap]
    float *part = sc + a.chunk_cap;          // [kAttnWarps * rows_per_warp][hd]

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float *cr = a.rope_cos + (size_t)pos * (hd / 2), *ci = a.rope_sin + (size_t)pos * (hd / 2);

    for (uint32_t i = threadIdx.x; i < kvm * hd; i += kAttnThreads) qs[i] = a.q[(size_t)g * kvm * hd + i];
    if (owner) for (uint32_t i = threadIdx.x; i < hd; i += kAttnThreads) krow[i] = a.kraw[(size_t)g * hd + i];
    __syncthreads();
    for (uint32_t m = warp; m < kvm + (owner ? 1u : 0u); m += kAttnWarps) {
        if (m < kvm) head_norm_rope(qs + m * hd, a.qnorm, cr, ci, d, exact);
        else head_norm_rope(krow, a.knorm, cr, ci, d, exact);
    }
    __syncthreads();
    float *kbase = a.kc + (size_t)g * d.max_seq * hd, *vbase = a.vc + (size_t)g * d.max_seq * hd;
    if (owner) for (uint32_t i = threadIdx.x; i < hd; i += kAttnThreads) kbase[(size_t)pos * hd + i] = krow[i];

    // lanes per cache row: smallest power of two >= hd/4 (float4 per lane)
    uint32_t lpr = 1; while (lpr * 4 < hd) lpr <<= 1; if (lpr > 32) lpr = 32;
    const uint32_t rpw = 32 / lpr;                      // rows per warp-iteration
    const uint32_t sub = lane / lpr, li = lane % lpr;
    const float inv_div = sqrtf((float)hd);

    for (uint32_t m = 0; m < kvm; m++) {
        const uint32_t h = g * kvm + m;
        const float *qh = qs + m * hd;
        // ---- scores ----
        for (uint32_t tb = warp * rpw; tb < len; tb += kAttnWarps * rpw) {
            const uint32_t tl = tb + sub;
            float acc = 0.0f;
            if (tl < len) {
                const uint32_t t = t0 + tl;
                const float *kr = (t == pos) ? krow : kbase + (size_t)t * hd;
                for (uint32_t c = li * 4; c < hd; c += lpr * 4) {
                    const float4 kv = *reinterpret_cast<const float4 *>(kr + c);
                    const float4 qv = *reinterpret_cast<const float4 *>(qh + c);
                    acc = fmaf(kv.x, qv.x, acc); acc = fmaf(kv.y, qv.y, acc);
                    acc = fmaf(kv.z, qv.z, acc); acc = fmaf(kv.w, qv.w, acc);
                }
            }
            for (uint32_t o = lpr >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (tl < len && li == 0) sc[tl] = __fdiv_rn(acc, inv_div);
        }
        __syncthreads();
        // ---- local softmax statistics ----
        float mx = -FLT_MAX;
        for (uint32_t t = threadIdx.x; t < len; t += kAttnThreads) mx = fmaxf(mx, sc[t]);
        mx = block_max<kAttnThreads>(mx, red);
        float lsum = 0.0f;
        for (uint32_t t = threadIdx.x; t < len; t += kAttnThreads) { const float e = expf(sc[t] - mx); sc[t] = e; lsum += e; }
        lsum = block_sum<kAttnThreads>(lsum, red);
        // ---- weighted V ----
        float4 av[4];                                   // hd <= 512 : up to 4 float4 per lane at lpr = 32
#pragma unroll
        for (int c = 0; c < 4; c++) av[c] = make_float4(0, 0, 0, 0);
        for (uint32_t tb = warp * rpw; tb < len; tb += kAttnWarps * rpw) {
            const uint32_t tl = tb + sub;
            if (tl < len) {
                const float e = sc[tl];
                const float *vr = vbase + (size_t)(t0 + tl) * hd;
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const uint32_t col = (li + c * lpr) * 4;
                    if (col < hd) {
                        const float4 vv = *reinterpret_cast<const float4 *>(vr + col);
                        av[c].x = fmaf(e, vv.x, av[c].x); av[c].y = fmaf(e, vv.y, av[c].y);
                        av[c].z = fmaf(e, vv.z, av[c].z); av[c].w = fmaf(e, vv.w, av[c].w);
                    }
                }
            }
        }
        float *mypart = part + (size_t)(warp * rpw + sub) * hd;
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const uint32_t col = (li + c * lpr) * 4;
            if (col < hd) *reinterpret_cast<float4 *>(mypart + col) = av[c];
        }
        __syncthreads();
        const size_t slot = (size_t)h * a.nsplit_max + split;
        for (uint32_t i = threadIdx.x; i < hd; i += kAttnThreads) {
            float s = 0.0f;
            for (uint32_t p = 0; p < kAttnWarps * rpw; p++) s += part[(size_t)p * hd + i];
            a.ws_acc[slot * hd + i] = s;
        }
        if (threadIdx.x == 0) { a.ws_m[slot] = mx; a.ws_l[slot] = lsum; }
        __syncthreads();
    }

    // ---- last CTA of this kv head merges the splits ----
    if (threadIdx.x == 0) {
        __threadfence();
        const uint32_t t = atomicAdd(a.ticket + g, 1u);
        is_last = (t == nsplit - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    for (uint32_t m = 0; m < kvm; m++) {
        const uint32_t h = g * kvm + m;
        float M = -FLT_MAX;
        for (uint32_t s = 0; s < nsplit; s++) M = fmaxf(M, __ldcg(a.ws_m + (size_t)h * a.nsplit_max + s));
        float Lsum = 0.0f;
        for (uint32_t s = 0; s < nsplit; s++) {
            const size_t slot = (size_t)h * a.nsplit_max + s;
            Lsum += __ldcg(a.ws_l + slot) * expf(__ldcg(a.ws_m + slot) - M);
        }
        for (uint32_t i = threadIdx.x; i < hd; i += kAttnThreads) {
            float o = 0.0f;
            for (uint32_t s = 0; s < nsplit; s++) {
                const size_t slot = (size_t)h * a.nsplit_max + s;
                o += __ldcg(a.ws_acc + slot * hd + i) * expf(__ldcg(a.ws_m + slot) - M);
            }
            a.xba[(size_t)h * hd + i] = __fdiv_rn(o, Lsum);
        }
    }
    if (threadIdx.x == 0) a.ticket[g] = 0;
}

// exact-mode attention: one CTA per q head, the reference's loop order (infer.c:841-879).
// att: [H][max_seq] scratch in HBM.
struct AttnExactArgs {
    const float *q, *kraw; float *kc, *vc; const float *qnorm, *knorm, *rope_cos, *rope_sin;
    float *xba; float *att; const DevState *st; Dims d;
};

NB_K __global__ void __launch_bounds__(kAttnThreads) k_attention_exact(const AttnExactArgs a) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float red[32];
    pdl_launch_dependents();
    pdl_wait();
    const Dims &d = a.d;
    const uint32_t hd = d.hd, h = blockIdx.x, g = h / d.kv_mul;
    const uint32_t pos = a.st->pos;
    const uint32_t range = a.st->is_causal ? pos + 1 : d.max_seq;
    float *qs = sm, *krow = sm + hd;
    const int warp = threadIdx.x >> 5;
    const float *cr = a.rope_cos + (size_t)pos * (hd / 2), *ci = a.rope_sin + (size_t)pos * (hd / 2);
    for (uint32_t i = threadIdx.x; i < hd; i += kAttnThreads) { qs[i] = a.q[(size_t)h * hd + i]; krow[i] = a.kraw[(size_t)g * hd + i]; }
    __syncthreads();
    if (warp == 0) head_norm_rope(qs, a.qnorm, cr, ci, d, true);
    if (warp == 1) head_norm_rope(krow, a.knorm, cr, ci, d, true);
    __syncthreads();
    float *kbase = a.kc + (size_t)g * d.max_seq * hd, *vbase = a.vc + (size_t)g * d.max_seq * hd;
    if (h % d.kv_mul == 0) for (uint32_t i = threadIdx.x; i < hd; i += kAttnThreads) kbase[(size_t)pos * hd + i] = krow[i];
    float *att = a.att + (size_t)h * d.max_seq;
    const float dv = sqrtf((float)hd);
    for (uint32_t t = threadIdx.x; t < range; t += kAttnThreads) {
        const float *kr = (t == pos) ? krow : kbase + (size_t)t * hd;
        float s = 0.0f;
        for (uint32_t i = 0; i < hd; i++) s = __fadd_rn(s, __fmul_rn(qs[i], kr[i]));
        att[t] = __fdiv_rn(s, dv);
    }
    __syncthreads();
    float mx = -FLT_MAX;
    for (uint32_t t = threadIdx.x; t < range; t += kAttnThreads) mx = fmaxf(mx, att[t]);
    mx = block_max<kAttnThreads>(mx, red);
    for (uint32_t t = threadIdx.x; t < range; t += kAttnThreads) att[t] = expf_ref(__fsub_rn(att[t], mx));
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.0f;
        for (uint32_t t = 0; t < range; t++) s = __fadd_rn(s, att[t]);
        red[0] = s;
    }
    __syncthreads();
    const float total = red[0];
    for (uint32_t t = threadIdx.x; t < range; t += kAttnThreads) att[t] = __fdiv_rn(att[t], total);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < hd; i += kAttnThreads) {
        float o = 0.0f;
        for (uint32_t t = 0; t < range; t++) {
            const float v = vbase[(size_t)t * hd + i];
            o = __fadd_rn(o, __fmul_rn(att[t], v));
        }
        a.xba[(size_t)h * hd + i] = o;
    }
}

// penalty + first-max argmax + state update over logits already in HBM (exact-mode F32 classifier)
struct FinalizeArgs { float *logits; uint32_t V; const uint8_t *seen; uint8_t *seen_rw; uint32_t *ids; DevState *st; };

NB_K __global__ void __launch_bounds__(1024) k_cls_finalize(const FinalizeArgs a) {
    float *logits = a.logits; const uint32_t V = a.V; const uint8_t *seen = a.seen; uint8_t *seen_rw = a.seen_rw;
    uint32_t *ids = a.ids; DevState *st = a.st;
    __shared__ float bvs[32];
    __shared__ uint32_t bis[32];
    pdl_launch_dependents();
    pdl_wait();
    const float pen = st->penalty;
    float bv = -FLT_MAX; uint32_t bi = 0xffffffffu;
    for (uint32_t i = threadIdx.x; i < V; i += 1024) {
        float v = logits[i];
        if (seen[i]) { v = __fdiv_rn(v, pen); logits[i] = v; }
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
        if (bi == 0xffffffffu) bi = 0;
        const uint32_t p = st->pos;
        if (st->advance) {
            const uint32_t tok_in = ids[p];
            seen_rw[tok_in] = 1;
            const bool forced = (p + 1 < st->n_prompt);
            if (!forced) ids[p + 1] = bi;
            st->next_token = forced ? ids[p + 1] : bi;
            st->pos = p + 1;
        } else st->next_token = bi;
    }
}

// marks seen[ids[i]] for i in [lo, hi) (repetition-penalty bookkeeping in API mode)
NB_K __global__ void k_mark_seen(uint8_t *seen, const uint32_t *ids, uint32_t lo, uint32_t hi) {
    for (uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += gridDim.x * blockDim.x) seen[ids[i]] = 1;
}

// standalone prep kernels for the op-level C-ABI (same device functions as the fused prologues)
NB_K __global__ void __launch_bounds__(kThreads) k_op_prep(const float *src, const float *gain, uint32_t n, uint32_t gs, uint32_t quant,
                                                     uint32_t exact, float *out_f32, int8_t *dump_codes, float *dump_scales) {
    extern __shared__ __align__(16) unsigned char act[];
    __shared__ float red[32];
    float *stage = reinterpret_cast<float *>(act + act_region_bytes(quant, n, gs ? gs : 1));
    if (quant == 0x00u) {
        prep_f32<kThreads>(src, gain, n, exact != 0, reinterpret_cast<float *>(act), stage, red);
        for (uint32_t i = threadIdx.x; i < n; i += kThreads) out_f32[i] = reinterpret_cast<float *>(act)[i];
    } else if (quant == 0x80u) prep_q80<kThreads>(src, gain, n, gs, exact != 0, act, stage, red, dump_codes, dump_scales);
    else prep_q4k<kThreads>(src, gain, n, exact != 0, act, stage, red, dump_codes, dump_scales);
}

// helpers shared with the persistent streaming kernel (stream.cuh)
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int *p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// embedding row -> x (infer.c:987-988 + load-time dequantisation), by one CTA
template <int NT>
__device__ __forceinline__ void embed_row(const void *w, const void *aux, float *x, uint32_t tok, const Dims &d) {
    const uint32_t E = d.E;
    for (uint32_t i = threadIdx.x; i < E; i += NT) {
        float v;
        if (d.quant == 0x00u) v = __ldg(static_cast<const float *>(w) + (size_t)tok * E + i);
        else if (d.quant == 0x80u) {
            const int8_t c = __ldg(static_cast<const int8_t *>(w) + (size_t)tok * E + i);
            const float s = __ldg(static_cast<const float *>(aux) + ((size_t)tok * E + i) / d.gs);
            v = __fmul_rn((float)c, s);                                  // tensor.c:15-19
        } else {
            const uint32_t bpr = E / 256, blk = i >> 8, e = i & 255, g = e >> 5, j = g & 3;
            const uint8_t byte = __ldg(static_cast<const uint8_t *>(w) + (size_t)tok * (E / 2) + (i >> 1));
            const uint32_t c = (i & 1) ? (byte >> 4) : (byte & 0x0f);
            const uint32_t *rec = reinterpret_cast<const uint32_t *>(static_cast<const uint8_t *>(aux) + ((size_t)tok * bpr + blk) * 20);
            const float ss = __uint_as_float(__ldg(rec)), sbi = __uint_as_float(__ldg(rec + 1));
            const uint32_t bs = (__ldg(rec + 2) >> (8 * j)) & 0xff, bb = (__ldg(rec + 3) >> (8 * j)) & 0xff, bh = (__ldg(rec + 4) >> (8 * j)) & 0xff;
            const uint32_t s6 = (g < 4) ? (bs & 0x3f) : ((((bs >> 6) << 4) | (bh & 0x0f)) & 0x3f);
            const uint32_t b6 = (g < 4) ? (bb & 0x3f) : ((((bb >> 6) << 4) | (bh >> 4)) & 0x3f);
            v = __fsub_rn(__fmul_rn((float)c, __fmul_rn((float)s6, ss)), __fmul_rn((float)b6, sbi));   // tensor.c:274
        }
        x[i] = v;
    }
}

}  // namespace nb
