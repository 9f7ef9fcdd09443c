// row_dot_probe.cu -- test harness for the row dots of both decode paths, one row at a time.
//
// Streaming kernel (stream.cuh): one CTA of the kernel's shape (512 threads; warps 0-14 consume) runs st_prep<QUANT, LPG>
// on an fp32 vector held in shared memory, so the operand region is the prologue's own, then lays R weight rows out as ring
// tiles (row_stride = row bytes + 16, aux_stride as setup_stream computes it; the 16 pad bytes of a row and the pad of its
// aux record are filled with 0x5a, so a dot that reads past its row is wrong) and runs one of
//   form 0: st_row_q80_lpg<LPG>           with a given (lg2, gteam) lane geometry, rows spread over lane teams as st_consume's
//                                          shared tiles do; every lane of a team must hold the same bits;
//   form 1: st_rows_q80_warp<LPG, RB>     rows [0, shift) and the tail one at a time, the rest in blocks of RB (owned tiles);
//   form 2: st_row_q4k, form 3: st_row_f32 one warp per row.
// Multi-kernel path (kernels.cuh): a probe kernel copies an operand region built by the caller to shared memory and runs,
// per warp-owned block of RB rows, the row loops of matvec_phase: q80_load + q80_consume<RB, LPG, ORD> (+ warp_sum when
// !ORD), rows_f32<RB> or rows_q4k<RB>, with weights in global memory.
// Both write one fp32 per row.  Built by tests/test_row_dots.py with nvcc from the repository's headers.
#define NB_K static
#include "stream.cuh"

using namespace nb;

namespace {

constexpr uint32_t kEpoch = 0x5eedu;
constexpr unsigned char kPad = 0x5a;
constexpr uint32_t kSmemMax = 227u * 1024u;

__device__ __forceinline__ void check_same(float v, uint32_t src, bool on, uint32_t *mismatch) {
    const float v0 = __shfl_sync(0xffffffffu, v, src);
    if (on && __float_as_uint(v) != __float_as_uint(v0)) atomicAdd(mismatch, 1u);
}

template <int QUANT, int LPG, int RB>
__global__ void __launch_bounds__(kThreads, 1) k_stream_dots(const float *x, uint32_t n, const unsigned char *wmain, uint32_t main_b,
                                                             const unsigned char *waux, uint32_t aux_b, uint32_t R, uint32_t T,
                                                             uint32_t row_stride, uint32_t aux_stride, uint32_t act_bytes, uint32_t tile_off,
                                                             int form, uint32_t lg2, uint32_t gteam, uint32_t shift,
                                                             float *out, unsigned char *act_out, uint32_t *mismatch, uint32_t *err) {
    extern __shared__ __align__(128) unsigned char sm[];
    __shared__ __align__(16) StreamArgs sg;
    __shared__ float red[kWarps];
    for (uint32_t i = threadIdx.x; i < sizeof(StreamArgs) / 4; i += kThreads) reinterpret_cast<uint32_t *>(&sg)[i] = 0u;
    __syncthreads();
    if (threadIdx.x == 0) sg.err = err;
    float *ssrc = reinterpret_cast<float *>(sm + tile_off);        // the tiles reuse the source's space once the prologue is done
    for (uint32_t i = threadIdx.x; i < n; i += kThreads) ssrc[i] = x[i];
    __syncthreads();
    if (threadIdx.x >= (uint32_t)kConsThreads) return;
    st_prep<QUANT, LPG>(sg, nullptr, ssrc, kEpoch, nullptr, n, sm, red, nullptr);     // ends with a consumer barrier
    const unsigned char *act = sm;
    for (uint32_t i = threadIdx.x; i < act_bytes; i += kConsThreads) act_out[i] = act[i];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    unsigned char *tile = sm + tile_off;
    for (uint32_t t0 = 0; t0 < R; t0 += T) {
        const uint32_t tr = min(T, R - t0);
        const uint32_t tile_b = tr * (row_stride + aux_stride);
        cbar();
        for (uint32_t i = threadIdx.x; i < tile_b + 16u; i += kConsThreads) tile[i] = kPad;
        cbar();
        for (uint32_t i = threadIdx.x; i < tr * main_b; i += kConsThreads)
            tile[(i / main_b) * row_stride + i % main_b] = wmain[(size_t)t0 * main_b + i];
        for (uint32_t i = threadIdx.x; i < tr * aux_b; i += kConsThreads)
            tile[tr * row_stride + (i / aux_b) * aux_stride + i % aux_b] = waux[(size_t)t0 * aux_b + i];
        cbar();
        const unsigned char *aux = tile + (size_t)tr * row_stride;
        if constexpr (QUANT == 0x80) {
            if (form == 0) {
                // st_consume's shared tiles: a team of gteam * lg2 lanes per row, rw rows per warp pass
                const uint32_t TS = gteam * lg2, RW = 32u / TS;
                const uint32_t tm = lane / TS, team = tm < RW ? tm : RW - 1u, tl = lane % TS, gl = tl / lg2, ul = tl % lg2;
                const bool lane_on = lane < RW * TS;
                for (uint32_t rb = warp * RW; rb < tr; rb += kConsWarps * RW) {
                    const uint32_t rr = rb + team, rc = rr < tr ? rr : tr - 1u;
                    const float v = st_row_q80_lpg<LPG>(tile + (size_t)rc * row_stride, reinterpret_cast<const float *>(aux + (size_t)rc * aux_stride),
                                                        n, act, lg2, gteam, gl, ul, team * TS);
                    check_same(v, team * TS, lane_on && rr < tr, mismatch);
                    if (lane_on && rr < tr && tl == 0) out[t0 + rc] = v;
                }
            } else {
                // st_consume's owned tiles: whole-warp rows, one at a time before `shift` and at the tail, else in blocks of RB
                uint32_t r = 0, u = 0;
                auto single = [&](uint32_t r1) {
                    float v[1];
                    st_rows_q80_warp<LPG, 1>(tile + (size_t)r1 * row_stride, row_stride, aux + (size_t)r1 * aux_stride, aux_stride, n, act, v);
                    check_same(v[0], 0u, true, mismatch);
                    if (lane == 0) out[t0 + r1] = v[0];
                };
                for (; r < tr && r < shift; r++, u++) if (u % kConsWarps == warp) single(r);
                for (; r + RB <= tr; r += RB, u++) {
                    if (u % kConsWarps != warp) continue;
                    float v[RB];
                    st_rows_q80_warp<LPG, RB>(tile + (size_t)r * row_stride, row_stride, aux + (size_t)r * aux_stride, aux_stride, n, act, v);
#pragma unroll
                    for (int q = 0; q < RB; q++) {
                        check_same(v[q], 0u, true, mismatch);
                        if (lane == 0) out[t0 + r + q] = v[q];
                    }
                }
                for (; r < tr; r++, u++) if (u % kConsWarps == warp) single(r);
            }
        } else {
            for (uint32_t r = warp; r < tr; r += kConsWarps) {
                float v;
                if constexpr (QUANT == 0x42) v = st_row_q4k(tile + (size_t)r * row_stride, aux + (size_t)r * aux_stride, n, act);
                else v = st_row_f32(tile + (size_t)r * row_stride, n, act);
                check_same(v, 0u, true, mismatch);
                if (lane == 0) out[t0 + r] = v;
            }
        }
    }
}

template <int QUANT, int LPG, int RB>
cudaError_t launch_stream(const float *x, uint32_t n, const unsigned char *wm, uint32_t main_b, const unsigned char *wa, uint32_t aux_b,
                          uint32_t R, uint32_t T, uint32_t rs, uint32_t as, uint32_t act_bytes, uint32_t tile_off, uint32_t smem,
                          int form, uint32_t lg2, uint32_t gteam, uint32_t shift, float *out, unsigned char *act_out, uint32_t *mm, uint32_t *err) {
    cudaError_t e = cudaFuncSetAttribute((const void *)k_stream_dots<QUANT, LPG, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k_stream_dots<QUANT, LPG, RB><<<1, kThreads, smem>>>(x, n, wm, main_b, wa, aux_b, R, T, rs, as, act_bytes, tile_off, form, lg2, gteam, shift,
                                                         out, act_out, mm, err);
    return cudaGetLastError();
}

template <int QUANT, int RB, int LPG, bool ORD>
__global__ void __launch_bounds__(kThreads, 1) k_mk_dots(const void *w, const void *w_aux, uint32_t rows, uint32_t n,
                                                         const unsigned char *act_in, uint32_t act_bytes, float *out, uint32_t *mismatch) {
    extern __shared__ __align__(16) unsigned char act[];
    for (uint32_t i = threadIdx.x; i < act_bytes; i += kThreads) act[i] = act_in[i];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t nblocks = (rows + RB - 1) / RB, nwarps = gridDim.x * kWarps;
    for (uint32_t rb = blockIdx.x * kWarps + (threadIdx.x >> 5); rb < nblocks; rb += nwarps) {
        const uint32_t row0 = rb * RB;
        float val[RB];
        if constexpr (QUANT == 0x00) rows_f32<RB>(static_cast<const float *>(w), row0, rows, n, act, val);
        else if constexpr (QUANT == 0x42) rows_q4k<RB>(static_cast<const uint8_t *>(w), static_cast<const uint8_t *>(w_aux), row0, rows, n, act, val);
        else {
            // matvec_phase's K loop (the tiles it keeps in flight do not change the order of the consumes)
#pragma unroll
            for (int r = 0; r < RB; r++) val[r] = 0.0f;
            for (uint32_t k0 = 0; k0 < n; k0 += 1024u) {
                Q80Tile<RB> t;
                q80_load<RB, LPG>(t, static_cast<const int8_t *>(w), static_cast<const float *>(w_aux), row0, rows, n, k0);
                q80_consume<RB, LPG, ORD>(t, n, k0, act, val);
            }
            if (!ORD) {
#pragma unroll
                for (int r = 0; r < RB; r++) val[r] = warp_sum(val[r]);
            }
        }
#pragma unroll
        for (int r = 0; r < RB; r++) {
            check_same(val[r], 0u, true, mismatch);
            if (lane == 0 && row0 + r < rows) out[row0 + r] = val[r];
        }
    }
}

template <int QUANT, int RB, int LPG, bool ORD>
cudaError_t launch_mk(const void *w, const void *wa, uint32_t rows, uint32_t n, const unsigned char *act, uint32_t act_bytes, float *out, uint32_t *mm) {
    const uint32_t smem = (act_bytes + 127u) & ~127u;
    cudaError_t e = cudaFuncSetAttribute((const void *)k_mk_dots<QUANT, RB, LPG, ORD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const uint32_t nblocks = (rows + RB - 1) / RB, grid = (nblocks + kWarps - 1) / kWarps < 4u ? (nblocks + kWarps - 1) / kWarps : 4u;
    k_mk_dots<QUANT, RB, LPG, ORD><<<grid, kThreads, smem>>>(w, wa, rows, n, act, act_bytes, out, mm);
    return cudaGetLastError();
}

struct Dev {           // device copies of the probe's buffers, freed on every path
    void *p[8] = {};
    int k = 0;
    template <class T> cudaError_t put(T *&d, const void *h, size_t bytes) {
        cudaError_t e = cudaMalloc((void **)&d, bytes ? bytes : 16);
        if (e != cudaSuccess) return e;
        p[k++] = (void *)d;
        return h ? cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice) : cudaMemset(d, 0, bytes ? bytes : 16);
    }
    ~Dev() { for (int i = 0; i < k; i++) cudaFree(p[i]); }
};

}  // namespace

// Streaming-kernel row dots.  quant 0x80 (lpg 4 or 8), 0x42 or 0x00 (lpg 8); form as above (0 / 1 for Q80; 2 for Q4K,
// 3 for F32); rb 1, 2 or 4 (form 1).  x: the fp32 vector given to st_prep (no gain).  wmain: R rows of main_b bytes (Q80
// codes, Q4K nibble plane, F32 values), waux: R rows of aux_b bytes (Q80 scales, Q4K 20-byte side records).  tile_rows:
// rows per ring tile (0: as many as fit).  out: R floats; act_out: the operand region (act_region_bytes); *mismatch: rows
// whose value differs between the lanes meant to hold it.  Returns 0, a CUDA error code, or -1 for arguments the probe
// does not take.
extern "C" int probe_stream_dots(int quant, int lpg, int form, int rb, uint32_t lg2, uint32_t gteam, uint32_t shift, uint32_t tile_rows,
                                 const float *x, uint32_t n, const unsigned char *wmain, uint32_t main_b, const unsigned char *waux,
                                 uint32_t aux_b, uint32_t R, float *out, unsigned char *act_out, uint32_t act_cap, uint32_t *mismatch) {
    const uint32_t gs = quant == 0x80 ? (uint32_t)lpg * 16u : 1u;
    const uint32_t act_bytes = act_region_bytes((uint32_t)quant, n, gs);
    if (n == 0 || R == 0 || n > st_prep_max_n((uint32_t)quant, gs) || act_cap < act_bytes) return -1;
    if ((quant == 0x80 && (n % gs || (form != 0 && form != 1))) || (quant == 0x42 && (n % 256u || form != 2)) ||
        (quant == 0x00 && (n % 4u || form != 3)))
        return -1;
    const uint32_t want_main = quant == 0x80 ? n : quant == 0x42 ? n / 2u : n * 4u;
    const uint32_t want_aux = quant == 0x80 ? (n / gs) * 4u : quant == 0x42 ? (n / 256u) * 20u : 0u;
    if (main_b != want_main || aux_b != want_aux) return -1;
    const uint32_t row_stride = main_b + 16u;                                             // setup_stream's strides
    const uint32_t aux_stride = quant == 0x80 ? ((n / gs) | 1u) * 4u : aux_b;
    const uint32_t tile_off = (act_bytes + 127u) & ~127u;
    if (tile_off + 16u + row_stride + aux_stride > kSmemMax) return -1;
    const uint32_t fit = (kSmemMax - tile_off - 16u) / (row_stride + aux_stride);
    const uint32_t T = tile_rows ? tile_rows : (fit < R ? fit : R);
    if (T > fit) return -1;
    uint32_t need = T * (row_stride + aux_stride) + 16u;
    if (need < n * 4u) need = n * 4u;
    const uint32_t smem = tile_off + ((need + 127u) & ~127u);
    if (smem > kSmemMax) return -1;
    Dev dv;
    float *dx, *dout; unsigned char *dm, *da, *dact; uint32_t *dmm, *derr;
    cudaError_t e = dv.put(dx, x, n * 4ull);
    if (e == cudaSuccess) e = dv.put(dm, wmain, (size_t)R * main_b);
    if (e == cudaSuccess) e = dv.put(da, waux, (size_t)R * aux_b);
    if (e == cudaSuccess) e = dv.put(dout, nullptr, R * 4ull);
    if (e == cudaSuccess) e = dv.put(dact, nullptr, act_bytes);
    if (e == cudaSuccess) e = dv.put(dmm, nullptr, 4);
    if (e == cudaSuccess) e = dv.put(derr, nullptr, 4);
    if (e != cudaSuccess) return (int)e;
#define NB_ST(Q, L, B) launch_stream<Q, L, B>(dx, n, dm, main_b, da, aux_b, R, T, row_stride, aux_stride, act_bytes, tile_off, smem, form, lg2, gteam, shift, dout, dact, dmm, derr)
    if (quant == 0x80 && lpg == 8 && rb == 1) e = NB_ST(0x80, 8, 1);
    else if (quant == 0x80 && lpg == 8 && rb == 2) e = NB_ST(0x80, 8, 2);
    else if (quant == 0x80 && lpg == 8 && rb == 4) e = NB_ST(0x80, 8, 4);
    else if (quant == 0x80 && lpg == 4 && rb == 1) e = NB_ST(0x80, 4, 1);
    else if (quant == 0x80 && lpg == 4 && rb == 2) e = NB_ST(0x80, 4, 2);
    else if (quant == 0x80 && lpg == 4 && rb == 4) e = NB_ST(0x80, 4, 4);
    else if (quant == 0x42 && lpg == 8) e = NB_ST(0x42, 8, 1);
    else if (quant == 0x00 && lpg == 8) e = NB_ST(0x00, 8, 1);
    else return -1;
#undef NB_ST
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, R * 4ull, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(act_out, dact, act_bytes, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(mismatch, dmm, 4, cudaMemcpyDeviceToHost);
    return (int)e;
}

// Multi-kernel row dots.  quant 0x80 (lpg 2, 4, 8 or 16; ordered: q80_consume's ORD), 0x00 or 0x42 (lpg and ordered
// ignored); rb 1, 2 or 4.  w / w_aux: the matrix as the engine holds it (Q80 codes [rows][n] + scales [rows][n/gs]; F32
// [rows][n]; Q4K nibble plane [rows][n/2] + side records [rows][n/256][20]).  act: the operand region (act_region_bytes).
extern "C" int probe_mk_dots(int quant, int lpg, int ordered, int rb, const void *w, uint64_t w_bytes, const void *w_aux, uint64_t aux_bytes,
                             uint32_t rows, uint32_t n, const unsigned char *act, uint32_t act_bytes, float *out, uint32_t *mismatch) {
    const uint32_t gs = quant == 0x80 ? (uint32_t)lpg * 16u : 1u;
    if (rows == 0 || n == 0 || act_bytes != act_region_bytes((uint32_t)quant, n, gs) || act_bytes > kSmemMax) return -1;
    if ((quant == 0x80 && n % gs) || (quant == 0x42 && n % 256u) || (quant == 0x00 && n % 4u)) return -1;
    Dev dv;
    unsigned char *dw, *da, *dact; float *dout; uint32_t *dmm;
    cudaError_t e = dv.put(dw, w, w_bytes);
    if (e == cudaSuccess) e = dv.put(da, w_aux, aux_bytes);
    if (e == cudaSuccess) e = dv.put(dact, act, act_bytes);
    if (e == cudaSuccess) e = dv.put(dout, nullptr, rows * 4ull);
    if (e == cudaSuccess) e = dv.put(dmm, nullptr, 4);
    if (e != cudaSuccess) return (int)e;
#define NB_MK(Q, B, L, O) launch_mk<Q, B, L, O>(dw, da, rows, n, dact, act_bytes, dout, dmm)
#define NB_MK_RB(Q, L, O) (rb == 1 ? NB_MK(Q, 1, L, O) : rb == 2 ? NB_MK(Q, 2, L, O) : NB_MK(Q, 4, L, O))
#define NB_MK_ORD(L) (ordered ? NB_MK_RB(0x80, L, true) : NB_MK_RB(0x80, L, false))
    if (rb != 1 && rb != 2 && rb != 4) return -1;
    if (quant == 0x80 && lpg == 2) e = NB_MK_ORD(2);
    else if (quant == 0x80 && lpg == 4) e = NB_MK_ORD(4);
    else if (quant == 0x80 && lpg == 8) e = NB_MK_ORD(8);
    else if (quant == 0x80 && lpg == 16) e = NB_MK_ORD(16);
    else if (quant == 0x00) e = NB_MK_RB(0x00, 8, false);
    else if (quant == 0x42) e = NB_MK_RB(0x42, 8, false);
    else return -1;
#undef NB_MK_ORD
#undef NB_MK_RB
#undef NB_MK
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, rows * 4ull, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(mismatch, dmm, 4, cudaMemcpyDeviceToHost);
    return (int)e;
}
