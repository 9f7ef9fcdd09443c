// sample.cu -- temperature / top-p sampling on the device (SURVEY 8(f3)).
//
// Reference: generate_next_token, temperature > 0 branch (infer/infer.c:1170-1189): logits /= temperature, softmax (:616-634),
// coin = random_f32 (utils.c:959-970, drawn by the host shim from the Sampler's xorshift state), sample_top_p (:1062-1109).
// Everything that decides the sampled id is reproduced operation by operation:
//   * division by the temperature, max, expf (the glibc-equivalent expf_ref), the SEQUENTIAL sum of the exponentials in index order,
//     the division by that sum -- bit-identical probabilities whenever the logits are (exact mode);
//   * the cutoff filter; candidates sorted by probability, descending, ties in index order -- what glibc's stable (merge-sort) qsort
//     gives the reference -- with a stable LSD radix sort (cub::DeviceRadixSort; rejected entries carry the key -1 and sort last);
//   * the sequential cumulative sum up to top_p and the sequential CDF walk with r = coin * cumulative.
// Only the sampled id (and the six most probable ids, for the observation hook) leave the device: 32 bytes instead of V * 4.
#define NB_K static
#include <cub/device/device_radix_sort.cuh>

#include "kernels.cuh"
#include "sample_host.h"

namespace nb {

constexpr int kSampThreads = 1024;
constexpr int kSampChunk = 4096;       // floats staged in shared memory per step of a sequential scan

// pass 1: y = logit / T, max; p = expf(y - max); sequential sum; p /= sum; key = p >= cutoff ? p : -1; out[7] = n0 = #candidates,
// out[8] = the first index of the largest p
__global__ void __launch_bounds__(kSampThreads) k_sample_prepare(const float *__restrict__ logits, uint32_t V, float temperature, float top_p,
                                                                 float *keys, uint32_t *vals, uint32_t *out) {
    __shared__ float red[32];
    __shared__ float chunk[kSampChunk];
    __shared__ float s_total;
    __shared__ uint32_t s_cnt, s_best[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float mx = -FLT_MAX;
    for (uint32_t i = threadIdx.x; i < V; i += kSampThreads) {
        const float y = __fdiv_rn(logits[i], temperature);           // infer.c:1172-1174
        keys[i] = y;
        mx = fmaxf(mx, y);
    }
    mx = block_max<kSampThreads>(mx, red);
    for (uint32_t i = threadIdx.x; i < V; i += kSampThreads) keys[i] = expf_ref(__fsub_rn(keys[i], mx));      // infer.c:627
    __syncthreads();
    // sum += x[i] in index order (infer.c:628): staged through shared memory, added by one thread
    float total = 0.0f;
    for (uint32_t c0 = 0; c0 < V; c0 += kSampChunk) {
        const uint32_t n = min((uint32_t)kSampChunk, V - c0);
        for (uint32_t i = threadIdx.x; i < n; i += kSampThreads) chunk[i] = keys[c0 + i];
        __syncthreads();
        if (threadIdx.x == 0) {
#pragma unroll 8
            for (uint32_t i = 0; i < n; i++) total = __fadd_rn(total, chunk[i]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { s_total = total; s_cnt = 0; }
    __syncthreads();
    total = s_total;
    const float cutoff = __fdiv_rn(__fsub_rn(1.0f, top_p), (float)(int)(V - 1));        // infer.c:1064
    uint32_t cnt = 0;
    float bp = -1.0f;                 // first-max argmax of the probabilities: the pick when no candidate passes the cutoff
    uint32_t bi = 0;
    for (uint32_t i = threadIdx.x; i < V; i += kSampThreads) {
        const float p = __fdiv_rn(keys[i], total);                   // infer.c:632
        const bool in = p >= cutoff;
        keys[i] = in ? p : -1.0f;
        vals[i] = i;
        cnt += in ? 1u : 0u;
        if (p > bp) { bp = p; bi = i; }                              // ascending i per thread: the thread's first max
    }
    for (int o = 16; o > 0; o >>= 1) {
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        const float op = __shfl_xor_sync(0xffffffffu, bp, o);
        const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (op > bp || (op == bp && oi < bi)) { bp = op; bi = oi; }
    }
    if (lane == 0) { red[warp] = bp; s_best[warp] = bi; }
    if (lane == 0 && cnt) atomicAdd(&s_cnt, cnt);
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kSampThreads / 32; w++)
            if (red[w] > bp || (red[w] == bp && s_best[w] < bi)) { bp = red[w]; bi = s_best[w]; }
        out[7] = s_cnt;
        out[8] = bi;
    }
}

// pass 2 (after the sort): cumulative sum to top_p, then the CDF walk (infer.c:1076-1106), both sequential
__global__ void __launch_bounds__(256) k_sample_pick(const float *__restrict__ keys, const uint32_t *__restrict__ vals, float top_p, float coin,
                                                     uint32_t *out, DevState *st) {
    __shared__ float chunk[kSampChunk];
    __shared__ uint32_t s_stop, s_last;
    __shared__ float s_cum;
    const uint32_t n0 = out[7];
    if (n0 == 0) {
        // No probability reaches the cutoff (top_p < 1/V over a near-flat distribution).  The reference then reads
        // probindex[-1] (undefined); this sampler returns the first-max argmax of the probabilities and six zero ids.
        if (threadIdx.x == 0) {
            const uint32_t tok = out[8];
            out[0] = tok;
            for (uint32_t i = 0; i < 6; i++) out[1 + i] = 0u;
            if (st) st->next_token = tok;
        }
        return;
    }
    if (threadIdx.x == 0) { s_stop = 0; s_last = n0 - 1; s_cum = 0.0f; }
    __syncthreads();
    float cum = 0.0f;
    for (uint32_t c0 = 0; c0 < n0 && !s_stop; c0 += kSampChunk) {
        const uint32_t n = min((uint32_t)kSampChunk, n0 - c0);
        for (uint32_t i = threadIdx.x; i < n; i += 256) chunk[i] = keys[c0 + i];
        __syncthreads();
        if (threadIdx.x == 0) {
            for (uint32_t i = 0; i < n; i++) {
                cum = __fadd_rn(cum, chunk[i]);
                if (cum > top_p) { s_last = c0 + i; s_stop = 1; break; }
            }
            s_cum = cum;
        }
        __syncthreads();
    }
    const uint32_t last = s_last;
    const float r = __fmul_rn(coin, s_cum);
    __syncthreads();                  // every warp has read s_stop in its loop test before it is cleared for the CDF walk
    if (threadIdx.x == 0) s_stop = 0;
    __syncthreads();
    float cdf = 0.0f;
    uint32_t pick = last;
    for (uint32_t c0 = 0; c0 <= last && !s_stop; c0 += kSampChunk) {
        const uint32_t n = min((uint32_t)kSampChunk, last + 1 - c0);
        for (uint32_t i = threadIdx.x; i < n; i += 256) chunk[i] = keys[c0 + i];
        __syncthreads();
        if (threadIdx.x == 0) {
            for (uint32_t i = 0; i < n; i++) {
                cdf = __fadd_rn(cdf, chunk[i]);
                if (r < cdf) { pick = c0 + i; s_stop = 1; break; }
            }
            s_last = pick;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const uint32_t tok = vals[s_stop ? s_last : last];
        out[0] = tok;
        for (uint32_t i = 0; i < 6; i++) out[1 + i] = (n0 > i) ? vals[i] : 0u;        // the observation hook's token_0..5 (infer.c:1086-1096)
        if (st) st->next_token = tok;
    }
}

// The workspace: keys and values in and out (V words each, 256-byte aligned), the sort's temporary storage, then the result
// words {token, top-6 ids, n0, first-max index} in the last 256 bytes.
struct SampleWorkspace {
    float *keys_in, *keys_out;
    uint32_t *vals_in, *vals_out;
    void *tmp;
    uint32_t *out;
};

static inline SampleWorkspace sample_workspace(void *workspace, uint32_t V, size_t cub_bytes) {
    const size_t a = ((size_t)V * 4 + 255) & ~(size_t)255;
    unsigned char *w = static_cast<unsigned char *>(workspace);
    return {reinterpret_cast<float *>(w), reinterpret_cast<float *>(w + a), reinterpret_cast<uint32_t *>(w + 2 * a),
            reinterpret_cast<uint32_t *>(w + 3 * a), w + 4 * a, reinterpret_cast<uint32_t *>(w + 4 * a + ((cub_bytes + 255) & ~(size_t)255))};
}

size_t sample_workspace_bytes(uint32_t V, size_t *cub_bytes) {
    size_t tmp = 0;
    cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp, (const float *)nullptr, (float *)nullptr, (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)V);
    if (cub_bytes) *cub_bytes = tmp;
    const size_t a = ((size_t)V * 4 + 255) & ~(size_t)255;
    return 4 * a + ((tmp + 255) & ~(size_t)255) + 256;
}

cudaError_t sample_top_p_launch(void *workspace, size_t cub_bytes, const float *logits, uint32_t V, float temperature, float top_p, float coin,
                                DevState *st, uint32_t **out_dev, cudaStream_t stream) {
    const SampleWorkspace w = sample_workspace(workspace, V, cub_bytes);
    k_sample_prepare<<<1, kSampThreads, 0, stream>>>(logits, V, temperature, top_p, w.keys_in, w.vals_in, w.out);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t tb = cub_bytes;
    e = cub::DeviceRadixSort::SortPairsDescending(w.tmp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, (int)V, 0, 32, stream);
    if (e != cudaSuccess) return e;
    k_sample_pick<<<1, 256, 0, stream>>>(w.keys_out, w.vals_out, top_p, coin, w.out, st);
    *out_dev = w.out;
    return cudaGetLastError();
}

}  // namespace nb
