// stream_prep_probe.cu -- test harness for the streaming kernel's activation prologue (st_prep, stream.cuh) on its own.
//
// The prologue keeps what it produces (Q80 codes + scales, Q4K nibble codes + group records, F32 normalised values) in
// shared memory, where no engine entry point can read it.  Here one CTA of the kernel's shape (512 threads; warps 0-14
// are the consumers, warp 15 only takes part in the set-up) runs st_prep<QUANT, LPG> on a vector given either as exchange
// words or in shared memory, and copies the operand region (layout: act_region_bytes, kernels.cuh) to global memory.
// Every exchange word carries the awaited epoch before the launch, so no poll ever waits.
// Built by tests/test_stream_prep_probe.py with nvcc from the repository's headers.
#define NB_K static
#include "stream.cuh"

using namespace nb;

namespace {

constexpr uint32_t kEpoch = 0x5eedu;

template <int QUANT, int LPG>
__global__ void __launch_bounds__(kThreads, 1) k_prep_probe(const unsigned long long *xw, const float *xs, const float *gain, uint32_t n,
                                                            uint32_t act_bytes, uint32_t src_off, unsigned char *out, uint32_t *err) {
    extern __shared__ __align__(128) unsigned char sm[];
    __shared__ __align__(16) StreamArgs sg;
    __shared__ float red[kWarps];
    for (uint32_t i = threadIdx.x; i < sizeof(StreamArgs) / 4; i += kThreads) reinterpret_cast<uint32_t *>(&sg)[i] = 0u;
    __syncthreads();
    if (threadIdx.x == 0) sg.err = err;
    float *ssrc = xs ? reinterpret_cast<float *>(sm + src_off) : nullptr;
    if (ssrc)
        for (uint32_t i = threadIdx.x; i < n; i += kThreads) ssrc[i] = xs[i];
    __syncthreads();
    if (threadIdx.x >= (uint32_t)kConsThreads) return;       // the producer warp has no part in the prologue
    st_prep<QUANT, LPG>(sg, ssrc ? nullptr : xw, ssrc, kEpoch, gain, n, sm, red, nullptr);
    for (uint32_t i = threadIdx.x; i < act_bytes; i += kConsThreads) out[i] = sm[i];
}

template <int QUANT, int LPG>
cudaError_t launch(const unsigned long long *xw, const float *xs, const float *gain, uint32_t n, uint32_t act_bytes, uint32_t src_off,
                   uint32_t smem, unsigned char *out, uint32_t *err) {
    cudaError_t e = cudaFuncSetAttribute((const void *)k_prep_probe<QUANT, LPG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k_prep_probe<QUANT, LPG><<<1, kThreads, smem>>>(xw, xs, gain, n, act_bytes, src_off, out, err);
    return cudaGetLastError();
}

}  // namespace

// quant 0x80 (lpg 8: groups of 128, lpg 4: groups of 64), 0x00 or 0x42; shared_src: the vector is read from shared memory
// instead of exchange words; gain may be null (no rmsnorm).  out receives act_region_bytes(quant, n, gs) bytes.
// Returns 0, or a CUDA error code, or -1 for arguments the prologue does not take.
extern "C" int probe_prep(int quant, int lpg, int shared_src, const float *x, const float *gain, uint32_t n, unsigned char *out, uint32_t out_bytes) {
    const uint32_t gs = quant == 0x80 ? (uint32_t)lpg * 16u : 1u;
    const uint32_t act_bytes = act_region_bytes((uint32_t)quant, n, gs);
    if (n == 0 || n > st_prep_max_n((uint32_t)quant, gs) || out_bytes < act_bytes) return -1;
    if ((quant == 0x80 && n % gs) || (quant == 0x42 && n % 256u) || (quant == 0x00 && n % 4u)) return -1;
    const uint32_t nw = (n + 3u) & ~3u;
    unsigned long long *hw = (unsigned long long *)malloc(nw * 8ull);
    for (uint32_t i = 0; i < nw; i++) {
        uint32_t bits = 0;
        if (i < n) memcpy(&bits, x + i, 4);
        hw[i] = ((unsigned long long)kEpoch << 32) | bits;
    }
    unsigned long long *dw = nullptr; float *dx = nullptr, *dg = nullptr; unsigned char *dout = nullptr; uint32_t *derr = nullptr;
    cudaError_t e = cudaMalloc(&dw, nw * 8ull);
    if (e == cudaSuccess) e = cudaMalloc(&dx, nw * 4ull);
    if (e == cudaSuccess && gain) e = cudaMalloc(&dg, nw * 4ull);
    if (e == cudaSuccess) e = cudaMalloc(&dout, act_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&derr, 4);
    if (e == cudaSuccess) e = cudaMemcpy(dw, hw, nw * 8ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(dx, x, n * 4ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && gain) e = cudaMemcpy(dg, gain, n * 4ull, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(derr, 0, 4);
    const uint32_t src_off = (act_bytes + 127u) & ~127u, smem = src_off + ((n * 4u + 127u) & ~127u);
    if (e == cudaSuccess) {
        const float *xs = shared_src ? dx : nullptr;
        if (quant == 0x80 && lpg == 8) e = launch<0x80, 8>(dw, xs, dg, n, act_bytes, src_off, smem, dout, derr);
        else if (quant == 0x80 && lpg == 4) e = launch<0x80, 4>(dw, xs, dg, n, act_bytes, src_off, smem, dout, derr);
        else if (quant == 0x00) e = launch<0x00, 8>(dw, xs, dg, n, act_bytes, src_off, smem, dout, derr);
        else if (quant == 0x42) e = launch<0x42, 8>(dw, xs, dg, n, act_bytes, src_off, smem, dout, derr);
        else e = cudaErrorInvalidValue;
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out, dout, act_bytes, cudaMemcpyDeviceToHost);
    cudaFree(dw); cudaFree(dx); cudaFree(dg); cudaFree(dout); cudaFree(derr);
    free(hw);
    return e == cudaSuccess ? 0 : (int)e;
}
