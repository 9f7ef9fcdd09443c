// Microbenchmark: cost of grid-barrier variants (one CTA per SM x 512 threads, cooperative launch; flags sized for up to 148 SMs).
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ unsigned ld_acq(const unsigned *p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_rlx(const unsigned *p) { unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_vol(const unsigned *p) { unsigned v; asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }

template <int V>
__device__ __forceinline__ void bar(unsigned *ctr, unsigned &target, unsigned ncta, unsigned *flags, unsigned *go) {
    __syncthreads();
    if (V == 4) {   // two-level flags: each CTA stores its epoch; CTA 0's threads poll them; then a go flag
        target += 1;
        if (threadIdx.x == 0) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flags + blockIdx.x * 32), "r"(target) : "memory"); }
        if (blockIdx.x == 0) {
            if (threadIdx.x < ncta) while (ld_acq(flags + threadIdx.x * 32) < target) { }
            __syncthreads();
            if (threadIdx.x == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(go), "r"(target) : "memory");
        } else if (threadIdx.x == 0) {
            while (ld_acq(go) < target) { }
        }
        __syncthreads();
        return;
    }
    if (threadIdx.x == 0) {
        target += ncta;
        if (V == 0) { asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory"); while (ld_acq(ctr) < target) { } }
        if (V == 1) { __threadfence(); atomicAdd(ctr, 1u); while (ld_vol(ctr) < target) { } __threadfence(); }
        if (V == 2) { asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory"); while (ld_rlx(ctr) < target) { } }
        if (V == 3) { asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory"); while (ld_rlx(ctr) < target) { } asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
    }
    __syncthreads();
}

template <int V, int STORES>
__global__ void __launch_bounds__(512, 1) k(unsigned *ctr, unsigned *flags, unsigned *go, float *buf, long long *out, int iters) {
    unsigned target = 0;
    long long t0 = 0;
    for (int i = 0; i < iters + 10; i++) {
        if (i == 10) t0 = clock64();
        if (STORES) buf[(size_t)blockIdx.x * 512 + threadIdx.x] = (float)i;
        bar<V>(ctr, target, gridDim.x, flags, go);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) out[0] = (clock64() - t0) / iters;
}

template <int V, int STORES>
int run(const char *name, unsigned *ctr, unsigned *flags, unsigned *go, float *buf, long long *out, int ncta) {
    int iters = 2000;
    CK(cudaMemset(ctr, 0, 4)); CK(cudaMemset(flags, 0, 148 * 128)); CK(cudaMemset(go, 0, 4));
    void *args[] = {&ctr, &flags, &go, &buf, &out, &iters};
    CK(cudaLaunchCooperativeKernel((const void *)k<V, STORES>, dim3(ncta), dim3(512), args, 0, 0));
    CK(cudaDeviceSynchronize());
    long long h; CK(cudaMemcpy(&h, out, 8, cudaMemcpyDeviceToHost));
    printf("%-52s stores=%d  ncta=%d : %lld cycles/barrier\n", name, STORES, ncta, h);
    return 0;
}

int main() {
    unsigned *ctr, *flags, *go; float *buf; long long *out;
    CK(cudaMalloc(&ctr, 256)); CK(cudaMalloc(&flags, 148 * 128)); CK(cudaMalloc(&go, 256)); CK(cudaMalloc(&buf, 148 * 512 * 4)); CK(cudaMalloc(&out, 64));
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    for (int ncta : {sms, sms / 2, 8}) {
        run<0, 0>("red.release + ld.acquire poll", ctr, flags, go, buf, out, ncta);
        run<0, 1>("red.release + ld.acquire poll", ctr, flags, go, buf, out, ncta);
        run<1, 1>("threadfence + atomicAdd + ld.volatile + threadfence", ctr, flags, go, buf, out, ncta);
        run<2, 1>("relaxed red + relaxed poll (no ordering: floor)", ctr, flags, go, buf, out, ncta);
        run<3, 1>("red.release + relaxed poll + one fence.acq_rel", ctr, flags, go, buf, out, ncta);
        run<4, 1>("per-CTA flags (st.release) + master poll + go flag", ctr, flags, go, buf, out, ncta);
    }
    return 0;
}
