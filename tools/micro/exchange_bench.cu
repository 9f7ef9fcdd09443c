// Microbenchmark: the bare activation-exchange protocol of k_decode_stream.  One CTA per SM x 480 threads; per round every CTA publishes
// its share of an n-element vector as {value, epoch} words into R replicas (st.relaxed.gpu), then all its threads poll the words
// of their slot in "their" replica until the round's epoch has arrived (ld.relaxed.gpu.v2.u64 x 2), bar.sync, next round.
// Reports cycles per round = the floor of a decode phase with no arithmetic at all.
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)
__device__ __forceinline__ void ld2(const unsigned long long *p, unsigned long long &a, unsigned long long &b) {
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void st1(unsigned long long *p, unsigned long long v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__global__ void __launch_bounds__(512, 1) k_xchg(unsigned long long *buf, uint32_t n, uint32_t R, uint32_t rs, int rounds, int sleep_ns, int pollers, long long *out) {
    if (threadIdx.x >= 480) return;
    const uint32_t cta = blockIdx.x, ncta = gridDim.x;
    const uint32_t r0 = (uint32_t)((uint64_t)cta * n / ncta), r1 = (uint32_t)((uint64_t)(cta + 1) * n / ncta);
    const unsigned long long *mine = buf + (size_t)(cta % R) * rs;
    const uint32_t i = threadIdx.x * 4;          // this thread's slot (n <= 1920)
    long long t0 = 0;
    for (int it = 0; it < rounds + 5; it++) {
        if (it == 5) t0 = clock64();
        const uint32_t epoch = (uint32_t)it + 1;
        // publish: warp w's lanes 0..R-1 write element r0 + w to the R replicas
        const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (uint32_t e = r0 + w; e < r1; e += 15) if (lane < R) st1(buf + (size_t)lane * rs + e, ((unsigned long long)epoch << 32) | e);
        // poll
        if (i < n && (int)threadIdx.x < pollers) {
            unsigned long long a, b, c, d;
            for (uint32_t j = i; j < n; j += (uint32_t)pollers * 4) {       // pollers < 480: fewer threads cover the whole vector
                for (;;) {
                    ld2(mine + j, a, b); ld2(mine + j + 2, c, d);
                    if ((uint32_t)(a >> 32) >= epoch && (uint32_t)(b >> 32) >= epoch && (uint32_t)(c >> 32) >= epoch && (uint32_t)(d >> 32) >= epoch) break;       // >=: a fast CTA may already have published the next round
                    if (sleep_ns) __nanosleep(sleep_ns);
                }
            }
        }
        asm volatile("bar.sync 1, 480;" ::: "memory");
    }
    if (cta == 0 && threadIdx.x == 0) out[0] = (clock64() - t0) / rounds;
}
int main() {
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    unsigned long long *buf; long long *out;
    CK(cudaMalloc(&buf, 8 * 4096 * 8)); CK(cudaMalloc(&out, 64));
    for (uint32_t n : {768u, 1920u})
        for (uint32_t R : {1u, 4u, 8u})
            for (int sl : {0, 50})
                for (int pollers : {480, 64}) {
                    CK(cudaMemset(buf, 0, 8 * 4096 * 8));
                    uint32_t rs = 4096; int rounds = 2000;
                    void *args[] = {&buf, &n, &R, &rs, &rounds, &sl, &pollers, &out};
                    CK(cudaLaunchCooperativeKernel((const void *)k_xchg, dim3(sms), dim3(512), args, 0, 0));
                    CK(cudaDeviceSynchronize());
                    long long h; CK(cudaMemcpy(&h, out, 8, cudaMemcpyDeviceToHost));
                    printf("n=%4u replicas=%u poll back-off %3d ns, %3d polling threads/CTA: %6lld cycles per exchange round\n", n, R, sl, pollers, h);
                }
    return 0;
}
