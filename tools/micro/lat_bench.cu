// Microbenchmark: the latencies the persistent decode kernel is made of, measured on an otherwise idle GPU and with
// all other SMs polling L2 (the situation inside a grid barrier).
//   * dependent ld.global.cg / ld.relaxed.gpu / ld.acquire.gpu chain through an L2-resident buffer (cycles per load)
//   * st.global + fence (membar.gl) drain time, atomicAdd round trip
//   * cp.async.bulk of 8 KB: issue -> mbarrier completion, source in L2 and in HBM
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ unsigned ld_cg(const unsigned *p) { unsigned v; asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_rlx(const unsigned *p) { unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_acq(const unsigned *p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// out[0..]: results of CTA 0; other CTAs (if any) poll `noise` until told to stop
__global__ void __launch_bounds__(512, 1) k_lat(unsigned *chain, unsigned nchain, unsigned *scratch, unsigned *noise, volatile unsigned *stop,
                                                const unsigned char *bulk_src, long long *out) {
    __shared__ __align__(128) unsigned char buf[16384];
    __shared__ uint64_t mbar;
    if (blockIdx.x != 0) {
        if (threadIdx.x == 0) { while (!*stop) { (void)ld_rlx(noise); } }
        return;
    }
    if (threadIdx.x == 0) {
        const int N = 256;
        unsigned idx = 0;
        for (int i = 0; i < 64; i++) idx = ld_cg(chain + idx);           // warm (into L2)
        long long t0 = clock64();
        for (int i = 0; i < N; i++) idx = ld_cg(chain + idx);
        out[0] = (clock64() - t0) / N;
        t0 = clock64();
        for (int i = 0; i < N; i++) idx = ld_rlx(chain + idx);
        out[1] = (clock64() - t0) / N;
        t0 = clock64();
        for (int i = 0; i < N; i++) idx = ld_acq(chain + idx);
        out[2] = (clock64() - t0) / N;
        // store + fence
        t0 = clock64();
        for (int i = 0; i < N; i++) { scratch[(i * 97) & 4095] = idx + i; __threadfence(); }
        out[3] = (clock64() - t0) / N;
        // atomic round trip
        unsigned a = 0;
        t0 = clock64();
        for (int i = 0; i < N; i++) a += atomicAdd(scratch + 8192 + ((a + i) & 1023), 1u);
        out[4] = (clock64() - t0) / N;
        // red.release (fence + fire-and-forget atomic) after one store
        t0 = clock64();
        for (int i = 0; i < N; i++) { scratch[(i * 97) & 4095] = idx + i; asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(scratch + 16384) : "memory"); }
        out[5] = (clock64() - t0) / N;
        // bulk copy latency, 8 KB
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&mbar)) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        unsigned par = 0;
        for (int rep = 0; rep < 2; rep++) {        // rep 0: source far apart (HBM, cold), rep 1: same 8 KB again and again (L2)
            long long acc = 0;
            for (int i = 0; i < 64; i++) {
                const unsigned char *src = bulk_src + (rep == 0 ? (size_t)i * (1u << 20) : 0);
                t0 = clock64();
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&mbar)), "r"(8192u) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_u32(buf)), "l"(src), "r"(8192u), "r"(smem_u32(&mbar)) : "memory");
                unsigned ok = 0;
                while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(&mbar)), "r"(par) : "memory");
                acc += clock64() - t0;
                par ^= 1u;
            }
            out[6 + rep] = acc / 64;
        }
        out[15] = idx + a + buf[0];
        *stop = 1;
        __threadfence();
    }
}

int main() {
    unsigned *chain, *scratch, *noise, *stop; unsigned char *bulk; long long *out;
    const unsigned nchain = 1u << 18;      // 1 MB of indices: L2-resident, far beyond L1
    CK(cudaMalloc(&chain, nchain * 4)); CK(cudaMalloc(&scratch, 1 << 20)); CK(cudaMalloc(&noise, 256)); CK(cudaMalloc(&stop, 256));
    CK(cudaMalloc(&bulk, 128u << 20)); CK(cudaMalloc(&out, 256));
    CK(cudaMemset(bulk, 1, 128u << 20)); CK(cudaMemset(scratch, 0, 1 << 20)); CK(cudaMemset(noise, 0, 256));
    unsigned *h = (unsigned *)malloc(nchain * 4);
    for (unsigned i = 0; i < nchain; i++) h[i] = (unsigned)(((unsigned long long)i * 40503u + 12345u) % nchain);   // scattered, 4-byte stride jumps >> 128 B
    CK(cudaMemcpy(chain, h, nchain * 4, cudaMemcpyHostToDevice));
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const char *names[8] = {"ld.global.cg chain", "ld.relaxed.gpu chain", "ld.acquire.gpu chain", "st + __threadfence", "atomicAdd round trip",
                            "st + red.release.gpu", "bulk 8 KB from HBM (issue->complete)", "bulk 8 KB from L2 (issue->complete)"};
    for (int ncta : {1, sms}) {
        CK(cudaMemset(stop, 0, 256));
        void *args[] = {&chain, (void *)&nchain, &scratch, &noise, &stop, &bulk, &out};
        CK(cudaLaunchCooperativeKernel((const void *)k_lat, dim3(ncta), dim3(512), args, 0, 0));
        CK(cudaDeviceSynchronize());
        long long r[16]; CK(cudaMemcpy(r, out, 128, cudaMemcpyDeviceToHost));
        for (int i = 0; i < 8; i++) printf("ncta=%3d  %-40s %6lld cycles\n", ncta, names[i], r[i]);
    }
    return 0;
}
