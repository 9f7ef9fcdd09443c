// Microbenchmark: how long do the short dependent instruction chains of a decode phase take when nothing else runs?
// One CTA of 480 threads (the consumer warps of k_decode_stream), hot instruction cache, data in shared memory.
//   A: block reduce for the rmsnorm inverse (warp_sum + smem + named barrier + 15 adds + div/sqrt/div)
//   B: Q80 quantise of one 128-element group per warp (amax shuffles, scale, 4 codes per lane, pack)
//   C: Q80 row dot by an 8-lane team, 6 / 16 groups (LDS.128 x2, 4 dp4a, 3 shuffles, ordered fp32 sum)
//   D: 4-word poll of ready data in L2 (ld.relaxed.gpu.v2.u64 x2 + epoch check)
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, 480;" ::: "memory"); }
static __device__ __noinline__ int q80_code_slow(float v, float sc) { return (int)roundf(__fdiv_rn(v, sc)); }
__device__ __forceinline__ int q80_code(float v, float sc, float rinv) {
    const float q = v * rinv;
    const float a = fabsf(q), fl = floorf(a), frac = a - fl;
    if (fabsf(frac - 0.5f) < 1e-3f) return q80_code_slow(v, sc);
    const int c = (int)fl + (frac > 0.5f ? 1 : 0);
    return q < 0.0f ? -c : c;
}
// branch-free variant: round half away via trunc(|q| + 0.5); a warp vote sends rare ties to the exact path
__device__ __forceinline__ int q80_code_bf(float v, float sc, float rinv, bool &tie) {
    const float q = v * rinv, a = fabsf(q);
    const float t = a + 0.5f;
    const int c = __float2int_rz(t);
    const float f = t - (float)c;
    tie = tie || (f < 1e-3f) || (f > 0.999f);
    return q < 0.0f ? -c : c;
}

__global__ void __launch_bounds__(512, 1) k_chain(const float *xin, unsigned long long *words, long long *out, int iters) {
    __shared__ float red[32];
    __shared__ __align__(16) unsigned char act[4096];
    __shared__ __align__(16) unsigned char tile[16 * 2080];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x >= 480) return;
    for (int i = threadIdx.x; i < 4096 / 4; i += 480) reinterpret_cast<uint32_t *>(act)[i] = 0x01020304u * (i + 1);
    for (int i = threadIdx.x; i < 16 * 2080 / 4; i += 480) reinterpret_cast<uint32_t *>(tile)[i] = 0x03fe01ffu * (i + 3);
    cbar();
    float4 v = reinterpret_cast<const float4 *>(xin)[threadIdx.x];
    long long tA = 0, tB = 0, tB2 = 0, tC6 = 0, tC16 = 0, tD = 0, tV[4] = {0, 0, 0, 0};
    float sink = 0.0f;
    for (int it = 0; it < iters + 2; it++) {
        const bool on = it >= 2;
        // ---- A ----
        cbar();
        long long t0 = clock64();
        float ss = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, v.w * v.w)));
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
        cbar();
        float tot = 0.0f;
#pragma unroll
        for (int w = 0; w < 15; w++) tot += red[w];
        tot = __fdiv_rn(tot, 768.0f); tot = __fadd_rn(tot, 1e-5f);
        const float inv = __fdiv_rn(1.0f, __fsqrt_rn(tot));
        long long t1 = clock64();
        if (on) tA += t1 - t0;
        // ---- B ----
        float4 a = make_float4(v.x * inv, v.y * inv, v.z * inv, v.w * inv);
        t0 = clock64();
        {
            float amax = fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w)));
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
            const float sc = __fdiv_rn(amax, 127.0f), rinv = __fdividef(127.0f, amax);
            uint32_t pk = 0;
            if (sc != 0.0f)
                pk = ((uint32_t)q80_code(a.x, sc, rinv) & 0xffu) | (((uint32_t)q80_code(a.y, sc, rinv) & 0xffu) << 8) |
                     (((uint32_t)q80_code(a.z, sc, rinv) & 0xffu) << 16) | (((uint32_t)q80_code(a.w, sc, rinv) & 0xffu) << 24);
            reinterpret_cast<uint32_t *>(act)[threadIdx.x] = pk;
            if (lane == 0) reinterpret_cast<float *>(act + 2048)[warp] = sc;
        }
        t1 = clock64();
        if (on) tB += t1 - t0;
        // ---- B2: redux max + branch-free codes ----
        t0 = clock64();
        {
            float amax = fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w)));
            amax = __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(amax)));
            const float sc = __fdiv_rn(amax, 127.0f), rinv = __fdividef(127.0f, amax);
            bool tie = false;
            int c0 = q80_code_bf(a.x, sc, rinv, tie), c1 = q80_code_bf(a.y, sc, rinv, tie), c2 = q80_code_bf(a.z, sc, rinv, tie), c3 = q80_code_bf(a.w, sc, rinv, tie);
            if (tie) { c0 = q80_code_slow(a.x, sc); c1 = q80_code_slow(a.y, sc); c2 = q80_code_slow(a.z, sc); c3 = q80_code_slow(a.w, sc); }
            uint32_t pk = (sc != 0.0f) ? ((uint32_t)c0 & 0xffu) | (((uint32_t)c1 & 0xffu) << 8) | (((uint32_t)c2 & 0xffu) << 16) | (((uint32_t)c3 & 0xffu) << 24) : 0u;
            reinterpret_cast<uint32_t *>(act)[threadIdx.x] = pk;
            if (lane == 0) reinterpret_cast<float *>(act + 2048)[warp] = sc;
        }
        t1 = clock64();
        if (on) tB2 += t1 - t0;
        cbar();
        // ---- C: team row dots ----
        for (int G : {6, 16}) {
            t0 = clock64();
            const uint32_t tl = lane % 8, team = lane / 8;
            const unsigned char *wrow = tile + (size_t)((warp * 4 + team) % 16) * 2080;
            const float *srow = reinterpret_cast<const float *>(act + 2048), *xs = reinterpret_cast<const float *>(act + 2048 + 64);
            float val = 0.0f;
#pragma unroll 4
            for (int gi = 0; gi < G; gi++) {
                const int4 w = *reinterpret_cast<const int4 *>(wrow + gi * 128 + tl * 16), xq = *reinterpret_cast<const int4 *>(act + gi * 128 + tl * 16);
                int isum = __dp4a(w.x, xq.x, 0);
                isum = __dp4a(w.y, xq.y, isum); isum = __dp4a(w.z, xq.z, isum); isum = __dp4a(w.w, xq.w, isum);
#pragma unroll
                for (int o = 1; o < 8; o <<= 1) isum += __shfl_xor_sync(0xffffffffu, isum, o);
                val = __fadd_rn(val, __fmul_rn(__fmul_rn((float)isum, srow[gi & 15]), xs[gi & 15]));
            }
            sink += val;
            t1 = clock64();
            if (on) { if (G == 6) tC6 += t1 - t0; else tC16 += t1 - t0; }
        }
        // ---- C2..C5: lane-per-group variants (6 groups, 5 rows per warp) ----
        for (int var = 0; var < 4; var++) {
            cbar();
            t0 = clock64();
            const uint32_t TS = 6, tl = lane % TS, team = min((uint32_t)lane / TS, 4u), team_base = team * TS;
            const unsigned char *wrow = tile + (size_t)((warp * 5 + team) % 16) * 2080;
            const float *srow = reinterpret_cast<const float *>(act + 2048), *xs = reinterpret_cast<const float *>(act + 2048 + 64);
            const unsigned char *wp = wrow + tl * 128, *xp = act + tl * 128;
            int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
            for (int c = 0; c < 8; c++) {
                const uint32_t off = ((uint32_t)(c + tl) % 8) * 16u;
                const int4 w = *reinterpret_cast<const int4 *>(wp + off), xq = *reinterpret_cast<const int4 *>(xp + off);
                a0 = __dp4a(w.x, xq.x, a0); a1 = __dp4a(w.y, xq.y, a1); a2 = __dp4a(w.z, xq.z, a2); a3 = __dp4a(w.w, xq.w, a3);
            }
            float val = 0.0f;
            if (var == 0) {            // C2: as in the kernel (runtime-count shuffle loop)
                const float term = __fmul_rn(__fmul_rn((float)((a0 + a1) + (a2 + a3)), srow[tl]), xs[tl]);
                const uint32_t cnt = min(TS, (uint32_t)(6 + (it >> 20)));
                for (uint32_t j = 0; j < cnt; j++) val = __fadd_rn(val, __shfl_sync(0xffffffffu, term, team_base + j));
            } else if (var == 1) {     // C3: unrolled-by-8 predicated shuffle gather
                const float term = __fmul_rn(__fmul_rn((float)((a0 + a1) + (a2 + a3)), srow[tl]), xs[tl]);
                const uint32_t cnt = min(TS, (uint32_t)(6 + (it >> 20)));
                float t8[8];
#pragma unroll
                for (int j = 0; j < 8; j++) t8[j] = __shfl_sync(0xffffffffu, term, team_base + j);
#pragma unroll
                for (int j = 0; j < 8; j++) if ((uint32_t)j < cnt) val = __fadd_rn(val, t8[j]);
            } else if (var == 2) {     // C4: no gather at all (integer sum -> float)
                val = __fmul_rn(__fmul_rn((float)((a0 + a1) + (a2 + a3)), srow[tl]), xs[tl]);
            } else {                   // C5: loads + dp4a only
                val = __int_as_float((a0 + a1) + (a2 + a3));
            }
            sink += val;
            t1 = clock64();
            if (on) tV[var] += t1 - t0;
        }
        // ---- D ----
        t0 = clock64();
        {
            unsigned long long w0, w1, w2, w3;
            const unsigned long long *p = words + (size_t)threadIdx.x * 4;
            asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(p) : "memory");
            asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(w2), "=l"(w3) : "l"(p + 2) : "memory");
            if ((uint32_t)(w0 >> 32) == 7u && (uint32_t)(w1 >> 32) == 7u && (uint32_t)(w2 >> 32) == 7u && (uint32_t)(w3 >> 32) == 7u) sink += __uint_as_float((uint32_t)w0);
        }
        t1 = clock64();
        if (on) tD += t1 - t0;
        v.x += sink * 1e-30f;
    }
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        out[0] = tA / iters; out[1] = tB / iters; out[2] = tB2 / iters; out[3] = tC6 / iters; out[4] = tC16 / iters; out[5] = tD / iters;
        out[7] = (long long)sink; for (int i = 0; i < 4; i++) out[8 + i] = tV[i] / iters;
    }
}

int main() {
    float *x; unsigned long long *words; long long *out;
    CK(cudaMalloc(&x, 4096 * 4)); CK(cudaMalloc(&words, 4096 * 8)); CK(cudaMalloc(&out, 256));
    float h[4096]; for (int i = 0; i < 4096; i++) h[i] = 0.01f * ((i * 37) % 101 - 50);
    CK(cudaMemcpy(x, h, sizeof h, cudaMemcpyHostToDevice));
    unsigned long long hw[4096]; for (int i = 0; i < 4096; i++) hw[i] = (7ull << 32) | (unsigned)i;
    CK(cudaMemcpy(words, hw, sizeof hw, cudaMemcpyHostToDevice));
    int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    for (int ncta : {1, sms}) {
        k_chain<<<ncta, 512>>>(x, words, out, 200);
        CK(cudaDeviceSynchronize());
        long long r[12]; CK(cudaMemcpy(r, out, 96, cudaMemcpyDeviceToHost));
        printf("ncta=%3d  A inverse(block reduce) %lld | B quantise group %lld | B2 redux+branch-free %lld | C row dot 6 groups %lld, 16 groups %lld | D poll4 ready %lld  cycles\n",
               ncta, r[0], r[1], r[2], r[3], r[4], r[5]);
        printf("          lane-per-group row dot (6 groups): C2 runtime shuffle loop %lld | C3 unrolled gather %lld | C4 no gather %lld | C5 loads+dp4a only %lld\n", r[8], r[9], r[10], r[11]);
    }
    return 0;
}
