// stream.cu -- translation unit of the grid-wide streaming decode kernel (stream.cuh): the plain launch's kernel instantiations
// + the load-time builder of the per-CTA weight streams.  Compiled beside engine.cu and stream_cl.cu (the cluster launch's
// instantiations) so that they build in parallel.
#define NB_K static
#include "stream_host.h"
#include "stream.cuh"

namespace nb {

// copy the rows a CTA owns of one fused matrix into its stream: tile = [rows x row_stride main][rows x aux_stride aux]
__global__ void k_build_stream(const uint8_t *__restrict__ mainp, const uint8_t *__restrict__ auxp, uint32_t main_bytes, uint32_t aux_bytes,
                               StKind k, uint8_t *stream, uint64_t cta_stride, uint64_t base_off) {
    const uint32_t cta = blockIdx.y, ncta = gridDim.y;
    const uint32_t u0 = (uint32_t)(((uint64_t)cta * k.units) / ncta), u1 = (uint32_t)(((uint64_t)(cta + 1) * k.units) / ncta);
    const uint32_t row0 = u0 * k.unit_rows, rows = (u1 - u0) * k.unit_rows;
    for (uint32_t lrow = blockIdx.x; lrow < rows; lrow += gridDim.x) {
        const uint32_t j = lrow / k.tile_rows, i = lrow % k.tile_rows;
        const uint32_t tr = min(k.tile_rows, rows - j * k.tile_rows);
        uint8_t *tile = stream + (uint64_t)cta * cta_stride + base_off + k.off + (uint64_t)j * k.tile_stride;
        const uint64_t grow = (uint64_t)row0 + lrow;
        const int4 *src = reinterpret_cast<const int4 *>(mainp + grow * main_bytes);
        int4 *dst = reinterpret_cast<int4 *>(tile + (uint64_t)i * k.row_stride);
        for (uint32_t c = threadIdx.x; c < main_bytes / 16; c += blockDim.x) dst[c] = src[c];
        if (aux_bytes) {
            const uint32_t *asrc = reinterpret_cast<const uint32_t *>(auxp + grow * aux_bytes);
            uint32_t *adst = reinterpret_cast<uint32_t *>(tile + (uint64_t)tr * k.row_stride + (uint64_t)i * k.aux_stride);
            for (uint32_t c = threadIdx.x; c < aux_bytes / 4; c += blockDim.x) adst[c] = asrc[c];
        }
    }
}

cudaError_t stream_build_launch(const uint8_t *mainp, const uint8_t *auxp, uint32_t main_bytes, uint32_t aux_bytes, const StKind &k,
                                uint8_t *stream, uint64_t cta_stride, uint64_t base_off, uint32_t grid_x, uint32_t ncta) {
    k_build_stream<<<dim3(grid_x, ncta), 128>>>(mainp, auxp, main_bytes, aux_bytes, k, stream, cta_stride, base_off);
    return cudaGetLastError();
}

StreamKern pick_stream(const Dims &d, bool cluster) {
    if (d.hd > 128 || (d.arch == 3u && (d.hd & (d.hd - 1)) != 0)) return nullptr;     // in-register half-split RoPE needs hd = 4 * 2^k
    return cluster ? pick_stream_cluster(d) : st_pick<0>(d);
}

}  // namespace nb
