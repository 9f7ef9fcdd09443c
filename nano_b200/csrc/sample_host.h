// sample_host.h -- host entry points of the device-side sampler (sample.cu)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace nb {
struct DevState;
// bytes of the workspace for a vocabulary of V entries (keys / values in and out + the sort's temporary storage + 9 result words)
size_t sample_workspace_bytes(uint32_t V, size_t *cub_bytes);
// temperature / top-p sampling over `logits` (device, penalty already applied); *out_dev -> {token, top-6 ids, n candidates, first-max index}
cudaError_t sample_top_p_launch(void *workspace, size_t cub_bytes, const float *logits, uint32_t V, float temperature, float top_p, float coin,
                                DevState *st, uint32_t **out_dev, cudaStream_t stream);

// Several rows at once (nb200_batch_next_sampled): row j samples logits row slot[j] with its own temperature, top_p and coin,
// exactly as sample_top_p_launch would, writes {token, six ids, n0, first-max index} to res[entry[j] * 16 ..] and the token to
// next[entry[j]].  Three launches (prepare, one device-wide sort, pick) for any n.
constexpr uint32_t kSampleRowsMax = 16;
struct SampleRows {
    uint32_t n;
    uint32_t slot[kSampleRowsMax], entry[kSampleRowsMax];
    float temperature[kSampleRowsMax], top_p[kSampleRowsMax], coin[kSampleRowsMax];
};
// bytes of the workspace for up to `rows` rows of V entries
size_t sample_rows_workspace_bytes(uint32_t V, uint32_t rows, size_t *cub_bytes);
cudaError_t sample_rows_launch(void *workspace, size_t cub_bytes, uint32_t rows, const float *logits, uint32_t V, const SampleRows &r,
                               uint32_t *res, uint32_t *next, cudaStream_t stream);
}  // namespace nb
