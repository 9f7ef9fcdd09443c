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
}  // namespace nb
