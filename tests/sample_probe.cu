// sample_probe.cu -- test harness for the device sampler (nano_b200/csrc/sample.cu) on host-given logits.
//
// Runs sample_top_p_launch with no engine state and returns the result words {id, six observed ids, n0, first-max index}
// and the sorted keys (probabilities, -1 for rejected entries) and values (vocabulary indices).
// Built by tests/test_gpu_sampler.py with nvcc from the repository's sources.
#include "sample.cu"

using namespace nb;

// out: 9 words; keys / vals: V entries each (may be null).  Returns 0 or a CUDA error code.
extern "C" int probe_sample(const float *logits, uint32_t V, float temperature, float top_p, float coin, uint32_t *out, float *keys,
                            uint32_t *vals) {
    size_t cub_bytes = 0;
    const size_t bytes = sample_workspace_bytes(V, &cub_bytes);
    void *ws = nullptr; float *dl = nullptr;
    cudaError_t e = cudaMalloc(&ws, bytes);
    if (e == cudaSuccess) e = cudaMalloc(&dl, (size_t)V * 4);
    if (e == cudaSuccess) e = cudaMemset(ws, 0xff, bytes);
    if (e == cudaSuccess) e = cudaMemcpy(dl, logits, (size_t)V * 4, cudaMemcpyHostToDevice);
    uint32_t *out_dev = nullptr;
    if (e == cudaSuccess) e = sample_top_p_launch(ws, cub_bytes, dl, V, temperature, top_p, coin, nullptr, &out_dev, 0);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    const SampleWorkspace w = sample_workspace(ws, V, cub_bytes);
    if (e == cudaSuccess && out_dev != w.out) e = cudaErrorInvalidValue;
    if (e == cudaSuccess) e = cudaMemcpy(out, w.out, 9 * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && keys) e = cudaMemcpy(keys, w.keys_out, (size_t)V * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && vals) e = cudaMemcpy(vals, w.vals_out, (size_t)V * 4, cudaMemcpyDeviceToHost);
    cudaFree(ws); cudaFree(dl);
    return e == cudaSuccess ? 0 : (int)e;
}
