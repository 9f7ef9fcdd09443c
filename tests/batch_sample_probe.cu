// batch_sample_probe.cu -- test harness for the several-row sampler (sample_rows_launch, nano_b200/csrc/sample.cu) on host-given
// logits.
//
// Row j of the call samples logits row slot[j] of `logits` ([n_rows][V]) with its own temperature, top_p and coin and reports
// under entry[j], as a batch pass does.  The workspace holds kSampleRowsMax rows whatever n is, as a batch's does.  Returns the
// result words res[16][16] and next[16] (by entry, filled with 0xffffffff first) and, per row j, the sorted keys decoded to
// floats (probabilities, -1 for rejected entries) and values (vocabulary indices).
// Built by tests/test_gpu_batch_sampling.py with nvcc from the repository's sources.
#include <vector>

#include "sample.cu"

using namespace nb;

extern "C" int probe_sample_rows(const float *logits, uint32_t n_rows, uint32_t V, uint32_t n, const uint32_t *slot, const uint32_t *entry,
                                 const float *temperature, const float *top_p, const float *coin, uint32_t *res, uint32_t *next, float *keys,
                                 uint32_t *vals) {
    if (n == 0 || n > kSampleRowsMax) return (int)cudaErrorInvalidValue;
    SampleRows r{};
    r.n = n;
    for (uint32_t j = 0; j < n; j++) {
        r.slot[j] = slot[j]; r.entry[j] = entry[j];
        r.temperature[j] = temperature[j]; r.top_p[j] = top_p[j]; r.coin[j] = coin[j];
    }
    size_t cub_bytes = 0;
    const size_t bytes = sample_rows_workspace_bytes(V, kSampleRowsMax, &cub_bytes);
    void *ws = nullptr; float *dl = nullptr; uint32_t *dres = nullptr, *dnext = nullptr;
    cudaError_t e = cudaMalloc(&ws, bytes);
    if (e == cudaSuccess) e = cudaMalloc(&dl, (size_t)n_rows * V * 4);
    if (e == cudaSuccess) e = cudaMalloc(&dres, 16 * 16 * 4);
    if (e == cudaSuccess) e = cudaMalloc(&dnext, 16 * 4);
    if (e == cudaSuccess) e = cudaMemset(ws, 0xff, bytes);
    if (e == cudaSuccess) e = cudaMemset(dres, 0xff, 16 * 16 * 4);
    if (e == cudaSuccess) e = cudaMemset(dnext, 0xff, 16 * 4);
    if (e == cudaSuccess) e = cudaMemcpy(dl, logits, (size_t)n_rows * V * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = sample_rows_launch(ws, cub_bytes, kSampleRowsMax, dl, V, r, dres, dnext, 0);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    const SampleRowsWorkspace w = sample_rows_workspace(ws, V, kSampleRowsMax);
    if (e == cudaSuccess) e = cudaMemcpy(res, dres, 16 * 16 * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(next, dnext, 16 * 4, cudaMemcpyDeviceToHost);
    std::vector<unsigned long long> k64((size_t)n * V);
    if (e == cudaSuccess) e = cudaMemcpy(k64.data(), w.keys_out, k64.size() * 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(vals, w.vals_out, (size_t)n * V * 4, cudaMemcpyDeviceToHost);
    for (size_t i = 0; e == cudaSuccess && i < k64.size(); i++) {
        const uint32_t row = n - 1 - (uint32_t)(i / V);               // the row field of the composite key
        if ((uint32_t)(k64[i] >> 32) != row) { e = cudaErrorInvalidValue; break; }
        keys[i] = key_float((uint32_t)k64[i]);
    }
    cudaFree(ws); cudaFree(dl); cudaFree(dres); cudaFree(dnext);
    return e == cudaSuccess ? 0 : (int)e;
}
