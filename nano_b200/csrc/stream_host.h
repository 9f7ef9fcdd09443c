// stream_host.h -- host-side entry points of the streaming-kernel translation unit (stream.cu)
#pragma once
#include "stream_args.h"

namespace nb {
typedef void (*StreamKern)(const StreamArgs);
// the k_decode_stream instantiation for a model shape, or nullptr when the streaming kernel does not take it
// (cluster: the one launched in clusters of kStCluster CTAs)
StreamKern pick_stream(const Dims &d, bool cluster);
StreamKern pick_stream_cluster(const Dims &d);          // stream_cl.cu (pick_stream checks the shape first)
// copies the rows every CTA owns of one fused matrix into its tile-ordered stream (one launch per matrix, at load time)
cudaError_t stream_build_launch(const uint8_t *mainp, const uint8_t *auxp, uint32_t main_bytes, uint32_t aux_bytes, const StKind &k,
                                uint8_t *stream, uint64_t cta_stride, uint64_t base_off, uint32_t grid_x, uint32_t ncta);
}  // namespace nb
