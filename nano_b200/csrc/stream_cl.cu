// stream_cl.cu -- the streaming decode kernel's instantiations for the cluster launch (stream.cuh, CL = kStCluster), in a
// translation unit of their own so that they compile in parallel with the plain launch's (stream.cu)
#define NB_K static
#include "stream_host.h"
#include "stream.cuh"

namespace nb {

StreamKern pick_stream_cluster(const Dims &d) { return st_pick<kStCluster>(d); }

}  // namespace nb
