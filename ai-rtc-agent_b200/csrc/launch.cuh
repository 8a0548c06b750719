// Kernel launch helper: programmatic dependent launch (PDL) + optional thread-block cluster.
//
// Every kernel of the frame program starts with `griddepcontrol.launch_dependents` (the next kernel of the stream /
// CUDA graph may be scheduled as soon as all CTAs of this one have started) and executes `griddepcontrol.wait`
// before touching global memory produced by its predecessor.  The successor's launch latency and prologue (barrier
// init, descriptor prefetch) then overlap this kernel's execution instead of sitting on the
// critical path -- with ~450 launches per frame that is a large fraction of the frame time.
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

namespace b2 {

__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

inline bool pdl_enabled() {
    static const bool on = getenv("B2_NO_PDL") == nullptr;
    return on;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kc(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_x,
                             int cluster_z, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (cluster_z > 1 || cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = (unsigned)(cluster_x > 1 ? cluster_x : 1);
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = (unsigned)(cluster_z > 1 ? cluster_z : 1);
        ++n;
    }
    if (pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_z,
                            Args&&... args) {
    return launch_kc(kernel, grid, block, smem, stream, 1, cluster_z, static_cast<Args&&>(args)...);
}

}  // namespace b2
