// Shared host-side plumbing for the C-ABI: last-error string, CUDA error checks, device buffers, graph capture.
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>
#include <string>
#include <vector>

namespace ara {

std::string& last_error_ref();
int set_error(const char* fmt, ...);

#define ARA_CUDA_OK(expr)                                                                          \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return ::ara::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    } while (0)

// Owner of device buffers: every allocation is zero-filled and recorded, and all of them are freed with the owner, on
// every return path.
class DeviceBuffers {
   public:
    DeviceBuffers() = default;
    ~DeviceBuffers() {
        for (void* p : ptrs_) cudaFree(p);
    }
    DeviceBuffers(const DeviceBuffers&) = delete;
    DeviceBuffers& operator=(const DeviceBuffers&) = delete;
    template <typename T>
    int dalloc(T** p, size_t count) {
        void* q = nullptr;
        ARA_CUDA_OK(cudaMalloc(&q, count * sizeof(T)));
        ptrs_.push_back(q);
        ARA_CUDA_OK(cudaMemset(q, 0, count * sizeof(T)));
        *p = static_cast<T*>(q);
        return 0;
    }

   private:
    std::vector<void*> ptrs_;
};

// Captures the work enqueue() (0 or -1 with the error set) puts on stream s into *exec.
template <typename F>
int capture_graph(cudaStream_t s, cudaGraphExec_t* exec, F&& enqueue) {
    cudaGraph_t g;
    ARA_CUDA_OK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue();
    const cudaError_t e = cudaStreamEndCapture(s, &g);
    if (e == cudaSuccess && rc != 0) cudaGraphDestroy(g);
    if (rc) return -1;
    ARA_CUDA_OK(e);
    const cudaError_t ie = cudaGraphInstantiate(exec, g, 0);
    cudaGraphDestroy(g);
    ARA_CUDA_OK(ie);
    return 0;
}

// Launch with programmatic stream serialization (PDL): the kernel may start while its predecessor in the stream is
// still draining; kernels call pdl_wait() before touching the predecessor's outputs.
bool pdl_enabled();
// While one lives on the calling thread, launch_pdl launches (and captures) plain kernels.  A search with Threads = 2 runs
// the network on a second stream beside the tree kernels; thread blocks of early-launched network kernels parked at
// their griddepcontrol.wait then delay the tree stream's launches (measured: 29.8 ms per headline search with the
// attribute, 21.4 ms without), so that mode captures the network without it.
struct PdlSuspend {
    explicit PdlSuspend(bool on);
    ~PdlSuspend();
    PdlSuspend(const PdlSuspend&) = delete;
    PdlSuspend& operator=(const PdlSuspend&) = delete;

   private:
    bool on_;
};
// launch_pdl with thread-block clusters of `cluster_x` CTAs along x (1: no cluster)
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                               unsigned cluster_x, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster_x;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    return launch_pdl_cluster(kernel, grid, block, smem, stream, 1u, args...);
}

}  // namespace ara
