// prof.cuh -- optional per-kernel-class timing with CUDA events on the launch stream (eager mode only; it is
// switched off while a step is captured into / replayed from a CUDA graph).  Used by bench.py's roofline probe.
#pragma once
#include <cuda_runtime.h>

namespace nats {

enum KClass {
    K_GEMM_BASE = 0,        // + cfg(0 big, 1 mid, 2 smallm) * 4 + transA * 2 + transB   (12 classes)
    K_GATES_FWD = 12,
    K_GATES_BWD,
    K_ATT_SCORES,
    K_ATT_CONTEXT,
    K_ATT_BWD_CTX,
    K_ATT_BWD_DALPHA,
    K_ATT_BWD_SOFTMAX,
    K_NLL,
    K_DLOGITS,
    K_SOFTMAX_SAMPLE,
    K_COLSUM,
    K_REDUCE_SPLITS,
    K_EMBED,
    K_ELEMWISE,
    K_OPTIM,
    K_BEAM,
    K_MEMSET,
    K_TC_GEMM,           // wgmma 3xTF32, 128 x 64 tiles
    K_TC_GEMM_SKINNY,    // wgmma 3xTF32, N side <= 64 (the batch, roles swapped)
    K_ENC_PERSIST_FWD,   // persistent weight-stationary wgmma bidirectional encoder recurrence (one launch per pass)
    K_ENC_PERSIST_BWD,
    K_COUNT
};

const char* kclass_name(int cls);
bool prof_enabled();
void prof_begin(cudaStream_t st, int cls, double flops, double bytes);
void prof_end(cudaStream_t st);

struct ProfScope {
    cudaStream_t st;
    bool on;
    ProfScope(cudaStream_t s, int cls, double flops = 0.0, double bytes = 0.0) : st(s), on(prof_enabled()) {
        if (on) prof_begin(st, cls, flops, bytes);
    }
    ~ProfScope() {
        if (on) prof_end(st);
    }
};

inline cudaError_t memset_async(cudaStream_t st, void* p, int v, size_t bytes) {
    ProfScope ps(st, K_MEMSET, 0.0, (double)bytes);
    return cudaMemsetAsync(p, v, bytes, st);
}

}  // namespace nats
