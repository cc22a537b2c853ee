// ops_optim.cu -- L2 term + global-norm clip (nats.py:1326-1353) and the optimisers (nats.py:1106-1206),
// all as flat, stream-ordered passes over the packed parameter / gradient buffers (no host sync).
#include "ops.cuh"

namespace nats {

namespace {

constexpr int kRedBlocks = 132 * 4;

__global__ void sumsq_stage1(const float* __restrict__ x, long long n, float* __restrict__ part) {
    __shared__ float red[32];
    float s = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = x[i];
        s = fmaf(v, v, s);
    }
    s = block_sum(s, red);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__global__ void sumsq_stage2(const float* __restrict__ part, int n, float* __restrict__ out) {
    __shared__ float red[32];
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += part[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) *out = s;
}
__global__ void add_decay_kernel(float* __restrict__ g, const float* __restrict__ p, long long n, float two_decay) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        g[i] = fmaf(two_decay, p[i], g[i]);
}
__global__ void clip_scale_kernel(float* __restrict__ g, long long n, const float* __restrict__ stats, float clip_c) {
    const float g2 = stats[0];
    if (!(clip_c > 0.f) || !(g2 > clip_c * clip_c)) return;        // nats.py:1350: switch(g2 > clip_c**2, ...)
    const float sc = clip_c / sqrtf(g2);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        g[i] *= sc;
}

__global__ void adadelta_gs_kernel(const float* __restrict__ zg, float* __restrict__ rg2, long long n, float rho) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float g = zg[i];
        rg2[i] = rho * rg2[i] + (1.f - rho) * (g * g);            // nats.py:1157
    }
}
__global__ void adadelta_up_kernel(float* __restrict__ p, const float* __restrict__ zg, float* __restrict__ ru2,
                                   const float* __restrict__ rg2, long long n, float rho, float eps) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float r = ru2[i];
        const float ud = -sqrtf(r + eps) / sqrtf(rg2[i] + eps) * zg[i];     // nats.py:1163
        ru2[i] = rho * r + (1.f - rho) * (ud * ud);                          // nats.py:1166
        p[i] = p[i] + ud;                                                    // nats.py:1168
    }
}
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, long long n, float b1, float b2, float e, float lr_t) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gi = g[i];
        const float mt = b1 * gi + (1.f - b1) * m[i];                        // nats.py:1130
        const float vt = b2 * (gi * gi) + (1.f - b2) * v[i];                 // nats.py:1131
        p[i] = p[i] - lr_t * (mt / (sqrtf(vt) + e));                         // nats.py:1132-1133
        m[i] = mt;
        v[i] = vt;
    }
}
__global__ void rmsprop_gs_kernel(const float* __restrict__ zg, float* __restrict__ rg, float* __restrict__ rg2,
                                  long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float g = zg[i];
        rg[i] = 0.95f * rg[i] + 0.05f * g;                                    // nats.py:1188
        rg2[i] = 0.95f * rg2[i] + 0.05f * (g * g);                            // nats.py:1189
    }
}
__global__ void rmsprop_up_kernel(float* __restrict__ p, const float* __restrict__ zg, float* __restrict__ ud,
                                  const float* __restrict__ rg, const float* __restrict__ rg2, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float r = rg[i];
        const float u = 0.9f * ud[i] - 1e-4f * zg[i] / sqrtf(rg2[i] - r * r + 1e-4f);   // nats.py:1198
        ud[i] = u;
        p[i] = p[i] + u;
    }
}

inline int flat_grid(long long n) {
    long long g = (n + 255) / 256;
    if (g > 148LL * 16) g = 148LL * 16;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace

int grad_clip(const nats_ctx* ctx, cudaStream_t st, long long n, const float* params, float* grads, float decay_c,
              float clip_c, float* stats) {
    if (n == 0) return 0;
    float* part = ctx->dev_scratch;
    ProfScope ps(st, K_OPTIM, 0.0, 4.0 * n * ((clip_c > 0.f ? 3 : 1) + (decay_c > 0.f ? 4 : 0)));
    if (decay_c > 0.f) {
        sumsq_stage1<<<kRedBlocks, 256, 0, st>>>(params, n, part);
        NATS_LAUNCH_OK();
        sumsq_stage2<<<1, 256, 0, st>>>(part, kRedBlocks, stats + 1);
        NATS_LAUNCH_OK();
        add_decay_kernel<<<flat_grid(n), 256, 0, st>>>(grads, params, n, 2.f * decay_c);
        NATS_LAUNCH_OK();
    }
    sumsq_stage1<<<kRedBlocks, 256, 0, st>>>(grads, n, part);
    NATS_LAUNCH_OK();
    sumsq_stage2<<<1, 256, 0, st>>>(part, kRedBlocks, stats);
    NATS_LAUNCH_OK();
    if (clip_c > 0.f) {
        clip_scale_kernel<<<flat_grid(n), 256, 0, st>>>(grads, n, stats, clip_c);
        NATS_LAUNCH_OK();
    }
    return 0;
}
int adadelta_grad_shared(cudaStream_t st, long long n, const float* zg, float* rg2, float rho) {
    if (n == 0) return 0;
    ProfScope ps(st, K_OPTIM, 0.0, 12.0 * n);
    adadelta_gs_kernel<<<flat_grid(n), 256, 0, st>>>(zg, rg2, n, rho);
    NATS_LAUNCH_OK();
    return 0;
}
int adadelta_update(cudaStream_t st, long long n, float* p, const float* zg, float* ru2, const float* rg2, float rho,
                    float eps) {
    if (n == 0) return 0;
    ProfScope ps(st, K_OPTIM, 0.0, 24.0 * n);
    adadelta_up_kernel<<<flat_grid(n), 256, 0, st>>>(p, zg, ru2, rg2, n, rho, eps);
    NATS_LAUNCH_OK();
    return 0;
}
int adam_update(cudaStream_t st, long long n, float* p, const float* g, float* m, float* v, long long step) {
    if (n == 0) return 0;
    const float lr0 = 0.0002f, b1 = 0.1f, b2 = 0.001f, e = 1e-8f;     // nats.py:1114-1117
    const float i_t = (float)step + 1.f;
    const float fix1 = 1.f - powf(b1, i_t), fix2 = 1.f - powf(b2, i_t);
    const float lr_t = lr0 * (sqrtf(fix2) / fix1);                     // nats.py:1123-1125
    ProfScope ps(st, K_OPTIM, 0.0, 28.0 * n);
    adam_kernel<<<flat_grid(n), 256, 0, st>>>(p, g, m, v, n, b1, b2, e, lr_t);
    NATS_LAUNCH_OK();
    return 0;
}
int rmsprop_grad_shared(cudaStream_t st, long long n, const float* zg, float* rg, float* rg2) {
    if (n == 0) return 0;
    ProfScope ps(st, K_OPTIM, 0.0, 20.0 * n);
    rmsprop_gs_kernel<<<flat_grid(n), 256, 0, st>>>(zg, rg, rg2, n);
    NATS_LAUNCH_OK();
    return 0;
}
int rmsprop_update(cudaStream_t st, long long n, float* p, const float* zg, float* ud, const float* rg,
                   const float* rg2) {
    if (n == 0) return 0;
    ProfScope ps(st, K_OPTIM, 0.0, 28.0 * n);
    rmsprop_up_kernel<<<flat_grid(n), 256, 0, st>>>(p, zg, ud, rg, rg2, n);
    NATS_LAUNCH_OK();
    return 0;
}

}  // namespace nats
