// enc_tc.cu -- the bidirectional GRU encoder recurrence (nats.py:336-372, both directions) and its reverse mode as ONE
// persistent, WEIGHT-STATIONARY tensor-core kernel per pass.
//
// Why.  A recurrent step is  h[n,D] x [U|Ux][D,3D]  with n = 32: launched per step it costs a split-K product kernel + a
// gate kernel, two kernel boundaries and 24 MB of weights re-streamed from L2 per step, and the 2 x 400 dependent steps
// dominate the training step.  Here the weights never move after the prologue:
//   * one CTA per SM, at most 66 CTAs per direction on the 132 SMs of an H100.  The swapped product (rows = weight columns,
//     N = batch) is cut into row tiles of <= 192 rows (three warpgroups of 64) x Kc deep; at D = 1000:
//       forward : 16 row tiles (the r|u|c gate columns of 63 hidden units each) x 4 K chunks of D;
//       backward:  8 row tiles (125 hidden units of d h_{t-1})                  x 8 K chunks of 3D.
//   * each CTA keeps its tile of [U|Ux] (forward) / [U|Ux]^T (backward) as RAW fp32 in shared memory in the K-major
//     SWIZZLE_128B layout of the wgmma descriptors (<= 192 KB).  The tensor core reads the upper 19 bits of an fp32 word,
//     so the raw tile IS the "hi" operand; its residual  lo = x - trunc_tf32(x)  is formed in registers from the same
//     shared-memory words right before each k-step and fed as the register A operand.  3xTF32 per k-step of 8:
//       acc_hh += A_raw(smem) x B_raw,   acc_x += A_raw(smem) x B_lo  +  A_lo(registers) x B_raw.
//   * per step the only moving operand is B = h_{t-1} (forward; raw = the context row itself) / dG_{t+1} (backward; raw =
//     the saved gate-derivative row itself), plus its residual in a 2-deep side buffer written by the gate warps: TMA
//     boxes of 32 k x n rows into a ring of stages, gated by ONE monotonic counter per row tile in L2 (red.release /
//     ld.acquire).
//   * the K partials of a row tile are exchanged through L2 (fixed summation order: deterministic): every CTA writes
//     its partial slab, bumps the tile's counter, waits for its S-1 peers and finishes the gate arithmetic (forward:
//     nats.py:336-356; backward: its reverse) for ITS share of the tile's units in registers; it stores h_t straight
//     into the concatenated context [Tx,n,2D] (nats.py:713 needs no copy) / dG_t into the saved arrays the weight-gradient
//     products read, publishes the residuals, bumps the counter, and only then writes what nobody waits for.
// Every spin is bounded (a stuck CTA traps after ~1 s instead of hanging the GPU).  The grid must be co-resident: the
// host checks the occupancy before choosing this path.
#include <cuda.h>

#include "ops.cuh"
#include "tc_common.cuh"

namespace nats {

namespace {

using namespace tc;

constexpr int kMmaWG = 3;               // warps 0-11: three MMA warpgroups (rows 64w..64w+63 of the row tile) + epilogue
constexpr int kMmaThreads = kMmaWG * 128;
constexpr int kProdWarp = kMmaWG * 4;   // warp 12: flag poll + TMA producer
constexpr int kGateWarp0 = kProdWarp + 1;   // warps 13-20: gates
constexpr int kGateThreads = 256;
constexpr int kThreads = kGateWarp0 * 32 + kGateThreads;
constexpr int kMaxRows = 64 * kMmaWG;
constexpr int kMaxNS = 8;
constexpr int kMaxWords = 12;           // K chunks x gate groups summed per gate element
constexpr int kMaxDps = 16;             // units finished per CTA and step
constexpr int kMaxCtasPerDir = 74;      // bound of the device-independent scratch sizes
constexpr long long kSpinLimit = 2000000000LL;
constexpr int kCtrStride = 32;          // counters live in separate 128-byte lines

struct EncTc {
    CUtensorMap map_raw[2];     // B operand, raw: forward = view of cc (+dir*D): dims (D, n, Tx); backward = dG[dir]: dims (3D, n, Tx)
    CUtensorMap map_lo[2];      // B operand, residual side buffer of the direction: dims (K, n, 2)
    const float* Ucat[2];       // [D,3D]
    const float* mask;          // [Tx,n] or NULL
    // ---- forward
    const float* xproj[2];      // [Tx*n,3D] by source position
    float* cc;                  // [Tx,n,2D]
    float* r[2]; float* u[2]; float* c[2]; float* p[2];   // saved gates [Tx*n,D] by position (forward: outputs or NULL)
    float* ctxsum;              // [n,2D]
    // ---- backward
    const float* dcc;           // [Tx,n,2D]  d cost / d context
    const float* mean_grad;     // [n,2D] or NULL
    const float* coef;          // [n]
    float* dG[2]; float* dGx[2];   // [Tx*n,3D] by position
    // ---- exchange
    float* lo;                  // [2 dir][2 parity][n][Kp]
    unsigned long long* slab;   // [2 dir][NT][S][NG][BN][dpc] K partials as {value, step tag} words (filled with 0xff before the launch)
    unsigned* bar;              // [32 * (dir*NT + tile)]: arrivals of the tile's CTAs (zero-initialised)
    unsigned long long* dbg;    // optional phase stamps of CTA 0 (NULL = off)
    int Tx, n, D, Kp;
    int NT, S, dpc, dps, Kc, nkbA, NS, nwg;   // nwg: warpgroups holding rows of the tile (k-block = nwg * 8 KB of shared memory)
};

// bounded waits: a protocol error becomes a trap (context error), never a hung GPU
__device__ __forceinline__ void mbar_wait_b(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    const long long t0 = clock64();
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
        if (!ok && clock64() - t0 > kSpinLimit) __trap();
    } while (!ok);
}
__device__ __forceinline__ void flag_arrive(unsigned* ctr) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
}
// K-partial exchange words: {fp32 value, step tag} in ONE naturally aligned 64-bit word (single-copy atomic), written with
// a relaxed gpu-scope store and polled with relaxed gpu-scope loads: no fence, no counter, one L2 round trip.
__device__ __forceinline__ void st_word(unsigned long long* p, float v, uint32_t tag) {
    const unsigned long long w = ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(v);
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ unsigned long long ld_word(const unsigned long long* p) {
    unsigned long long w;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
    return w;
}

// shared-memory byte offset of element (row m, k) inside a K-major SWIZZLE_128B operand made of 32-deep k-blocks of
// kb_bytes (rows of 128 B, 8-row groups 1024 B apart, 16-byte chunks XOR (m & 7))
__device__ __forceinline__ uint32_t a_off(int m, int k, uint32_t kb_bytes) {
    const int kb = k >> 5, kk = k & 31;
    return (uint32_t)kb * kb_bytes + (uint32_t)m * 128u + (uint32_t)(((kk >> 2) ^ (m & 7)) << 4) + (uint32_t)((kk & 3) << 2);
}

template <int BN>
__device__ __forceinline__ void mma_ss(float (&d)[BN / 2], uint64_t da, uint64_t db) {
    if constexpr (BN == 32) wgmma_ss_n32(d, da, db);
    else wgmma_ss_n64(d, da, db);
}
template <int BN>
__device__ __forceinline__ void mma_rs(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t db) {
    if constexpr (BN == 32) wgmma_rs_n32(d, a, db);
    else wgmma_rs_n64(d, a, db);
}

template <int BN, bool BWD>
__global__ void __launch_bounds__(kThreads, 1) enc_tc_kernel(const __grid_constant__ EncTc a) {
    constexpr uint32_t kStage = 2u * BN * 128u;             // [B_raw BN rows x 128 B | B_lo]
    constexpr int EPT = (kMaxDps * BN + kGateThreads - 1) / kGateThreads;   // gate elements per gate thread
    constexpr int NG = BWD ? 1 : 3;                         // gate column groups inside a row tile
    constexpr int R = BN / 2;                               // accumulator registers per MMA thread

    extern __shared__ __align__(1024) unsigned char smem[];
    __shared__ __align__(8) uint64_t full[kMaxNS];
    __shared__ __align__(8) uint64_t empty[kMaxNS];

    // the warp index as a shuffled (provably warp-uniform) value: role branches on it are not divergent for the compiler,
    // which would otherwise serialize the wgmma instructions inside them
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
    const int D = a.D, n = a.n, Tx = a.Tx, D3 = 3 * a.D, C = 2 * a.D;
    const int S = a.S, NT = a.NT, dpc = a.dpc, dps = a.dps;
    const int dir = blockIdx.x / (NT * S);
    const int rem = blockIdx.x - dir * NT * S;
    const int tile = rem / S, crank = rem - tile * S;
    const int d0 = tile * dpc;
    const int nd = min(dpc, D - d0);                         // units of this row tile (>= 1)
    const int Ktot = BWD ? D3 : D;
    const int kbeg = crank * a.Kc;
    const int kend = min(Ktot, kbeg + a.Kc);
    const int klen = max(0, kend - kbeg);
    const int nkb = (klen + 31) >> 5;
    const int NS = a.NS;
    const uint32_t kb_bytes = (uint32_t)a.nwg * 8192u;

    const uint32_t sA = (smem_u32(smem) + 1023u) & ~1023u;   // the wgmma / TMA swizzle atoms need 1024-byte alignment
    const uint32_t sRing = sA + (uint32_t)a.nkbA * kb_bytes;

    // ------------------------------------------------------------------ prologue: weights -> shared (raw)
    {
        const uint32_t words = (uint32_t)a.nkbA * kb_bytes / 4u;
        for (uint32_t i = tid; i < words / 4; i += kThreads)
            asm volatile("st.shared.v4.f32 [%0], {%1,%1,%1,%1};" ::"r"(sA + i * 16u), "f"(0.f) : "memory");
    }
    if (tid == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&a.map_raw[dir]) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&a.map_lo[dir]) : "memory");
        for (int s = 0; s < NS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kMmaThreads / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    {
        const float* __restrict__ W = a.Ucat[dir];
        if (!BWD) {                                          // rows = gate columns g*D + d0 + dl of [U|Ux], k = input unit
            const int rows = 3 * nd;
            const int total = klen * rows;
            for (int e = tid; e < total; e += kThreads) {
                const int kl = e / rows, mm = e - kl * rows;
                const int g = mm / nd, dl = mm - g * nd;
                const float v = __ldg(W + (long long)(kbeg + kl) * D3 + g * D + d0 + dl);
                asm volatile("st.shared.f32 [%0], %1;" ::"r"(sA + a_off(g * dpc + dl, kl, kb_bytes)), "f"(v) : "memory");
            }
        } else {                                             // rows = units d0 + m of d h_{t-1}, k = gate column: [U|Ux]^T
            const int total = nd * klen;
            for (int e = tid; e < total; e += kThreads) {
                const int m = e / klen, kl = e - m * klen;
                const float v = __ldg(W + (long long)(d0 + m) * D3 + kbeg + kl);
                asm volatile("st.shared.f32 [%0], %1;" ::"r"(sA + a_off(m, kl, kb_bytes)), "f"(v) : "memory");
            }
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // the raw tiles were written by generic stores
    __syncthreads();

    unsigned* tctr = a.bar + (dir * NT + tile) * kCtrStride;      // arrivals of this row tile's gate warps (S * 8 per step)
    const bool stamp = a.dbg != nullptr && blockIdx.x == 0;
#define ENC_STAMP(i) do { a.dbg[i] = gtimer(); a.dbg[32 + (i)] = (unsigned long long)clock64(); } while (0)

    // Ring protocol: k-block j of the CTA's whole run (all steps) uses stage j % NS; the producer refills a stage once all
    // twelve MMA warps have arrived on its `empty` barrier (after the wgmmas that read it completed).
    if (warp == kProdWarp) {
        // ============================================================ flag poll + TMA producer
        // Dependencies are tracked per ROW TILE (S arrivals per step each): this CTA's operand columns [kbeg, kcov) are
        // produced by a few tiles only, so it does not wait for the slowest CTA of the whole direction.  Lane l polls the
        // counter of tile l; the warp proceeds when every needed tile is complete.
        const int kcov = min(Ktot, kbeg + 32 * nkb);
        bool need = false;
        if (lane < NT) {
            const int u0 = lane * dpc, u1 = min(D, u0 + dpc);          // units finished by tile `lane`
            for (int g = 0; g < (BWD ? 3 : 1); ++g) need = need || (g * D + u0 < kcov && g * D + u1 > kbeg);
        }
        const unsigned* pctr = a.bar + (dir * NT + lane) * kCtrStride;
        uint32_t it = 0;
        for (int s = 1; s < Tx; ++s) {
            {
                const unsigned target = (unsigned)(S * (kGateThreads / 32) * s);
                const long long t0 = clock64();
                bool ok;
                do {
                    ok = true;
                    if (need) {
                        unsigned v;
                        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(pctr) : "memory");
                        ok = v >= target;
                    }
                    if (!ok && clock64() - t0 > kSpinLimit) __trap();
                } while (!__all_sync(0xffffffffu, ok));
            }
            if (lane == 0) {
                // row of the raw operand: forward h_{t-1} = context row of the previous position of this direction;
                // backward dG of the step processed just before
                const int brow = BWD ? (dir == 0 ? Tx - s : s - 1) : (dir == 0 ? s - 1 : Tx - s);
                asm volatile("fence.proxy.async;" ::: "memory");      // the operand was written by generic stores of other SMs
                if (stamp && s == 8) ENC_STAMP(0);
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const uint32_t slot = it % (uint32_t)NS;
                    if (it >= (uint32_t)NS) mbar_wait_b(&empty[slot], ((it / (uint32_t)NS) - 1u) & 1u);
                    mbar_expect_tx(&full[slot], kStage);
                    const uint32_t dst = sRing + slot * kStage;
                    tma_load_3d(dst, &a.map_raw[dir], &full[slot], kbeg + 32 * kb, 0, brow);
                    tma_load_3d(dst + BN * 128u, &a.map_lo[dir], &full[slot], kbeg + 32 * kb, 0, (s - 1) & 1);
                }
            }
            __syncwarp();
        }
    } else if (warp < kProdWarp) {
        // ============================================================ MMA warpgroups: K partials of this CTA's chunk
        const int wg = warp >> 2;
        const bool active = wg < a.nwg;                      // warpgroup-uniform: rows 64wg.. hold weights
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);       // fragment rows r0, r0 + 8
        const int q = lane & 3;
        int g_row[2], dl_row[2];
        bool row_ok[2];
        unsigned long long* slab_w[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int mrow = r0 + 8 * h;
            g_row[h] = BWD ? 0 : mrow / dpc;
            dl_row[h] = mrow - g_row[h] * dpc;
            row_ok[h] = g_row[h] < NG && dl_row[h] < nd;
            slab_w[h] = a.slab + (long long)(dir * NT + tile) * S * NG * BN * dpc +
                        (long long)((crank * NG + g_row[h]) * BN) * dpc + dl_row[h];      // + b*dpc
        }
        const uint32_t a_row0 = sA + (uint32_t)r0 * 128u, a_row1 = a_row0 + 1024u;  // rows r0 and r0 + 8: same (m & 7)
        const uint32_t sw = (uint32_t)(r0 & 7);
        const uint64_t adesc0 = desc_sw128(sA + (uint32_t)wg * 8192u);
        const uint64_t bdesc0 = desc_sw128(sRing);
        uint32_t it = 0;
        for (int s = 1; s < Tx; ++s) {
            float acc_hh[R], acc_x[R];
#pragma unroll
            for (int i = 0; i < R; ++i) { acc_hh[i] = 0.f; acc_x[i] = 0.f; }
            for (int kb = 0; kb < nkb; ++kb, ++it) {
                const uint32_t slot = it % (uint32_t)NS;
                // residual A fragments of the 4 k-steps (rows r0 / r0+8, k = 8kk + q and 8kk + q + 4)
                uint32_t alo[4][4];
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    const uint32_t c0 = (((uint32_t)(2 * kk) ^ sw) << 4) + (uint32_t)(q << 2);
                    const uint32_t c1 = (((uint32_t)(2 * kk + 1) ^ sw) << 4) + (uint32_t)(q << 2);
                    const uint32_t kbo = (uint32_t)kb * kb_bytes;
                    float v0, v1, v2, v3;
                    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v0) : "r"(a_row0 + kbo + c0));
                    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v1) : "r"(a_row1 + kbo + c0));
                    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v2) : "r"(a_row0 + kbo + c1));
                    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v3) : "r"(a_row1 + kbo + c1));
                    alo[kk][0] = __float_as_uint(resid(v0)); alo[kk][1] = __float_as_uint(resid(v1));
                    alo[kk][2] = __float_as_uint(resid(v2)); alo[kk][3] = __float_as_uint(resid(v3));
                }
                mbar_wait_b(&full[slot], (it / (uint32_t)NS) & 1u);
                if (active) {
                    const uint64_t ad = adesc0 + (uint64_t)((kb * kb_bytes) >> 4);
                    const uint64_t braw = bdesc0 + (uint64_t)((slot * kStage) >> 4), blo = braw + (uint64_t)((BN * 128u) >> 4);
                    wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        mma_ss<BN>(acc_hh, ad + 2 * kk, braw + 2 * kk);
                        mma_ss<BN>(acc_x, ad + 2 * kk, blo + 2 * kk);
                        mma_rs<BN>(acc_x, alo[kk], braw + 2 * kk);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    reg_fence(acc_hh); reg_fence(acc_x);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[slot]);
            }
            if (stamp && s == 8 && tid == 0) ENC_STAMP(3);
            // fragment i of this thread: row r0 + 8*((i>>1)&1), batch column 8*(i>>2) + 2q + (i&1)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!row_ok[h]) continue;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int i = 4 * j + 2 * h + e;
                        st_word(slab_w[h] + (long long)(8 * j + 2 * q + e) * dpc, acc_hh[i] + acc_x[i], (uint32_t)s);
                    }
            }
            if (stamp && s == 8 && tid == 0) ENC_STAMP(6);
            // the peers' partials are written at about the same time as ours: only now do the gate warps start polling
            asm volatile("bar.arrive 2, %0;" ::"r"(kMmaThreads + kGateThreads) : "memory");
        }
    } else {
        // ============================================================ gate warps: K partials of the tile -> gates of this CTA's units
        const int gtid = tid - kGateWarp0 * 32;
        const unsigned long long* slab_tile = a.slab + (long long)(dir * NT + tile) * S * NG * BN * dpc;
        const int nw = S * NG;                               // exchange words per gate element
        // gate elements of this thread: e = gtid + 256*i -> (b = e / dps, dlo = e % dps): consecutive lanes = consecutive units
        const int nds = max(0, min(dps, nd - crank * dps));
        const int dbase = d0 + crank * dps;                  // first unit finished by this CTA
        int eb[EPT], ed[EPT];
        bool ev[EPT];
        float carry[EPT], csum[EPT];                         // forward: h_{t-1} / running sum_t mask*h;  backward: elementwise part of d h
#pragma unroll
        for (int i = 0; i < EPT; ++i) {
            const int e = gtid + kGateThreads * i;
            eb[i] = e / dps;
            ed[i] = e - eb[i] * dps;
            ev[i] = eb[i] < n && ed[i] < nds;
            carry[i] = 0.f; csum[i] = 0.f;
        }
        for (int s = 0; s < Tx; ++s) {
            const int pos = BWD ? (dir == 0 ? Tx - 1 - s : s) : (dir == 0 ? s : Tx - 1 - s);
            // inputs that do not depend on the recurrence: in flight while the product of this step runs
            float x0[EPT], x1[EPT], x2[EPT], mk[EPT];
            float sr_[EPT], su_[EPT], sc_[EPT], sp_[EPT];     // backward: saved gates
#pragma unroll
            for (int i = 0; i < EPT; ++i) {
                x0[i] = x1[i] = x2[i] = 0.f; mk[i] = 1.f;
                sr_[i] = su_[i] = sc_[i] = sp_[i] = 0.f;
                if (ev[i]) {
                    const long long row = (long long)pos * n + eb[i];
                    const int d = dbase + ed[i];
                    if (a.mask) mk[i] = __ldg(a.mask + row);
                    if (!BWD) {
                        const float* xp = a.xproj[dir] + row * D3 + d;
                        x0[i] = __ldg(xp); x1[i] = __ldg(xp + D); x2[i] = __ldg(xp + 2 * D);
                    } else {
                        const long long o = row * D + d;
                        sr_[i] = __ldg(a.r[dir] + o); su_[i] = __ldg(a.u[dir] + o); sc_[i] = __ldg(a.c[dir] + o); sp_[i] = __ldg(a.p[dir] + o);
                        x0[i] = __ldg(a.dcc + row * C + dir * D + d);                                  // d cost / d context
                        const int prev = dir == 0 ? pos - 1 : pos + 1;                                 // h_{t-1} of this direction
                        x1[i] = (s < Tx - 1) ? __ldg(a.cc + ((long long)prev * n + eb[i]) * C + dir * D + d) : 0.f;
                        x2[i] = a.mean_grad ? __ldg(a.coef + eb[i]) * __ldg(a.mean_grad + (long long)eb[i] * C + dir * D + d) : 0.f;
                    }
                }
            }
            // K partials of this thread's gate elements, two elements at a time: all their loads are issued before the first
            // tag is looked at (one L2 round trip per pair); a word whose tag is not this step's yet is simply read again.
            // Sums in ascending chunk order: deterministic.
            // With more than two elements per thread (batch 64) the registers do not hold every element's partial words,
            // sums and outputs at once: each pair is then finished (gates + stores) right after its words arrived, and the
            // saved gates are written immediately instead of after the release.
            constexpr bool kDefer = EPT <= 2;
            float o0[kDefer ? EPT : 1], o1[kDefer ? EPT : 1], o2[kDefer ? EPT : 1], o3[kDefer ? EPT : 1];
            auto finish = [&](int i, float s0, float s1, float s2) {
                const long long row = (long long)pos * n + eb[i];
                const int d = dbase + ed[i];
                float q0, q1, q2, q3 = 0.f;
                if (!BWD) {                                                           // nats.py:336-356
                    const float r = sigmoidf_(s0 + x0[i]), u = sigmoidf_(s1 + x1[i]);
                    const float cnd = tanhf(s2 * r + x2[i]);
                    const float hn = u * carry[i] + (1.f - u) * cnd;
                    const float h = mk[i] * hn + (1.f - mk[i]) * carry[i];
                    a.cc[row * C + dir * D + d] = h;
                    a.lo[((long long)(dir * 2 + (s & 1)) * n + eb[i]) * a.Kp + d] = resid(h);
                    carry[i] = h;
                    csum[i] += mk[i] * h;
                    q0 = r; q1 = u; q2 = cnd; q3 = s2;
                } else {                                                              // reverse of the above
                    const float m = mk[i], r = sr_[i], u = su_[i], cnd = sc_[i], pp = sp_[i], hp = x1[i];
                    float dh = x0[i];
                    if (s > 0) { dh += carry[i]; dh += s0; }
                    if (a.mean_grad) dh += m * x2[i];
                    const float dhn = m * dh;
                    const float du = dhn * (hp - cnd);
                    const float dc = dhn * (1.f - u);
                    const float dpc_ = dc * (1.f - cnd * cnd);
                    const float dp = dpc_ * r;
                    const float dr = dpc_ * pp;
                    const float dgr = dr * r * (1.f - r);
                    const float dgu = du * u * (1.f - u);
                    float* g = a.dG[dir] + row * D3 + d;
                    g[0] = dgr; g[D] = dgu; g[2 * D] = dp;
                    float* gl = a.lo + ((long long)(dir * 2 + (s & 1)) * n + eb[i]) * a.Kp + d;
                    gl[0] = resid(dgr); gl[D] = resid(dgu); gl[2 * D] = resid(dp);
                    carry[i] = (1.f - m) * dh + dhn * u;
                    q0 = dgr; q1 = dgu; q2 = dpc_;
                }
                if (kDefer) {
                    o0[kDefer ? i : 0] = q0; o1[kDefer ? i : 0] = q1; o2[kDefer ? i : 0] = q2; o3[kDefer ? i : 0] = q3;
                } else if (!BWD) {
                    if (a.r[dir]) {
                        const long long o = row * D + d;
                        a.r[dir][o] = q0; a.u[dir][o] = q1; a.c[dir][o] = q2; a.p[dir][o] = q3;
                    }
                } else {
                    float* gx = a.dGx[dir] + row * D3 + d;
                    gx[0] = q0; gx[D] = q1; gx[2 * D] = q2;
                }
            };
            if (s > 0) {
                named_bar_sync(2, kMmaThreads + kGateThreads);       // (256 pollers spinning through the whole product would starve the MMA warps' stores)
#pragma unroll
                for (int i0 = 0; i0 < EPT; i0 += 2) {
                    unsigned long long w[2][kMaxWords];
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        if (i0 + j < EPT) {
                            const unsigned long long* rp = slab_tile + (long long)eb[i0 + j] * dpc + crank * dps + ed[i0 + j];
#pragma unroll
                            for (int k = 0; k < kMaxWords; ++k)
                                if (ev[i0 + j] && k < nw) w[j][k] = ld_word(rp + (long long)(k * BN) * dpc);
                        }
                    }
                    const long long t0 = clock64();
                    bool again;
                    do {
                        again = false;
#pragma unroll
                        for (int j = 0; j < 2; ++j) {
                            if (i0 + j < EPT) {
                                const unsigned long long* rp = slab_tile + (long long)eb[i0 + j] * dpc + crank * dps + ed[i0 + j];
#pragma unroll
                                for (int k = 0; k < kMaxWords; ++k)
                                    if (ev[i0 + j] && k < nw && (uint32_t)(w[j][k] >> 32) != (uint32_t)s) {
                                        w[j][k] = ld_word(rp + (long long)(k * BN) * dpc);
                                        again = true;
                                    }
                            }
                        }
                        if (again && clock64() - t0 > kSpinLimit) __trap();
                    } while (again);
                    if (stamp && s == 8 && gtid == 0 && i0 + 2 >= EPT) ENC_STAMP(4);
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        if (i0 + j < EPT && ev[i0 + j]) {
                            float p0 = 0.f, p1 = 0.f, p2 = 0.f;                       // ascending chunk order: deterministic
#pragma unroll
                            for (int k = 0; k < kMaxWords; k += NG) {
                                if (k < nw) {
                                    p0 += __uint_as_float((uint32_t)w[j][k]);
                                    if (NG == 3) {
                                        p1 += __uint_as_float((uint32_t)w[j][k + NG - 2]);
                                        p2 += __uint_as_float((uint32_t)w[j][k + NG - 1]);
                                    }
                                }
                            }
                            finish(i0 + j, p0, p1, p2);
                        }
                    }
                }
            } else {
#pragma unroll
                for (int i = 0; i < EPT; ++i)
                    if (ev[i]) finish(i, 0.f, 0.f, 0.f);
            }
            if (stamp && s == 8 && gtid == 0) ENC_STAMP(9);
            // every gate warp releases its own stores (no CTA-wide barrier in front of the fence): the tile counter counts
            // S * 8 arrivals per step
            __syncwarp();
            if (lane == 0) {
                flag_arrive(tctr);                            // release: cumulative over the warp's stores ordered before __syncwarp
                if (stamp && s == 8 && gtid == 0) ENC_STAMP(5);
            }
            // what no other CTA waits for
            if (kDefer) {
#pragma unroll
                for (int i = 0; i < EPT; ++i) {
                    if (ev[i]) {
                        const long long row = (long long)pos * n + eb[i];
                        const int d = dbase + ed[i];
                        if (!BWD) {
                            if (a.r[dir]) {
                                const long long o = row * D + d;
                                a.r[dir][o] = o0[kDefer ? i : 0]; a.u[dir][o] = o1[kDefer ? i : 0];
                                a.c[dir][o] = o2[kDefer ? i : 0]; a.p[dir][o] = o3[kDefer ? i : 0];
                            }
                        } else {
                            float* gx = a.dGx[dir] + row * D3 + d;
                            gx[0] = o0[kDefer ? i : 0]; gx[D] = o1[kDefer ? i : 0]; gx[2 * D] = o2[kDefer ? i : 0];
                        }
                    }
                }
            }
        }
        if (!BWD && a.ctxsum) {
#pragma unroll
            for (int i = 0; i < EPT; ++i)
                if (ev[i]) a.ctxsum[(long long)eb[i] * C + dir * D + dbase + ed[i]] = csum[i];
        }
    }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_enc = nullptr;
int g_enable = 1;                        // 0 off, 1 both passes, 2 forward only, 3 backward only
size_t g_static_smem = 1024;
int g_resident = -1;                     // CTAs of the largest configuration that fit on one SM (queried once; must be >= 1)

int make_map(const float* ptr, long long inner, long long rows, long long outer, long long row_stride, long long outer_stride,
             int box_rows, CUtensorMap* out) {
    cuuint64_t gdim[3] = {(cuuint64_t)inner, (cuuint64_t)rows, (cuuint64_t)outer};
    cuuint64_t gstr[2] = {(cuuint64_t)row_stride * 4, (cuuint64_t)outer_stride * 4};
    cuuint32_t box[3] = {32, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = g_enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), gdim, gstr, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("enc_tc: cuTensorMapEncodeTiled failed (%d): ptr=%p inner=%lld rows=%lld outer=%lld", (int)r, ptr, inner, rows, outer);
        return 1;
    }
    return 0;
}

struct TcPlan {
    bool ok;
    int BN, NT, S, NG, dpc, dps, Kc, nkbA, NS, Ktot, nwg;
    size_t smem;
    long long slab_floats, lo_floats, counter_ints;
};

// Row tiles of <= 192 rows (forward: 3 gate columns x dpc units; backward: dpc units), K cut into S chunks.  Among the S whose
// weight tile fits next to a ring of at least two stages in shared memory, the one with the fewest k-blocks per CTA wins
// (the k-blocks of a step are a serial chain of MMAs, the exchange words grow only linearly), ties to the smaller S.
TcPlan plan(const nats_ctx* ctx, int n, int D, int pass) {
    TcPlan p;
    memset(&p, 0, sizeof(p));
    if (g_enc == nullptr || n < 1 || n > 64 || D < 96 || (D & 3)) return p;
    p.BN = n <= 32 ? 32 : 64;
    const int per_dir = min(ctx->num_sms / 2, kMaxCtasPerDir);
    const size_t lim = (size_t)ctx->max_smem_optin - g_static_smem - 1024;     // 1 KB: alignment of the dynamic base
    const size_t stage = (size_t)2 * p.BN * 128;
    p.NG = pass == 0 ? 3 : 1;
    p.Ktot = pass == 0 ? D : 3 * D;
    TcPlan best = p;
    for (int S = 2; S <= kMaxWords / p.NG; ++S) {
        const int NT0 = per_dir / S;
        if (NT0 < 1) break;
        const int dpc = (D + NT0 - 1) / NT0;
        const int NT = (D + dpc - 1) / dpc;
        const int rows = p.NG * dpc;
        if (rows > kMaxRows || NT > 32) continue;
        const int dps = (dpc + S - 1) / S;
        if (dps > kMaxDps) continue;
        const int Kc = (((p.Ktot + S - 1) / S + 31) / 32) * 32;
        if (p.Ktot - Kc * (S - 1) < 8) continue;                  // every CTA owns at least one k-step
        const int nwg = (rows + 63) / 64;
        const size_t fixed = (size_t)(Kc / 32) * nwg * 8192;
        if (fixed + 2 * stage > lim) continue;
        if (best.ok && Kc / 32 >= best.nkbA) continue;
        p.S = S; p.NT = NT; p.dpc = dpc; p.dps = dps; p.Kc = Kc; p.nkbA = Kc / 32; p.nwg = nwg;
        p.NS = (int)((lim - fixed) / stage);
        if (p.NS > kMaxNS) p.NS = kMaxNS;
        if (p.NS > p.nkbA) p.NS = max(2, p.nkbA);
        p.smem = fixed + (size_t)p.NS * stage + 1024;
        const long long Kp = (p.Ktot + 3) / 4 * 4;
        p.lo_floats = (4LL * n * Kp + 3) / 4 * 4;
        p.slab_floats = 2LL * (2LL * p.NT * p.S * p.NG * p.BN * p.dpc);      // 64-bit words
        p.counter_ints = 2LL * p.NT * kCtrStride;
        p.ok = true;
        best = p;
    }
    return best;
}

template <int BN, bool BWD>
int launch(cudaStream_t st, const TcPlan& pl, const EncTc& a) {
    enc_tc_kernel<BN, BWD><<<dim3(2 * pl.NT * pl.S), dim3(kThreads), pl.smem, st>>>(a);
    NATS_LAUNCH_OK();
    return 0;
}

}  // namespace

void enc_tc_enable(int on) { g_enable = on; }

int enc_tc_setup(const nats_ctx* ctx) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    NATS_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    if (fn == nullptr || q != cudaDriverEntryPointSuccess) return 0;          // path stays ineligible
    cudaFuncAttributes fa;
    size_t st = 0;
    NATS_CUDA_OK(cudaFuncGetAttributes(&fa, enc_tc_kernel<32, false>)); st = st > fa.sharedSizeBytes ? st : fa.sharedSizeBytes;
    NATS_CUDA_OK(cudaFuncGetAttributes(&fa, enc_tc_kernel<64, false>)); st = st > fa.sharedSizeBytes ? st : fa.sharedSizeBytes;
    NATS_CUDA_OK(cudaFuncGetAttributes(&fa, enc_tc_kernel<32, true>)); st = st > fa.sharedSizeBytes ? st : fa.sharedSizeBytes;
    NATS_CUDA_OK(cudaFuncGetAttributes(&fa, enc_tc_kernel<64, true>)); st = st > fa.sharedSizeBytes ? st : fa.sharedSizeBytes;
    g_static_smem = st;
    const int dyn = ctx->max_smem_optin - (int)g_static_smem;
    NATS_CUDA_OK(cudaFuncSetAttribute(enc_tc_kernel<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
    NATS_CUDA_OK(cudaFuncSetAttribute(enc_tc_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
    NATS_CUDA_OK(cudaFuncSetAttribute(enc_tc_kernel<32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
    NATS_CUDA_OK(cudaFuncSetAttribute(enc_tc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
    int r = 0;
    NATS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&r, enc_tc_kernel<32, false>, kThreads, dyn));
    g_resident = r;
    g_enc = reinterpret_cast<EncodeTiledFn>(fn);
    return 0;
}

// pass: 0 forward, 1 backward
bool enc_tc_eligible(const nats_ctx* ctx, int n, int D, int pass) {
    if (!(g_enable == 1 || (g_enable == 2 && pass == 0) || (g_enable == 3 && pass == 1))) return false;
    if (g_resident < 1) return false;
    const TcPlan p = plan(ctx, n, D, pass);
    return p.ok && 2 * p.NT * p.S <= ctx->num_sms;           // one CTA per SM, all co-resident
}

// upper bounds that do not depend on the device (workspace carving happens without a context):
// residual side buffer 4*n*(3D+4) floats + K-partial words: 2 directions x <= 74 CTAs x 192 rows x BN batch columns
long long enc_tc_scratch_floats(int n, int D) {
    const long long BN = n <= 32 ? 32 : 64;
    return 4LL * n * (3LL * D + 4) + 2LL * (2LL * kMaxCtasPerDir * kMaxRows * BN) + 64;
}
long long enc_tc_counter_ints() { return 2LL * 32 * kCtrStride + 64; }

int enc_tc_fwd(const nats_ctx* ctx, cudaStream_t st, const EncTcFwdArgs& g) {
    const TcPlan pl = plan(ctx, g.n, g.D, 0);
    NATS_REQUIRE(pl.ok && 2 * pl.NT * pl.S <= ctx->num_sms, "tensor-core persistent encoder not applicable");
    NATS_REQUIRE((reinterpret_cast<uintptr_t>(g.cc) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.scratch) & 15) == 0, "alignment");
    NATS_REQUIRE(g.scratch_floats >= pl.lo_floats + pl.slab_floats && g.bar_ints >= pl.counter_ints, "scratch size");
    EncTc a;
    memset(&a, 0, sizeof(a));
    const int D = g.D, n = g.n, Kp = (D + 3) / 4 * 4;
    for (int d = 0; d < 2; ++d) {
        a.Ucat[d] = g.Ucat[d]; a.xproj[d] = g.xproj[d];
        a.r[d] = g.r[d]; a.u[d] = g.u[d]; a.c[d] = g.c[d]; a.p[d] = g.p[d];
        NATS_TRY(make_map(g.cc + (long long)d * D, D, n, g.Tx, 2LL * D, 2LL * D * n, pl.BN, &a.map_raw[d]));
        NATS_TRY(make_map(g.scratch + (long long)d * 2 * n * Kp, D, n, 2, Kp, (long long)n * Kp, pl.BN, &a.map_lo[d]));
    }
    a.mask = g.mask; a.cc = g.cc; a.lo = g.scratch; a.slab = reinterpret_cast<unsigned long long*>(g.scratch + pl.lo_floats); a.ctxsum = g.ctxsum; a.bar = g.bar; a.dbg = g.dbg;
    a.Tx = g.Tx; a.n = n; a.D = D; a.Kp = Kp;
    a.NT = pl.NT; a.S = pl.S; a.dpc = pl.dpc; a.dps = pl.dps; a.Kc = pl.Kc; a.nkbA = pl.nkbA; a.NS = pl.NS; a.nwg = pl.nwg;
    NATS_CUDA_OK(memset_async(st, g.bar, 0, (size_t)pl.counter_ints * sizeof(unsigned)));
    NATS_CUDA_OK(memset_async(st, g.scratch + pl.lo_floats, 0xff, (size_t)pl.slab_floats * sizeof(float)));     // no stale step tags
    ProfScope ps(st, K_ENC_PERSIST_FWD, 2.0 * 2 * g.Tx * (double)n * 3.0 * D * D, 4.0 * 2 * 3.0 * D * D);
    return pl.BN == 32 ? launch<32, false>(st, pl, a) : launch<64, false>(st, pl, a);
}

int enc_tc_bwd(const nats_ctx* ctx, cudaStream_t st, const EncTcBwdArgs& g) {
    const TcPlan pl = plan(ctx, g.n, g.D, 1);
    NATS_REQUIRE(pl.ok && 2 * pl.NT * pl.S <= ctx->num_sms, "tensor-core persistent encoder (backward) not applicable");
    NATS_REQUIRE((reinterpret_cast<uintptr_t>(g.dG[0]) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.dG[1]) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(g.scratch) & 15) == 0, "alignment");
    NATS_REQUIRE(g.scratch_floats >= pl.lo_floats + pl.slab_floats && g.bar_ints >= pl.counter_ints, "scratch size");
    EncTc a;
    memset(&a, 0, sizeof(a));
    const int D = g.D, n = g.n, K = 3 * D, Kp = (K + 3) / 4 * 4;
    for (int d = 0; d < 2; ++d) {
        a.Ucat[d] = g.Ucat[d];
        a.r[d] = const_cast<float*>(g.r[d]); a.u[d] = const_cast<float*>(g.u[d]);
        a.c[d] = const_cast<float*>(g.c[d]); a.p[d] = const_cast<float*>(g.p[d]);
        a.dG[d] = g.dG[d]; a.dGx[d] = g.dGx[d];
        NATS_TRY(make_map(g.dG[d], K, n, g.Tx, K, (long long)K * n, pl.BN, &a.map_raw[d]));
        NATS_TRY(make_map(g.scratch + (long long)d * 2 * n * Kp, K, n, 2, Kp, (long long)n * Kp, pl.BN, &a.map_lo[d]));
    }
    a.mask = g.mask; a.cc = const_cast<float*>(g.cc); a.dcc = g.dcc; a.mean_grad = g.mean_grad; a.coef = g.coef;
    a.lo = g.scratch; a.slab = reinterpret_cast<unsigned long long*>(g.scratch + pl.lo_floats); a.bar = g.bar; a.dbg = g.dbg;
    a.Tx = g.Tx; a.n = n; a.D = D; a.Kp = Kp;
    a.NT = pl.NT; a.S = pl.S; a.dpc = pl.dpc; a.dps = pl.dps; a.Kc = pl.Kc; a.nkbA = pl.nkbA; a.NS = pl.NS; a.nwg = pl.nwg;
    NATS_CUDA_OK(memset_async(st, g.bar, 0, (size_t)pl.counter_ints * sizeof(unsigned)));
    NATS_CUDA_OK(memset_async(st, g.scratch + pl.lo_floats, 0xff, (size_t)pl.slab_floats * sizeof(float)));     // no stale step tags
    ProfScope ps(st, K_ENC_PERSIST_BWD, 2.0 * 2 * g.Tx * (double)n * 3.0 * D * D, 4.0 * 2 * 3.0 * D * D);
    return pl.BN == 32 ? launch<32, true>(st, pl, a) : launch<64, true>(st, pl, a);
}

}  // namespace nats
