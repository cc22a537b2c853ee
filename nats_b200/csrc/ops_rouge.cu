// ops_rouge.cu -- ROUGE-1 / ROUGE-2 / ROUGE-L F of token-id sequences (the scores of nats_b200/evaluate.py, the rules of
// ROUGE.pl without its 5-decimal rounding), one CTA per candidate row.  Integer counting throughout; the one division
// is the F value itself, so the result is exactly (float)(2 h) / (float)(m + c).
#include "ops.cuh"

namespace nats {

namespace {

constexpr int kRougeThreads = 256;
constexpr int kUnk = 1;

// hits of candidate n-gram i (N = 1 or 2): it is a hit when its rank among the equal candidate n-grams before it is
// below its count in the reference -- summed over i this is ROUGE.pl's clipped sum_g min(c_ref(g), c_cand(g)).
// An n-gram holding UNK matches nothing.
template <int N>
__device__ int ngram_hits(const int* __restrict__ a, int m, const int* __restrict__ b, int c) {
    const int nm = m - N + 1, nc = c - N + 1;
    int hits = 0;
    for (int i = threadIdx.x; i < nc; i += blockDim.x) {
        const int g0 = b[i], g1 = N == 2 ? b[i + 1] : 0;
        if (g0 == kUnk || (N == 2 && g1 == kUnk)) continue;
        int rank = 0;
        for (int k = 0; k < i; ++k) rank += (b[k] == g0 && (N == 1 || b[k + 1] == g1)) ? 1 : 0;
        int cnt = 0;
        for (int j = 0; j < nm && cnt <= rank; ++j) cnt += (a[j] == g0 && (N == 1 || a[j + 1] == g1)) ? 1 : 0;
        hits += rank < cnt ? 1 : 0;
    }
    return hits;
}

__device__ __forceinline__ float rouge_fval(int h, int m, int c) {
    return h == 0 ? 0.f : (float)(2 * h) / (float)(m + c);
}

// shared memory: ref [ref_cap] | cand [cand_cap] | three LCS anti-diagonals [ref_cap + 1] each
__global__ void __launch_bounds__(kRougeThreads) rouge_kernel(const int32_t* __restrict__ cand, int cand_cap,
                                                              const int32_t* __restrict__ cand_len, int n,
                                                              const int32_t* __restrict__ ref, int ref_cap,
                                                              const int32_t* __restrict__ ref_len, int rows_per_ref,
                                                              float* __restrict__ out) {
    extern __shared__ int sm[];
    __shared__ int s_m, s_c, s_hit[2];
    int* a = sm;
    int* b = a + ref_cap;
    int* dg = b + cand_cap;
    const int ld = ref_cap + 1;
    const int r = blockIdx.x, q = r / rows_per_ref, tid = threadIdx.x;
    const int32_t* ar = ref + (long long)q * ref_cap;
    const int32_t* br = cand + (long long)r * cand_cap;
    const int lm = min(max(ref_len[q], 0), ref_cap);          // device lengths are clamped: no index leaves the row
    const int lc = min(max(cand_len[r], 0), cand_cap);
    if (tid == 0) { s_m = lm; s_c = lc; s_hit[0] = 0; s_hit[1] = 0; }
    for (int i = tid; i < 3 * ld; i += blockDim.x) dg[i] = 0;
    __syncthreads();
    for (int i = tid; i < lm; i += blockDim.x) {
        const int v = ar[i];
        a[i] = v;
        if (v == 0) atomicMin(&s_m, i);                        // the words end at the first EOS
    }
    for (int i = tid; i < lc; i += blockDim.x) {
        const int v = br[i];
        b[i] = v;
        if (v == 0) atomicMin(&s_c, i);
    }
    __syncthreads();
    const int m = s_m, c = s_c;
    const int h1 = ngram_hits<1>(a, m, b, c);
    const int h2 = ngram_hits<2>(a, m, b, c);
    if (h1) atomicAdd(&s_hit[0], h1);                          // integer sums: exact in any order
    if (h2) atomicAdd(&s_hit[1], h2);
    // LCS by anti-diagonals d = i + j of the table L[i][j] (i over the reference, j over the candidate); L[0][.] =
    // L[.][0] = 0.  Diagonal d lives in dg[(d % 3) * ld + i]; one barrier per diagonal.
    for (int d = 2; d <= m + c; ++d) {
        int* cur = dg + (d % 3) * ld;
        const int* p1 = dg + ((d - 1) % 3) * ld;
        const int* p2 = dg + ((d - 2) % 3) * ld;
        const int lo = max(1, d - c), hi = min(m, d - 1);
        for (int i = lo + tid; i <= hi; i += blockDim.x) {
            const int j = d - i;
            const int ai = a[i - 1];
            int v;
            if (ai == b[j - 1] && ai != kUnk) {
                v = ((i > 1 && j > 1) ? p2[i - 1] : 0) + 1;
            } else {
                const int up = i > 1 ? p1[i - 1] : 0, left = j > 1 ? p1[i] : 0;
                v = up > left ? up : left;
            }
            cur[i] = v;
        }
        __syncthreads();
    }
    __syncthreads();
    if (tid == 0) {
        const int lcs = (m > 0 && c > 0) ? dg[((m + c) % 3) * ld + m] : 0;
        out[r] = rouge_fval(s_hit[0], m, c);
        out[(long long)n + r] = rouge_fval(s_hit[1], max(0, m - 1), max(0, c - 1));
        out[2LL * n + r] = rouge_fval(lcs, m, c);
    }
}

}  // namespace

int rouge_f(cudaStream_t st, const int32_t* cand, int cand_cap, const int32_t* cand_len, int n, const int32_t* ref,
            int ref_cap, const int32_t* ref_len, int rows_per_ref, float* out) {
    NATS_REQUIRE(n >= 1 && rows_per_ref >= 1 && cand_cap >= 1 && ref_cap >= 1, "rouge_f shape");
    NATS_REQUIRE(cand_cap + ref_cap <= kRougeMaxCap, "rouge_f: ref_cap + cand_cap must be <= 4096");
    const size_t smem = (size_t)(cand_cap + ref_cap + 3 * (ref_cap + 1)) * sizeof(int);
    if (smem > 48 * 1024) {
        NATS_CUDA_OK(cudaFuncSetAttribute(rouge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    ProfScope ps(st, K_ROUGE, 0.0, 4.0 * ((double)n * cand_cap + (double)(n / rows_per_ref) * ref_cap));
    rouge_kernel<<<n, kRougeThreads, smem, st>>>(cand, cand_cap, cand_len, n, ref, ref_cap, ref_len, rows_per_ref, out);
    NATS_LAUNCH_OK();
    return 0;
}

}  // namespace nats
