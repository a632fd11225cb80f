// CMA-ES rank-mu covariance update (the arithmetic inside es.tell, cma_es.py:90; Hansen tutorial
// arXiv:1604.00772 eq. 47):   dC = sum_i w_i y_i y_i^T = Y^T diag(w) Y,    C <- decay*C + c1 pc pc^T + cmu dC
//
// SYRK-shaped: only tiles on or above the diagonal are computed and mirrored on store.  fp32 FFMA
// (the 1e-5 parity bar rules out single-pass TF32/BF16 tensor cores here; see DESIGN.md), register
// micro-tiles fed from shared memory, k-panels of 16 members.
// Bound: CUDA-core FMA, lambda*n*(n+tile) flop with symmetry; traffic 4*lambda*n (Y) + 4*n*n (dC).
#include "des_common.cuh"

namespace des {

constexpr int kCmaThreads = 256;
constexpr int kCmaKP = 16;   // members per k-panel
constexpr int kCmaTile = 64; // output tile side; the kernel runs for n < kCmaTcMinN, where it is the packed tile side
static_assert(cma_packed_tile(kCmaTcMinN - 1) == kCmaTile, "packed output of the FFMA kernel needs tiles of its side");

// 64 x 64 outputs per CTA, 256 threads as 16 x 16.  Each thread owns a 4 x 4 block (rows ty*4 + {0..3}, columns
// tx*4 + {0..3}), so every shared-memory operand read is one conflict-free LDS.128.  k-panels of 16 members are double
// buffered: the next panel's global loads are in flight while the current one is multiplied.
// The body of the kernel, shared with the run-batched kernel (des_cma_rank_mu_runs): dC, Y and w are the CTA's run's.
__device__ __forceinline__ void cma_rank_mu_tile(float *__restrict__ dC, const float *__restrict__ Y,
                                                 const float *__restrict__ w, int64_t lambda, int64_t n, int tiles_per_side,
                                                 int packed) {
    constexpr int MT = 4;
    constexpr int LD = kCmaKP * kCmaTile / kCmaThreads;   // elements each thread stages per operand and panel
    __shared__ __align__(16) float As[2][kCmaKP][kCmaTile];   // w_k * Y[k][i0 + i]
    __shared__ __align__(16) float Bs[2][kCmaKP][kCmaTile];   //       Y[k][j0 + j]
    int bi = 0, rem = blockIdx.x;
    while (rem >= tiles_per_side - bi) { rem -= tiles_per_side - bi; ++bi; }
    const int bj = bi + rem;
    const int64_t i0 = (int64_t)bi * kCmaTile, j0 = (int64_t)bj * kCmaTile;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;

    float acc[MT][MT];
#pragma unroll
    for (int a = 0; a < MT; ++a)
#pragma unroll
        for (int b = 0; b < MT; ++b) acc[a][b] = 0.f;

    float ra[LD], rb[LD];
    auto fetch = [&](int64_t k0) {
#pragma unroll
        for (int e = 0; e < LD; ++e) {
            const int idx = threadIdx.x + e * kCmaThreads;
            const int kk = idx / kCmaTile, c = idx - kk * kCmaTile;
            const int64_t k = k0 + kk;
            float a = 0.f, b = 0.f;
            if (k < lambda) {
                const float wk = __ldg(w + k);
                if (i0 + c < n) a = wk * __ldg(Y + k * n + i0 + c);
                if (j0 + c < n) b = __ldg(Y + k * n + j0 + c);
            }
            ra[e] = a;
            rb[e] = b;
        }
    };
    auto stage = [&](int buf) {
#pragma unroll
        for (int e = 0; e < LD; ++e) {
            const int idx = threadIdx.x + e * kCmaThreads;
            const int kk = idx / kCmaTile, c = idx - kk * kCmaTile;
            As[buf][kk][c] = ra[e];
            Bs[buf][kk][c] = rb[e];
        }
    };
    fetch(0);
    stage(0);
    __syncthreads();
    int buf = 0;
    for (int64_t k0 = 0; k0 < lambda; k0 += kCmaKP) {
        const bool more = k0 + kCmaKP < lambda;
        if (more) fetch(k0 + kCmaKP);            // global loads overlap the multiply below
#pragma unroll
        for (int kk = 0; kk < kCmaKP; ++kk) {
            const float4 a4 = *reinterpret_cast<const float4 *>(&As[buf][kk][ty * 4]);
            const float4 b4 = *reinterpret_cast<const float4 *>(&Bs[buf][kk][tx * 4]);
            const float av[MT] = {a4.x, a4.y, a4.z, a4.w}, bv[MT] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int a = 0; a < MT; ++a)
#pragma unroll
                for (int b = 0; b < MT; ++b) acc[a][b] = __fmaf_rn(av[a], bv[b], acc[a][b]);
        }
        if (more) {
            stage(buf ^ 1);
            __syncthreads();
            buf ^= 1;
        }
    }
    if (packed) {
        // upper-triangular tiles only, tile after tile ([tile][64][64], the collective's payload: half the bytes of
        // the full matrix); entries beyond n are zero so that partial sums of different ranks can be added blindly
        float *tile = dC + (int64_t)blockIdx.x * kCmaTile * kCmaTile;
        const int lj = tx * 4;
#pragma unroll
        for (int a = 0; a < MT; ++a) {
            const int li = ty * 4 + a;
            float4 v = make_float4(acc[a][0], acc[a][1], acc[a][2], acc[a][3]);
            if (i0 + li >= n) v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (j0 + lj + 0 >= n) v.x = 0.f;
            if (j0 + lj + 1 >= n) v.y = 0.f;
            if (j0 + lj + 2 >= n) v.z = 0.f;
            if (j0 + lj + 3 >= n) v.w = 0.f;
            *reinterpret_cast<float4 *>(tile + li * kCmaTile + lj) = v;
        }
        return;
    }
#pragma unroll
    for (int a = 0; a < MT; ++a) {
        const int64_t i = i0 + ty * 4 + a;
#pragma unroll
        for (int b = 0; b < MT; ++b) {
            const int64_t j = j0 + tx * 4 + b;
            if (i < n && j < n) {
                if (bi != bj) {
                    dC[i * n + j] = acc[a][b];
                    dC[j * n + i] = acc[a][b];
                } else if (j >= i) {
                    // diagonal tile: (i,j) and (j,i) are both computed; keep the j >= i one for exact symmetry
                    dC[i * n + j] = acc[a][b];
                    dC[j * n + i] = acc[a][b];
                }
            }
        }
    }
}

__global__ void __launch_bounds__(kCmaThreads) cma_rank_mu_kernel(float *__restrict__ dC, const float *__restrict__ Y,
                                                                  const float *__restrict__ w, int64_t lambda, int64_t n,
                                                                  int tiles_per_side, int packed) {
    cma_rank_mu_tile(dC, Y, w, lambda, n, tiles_per_side, packed);
}

// A batch of runs (des_cma_rank_mu_runs): CTA row y is run y's cma_rank_mu_kernel, full matrix, on its rows of dC, Y, w.
__global__ void __launch_bounds__(kCmaThreads) cma_rank_mu_runs_kernel(float *__restrict__ dC, const float *__restrict__ Y,
                                                                       const float *__restrict__ w, int64_t lambda,
                                                                       int64_t n, int tiles_per_side) {
    const int64_t run = blockIdx.y;
    cma_rank_mu_tile(dC + run * n * n, Y + run * lambda * n, w + run * lambda, lambda, n, tiles_per_side, 0);
}

// The covariance update of one entry, shared with the run-batched kernel (des_cma_cov_apply_runs).
__device__ __forceinline__ void cma_cov_apply_at(float *__restrict__ C, const float *__restrict__ dC,
                                                 const float *__restrict__ pc, int64_t n, float decay, float c1, float cmu) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * n) return;
    const int64_t i = idx / n, j = idx - i * n;
    float v = decay * C[idx];
    if (pc) v = __fmaf_rn(c1 * __ldg(pc + i), __ldg(pc + j), v);
    C[idx] = __fmaf_rn(cmu, dC[idx], v);
}

__global__ void cma_cov_apply_kernel(float *__restrict__ C, const float *__restrict__ dC, const float *__restrict__ pc,
                                     int64_t n, float decay, float c1, float cmu) {
    cma_cov_apply_at(C, dC, pc, n, decay, c1, cmu);
}

// A batch of runs (des_cma_cov_apply_runs): CTA row y updates run y's C with its dC, pc and decay; decay is converted to
// fp32 as the host converts the single call's.
__global__ void cma_cov_runs_kernel(float *__restrict__ C, const float *__restrict__ dC, const float *__restrict__ pc,
                                          const double *__restrict__ decay, int64_t n, float c1, float cmu) {
    const int64_t run = blockIdx.y;
    cma_cov_apply_at(C + run * n * n, dC + run * n * n, pc ? pc + run * n : nullptr, n, (float)decay[run], c1, cmu);
}

// C <- decay*C + c1 pc pc^T + cmu*dC with dC given as packed upper-triangular tiles (cma_rank_mu_kernel, packed = 1).
// One CTA per 64 x 64 block of an upper tile: the block is staged in shared memory, applied to C[i-block][j-block] and,
// transposed, to C[j-block][i-block] — both coalesced.  Diagonal blocks take the j >= i entry for both sides, so C stays
// exactly symmetric.
template <int TILE>
__global__ void __launch_bounds__(256) cma_cov_apply_packed_kernel(float *__restrict__ C, const float *__restrict__ tiles,
                                                                   const float *__restrict__ pc, int64_t n, float decay,
                                                                   float c1, float cmu, int tiles_per_side) {
    constexpr int SB = TILE / 64;                     // 64 x 64 sub-blocks per tile side
    __shared__ float blk[64][65];
    int bi = 0, rem = blockIdx.x / (SB * SB);
    while (rem >= tiles_per_side - bi) { rem -= tiles_per_side - bi; ++bi; }
    const int bj = bi + rem;
    const int sub = blockIdx.x % (SB * SB), si = sub / SB, sj = sub % SB;
    const float *tile = tiles + (int64_t)(blockIdx.x / (SB * SB)) * TILE * TILE;
    const int64_t i0 = (int64_t)bi * TILE + si * 64, j0 = (int64_t)bj * TILE + sj * 64;
    if (bi == bj && sj < si) return;                  // lower sub-block of a diagonal tile: written by its mirror
    const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;       // 64 x 4
    for (int r = ty; r < 64; r += 4) blk[r][tx] = tile[(si * 64 + r) * TILE + sj * 64 + tx];
    __syncthreads();
    const bool diag = (i0 == j0);
    for (int r = ty; r < 64; r += 4) {                // C[i0 + r][j0 + tx]
        const int64_t i = i0 + r, j = j0 + tx;
        if (i < n && j < n) {
            const float d = diag ? blk[min(r, tx)][max(r, tx)] : blk[r][tx];
            float v = decay * C[i * n + j];
            if (pc) v = __fmaf_rn(c1 * __ldg(pc + i), __ldg(pc + j), v);
            C[i * n + j] = __fmaf_rn(cmu, d, v);
        }
    }
    if (!diag) {
        for (int r = ty; r < 64; r += 4) {            // mirror: C[j0 + r][i0 + tx] = f(blk[tx][r])
            const int64_t i = j0 + r, j = i0 + tx;
            if (i < n && j < n) {
                float v = decay * C[i * n + j];
                if (pc) v = __fmaf_rn(c1 * __ldg(pc + i), __ldg(pc + j), v);
                C[i * n + j] = __fmaf_rn(cmu, blk[tx][r], v);
            }
        }
    }
}

}  // namespace des

extern "C" DES_API int64_t des_cma_packed_elems(int64_t n) {
    if (n <= 0) return 0;
    const int64_t tile = des::cma_packed_tile(n), t = (n + tile - 1) / tile;
    return t * (t + 1) / 2 * tile * tile;
}

extern "C" DES_API size_t des_cma_rank_mu_workspace_bytes(int64_t n, int64_t lambda_local) {
    return n >= des::kCmaTcMinN && lambda_local > 0 ? des::cma_tc_workspace_bytes(n, lambda_local) : 0;
}

extern "C" DES_API int des_cma_rank_mu(float *out_dev, const float *Y_dev, const float *w_dev, int64_t lambda_local, int64_t n,
                                       int packed, void *workspace_dev, size_t workspace_bytes, void *stream) {
    using namespace des;
    DES_REQUIRE(n > 0 && lambda_local >= 0, "des_cma_rank_mu: bad sizes lambda=%lld n=%lld", (long long)lambda_local,
                (long long)n);
    DES_REQUIRE(n <= 46340 * 16, "des_cma_rank_mu: n too large");
    DES_REQUIRE(out_dev && (lambda_local == 0 || (Y_dev && w_dev)), "des_cma_rank_mu: NULL pointer");
    const size_t need = des_cma_rank_mu_workspace_bytes(n, lambda_local);
    if (need && (!workspace_dev || workspace_bytes < need)) {
        set_error("des_cma_rank_mu: workspace %zu B < required %zu B", workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (lambda_local == 0) {
        const size_t elems = packed ? (size_t)des_cma_packed_elems(n) : (size_t)n * n;
        DES_CUDA(cudaMemsetAsync(out_dev, 0, elems * sizeof(float), st));
        return DES_OK;
    }
    if (n >= kCmaTcMinN) return cma_rank_mu_tc(out_dev, Y_dev, w_dev, lambda_local, n, packed, workspace_dev, st);
    const int t = (int)((n + kCmaTile - 1) / kCmaTile);
    cma_rank_mu_kernel<<<(unsigned)(t * (t + 1) / 2), kCmaThreads, 0, st>>>(out_dev, Y_dev, w_dev, lambda_local, n, t,
                                                                            packed ? 1 : 0);
    DES_LAUNCH_CHECK("cma_rank_mu_kernel");
    return DES_OK;
}

extern "C" DES_API int des_cma_cov_apply_packed(float *C_dev, const float *tiles_dev, const float *pc_dev, int64_t n, double decay,
                                                double c1, double cmu, void *stream) {
    using namespace des;
    DES_REQUIRE(n > 0, "des_cma_cov_apply_packed: n=%lld", (long long)n);
    DES_REQUIRE(C_dev && tiles_dev, "des_cma_cov_apply_packed: NULL pointer");
    const int tile = cma_packed_tile(n), t = (int)((n + tile - 1) / tile);
    const unsigned upper = (unsigned)(t * (t + 1) / 2);
    if (tile == 64)
        cma_cov_apply_packed_kernel<64><<<upper, 256, 0, (cudaStream_t)stream>>>(C_dev, tiles_dev, pc_dev, n, (float)decay, (float)c1, (float)cmu, t);
    else
        cma_cov_apply_packed_kernel<128><<<upper * 4, 256, 0, (cudaStream_t)stream>>>(C_dev, tiles_dev, pc_dev, n, (float)decay, (float)c1, (float)cmu, t);
    DES_LAUNCH_CHECK("cma_cov_apply_packed_kernel");
    return DES_OK;
}

extern "C" DES_API int des_cma_cov_apply(float *C_dev, const float *dC_dev, const float *pc_dev, int64_t n, double decay, double c1,
                                 double cmu, void *stream) {
    using namespace des;
    DES_REQUIRE(n > 0, "des_cma_cov_apply: n=%lld", (long long)n);
    DES_REQUIRE(C_dev && dC_dev, "des_cma_cov_apply: NULL pointer");
    const int64_t total = n * n;
    cma_cov_apply_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(C_dev, dC_dev, pc_dev, n,
                                                                                          (float)decay, (float)c1, (float)cmu);
    DES_LAUNCH_CHECK("cma_cov_apply_kernel");
    return DES_OK;
}

// ---- batches of runs: run r's Y, w, C, dC and pc are row r of [n_runs][...] arrays ----------------------------------------

extern "C" DES_API size_t des_cma_rank_mu_runs_workspace_bytes(int64_t n_runs, int64_t lambda, int64_t n) {
    return n_runs > 0 ? des_cma_rank_mu_workspace_bytes(n, lambda) : 0;      // the tensor-core runs reuse one workspace
}

extern "C" DES_API int des_cma_rank_mu_runs(float *out_dev, const float *Y_dev, const float *w_dev, int64_t n_runs,
                                            int64_t lambda, int64_t n, void *workspace_dev, size_t workspace_bytes,
                                            void *stream) {
    using namespace des;
    const char *who = "des_cma_rank_mu_runs";
    DES_REQUIRE(n_runs >= 0 && lambda >= 0 && n > 0, "%s: bad sizes n_runs=%lld lambda=%lld n=%lld", who,
                (long long)n_runs, (long long)lambda, (long long)n);
    DES_REQUIRE(n <= 46340 * 16, "%s: n too large", who);
    DES_REQUIRE(n_runs <= ((int64_t)1 << 40) / (n * n) && lambda <= ((int64_t)1 << 40) / n / (n_runs > 0 ? n_runs : 1),
                "%s: n_runs x n x n or n_runs x lambda x n (%lld, %lld, %lld) floats past 2^40", who, (long long)n_runs,
                (long long)lambda, (long long)n);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(out_dev && (lambda == 0 || (Y_dev && w_dev)), "%s: NULL pointer", who);
    const size_t need = des_cma_rank_mu_runs_workspace_bytes(n_runs, lambda, n);
    if (need && (!workspace_dev || workspace_bytes < need)) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (lambda == 0) {
        DES_CUDA(cudaMemsetAsync(out_dev, 0, (size_t)n_runs * n * n * sizeof(float), st));
        return DES_OK;
    }
    if (n >= kCmaTcMinN) {                 // one tensor-core SYRK per run, one workspace reused in stream order
        for (int64_t r = 0; r < n_runs; ++r) {
            const int rc = cma_rank_mu_tc(out_dev + r * n * n, Y_dev + r * lambda * n, w_dev + r * lambda, lambda, n, 0,
                                          workspace_dev, st);
            if (rc != DES_OK) return rc;
        }
        return DES_OK;
    }
    const int t = (int)((n + kCmaTile - 1) / kCmaTile);
    for (int64_t r0 = 0; r0 < n_runs; r0 += 65535) {            // grid y: up to 65535 runs per launch
        const int64_t nr = n_runs - r0 < 65535 ? n_runs - r0 : 65535;
        cma_rank_mu_runs_kernel<<<dim3((unsigned)(t * (t + 1) / 2), (unsigned)nr), kCmaThreads, 0, st>>>(
            out_dev + r0 * n * n, Y_dev + r0 * lambda * n, w_dev + r0 * lambda, lambda, n, t);
        DES_LAUNCH_CHECK("cma_rank_mu_runs_kernel");
    }
    return DES_OK;
}

extern "C" DES_API int des_cma_cov_apply_runs(float *C_dev, const float *dC_dev, const float *pc_dev,
                                              const double *decay_dev, double c1, double cmu, int64_t n_runs, int64_t n,
                                              void *stream) {
    using namespace des;
    const char *who = "des_cma_cov_apply_runs";
    DES_REQUIRE(n_runs >= 0 && n > 0, "%s: bad sizes n_runs=%lld n=%lld", who, (long long)n_runs, (long long)n);
    DES_REQUIRE(n <= 46340 * 16 && n_runs <= ((int64_t)1 << 40) / (n * n), "%s: n_runs x n x n past 2^40", who);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(C_dev && dC_dev && decay_dev, "%s: NULL pointer", who);
    const int64_t blocks = (n * n + 255) / 256;
    for (int64_t r0 = 0; r0 < n_runs; r0 += 65535) {            // grid y: up to 65535 runs per launch
        const int64_t nr = n_runs - r0 < 65535 ? n_runs - r0 : 65535;
        cma_cov_runs_kernel<<<dim3((unsigned)blocks, (unsigned)nr), 256, 0, (cudaStream_t)stream>>>(
            C_dev + r0 * n * n, dC_dev + r0 * n * n, pc_dev ? pc_dev + r0 * n : nullptr, decay_dev + r0, n, (float)c1,
            (float)cmu);
        DES_LAUNCH_CHECK("cma_cov_runs_kernel");
    }
    return DES_OK;
}
