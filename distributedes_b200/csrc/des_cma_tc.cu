// CMA-ES rank-mu covariance term on the tensor cores:  dC = sum_k w_k y_k y_k^T = Y^T diag(w) Y   (the arithmetic inside
// es.tell, cma_es.py:90; Hansen tutorial arXiv:1604.00772 eq. 47) as a symmetric rank-k update with split-fp16 operands.
//
//   Z  = diag(sqrt|w|) Y           (so that dC = Zs^T Z with Zs = diag(sign w) Z; both operands are O(|y|): no scaling)
//   pre-pass   Y [lambda][n] fp32 -> Zs_hi, Zs_lo, Z_hi, Z_lo  [n][lambda_pad] fp16, k contiguous (K-major), x = hi + lo
//   main       per 128 x 128 output tile touching the upper triangle:  D += A_hi B_hi^T + A_lo B_hi^T + A_hi B_lo^T
//              (wgmma m64n128k16, fp32 accumulation in registers; the dropped lo*lo term is 2^-22 relative), operand
//              tiles brought in by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B) through a three-stage mbarrier pipeline:
//              warps 0-7 = two consumer warpgroups (64 output rows each: wgmma, then registers -> global), warp 8 = TMA
//   output     the full symmetric matrix (upper entry written to both sides: exactly symmetric), or the packed
//              upper-triangular tiles (the payload of the cross-rank sum)
//
// des_cma_rank_mu (des_cma.cu) runs this for n >= kCmaTcMinN and the fp32 FFMA kernel below that.
// Accuracy: measured against the fp64 restatement in tests/test_gpu_cma.py at the same 1e-5 (both norms) bar.
#include <cuda.h>
#include <stddef.h>
#include "des_common.cuh"
#include "des_tc.cuh"

namespace des {
namespace cmatc {

using namespace tc;

constexpr int kBM = 128, kBN = 128, kBK = 64;
constexpr int kStages = 3;
constexpr int kABytes = kBM * kBK * 2, kBBytes = kBN * kBK * 2;
constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;             // A_hi | A_lo | B_hi | B_lo = 64 KB
constexpr int kThreads = 9 * 32;

// ---- pre-pass: transpose + scale + split --------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cma_split_kernel(__half *__restrict__ zs_hi, __half *__restrict__ zs_lo,
                                                        __half *__restrict__ z_hi, __half *__restrict__ z_lo,
                                                        const float *__restrict__ Y, const float *__restrict__ w,
                                                        int64_t lambda, int64_t lambda_pad, int64_t n) {
    __shared__ float tile[32][33];
    __shared__ float sgn[32];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8
    const int64_t k0 = (int64_t)blockIdx.y * 32, j0 = (int64_t)blockIdx.x * 32;
    for (int r = ty; r < 32; r += 8) {
        const int64_t k = k0 + r, j = j0 + tx;
        float v = 0.f;
        if (k < lambda && j < n) v = sqrtf(fabsf(__ldg(w + k))) * __ldg(Y + k * n + j);
        tile[r][tx] = v;
    }
    if (threadIdx.x < 32) sgn[threadIdx.x] = (k0 + threadIdx.x < lambda && __ldg(w + k0 + threadIdx.x) < 0.f) ? -1.f : 1.f;
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {                               // row j0 + r of the outputs, k = k0 + tx
        const int64_t j = j0 + r, k = k0 + tx;
        if (j < n && k < lambda_pad) {
            const float z = tile[tx][r];
            const __half h = __float2half_rn(z);
            const __half l = __float2half_rn(z - __half2float(h));
            const int64_t o = j * lambda_pad + k;
            z_hi[o] = h;
            z_lo[o] = l;
            const float s = sgn[tx];
            zs_hi[o] = __float2half_rn(s * __half2float(h));
            zs_lo[o] = __float2half_rn(s * __half2float(l));
        }
    }
}

struct Args {
    float *out;
    int64_t n;
    int k_stages;            // lambda_pad / 64
    int tiles;               // 128-row (and 128-column) blocks per side
    int packed, ptile, ptiles_per_side;
};

struct Bars {
    uint64_t full[kStages], empty[kStages];
};

__device__ __forceinline__ void store_out(const Args &a, int64_t i, int64_t j, float x) {
    const int64_t n = a.n;
    if (a.packed) {
        // packed upper tiles of side ptile: element (i, j) lives in tile (i / ptile, j / ptile), bi' <= bj'; the tiles are
        // padded to a multiple of their side and the padding is written too (zeros from the TMA fill)
        const int64_t lim = (int64_t)a.ptiles_per_side * a.ptile;
        const int64_t pb_i = i / a.ptile, pb_j = j / a.ptile;
        if (i < lim && j < lim && pb_i <= pb_j) {
            const int64_t t = pb_i * a.ptiles_per_side - pb_i * (pb_i - 1) / 2 + (pb_j - pb_i);
            a.out[t * a.ptile * a.ptile + (i % a.ptile) * a.ptile + (j % a.ptile)] = x;
        }
    } else if (i < n && j < n && j >= i) {
        a.out[i * n + j] = x;
        if (j > i) a.out[j * n + i] = x;                // mirrored: exactly symmetric
    }
}

__global__ void __launch_bounds__(kThreads, 1) cma_syrk_kernel(Args a, const __grid_constant__ CUtensorMap map_a_hi,
                                                               const __grid_constant__ CUtensorMap map_a_lo,
                                                               const __grid_constant__ CUtensorMap map_b_hi,
                                                               const __grid_constant__ CUtensorMap map_b_lo) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    Bars *bars = reinterpret_cast<Bars *>(smem + kStages * kStageBytes);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // tile (bi, bj): 128-row block bi, 128-column block bj >= bi (the blocks that touch the upper triangle)
    int bi = 0, rem = blockIdx.x;
    while (rem >= a.tiles - bi) { rem -= a.tiles - bi; ++bi; }
    const int bj = bi + rem;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(smem_u32(&bars->full[s]), 1);
            mbar_init(smem_u32(&bars->empty[s]), 2);          // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();

    const uint32_t smem_addr = smem_u32(smem), bars_addr = smem_u32(bars);
    if (warp == 8) {
        // ---- TMA producer (whole warp converged, one elected lane issues)
        for (int ks = 0; ks < a.k_stages; ++ks) {
            const int s = ks % kStages, use = ks / kStages;
            if (use > 0) mbar_wait(bars_addr + (uint32_t)offsetof(Bars, empty) + 8u * s, (use - 1) & 1);
            const uint32_t bar = bars_addr + (uint32_t)offsetof(Bars, full) + 8u * s;
            const uint32_t base = smem_addr + (uint32_t)(s * kStageBytes);
            if (elect_one()) {
                mbar_expect_tx(bar, kStageBytes);
                tma_load_2d(base, &map_a_hi, ks * kBK, bi * kBM, bar);
                tma_load_2d(base + kABytes, &map_a_lo, ks * kBK, bi * kBM, bar);
                tma_load_2d(base + 2 * kABytes, &map_b_hi, ks * kBK, bj * kBN, bar);
                tma_load_2d(base + 2 * kABytes + kBBytes, &map_b_lo, ks * kBK, bj * kBN, bar);
            }
            __syncwarp();
        }
    } else {
        // ---- consumer warpgroup wg: output rows [64 wg, 64 wg + 64) of the tile
        const int wg = warp >> 2;
        // two accumulators, one per half of K, added with round-to-nearest in the epilogue: the tensor cores
        // truncate when they align the fp32 accumulator, which biases long sums of same-sign terms (the diagonal)
        float acc0[64], acc1[64];
#pragma unroll
        for (int e = 0; e < 64; ++e) acc0[e] = acc1[e] = 0.f;
        // K stages [k0, k1) into acc: one loop per half of K, so that the accumulator each wgmma names is fixed per loop
        auto run_stages = [&](float (&acc)[64], int k0, int k1) {
            for (int ks = k0; ks < k1; ++ks) {
                const int s = ks % kStages, use = ks / kStages;
                mbar_wait(bars_addr + (uint32_t)offsetof(Bars, full) + 8u * s, use & 1);
                const uint32_t base = smem_addr + (uint32_t)(s * kStageBytes);
                const uint32_t a_hi = base + wg * (kABytes / 2), a_lo = a_hi + kABytes;
                const uint32_t b_hi = base + 2 * kABytes, b_lo = b_hi + kBBytes;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBK / 16; ++k) {
                    wgmma_ss_n128(acc, smem_desc_sw128(a_hi + k * 32), smem_desc_sw128(b_hi + k * 32), 1);
                    wgmma_ss_n128(acc, smem_desc_sw128(a_lo + k * 32), smem_desc_sw128(b_hi + k * 32), 1);
                    wgmma_ss_n128(acc, smem_desc_sw128(a_hi + k * 32), smem_desc_sw128(b_lo + k * 32), 1);
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(acc);
                // every MMA of this warpgroup that read the stage has completed: one arrival frees it for the producer
                if ((threadIdx.x & 127) == 0) mbar_arrive(bars_addr + (uint32_t)offsetof(Bars, empty) + 8u * s);
            }
        };
        const int k_half = (a.k_stages + 1) / 2;
        run_stages(acc0, 0, k_half);
        run_stages(acc1, k_half, a.k_stages);
        const int64_t i0 = (int64_t)bi * kBM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int64_t j0 = (int64_t)bj * kBN + (lane & 3) * 2;
#pragma unroll
        for (int jb = 0; jb < kBN / 8; ++jb) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int64_t i = i0 + 8 * (e >> 1), j = j0 + 8 * jb + (e & 1);
                store_out(a, i, j, acc0[4 * jb + e] + acc1[4 * jb + e]);
            }
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
        else
            cudaGetLastError();
    }
    return fn;
}

static int64_t lambda_pad_of(int64_t lambda) { return (lambda + kBK - 1) / kBK * kBK; }

}  // namespace cmatc

size_t cma_tc_workspace_bytes(int64_t n, int64_t lambda) {
    return 4 * (size_t)n * (size_t)cmatc::lambda_pad_of(lambda) * sizeof(__half) + 1024;
}

// Called by des_cma_rank_mu with validated sizes (n >= kCmaTcMinN, lambda >= 1) and a large enough workspace.
int cma_rank_mu_tc(float *out_dev, const float *Y_dev, const float *w_dev, int64_t lambda_local, int64_t n, int packed,
                   void *workspace_dev, cudaStream_t st) {
    using namespace cmatc;
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) {
        set_error("des_cma_rank_mu: cuTensorMapEncodeTiled is not available from this driver");
        return DES_ERR_UNSUPPORTED;
    }
    const int64_t lp = lambda_pad_of(lambda_local);
    __half *base = reinterpret_cast<__half *>(((uintptr_t)workspace_dev + 1023) & ~(uintptr_t)1023);
    __half *zs_hi = base, *zs_lo = base + n * lp, *z_hi = base + 2 * n * lp, *z_lo = base + 3 * n * lp;
    cma_split_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)(lp / 32)), 256, 0, st>>>(zs_hi, zs_lo, z_hi, z_lo, Y_dev, w_dev,
                                                                                          lambda_local, lp, n);
    DES_LAUNCH_CHECK("cma_split_kernel");
    CUtensorMap maps[4];
    __half *ptrs[4] = {zs_hi, zs_lo, z_hi, z_lo};
    for (int m = 0; m < 4; ++m) {
        const cuuint64_t gdim[2] = {(cuuint64_t)lp, (cuuint64_t)n};
        const cuuint64_t gstride[1] = {(cuuint64_t)lp * sizeof(__half)};
        const cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)(m < 2 ? kBM : kBN)};
        const cuuint32_t estr[2] = {1, 1};
        const CUresult cr = enc(&maps[m], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, ptrs[m], gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (cr != CUDA_SUCCESS) {
            set_error("des_cma_rank_mu: cuTensorMapEncodeTiled failed (%d)", (int)cr);
            return DES_ERR_CUDA;
        }
    }
    Args a;
    a.out = out_dev; a.n = n; a.k_stages = (int)(lp / kBK);
    a.tiles = (int)((n + kBM - 1) / kBM);
    a.packed = packed ? 1 : 0;
    a.ptile = cma_packed_tile(n);
    a.ptiles_per_side = (int)((n + a.ptile - 1) / a.ptile);
    const int64_t tiles = (int64_t)a.tiles * (a.tiles + 1) / 2;
    const size_t smem = 1024 + (size_t)kStages * kStageBytes + sizeof(Bars);
    return launch_smem("cma_syrk_kernel", cma_syrk_kernel, (unsigned)tiles, kThreads, smem, st, a, maps[0], maps[1], maps[2],
                       maps[3]);
}

}  // namespace des
