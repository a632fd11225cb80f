// CMA-ES rank-mu covariance term on the tensor cores:  dC = sum_k w_k y_k y_k^T = Y^T diag(w) Y   (the arithmetic inside
// es.tell, cma_es.py:90; Hansen tutorial arXiv:1604.00772 eq. 47) as a symmetric rank-k update with split-fp16 operands.
//
//   Z  = diag(sqrt|w|) Y           (so that dC = Zs^T Z with Zs = diag(sign w) Z)
//   column scale  e_j with max_k |Z_kj| * 2^-e_j in [2^14, 2^15) (0 for an all-zero column or a non-finite maximum), so
//              that fp16 hi + lo hold every column at the same relative precision whatever the scale of Y: unscaled, lo
//              goes subnormal below |z| ~ 2^-3, hi below 2^-14, and hi overflows above 65504.  Powers of two are exact,
//              so the scale changes no rounding but the split's, and dC of Y diag(2^s) is exactly 2^(s_i+s_j) dC of Y.
//   pre-pass   column maxima of |Z| over up to 32 slices of the members (integer max of the fp32 bit patterns), then
//              Y [lambda][n] fp32 -> Zs_hi, Zs_lo, Z_hi, Z_lo  [n][lambda_pad] fp16 of Z 2^-e, k contiguous (K-major),
//              and e [n] for the epilogue
//   main       per 128 x 128 output tile touching the upper triangle:  D += A_hi B_hi^T + A_lo B_hi^T + A_hi B_lo^T
//              (wgmma m64n128k16, fp32 accumulation in registers; the dropped lo*lo term is 2^-22 relative), operand
//              tiles brought in by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B) through a three-stage mbarrier pipeline:
//              warps 0-7 = two consumer warpgroups (64 output rows each: wgmma, then registers -> global), warp 8 = TMA
//   output     2^(e_i+e_j) D: the full symmetric matrix (upper entry written to both sides: exactly symmetric), or the
//              packed upper-triangular tiles (the payload of the cross-rank sum), bit-equal to each other
//
// des_cma_rank_mu (des_cma.cu) runs this for n >= kCmaTcMinN and the fp32 FFMA kernel below that.
// Accuracy: per entry within oracle/rank_mu_error.py's bound against the fp64 (Y w)^T Y of the same fp32 inputs
// (tests/test_gpu_rank_mu_entries.py), at every scale of Y's columns.
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
constexpr int kScaleExp = 15;            // a column's largest |z| is scaled into [2^14, 2^15): fp16 hi cannot overflow
constexpr int kMaxParts = 32;            // slices of the members in the column-maximum pass (one CTA row each)

// e_j from the bit pattern of max_k |z_kj|: 2^-e_j puts the maximum into [2^(kScaleExp-1), 2^kScaleExp).  An all-zero
// column (bits 0) and a non-finite maximum (inf or NaN: bits >= 0x7f800000) keep e_j = 0, so NaN and inf reach dC as
// they do in the FFMA kernel.
__device__ __forceinline__ int col_exp(uint32_t bits) {
    if (bits == 0u || bits >= 0x7f800000u) return 0;
    const int be = (int)(bits >> 23);
    const int e = be ? be - 126 : -117 - __clz((int)bits);       // frexp's exponent, subnormals included
    return e - kScaleExp;
}

// 2^e x, exact whenever the result is a normal fp32 number (|e| <= 378): three normal factors 2^(e/3), all on the same
// side of 1, so no intermediate product leaves the normal range before the result does
__device__ __forceinline__ float pow2_scale(float x, int e) {
    const int e1 = e / 3, e2 = (e - e1) / 2, e3 = e - e1 - e2;
    return x * __int_as_float((e1 + 127) << 23) * __int_as_float((e2 + 127) << 23) * __int_as_float((e3 + 127) << 23);
}

__device__ __forceinline__ float z_of(const float *__restrict__ Y, const float *__restrict__ w, int64_t k, int64_t j,
                                      int64_t n) {
    return sqrtf(fabsf(__ldg(w + k))) * __ldg(Y + k * n + j);
}

// rows of Y per slice of the column-maximum pass: at least 128, at most kMaxParts slices (short slices keep the grid
// several waves deep at large lambda), each a multiple of the CTA's 8 rows
static int64_t max_rows_of(int64_t lambda) {
    const int64_t r = (lambda + kMaxParts - 1) / kMaxParts;
    return r < 128 ? 128 : (r + 7) / 8 * 8;
}

// ---- pre-pass 1: column maxima of |z| over one slice of the members ---------------------------------------------------
// As fp32 bit patterns: for non-negative floats the integer order is the numeric order, and inf and NaN (after fabsf)
// sort above every finite value, so a NaN is never dropped the way fmaxf drops it.  Slice p writes part[p][j] for every
// j < n, so the array needs no initialisation.
__global__ void __launch_bounds__(256) cma_colmax_kernel(uint32_t *__restrict__ part, const float *__restrict__ Y,
                                                         const float *__restrict__ w, int64_t lambda, int64_t n,
                                                         int64_t rows) {
    __shared__ uint32_t red[8][32];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 columns x 8 rows
    const int64_t j = (int64_t)blockIdx.x * 32 + tx, k0 = (int64_t)blockIdx.y * rows;
    const int64_t k1 = k0 + rows < lambda ? k0 + rows : lambda;
    uint32_t m = 0;
    if (j < n) {
#pragma unroll 8
        for (int64_t k = k0 + ty; k < k1; k += 8) m = max(m, __float_as_uint(fabsf(z_of(Y, w, k, j, n))));
    }
    red[ty][tx] = m;
    __syncthreads();
    if (ty == 0 && j < n) {
#pragma unroll
        for (int r = 1; r < 8; ++r) m = max(m, red[r][tx]);
        part[blockIdx.y * n + j] = m;
    }
}

// ---- pre-pass 2: transpose + scale + split -------------------------------------------------------------------------
// e_j from the slices' maxima; the CTAs of the first k-block also store it for the SYRK's epilogue.
__global__ void __launch_bounds__(256) cma_split_kernel(__half *__restrict__ zs_hi, __half *__restrict__ zs_lo,
                                                        __half *__restrict__ z_hi, __half *__restrict__ z_lo,
                                                        int *__restrict__ exps, const float *__restrict__ Y,
                                                        const float *__restrict__ w, const uint32_t *__restrict__ part,
                                                        int parts, int64_t lambda, int64_t lambda_pad, int64_t n) {
    __shared__ float tile[32][33];
    __shared__ float sgn[32];
    __shared__ int sexp[32];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8
    const int64_t k0 = (int64_t)blockIdx.y * 32, j0 = (int64_t)blockIdx.x * 32;
    for (int r = ty; r < 32; r += 8) {
        const int64_t k = k0 + r, j = j0 + tx;
        float v = 0.f;
        if (k < lambda && j < n) v = z_of(Y, w, k, j, n);
        tile[r][tx] = v;
    }
    if (threadIdx.x < 32) {
        sgn[tx] = (k0 + tx < lambda && __ldg(w + k0 + tx) < 0.f) ? -1.f : 1.f;
        const int64_t j = j0 + tx;
        uint32_t m = 0;
        if (j < n)
#pragma unroll 8
            for (int p = 0; p < parts; ++p) m = max(m, __ldg(part + p * n + j));
        sexp[tx] = col_exp(m);
        if (blockIdx.y == 0 && j < n) exps[j] = sexp[tx];
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {                               // row j0 + r of the outputs, k = k0 + tx
        const int64_t j = j0 + r, k = k0 + tx;
        if (j < n && k < lambda_pad) {
            const float z = pow2_scale(tile[tx][r], -sexp[r]);
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
    const int *exps;         // e_j of every column (cma_split_kernel): the epilogue's rescale
    int64_t n;
    int k_stages;            // lambda_pad / 64
    int tiles;               // 128-row (and 128-column) blocks per side
    int packed, ptile, ptiles_per_side;
};

struct Bars {
    uint64_t full[kStages], empty[kStages];
};

// x = the tile's acc0 + acc1 for entry (i, j), e = e_i + e_j: both layouts store the same 2^e x
__device__ __forceinline__ void store_out(const Args &a, int64_t i, int64_t j, float x, int e) {
    const int64_t n = a.n;
    x = pow2_scale(x, e);                                // exact unless dC_ij itself is below fp32's normal range
    if (a.packed) {
        // packed upper tiles of side ptile: element (i, j) lives in tile (i / ptile, j / ptile), bi' <= bj'; the tiles are
        // padded to a multiple of their side and the padding is written too (zeros from the TMA fill)
        const int64_t lim = (int64_t)a.ptiles_per_side * a.ptile;
        const int sh = __ffs(a.ptile) - 1;               // ptile is a power of two (cma_packed_tile): shifts, no division
        const int64_t pb_i = i >> sh, pb_j = j >> sh, m = a.ptile - 1;
        if (i < lim && j < lim && pb_i <= pb_j) {
            const int64_t t = pb_i * a.ptiles_per_side - pb_i * (pb_i - 1) / 2 + (pb_j - pb_i);
            a.out[t * a.ptile * a.ptile + (i & m) * a.ptile + (j & m)] = x;
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
        // e of the tile's 128 rows (sexp[0, 128)) and 128 columns (sexp[128, 256)), fetched while the first stages land;
        // 0 for the padding beyond n (whose entries are zero)
        int *sexp = reinterpret_cast<int *>(smem + kStages * kStageBytes + sizeof(Bars));
        {
            const int t = threadIdx.x;
            const int64_t g = t < kBM ? (int64_t)bi * kBM + t : (int64_t)bj * kBN + (t - kBM);
            sexp[t] = g < a.n ? __ldg(a.exps + g) : 0;
        }
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
        named_bar_sync(1, 256);                          // the consumers' sexp stores are visible
        const int li = wg * 64 + (warp & 3) * 16 + (lane >> 2), lj = (lane & 3) * 2;
        const int64_t i0 = (int64_t)bi * kBM + li;
        const int64_t j0 = (int64_t)bj * kBN + lj;
        const int ei0 = sexp[li], ei1 = sexp[li + 8];
#pragma unroll
        for (int jb = 0; jb < kBN / 8; ++jb) {
            const int ej0 = sexp[kBM + lj + 8 * jb], ej1 = sexp[kBM + lj + 8 * jb + 1];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int64_t i = i0 + 8 * (e >> 1), j = j0 + 8 * jb + (e & 1);
                store_out(a, i, j, acc0[4 * jb + e] + acc1[4 * jb + e], ((e >> 1) ? ei1 : ei0) + ((e & 1) ? ej1 : ej0));
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
    // zs_hi | zs_lo | z_hi | z_lo, the slices' column maxima, the column exponents
    return 4 * (size_t)n * (size_t)cmatc::lambda_pad_of(lambda) * sizeof(__half) +
           (size_t)(cmatc::kMaxParts + 1) * (size_t)n * sizeof(uint32_t) + 1024;
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
    uint32_t *part = reinterpret_cast<uint32_t *>(base + 4 * n * lp);
    int *exps = reinterpret_cast<int *>(part + kMaxParts * n);
    const int64_t rows = max_rows_of(lambda_local);
    const int parts = (int)((lambda_local + rows - 1) / rows);
    cma_colmax_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)parts), 256, 0, st>>>(part, Y_dev, w_dev, lambda_local, n,
                                                                                       rows);
    DES_LAUNCH_CHECK("cma_colmax_kernel");
    cma_split_kernel<<<dim3((unsigned)((n + 31) / 32), (unsigned)(lp / 32)), 256, 0, st>>>(zs_hi, zs_lo, z_hi, z_lo, exps, Y_dev,
                                                                                          w_dev, part, parts, lambda_local, lp, n);
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
    a.out = out_dev; a.exps = exps; a.n = n; a.k_stages = (int)(lp / kBK);
    a.tiles = (int)((n + kBM - 1) / kBM);
    a.packed = packed ? 1 : 0;
    a.ptile = cma_packed_tile(n);
    a.ptiles_per_side = (int)((n + a.ptile - 1) / a.ptile);
    const int64_t tiles = (int64_t)a.tiles * (a.tiles + 1) / 2;
    const size_t smem = 1024 + (size_t)kStages * kStageBytes + sizeof(Bars) + (kBM + kBN) * sizeof(int);
    return launch_smem("cma_syrk_kernel", cma_syrk_kernel, (unsigned)tiles, kThreads, smem, st, a, maps[0], maps[1], maps[2],
                       maps[3]);
}

}  // namespace des
