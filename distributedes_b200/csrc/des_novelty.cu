// Novelty search (include/des_b200.h, "novelty search" and "novelty-search sweeps"):
//   des_novelty        novelty_out[n]: the mean Euclidean distance of each query row to its k nearest rows of an archive
//   des_ns_shape       shaped_out[N]: the blend of the centered ranks of fitness and of novelty (NS-ES, NSR-ES, NSRA-ES)
//   des_novelty_runs   des_novelty of every run of a sweep against its own archive, one launch
//   des_ns_shape_runs  des_ns_shape of every run with its own reward weight, from a device table
#include "des_common.cuh"

namespace des {

constexpr int kNovTile = 256;                 // archive rows per shared-memory tile
constexpr uint32_t kNovNanKey = 0x7F800001u;  // a NaN distance's key: above +inf's bits, so NaN sorts after every number

// The order of a candidate: (d2, index) as one integer.  d2 is a sum of squares from +0, never negative or -0, so its
// bits order as its value does.
__device__ __forceinline__ uint64_t novelty_key(float d2, uint32_t i) {
    const uint32_t hi = isnan(d2) ? kNovNanKey : __float_as_uint(d2);
    return ((uint64_t)hi << 32) | i;
}

// One warp per query row, `blockDim.x / 32` queries per CTA; `block` is the CTA's index among the CTAs of its queries.
// The CTA streams the archive through shared memory in tiles of kNovTile rows (row stride d | 1 words: lanes reading
// consecutive rows hit distinct banks).  Lane l scores the rows l, l + 32, .. of each tile against the query, which every
// lane holds in registers, and keeps its KC smallest keys sorted in registers (KC >= k).  Then k rounds of a warp argmin
// pop the k nearest rows in order; lane 0 sums their distances in fp64 in that order.  Everything is indexed at compile
// time: no local memory.
template <int KC>
__device__ __forceinline__ void novelty_rows(float *__restrict__ out, const float *__restrict__ queries, int64_t n,
                                             const float *__restrict__ archive, int A, int d, int k, unsigned block) {
    extern __shared__ float tile[];          // [kNovTile][d | 1]
    const int ds = d | 1;
    const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int64_t row = (int64_t)block * nw + (threadIdx.x >> 5);
    const bool active = row < n;
    float q[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) q[j] = (active && j < d) ? __ldg(queries + row * d + j) : 0.f;
    uint64_t best[KC];
#pragma unroll
    for (int s = 0; s < KC; ++s) best[s] = ~0ull;
    // 64-bit tile arithmetic: the last tile of an archive of up to 2^31 - 1 rows starts within 256 rows of INT32_MAX,
    // and `base + kNovTile` would leave int32 there
    for (int64_t base = 0; base < A; base += kNovTile) {
        const int rows = (int)min((int64_t)kNovTile, (int64_t)A - base);
        __syncthreads();                     // the previous tile is read
        const float *src = archive + base * d;
        for (int e = threadIdx.x; e < rows * d; e += blockDim.x) {
            const int r = e / d;
            tile[r * ds + (e - r * d)] = __ldg(src + e);
        }
        __syncthreads();
        if (!active) continue;
        for (int r = lane; r < rows; r += 32) {
            const float *a = tile + r * ds;
            float d2 = 0.f;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                if (j >= d) break;
                const float diff = __fsub_rn(q[j], a[j]);
                d2 = __fmaf_rn(diff, diff, d2);
            }
            const uint64_t key = novelty_key(d2, (uint32_t)(base + r));
            if (key < best[KC - 1]) {        // sorted insertion; the largest key drops out
#pragma unroll
                for (int s = KC - 1; s > 0; --s) best[s] = key < best[s - 1] ? best[s - 1] : (key < best[s] ? key : best[s]);
                best[0] = key < best[0] ? key : best[0];
            }
        }
    }
    if (!active) return;
    const int keff = min(k, A);
    double sum = 0.0;
    for (int t = 0; t < keff; ++t) {
        uint64_t m = best[0];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const uint64_t o = __shfl_xor_sync(0xffffffffu, m, off);
            m = o < m ? o : m;
        }
        if (best[0] == m) {                  // keys are unique (the index is in them): one lane pops its head
#pragma unroll
            for (int s = 0; s < KC - 1; ++s) best[s] = best[s + 1];
            best[KC - 1] = ~0ull;
        }
        if (lane == 0) {
            const uint32_t hi = (uint32_t)(m >> 32);
            const float d2 = hi == kNovNanKey ? __int_as_float(0x7fffffff) : __uint_as_float(hi);
            sum += (double)__fsqrt_rn(d2);
        }
    }
    if (lane == 0) out[row] = (float)(sum / keff);
}

template <int KC>
__global__ void __launch_bounds__(256, 1) novelty_kernel(float *__restrict__ out, const float *__restrict__ queries, int64_t n,
                                                      const float *__restrict__ archive, int A, int d, int k) {
    novelty_rows<KC>(out, queries, n, archive, A, d, k, blockIdx.x);
}

// A sweep's novelty (des_novelty_runs): CTA b serves run b / blocks_per_run, whose queries, outputs and archive are its
// rows of queries [n_runs][n][d], out [n_runs][n] and archive [n_runs][capacity][d]; the rest is novelty_kernel's.
template <int KC>
__global__ void __launch_bounds__(256, 1) novelty_runs_kernel(float *__restrict__ out, const float *__restrict__ queries,
                                                           int64_t n, const float *__restrict__ archive, int64_t capacity,
                                                           int A, int d, int k, unsigned blocks_per_run) {
    const unsigned run = blockIdx.x / blocks_per_run;
    novelty_rows<KC>(out + (int64_t)run * n, queries + (int64_t)run * n * d, n, archive + (int64_t)run * capacity * d, A,
                     d, k, blockIdx.x - run * blocks_per_run);
}

// shaped = fmaf(w, s_f, w1 * s_n), with s_f already in shaped
__global__ void ns_blend_kernel(float *__restrict__ shaped, const float *__restrict__ s_n, int64_t N, float w, float w1) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) shaped[i] = __fmaf_rn(w, shaped[i], __fmul_rn(w1, s_n[i]));
}

// shaped = fmaf(w_r, s_f, w1_r * s_n) of every run r, (w_r, w1_r) its row of the weight table
__global__ void ns_blend_runs_kernel(float *__restrict__ shaped, const float *__restrict__ s_n, int64_t n_total,
                                     int64_t run_size, const float2 *__restrict__ weights) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_total) {
        const float2 w = weights[i / run_size];
        shaped[i] = __fmaf_rn(w.x, shaped[i], __fmul_rn(w.y, s_n[i]));
    }
}

static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

static bool overlaps(const void *a, int64_t na, const void *b, int64_t nb) {
    const uintptr_t a0 = (uintptr_t)a, a1 = a0 + (uintptr_t)na * sizeof(float);
    const uintptr_t b0 = (uintptr_t)b, b1 = b0 + (uintptr_t)nb * sizeof(float);
    return a0 < b1 && b0 < a1;
}

}  // namespace des

extern "C" DES_API int des_novelty(float *novelty_out_dev, const float *queries_dev, int64_t n, const float *archive_dev,
                                   int64_t A, int32_t d, int32_t k, void *stream) {
    using namespace des;
    const char *who = "des_novelty";
    DES_REQUIRE(n >= 0 && n <= INT32_MAX, "%s: n must be in [0, 2^31) (got %lld)", who, (long long)n);
    DES_REQUIRE(A >= 1 && A <= INT32_MAX, "%s: the archive must have [1, 2^31) rows (got %lld)", who, (long long)A);
    DES_REQUIRE(d >= 1 && d <= 32, "%s: d must be in [1, 32] (got %d)", who, d);
    DES_REQUIRE(k >= 1 && k <= 32, "%s: k must be in [1, 32] (got %d)", who, k);
    if (n == 0) return DES_OK;
    DES_REQUIRE(novelty_out_dev && queries_dev && archive_dev, "%s: NULL pointer", who);
    const int warps = n >= 2048 ? 8 : 2;     // small batches: more CTAs, so more SMs share the archive scan
    const unsigned blocks = (unsigned)((n + warps - 1) / warps);
    const size_t smem = sizeof(float) * kNovTile * (size_t)(d | 1);
    cudaStream_t st = (cudaStream_t)stream;
    if (k <= 8) novelty_kernel<8><<<blocks, 32 * warps, smem, st>>>(novelty_out_dev, queries_dev, n, archive_dev, (int)A, d, k);
    else if (k <= 16) novelty_kernel<16><<<blocks, 32 * warps, smem, st>>>(novelty_out_dev, queries_dev, n, archive_dev, (int)A, d, k);
    else novelty_kernel<32><<<blocks, 32 * warps, smem, st>>>(novelty_out_dev, queries_dev, n, archive_dev, (int)A, d, k);
    DES_LAUNCH_CHECK("novelty_kernel");
    return DES_OK;
}

extern "C" DES_API size_t des_ns_shape_workspace_bytes(int64_t N) {
    if (N < 2) return 0;
    return 256 + des::al256((size_t)N * 4) + des_rank_workspace_bytes(N, N);
}

extern "C" DES_API int des_ns_shape(float *shaped_out_dev, const float *fitness_dev, const float *novelty_dev, int64_t N,
                                    double reward_weight, void *workspace_dev, size_t workspace_bytes, void *stream) {
    using namespace des;
    const char *who = "des_ns_shape";
    DES_REQUIRE(N >= 2 && N <= INT32_MAX, "%s: N=%lld, need 2 <= N < 2^31", who, (long long)N);
    DES_REQUIRE(reward_weight >= 0.0 && reward_weight <= 1.0, "%s: reward_weight must be in [0, 1] (got %g)", who,
                reward_weight);
    DES_REQUIRE(shaped_out_dev && fitness_dev && novelty_dev, "%s: NULL pointer", who);
    DES_REQUIRE(!overlaps(shaped_out_dev, N, fitness_dev, N) && !overlaps(shaped_out_dev, N, novelty_dev, N),
                "%s: shaped_out overlaps an input", who);
    const size_t need = des_ns_shape_workspace_bytes(N);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    uint8_t *p = (uint8_t *)(((uintptr_t)workspace_dev + 255) & ~(uintptr_t)255);
    float *s_n = (float *)p;
    p += al256((size_t)N * 4);
    const size_t rank_bytes = (size_t)((const uint8_t *)workspace_dev + workspace_bytes - p);
    int rc = des_centered_rank(shaped_out_dev, nullptr, fitness_dev, N, 0, N, p, rank_bytes, stream);
    if (rc != DES_OK) return rc;
    rc = des_centered_rank(s_n, nullptr, novelty_dev, N, 0, N, p, rank_bytes, stream);
    if (rc != DES_OK) return rc;
    const float w = (float)reward_weight, w1 = (float)(1.0 - reward_weight);
    ns_blend_kernel<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)stream>>>(shaped_out_dev, s_n, N, w, w1);
    DES_LAUNCH_CHECK("ns_blend_kernel");
    return DES_OK;
}

extern "C" DES_API int des_novelty_runs(float *novelty_out_dev, const float *queries_dev, int64_t n_runs, int64_t n,
                                        const float *archive_dev, int64_t capacity, int64_t A, int32_t d, int32_t k,
                                        void *stream) {
    using namespace des;
    const char *who = "des_novelty_runs";
    const int rc = check_runs(who, n_runs, n, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(capacity >= 1 && capacity <= INT32_MAX, "%s: capacity must be in [1, 2^31) (got %lld)", who,
                (long long)capacity);
    DES_REQUIRE(A >= 1 && A <= capacity, "%s: the archives must have [1, capacity = %lld] rows (got %lld)", who,
                (long long)capacity, (long long)A);
    DES_REQUIRE(d >= 1 && d <= 32, "%s: d must be in [1, 32] (got %d)", who, d);
    DES_REQUIRE(k >= 1 && k <= 32, "%s: k must be in [1, 32] (got %d)", who, k);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(novelty_out_dev && queries_dev && archive_dev, "%s: NULL pointer", who);
    const int warps = n >= 2048 ? 8 : 2;     // des_novelty's CTA shape for a population of n
    const unsigned per_run = (unsigned)((n + warps - 1) / warps);
    const unsigned blocks = (unsigned)n_runs * per_run;    // n_runs * n <= 2^28
    const size_t smem = sizeof(float) * kNovTile * (size_t)(d | 1);
    cudaStream_t st = (cudaStream_t)stream;
    if (k <= 8)
        novelty_runs_kernel<8><<<blocks, 32 * warps, smem, st>>>(novelty_out_dev, queries_dev, n, archive_dev, capacity,
                                                                 (int)A, d, k, per_run);
    else if (k <= 16)
        novelty_runs_kernel<16><<<blocks, 32 * warps, smem, st>>>(novelty_out_dev, queries_dev, n, archive_dev, capacity,
                                                                  (int)A, d, k, per_run);
    else
        novelty_runs_kernel<32><<<blocks, 32 * warps, smem, st>>>(novelty_out_dev, queries_dev, n, archive_dev, capacity,
                                                                  (int)A, d, k, per_run);
    DES_LAUNCH_CHECK("novelty_runs_kernel");
    return DES_OK;
}

extern "C" DES_API size_t des_ns_shape_runs_workspace_bytes(int64_t n_runs, int64_t run_size) {
    if (n_runs < 1 || run_size < 2) return 0;
    return 256 + des::al256((size_t)(n_runs * run_size) * 4) + des_rank_runs_workspace_bytes(n_runs, run_size);
}

extern "C" DES_API int des_ns_shape_runs(float *shaped_out_dev, const float *fitness_dev, const float *novelty_dev,
                                         int64_t n_runs, int64_t run_size, const float *weights_dev, void *workspace_dev,
                                         size_t workspace_bytes, void *stream) {
    using namespace des;
    const char *who = "des_ns_shape_runs";
    const int rc = check_runs(who, n_runs, run_size, 2);
    if (rc != DES_OK) return rc;
    if (n_runs == 0) return DES_OK;
    const int64_t total = n_runs * run_size;
    DES_REQUIRE(shaped_out_dev && fitness_dev && novelty_dev && weights_dev, "%s: NULL pointer", who);
    DES_REQUIRE((uintptr_t)weights_dev % 8 == 0, "%s: the weight table must be 8-byte aligned (rows of two fp32)", who);
    DES_REQUIRE(!overlaps(shaped_out_dev, total, fitness_dev, total) && !overlaps(shaped_out_dev, total, novelty_dev, total),
                "%s: shaped_out overlaps an input", who);
    const size_t need = des_ns_shape_runs_workspace_bytes(n_runs, run_size);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    uint8_t *p = (uint8_t *)(((uintptr_t)workspace_dev + 255) & ~(uintptr_t)255);
    float *s_n = (float *)p;
    p += al256((size_t)total * 4);
    const size_t rank_bytes = (size_t)((const uint8_t *)workspace_dev + workspace_bytes - p);
    int r = des_centered_rank_runs(shaped_out_dev, nullptr, fitness_dev, n_runs, run_size, p, rank_bytes, stream);
    if (r != DES_OK) return r;
    r = des_centered_rank_runs(s_n, nullptr, novelty_dev, n_runs, run_size, p, rank_bytes, stream);
    if (r != DES_OK) return r;
    ns_blend_runs_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        shaped_out_dev, s_n, total, run_size, reinterpret_cast<const float2 *>(weights_dev));
    DES_LAUNCH_CHECK("ns_blend_runs_kernel");
    return DES_OK;
}
