// des_centered_rank: centered-rank fitness shaping, fitness_shift utils.py:142-148.
//
//   rank_i = #{j : f_j < f_i} + #{j < i : f_j == f_i}       (ascending; ties by index; NaN last)
//   s_i    = rank_i/(N-1) - 0.5
//
// Populations up to 2048: counting rank instead of a sort (larger ones take the bucketed path below).  A shard needs ranks only for ITS members but against ALL N
// fitnesses (ranks are global), so the work is n_local x N comparisons, embarrassingly parallel,
// integer-exact and deterministic.  Keys are order-preserving uint32 images of the floats; each
// (i, j) pair costs one 64-bit compare.  The j range is split over blockIdx.y, partial counts are
// combined with integer atomics (exact, order independent).
#include "des_common.cuh"

namespace des {

constexpr int kRankThreads = 256;
constexpr int kRankTile = 2048;   // keys staged in shared memory per step

// float -> uint32 whose unsigned order is the numpy sort order: -inf < ... < -0 == +0 < ... < +inf < NaN
__device__ __forceinline__ uint32_t order_key(float f) {
    uint32_t b = __float_as_uint(f);
    if ((b & 0x7FFFFFFFu) > 0x7F800000u) return 0xFFFFFFFFu;   // any NaN -> last
    if ((b << 1) == 0u) b = 0u;                                 // -0 -> +0
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// counts[il] += #{j in the CTA's j-slice : (key_j, j) < (key_i, i)} for member i = member_offset + il, il in member block bx
__device__ __forceinline__ void rank_count(int32_t *__restrict__ counts, const float *__restrict__ fitness, int64_t N,
                                           int64_t member_offset, int64_t n_local, int64_t j_per_block, unsigned bx) {
    __shared__ uint32_t keys[kRankTile];
    const int64_t il = (int64_t)bx * kRankThreads + threadIdx.x;
    const bool live = il < n_local;
    const int64_t ig = member_offset + il;
    const uint64_t mine = live ? (((uint64_t)order_key(__ldg(fitness + ig)) << 32) | (uint64_t)(uint32_t)ig) : 0;
    const int64_t j_begin = (int64_t)blockIdx.y * j_per_block;
    const int64_t j_end = min(N, j_begin + j_per_block);
    int32_t cnt = 0;
    for (int64_t j0 = j_begin; j0 < j_end; j0 += kRankTile) {
        const int n = (int)min((int64_t)kRankTile, j_end - j0);
        __syncthreads();
        for (int t = threadIdx.x; t < n; t += kRankThreads) keys[t] = order_key(__ldg(fitness + j0 + t));
        __syncthreads();
        if (live) {
            const uint32_t jb = (uint32_t)j0;
#pragma unroll 8
            for (int t = 0; t < n; ++t) {
                const uint64_t other = ((uint64_t)keys[t] << 32) | (uint64_t)(jb + (uint32_t)t);
                cnt += (other < mine) ? 1 : 0;
            }
        }
    }
    if (live && cnt) atomicAdd(counts + il, cnt);
}

__global__ void __launch_bounds__(kRankThreads) rank_count_kernel(int32_t *__restrict__ counts,
                                                                   const float *__restrict__ fitness, int64_t N,
                                                                   int64_t member_offset, int64_t n_local,
                                                                   int64_t j_per_block) {
    rank_count(counts, fitness, N, member_offset, n_local, j_per_block, blockIdx.x);
}

// A batch of runs of N members (des_centered_rank_runs): member blocks of all runs along x, blocks_per_run per run, each
// run ranked within itself exactly as des_centered_rank ranks a population of N.
__global__ void __launch_bounds__(kRankThreads) rank_count_runs_kernel(int32_t *__restrict__ counts,
                                                                        const float *__restrict__ fitness, int64_t N,
                                                                        int64_t j_per_block, unsigned blocks_per_run) {
    const int64_t run = blockIdx.x / blocks_per_run;
    rank_count(counts + run * N, fitness + run * N, N, 0, N, j_per_block, blockIdx.x % blocks_per_run);
}

// The counting path's grid: bx member blocks of n_local, by j-slices of j_per_block keys (a multiple of the smem tile).
struct CountPlan {
    unsigned bx, by;
    int64_t j_per_block;
};
static CountPlan count_plan(int64_t N, int64_t n_local) {
    CountPlan p;
    p.bx = (unsigned)((n_local + kRankThreads - 1) / kRankThreads);
    // enough j-slices to fill the machine a few times over, each a multiple of the smem tile
    int64_t want_blocks = 132 * 8;                 // 132 SMs (H100 SXM)
    int64_t by = (want_blocks + p.bx - 1) / p.bx;
    int64_t max_by = (N + kRankTile - 1) / kRankTile;
    if (by > max_by) by = max_by;
    if (by < 1) by = 1;
    if (by > 65535) by = 65535;
    int64_t j_per_block = (N + by - 1) / by;
    p.j_per_block = ((j_per_block + kRankTile - 1) / kRankTile) * kRankTile;
    p.by = (unsigned)((N + p.j_per_block - 1) / p.j_per_block);
    return p;
}

__global__ void rank_finish_kernel(float *__restrict__ shaped, int32_t *__restrict__ rank_out,
                                   const int32_t *__restrict__ counts, int64_t N, int64_t n_local) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_local) return;
    const int32_t r = counts[i];
    if (rank_out) rank_out[i] = r;
    // utils.py:146-147 in fp64, then one rounding to fp32
    shaped[i] = (float)((double)r / (double)(N - 1) - 0.5);
}

// ---------------------------------------------------------------------------------------------------------------
// Large populations (N > kBucketMinN): sample-sort style bucketing makes the work ~N * (N/1024) instead of n * N.
//   1. 4096 strided sample keys are sorted by one CTA (bitonic, shared memory) -> 1023 splitters
//   2. every member finds its bucket by binary search over the splitters; bucket histogram (integer atomics)
//   3. exclusive scan of the 1024 bucket counts
//   4. members are grouped by bucket (order inside a bucket is arbitrary; it does not matter below)
//   5. rank_i = bucket_start + #{j in bucket : (key_j, j) < (key_i, i)}     — exact, ties by index
// Degenerate inputs (all keys equal) put everything in one bucket: still exact, cost falls back to n * N.
constexpr int kBuckets = 1024;          // upper bound; populations up to 256k use 256 buckets / 1024 samples
constexpr int kSamples = 4096;
constexpr int64_t kBucketMinN = 2048;    // populations up to this size use the counting rank
__host__ __device__ inline int buckets_for(int64_t N) { return N <= 262144 ? 256 : kBuckets; }

// sample t of ns: the key of member floor(t N / ns)   (t < 4096, N < 2^31: the product fits 64 bits)
__device__ __forceinline__ uint32_t sample_key(const float *__restrict__ fitness, int64_t N, int t, int ns) {
    return order_key(__ldg(fitness + (int64_t)(((uint64_t)t * (uint64_t)N) / (uint64_t)ns)));
}

// ascending bitonic sort of 1024 keys, one per thread of a 1024-thread CTA: partner distances below 32 go through
// shuffles, the 15 wider steps through shared memory.  Returns with s[0..1023] sorted (and a barrier behind it).
__device__ __forceinline__ void sort1024(uint32_t v, uint32_t *s) {
    const int t = threadIdx.x;
    for (int k = 2; k <= 1024; k <<= 1) {
        const bool up = (t & k) == 0;
        for (int j = k >> 1; j > 0; j >>= 1) {
            uint32_t o;
            if (j >= 32) {
                s[t] = v;
                __syncthreads();
                o = s[t ^ j];
                __syncthreads();
            } else {
                o = __shfl_xor_sync(0xffffffffu, v, j);
            }
            const bool keep_min = ((t & j) == 0) == up;
            v = keep_min ? min(v, o) : max(v, o);
        }
    }
    s[t] = v;
    __syncthreads();
}

// bucket(key) = #{splitters <= key}  (monotone in key, so bucket order == key order)
__device__ __forceinline__ int bucket_of_key(const uint32_t *sp, uint32_t key, int nb) {
    int lo = 0, hi = nb - 1;                  // answer in [0, nb-1]
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sp[mid] <= key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// 256 buckets (N <= 256k): steps 1+2 in ONE kernel.  Every CTA sorts the same 1024 samples itself (2 us of redundant
// work instead of a separate single-CTA kernel and a launch dependency), then classifies its 1024 members; the bucket
// histogram is accumulated in shared memory first (one global atomic per bucket and CTA).
__global__ void __launch_bounds__(1024) rank_classify256_kernel(int32_t *__restrict__ bucket_count,
                                                                uint16_t *__restrict__ bucket_id, uint32_t *__restrict__ keys,
                                                                const float *__restrict__ fitness, int64_t N) {
    __shared__ uint32_t s[1024];
    __shared__ uint32_t sp[256];
    __shared__ int32_t hist[256];
    const int t = threadIdx.x;
    const int64_t i = (int64_t)blockIdx.x * 1024 + t;
    const uint32_t key = i < N ? order_key(__ldg(fitness + i)) : 0u;
    if (t < 256) hist[t] = 0;
    sort1024(sample_key(fitness, N, t, 1024), s);
    if (t < 255) sp[t] = s[(t + 1) * 4];
    __syncthreads();
    if (i < N) {
        const int b = bucket_of_key(sp, key, 256);
        keys[i] = key;
        bucket_id[i] = (uint16_t)b;
        atomicAdd(hist + b, 1);
    }
    __syncthreads();
    if (t < 256 && hist[t]) atomicAdd(bucket_count + t, hist[t]);
}

// 1024 buckets (N > 256k): 4096 samples sorted by one CTA (bitonic, shared memory) ...
__global__ void __launch_bounds__(1024) rank_splitters_kernel(uint32_t *__restrict__ splitters,
                                                              const float *__restrict__ fitness, int64_t N, int nb) {
    __shared__ uint32_t sk[kSamples];
    const int ns = 4 * nb;                   // samples
    for (int t = threadIdx.x; t < ns; t += 1024) sk[t] = sample_key(fitness, N, t, ns);
    __syncthreads();
    for (int k = 2; k <= ns; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < ns; t += 1024) {
                const int p = t ^ j;
                if (p > t) {
                    const uint32_t a = sk[t], b = sk[p];
                    const bool up = (t & k) == 0;
                    if ((a > b) == up) { sk[t] = b; sk[p] = a; }
                }
            }
            __syncthreads();
        }
    }
    for (int t = threadIdx.x; t < nb - 1; t += 1024) splitters[t] = sk[(t + 1) * 4];
}

// ... and a histogram kernel that reads the splitters back
__global__ void __launch_bounds__(256) rank_bucket_hist_kernel(int32_t *__restrict__ bucket_count,
                                                               uint16_t *__restrict__ bucket_id, uint32_t *__restrict__ keys,
                                                               const uint32_t *__restrict__ splitters,
                                                               const float *__restrict__ fitness, int64_t N, int nb) {
    __shared__ uint32_t sp[kBuckets];
    for (int t = threadIdx.x; t < nb - 1; t += 256) sp[t] = splitters[t];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= N) return;
    const uint32_t key = order_key(__ldg(fitness + i));
    const int b = bucket_of_key(sp, key, nb);
    keys[i] = key;
    bucket_id[i] = (uint16_t)b;
    atomicAdd(bucket_count + b, 1);
}

// steps 3+4: every CTA scans the (<= 1024) bucket counts itself, CTA 0 publishes the starts, then the members are
// scattered to their buckets.  bucket_fill must be zero on entry (one memset covers it together with bucket_count).
__global__ void __launch_bounds__(256) rank_bucket_group_kernel(uint32_t *__restrict__ g_key, int32_t *__restrict__ g_idx,
                                                                int32_t *__restrict__ bucket_fill,
                                                                int32_t *__restrict__ bucket_start,
                                                                const int32_t *__restrict__ bucket_count,
                                                                const uint16_t *__restrict__ bucket_id,
                                                                const uint32_t *__restrict__ keys, int64_t N, int nb) {
    __shared__ int32_t start[kBuckets];
    __shared__ int32_t warp_tot[8];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int per = nb / 256;                        // 1 or 4 consecutive buckets per thread
    int32_t c[4] = {0, 0, 0, 0}, tot = 0;
    for (int q = 0; q < per; ++q) { c[q] = bucket_count[t * per + q]; tot += c[q]; }
    int32_t inc = tot;                               // inclusive scan of the per-thread totals
    for (int o = 1; o < 32; o <<= 1) {
        const int32_t v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    int32_t base = inc - tot;
    for (int q = 0; q < w; ++q) base += warp_tot[q];
    for (int q = 0; q < per; ++q) {
        start[t * per + q] = base;
        if (blockIdx.x == 0) bucket_start[t * per + q] = base;
        base += c[q];
    }
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * 256 + t;
    if (i >= N) return;
    const int b = bucket_id[i];
    const int pos = start[b] + atomicAdd(bucket_fill + b, 1);
    g_key[pos] = keys[i];
    g_idx[pos] = (int32_t)i;
}

// step 5, by POSITION in the grouped array: a CTA takes 256 consecutive grouped members (a few neighbouring buckets),
// stages the union of their buckets in shared memory tile by tile and counts, for each member of the shard, the
// entries of its own bucket that sort before it.  No dependent global loads in the counting loop; in the degenerate
// all-equal case (one bucket) the N x N comparisons are still spread over all CTAs.
constexpr int kFinishTile = 1024;
__global__ void __launch_bounds__(256) rank_bucket_finish_kernel(float *__restrict__ shaped, int32_t *__restrict__ rank_out,
                                                                 const uint32_t *__restrict__ g_key,
                                                                 const int32_t *__restrict__ g_idx,
                                                                 const int32_t *__restrict__ bucket_start,
                                                                 const int32_t *__restrict__ bucket_count,
                                                                 const uint16_t *__restrict__ bucket_id, int64_t N,
                                                                 int64_t member_offset, int64_t n_local) {
    __shared__ uint64_t tile[kFinishTile];
    __shared__ int32_t range[2];
    const int t = threadIdx.x;
    const int64_t p = (int64_t)blockIdx.x * 256 + t;
    if (t == 0) { range[0] = 0x7FFFFFFF; range[1] = 0; }
    int32_t idx = 0, st = 0, en = 0;
    uint64_t mine = 0;
    bool local = false;
    if (p < N) {
        idx = g_idx[p];
        local = idx >= member_offset && idx < member_offset + n_local;
        if (local) {
            const int b = bucket_id[idx];
            st = bucket_start[b];
            en = st + bucket_count[b];
            mine = ((uint64_t)g_key[p] << 32) | (uint64_t)(uint32_t)idx;
        }
    }
    __syncthreads();
    if (local) { atomicMin(range + 0, st); atomicMax(range + 1, en); }
    __syncthreads();
    const int32_t lo = range[0], hi = range[1];
    int32_t r = st;
    for (int32_t base = lo; base < hi; base += kFinishTile) {
        const int n = min(kFinishTile, hi - base);
        __syncthreads();
        for (int q = t; q < n; q += 256)
            tile[q] = ((uint64_t)__ldg(g_key + base + q) << 32) | (uint64_t)(uint32_t)__ldg(g_idx + base + q);
        __syncthreads();
        if (local) {
            const int a = max(st, base) - base, e = min(en, base + n) - base;
#pragma unroll 4
            for (int q = a; q < e; ++q) r += (tile[q] < mine) ? 1 : 0;
        }
    }
    if (local) {
        const int64_t il = idx - member_offset;
        if (rank_out) rank_out[il] = r;
        shaped[il] = (float)((double)r / (double)(N - 1) - 0.5);
    }
}

struct BucketWs {        // carved out of the caller's workspace (all 16-byte aligned)
    uint32_t *splitters, *keys, *g_key;
    int32_t *bucket_count, *bucket_start, *bucket_fill, *g_idx;
    uint16_t *bucket_id;
};
static size_t bucket_ws_bytes(int64_t N) {
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    return al(kBuckets * 4) * 4 + al((size_t)N * 4) * 3 + al((size_t)N * 2) + 256;
}
static BucketWs carve(void *ws, int64_t N) {
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    uint8_t *p = (uint8_t *)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
    BucketWs w;
    w.splitters = (uint32_t *)p; p += al(kBuckets * 4);
    w.bucket_count = (int32_t *)p; p += al(kBuckets * 4);          // count and fill adjacent: one memset
    w.bucket_fill = (int32_t *)p; p += al(kBuckets * 4);
    w.bucket_start = (int32_t *)p; p += al(kBuckets * 4);
    w.keys = (uint32_t *)p; p += al((size_t)N * 4);
    w.g_key = (uint32_t *)p; p += al((size_t)N * 4);
    w.g_idx = (int32_t *)p; p += al((size_t)N * 4);
    w.bucket_id = (uint16_t *)p;
    return w;
}

}  // namespace des

extern "C" DES_API size_t des_rank_workspace_bytes(int64_t N, int64_t n_local) {
    if (N > des::kBucketMinN) return des::bucket_ws_bytes(N);
    return n_local > 0 ? (size_t)n_local * sizeof(int32_t) : 0;
}

extern "C" DES_API int des_centered_rank(float *shaped_out_dev, int32_t *rank_out_dev, const float *fitness_all_dev, int64_t N,
                                 int64_t member_offset, int64_t n_local, void *workspace_dev, size_t workspace_bytes,
                                 void *stream) {
    using namespace des;
    DES_REQUIRE(N >= 2, "des_centered_rank: N=%lld, need N >= 2 (utils.py:146 divides by N-1)", (long long)N);
    DES_REQUIRE(N <= ((int64_t)1 << 31) - 1, "des_centered_rank: N too large");
    DES_REQUIRE(member_offset >= 0 && n_local >= 0 && member_offset + n_local <= N,
                "des_centered_rank: shard [%lld, %lld) outside population of %lld", (long long)member_offset,
                (long long)(member_offset + n_local), (long long)N);
    if (n_local == 0) return DES_OK;
    DES_REQUIRE(shaped_out_dev && fitness_all_dev, "des_centered_rank: NULL pointer");
    const size_t need = des_rank_workspace_bytes(N, n_local);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("des_centered_rank: workspace %zu B < required %zu B", workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (N > kBucketMinN) {
        const BucketWs w = carve(workspace_dev, N);
        const unsigned gn = (unsigned)((N + 255) / 256);
        DES_CUDA(cudaMemsetAsync(w.bucket_count, 0, 2 * kBuckets * sizeof(int32_t), st));
        const int nb = buckets_for(N);
        if (nb == 256) {
            rank_classify256_kernel<<<(unsigned)((N + 1023) / 1024), 1024, 0, st>>>(w.bucket_count, w.bucket_id, w.keys,
                                                                                   fitness_all_dev, N);
        } else {
            rank_splitters_kernel<<<1, 1024, 0, st>>>(w.splitters, fitness_all_dev, N, nb);
            rank_bucket_hist_kernel<<<gn, 256, 0, st>>>(w.bucket_count, w.bucket_id, w.keys, w.splitters, fitness_all_dev, N, nb);
        }
        rank_bucket_group_kernel<<<gn, 256, 0, st>>>(w.g_key, w.g_idx, w.bucket_fill, w.bucket_start, w.bucket_count,
                                                     w.bucket_id, w.keys, N, nb);
        rank_bucket_finish_kernel<<<gn, 256, 0, st>>>(shaped_out_dev, rank_out_dev, w.g_key, w.g_idx, w.bucket_start,
                                                      w.bucket_count, w.bucket_id, N, member_offset, n_local);
        DES_LAUNCH_CHECK("rank_bucket kernels");
        return DES_OK;
    }
    int32_t *counts = (int32_t *)workspace_dev;
    DES_CUDA(cudaMemsetAsync(counts, 0, (size_t)n_local * sizeof(int32_t), st));
    const CountPlan p = count_plan(N, n_local);
    rank_count_kernel<<<dim3(p.bx, p.by), kRankThreads, 0, st>>>(counts, fitness_all_dev, N, member_offset, n_local,
                                                                 p.j_per_block);
    DES_LAUNCH_CHECK("rank_count_kernel");
    rank_finish_kernel<<<(unsigned)((n_local + 255) / 256), 256, 0, st>>>(shaped_out_dev, rank_out_dev, counts, N,
                                                                          n_local);
    DES_LAUNCH_CHECK("rank_finish_kernel");
    return DES_OK;
}

extern "C" DES_API size_t des_rank_runs_workspace_bytes(int64_t n_runs, int64_t run_size) {
    if (n_runs <= 0 || run_size <= 0 || run_size > des::kRunMaxSize || n_runs > ((int64_t)1 << 28) / run_size) return 0;
    return (size_t)(n_runs * run_size) * sizeof(int32_t);
}

extern "C" DES_API int des_centered_rank_runs(float *shaped_out_dev, int32_t *rank_out_dev, const float *fitness_dev,
                                              int64_t n_runs, int64_t run_size, void *workspace_dev, size_t workspace_bytes,
                                              void *stream) {
    using namespace des;
    const char *who = "des_centered_rank_runs";
    const int rc = check_runs(who, n_runs, run_size, 2);      // utils.py:146 divides by N-1
    if (rc != DES_OK) return rc;
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(shaped_out_dev && fitness_dev, "%s: NULL pointer", who);
    const size_t need = des_rank_runs_workspace_bytes(n_runs, run_size);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = n_runs * run_size;
    int32_t *counts = (int32_t *)workspace_dev;
    DES_CUDA(cudaMemsetAsync(counts, 0, (size_t)n * sizeof(int32_t), st));
    const CountPlan p = count_plan(run_size, run_size);       // one run's plan: a single j-slice up to 2048 members
    rank_count_runs_kernel<<<dim3((unsigned)(p.bx * n_runs), p.by), kRankThreads, 0, st>>>(counts, fitness_dev, run_size,
                                                                                          p.j_per_block, p.bx);
    DES_LAUNCH_CHECK("rank_count_runs_kernel");
    // the finishing step is elementwise in the rank: the batch is one vector of n ranks within runs of run_size
    rank_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(shaped_out_dev, rank_out_dev, counts, run_size, n);
    DES_LAUNCH_CHECK("rank_finish_kernel");
    return DES_OK;
}
