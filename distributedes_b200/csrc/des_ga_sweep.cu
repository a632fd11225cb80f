// The genetic algorithm's table operations for a sweep of runs (include/des_b200.h, "genetic-algorithm sweeps"):
//   des_ga_rows_sweep   every run's generation rows [R * N][P], or, with a members list [R][table_rows], every run's next
//                       parents table gathered from its selected members
//   des_ga_order_runs   order_out[R][table_rows]: run r's T_r best members, best first, then -1
// Each thread reads its run's seed and sigma from the sweep table and its counts from the des_ga_run table, clamped to
// the [R][table_rows][P] buffers.
#include "des_ga.cuh"

static_assert(sizeof(des_ga_run) == 16 && offsetof(des_ga_run, n_elites) == 4 && offsetof(des_ga_run, truncation) == 8,
              "des_ga_run: 16 bytes, the header's field offsets");

namespace des {

// One thread per (row, quad), as ga_rows_kernel.  Rows mode (members NULL): row i is member i % run_size of run
// i / run_size.  Gather mode: row i = (r, k) is member members[i] of run r = i / table_rows; a negative member is skipped.
__global__ void ga_rows_sweep_kernel(float *__restrict__ out, const float *__restrict__ parents,
                                     const des_ga_run *__restrict__ ga, int table_rows, int64_t n, int64_t P,
                                     const des_run_hp *__restrict__ hp, uint32_t gen, int64_t run_size,
                                     const int32_t *__restrict__ members) {
    const int64_t nq = (P + 3) >> 2;
    const int64_t total = n * nq;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx / nq;
        const int64_t q = idx - i * nq;
        int64_t r;
        uint32_t m;
        if (members) {
            const int32_t mm = __ldg(members + i);
            if (mm < 0) continue;
            r = i / table_rows;
            m = (uint32_t)mm;
        } else {
            r = i / run_size;
            m = (uint32_t)(i - r * run_size);
        }
        const des_run_hp h = hp[r];
        const des_ga_run g = ga[r];
        PhiloxKey key;
        philox_round_keys(h.seed, key);
        const int n_parents = min(max(g.n_parents, 1), table_rows);
        const int n_elites = min(max(g.n_elites, 0), n_parents);
        ga_row_quad(out + i * P, parents + r * table_rows * P, (uint32_t)n_parents, (uint32_t)n_elites, P, q,
                    (float)h.sigma, key, gen, m);
    }
}

// keys[i] = -fitness[i] over every run (ga_negate_kernel's order: ascending rank of -fitness = descending position)
__global__ void ga_negate_runs_kernel(float *__restrict__ keys, const float *__restrict__ fitness, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keys[i] = -fitness[i];
}

// order[r][rank_i] = i % run_size for run r's members whose rank is below its truncation, clamped to [1, table_rows]
__global__ void ga_scatter_runs_kernel(int32_t *__restrict__ order, const int32_t *__restrict__ rank,
                                       const des_ga_run *__restrict__ ga, int64_t n, int64_t run_size, int table_rows) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t r = i / run_size;
    const int T = min(max(ga[r].truncation, 1), table_rows);
    const int32_t k = rank[i];
    if (k >= 0 && k < T) order[r * table_rows + k] = (int32_t)(i - r * run_size);
}

static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace des

extern "C" DES_API int des_ga_rows_sweep(float *rows_out_dev, const float *parents_dev, const des_ga_run *ga_dev,
                                         int64_t table_rows, int64_t P, const des_run_hp *hp_dev, uint64_t generation,
                                         int64_t n_runs, int64_t run_size, const int32_t *members_dev, void *stream) {
    using namespace des;
    const char *who = "des_ga_rows_sweep";
    const int rc = check_runs(who, n_runs, run_size, 2);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(P >= 1 && P <= ((int64_t)1 << 34), "%s: bad size (P=%lld)", who, (long long)P);
    DES_REQUIRE(table_rows >= 1 && table_rows <= run_size, "%s: table_rows must be in [1, run_size = %lld] (got %lld)", who,
                (long long)run_size, (long long)table_rows);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(rows_out_dev && parents_dev && ga_dev && hp_dev, "%s: NULL pointer", who);
    const int64_t n = n_runs * (members_dev ? table_rows : run_size);
    {       // the tables are double-buffered: the rows may not overlap the parents they are built from
        const uintptr_t o0 = (uintptr_t)rows_out_dev, o1 = o0 + (uintptr_t)(n * P) * sizeof(float);
        const uintptr_t p0 = (uintptr_t)parents_dev, p1 = p0 + (uintptr_t)(n_runs * table_rows * P) * sizeof(float);
        DES_REQUIRE(o1 <= p0 || p1 <= o0, "%s: rows_out overlaps parents (the table is double-buffered)", who);
    }
    const int threads = 256;
    int64_t blocks = (n * ((P + 3) / 4) + threads - 1) / threads;
    if (blocks > 132 * 64) blocks = 132 * 64;      // 132 SMs (H100 SXM), as des_ga_rows
    ga_rows_sweep_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
        rows_out_dev, parents_dev, ga_dev, (int)table_rows, n, P, hp_dev, (uint32_t)generation, run_size, members_dev);
    DES_LAUNCH_CHECK("ga_rows_sweep_kernel");
    return DES_OK;
}

extern "C" DES_API size_t des_ga_order_runs_workspace_bytes(int64_t n_runs, int64_t run_size) {
    const size_t rank = des_rank_runs_workspace_bytes(n_runs, run_size);
    if (rank == 0 || run_size < 2) return 0;
    const size_t n = (size_t)(n_runs * run_size);
    return 256 + 3 * des::al256(n * 4) + rank;
}

extern "C" DES_API int des_ga_order_runs(int32_t *order_out_dev, const float *fitness_dev, const des_ga_run *ga_dev,
                                         int64_t table_rows, int64_t n_runs, int64_t run_size, void *workspace_dev,
                                         size_t workspace_bytes, void *stream) {
    using namespace des;
    const char *who = "des_ga_order_runs";
    const int rc = check_runs(who, n_runs, run_size, 2);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(table_rows >= 1 && table_rows <= run_size, "%s: table_rows must be in [1, run_size = %lld] (got %lld)", who,
                (long long)run_size, (long long)table_rows);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(order_out_dev && fitness_dev && ga_dev, "%s: NULL pointer", who);
    const size_t need = des_ga_order_runs_workspace_bytes(n_runs, run_size);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = n_runs * run_size;
    uint8_t *p = (uint8_t *)(((uintptr_t)workspace_dev + 255) & ~(uintptr_t)255);
    float *keys = (float *)p; p += al256((size_t)n * 4);
    float *shaped = (float *)p; p += al256((size_t)n * 4);
    int32_t *rank = (int32_t *)p; p += al256((size_t)n * 4);
    const uint8_t *end = (const uint8_t *)workspace_dev + workspace_bytes;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    ga_negate_runs_kernel<<<blocks, 256, 0, st>>>(keys, fitness_dev, n);
    DES_LAUNCH_CHECK("ga_negate_runs_kernel");
    const int rr = des_centered_rank_runs(shaped, rank, keys, n_runs, run_size, p, (size_t)(end - p), stream);
    if (rr != DES_OK) return rr;
    DES_CUDA(cudaMemsetAsync(order_out_dev, 0xFF, (size_t)(n_runs * table_rows) * sizeof(int32_t), st));   // -1
    ga_scatter_runs_kernel<<<blocks, 256, 0, st>>>(order_out_dev, rank, ga_dev, n, run_size, (int)table_rows);
    DES_LAUNCH_CHECK("ga_scatter_runs_kernel");
    return DES_OK;
}
