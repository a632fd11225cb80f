// The genetic algorithm's table operations (include/des_b200.h, "genetic algorithm"):
//   des_ga_rows   rows_out[n][P]: the weights of members of a generation, each an elite's parent row or a parent row
//                 plus sigma*eps of the member: a generation's rows (host-stepped and tape sources), or, with a members
//                 list, the next parents table gathered from the selected members
//   des_ga_order  order_out[T]: the members of the T best fitnesses, best first (truncation selection)
//   des_ns_ga_order  order_out[T]: the members of the T smallest keys of the blend of the fitness and novelty ranks
//                    (the genetic algorithm's novelty search), from des_ns_shape, the rank and des_ga_order's kernels
#include "des_ga.cuh"

namespace des {

// One thread per (row, quad), as noise_rows_kernel<true>.  Row i is member members[i] (or member_offset + i).
__global__ void ga_rows_kernel(float *__restrict__ out, const float *__restrict__ parents, uint32_t n_parents,
                               uint32_t n_elites, int64_t n, int64_t P, float sigma, PhiloxKey key, uint32_t gen,
                               uint64_t member_offset, const int32_t *__restrict__ members) {
    const int64_t nq = (P + 3) >> 2;
    const int64_t total = n * nq;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx / nq;
        const int64_t q = idx - i * nq;
        const uint32_t m = members ? (uint32_t)__ldg(members + i) : (uint32_t)(member_offset + i);
        ga_row_quad(out + i * P, parents, n_parents, n_elites, P, q, sigma, key, gen, m);
    }
}

// keys[i] = -fitness[i]: the ascending rank of the negated fitness is the descending position (ties by index, NaN last,
// -0 == +0, as des_centered_rank orders)
__global__ void ga_negate_kernel(float *__restrict__ keys, const float *__restrict__ fitness, int64_t N) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) keys[i] = -fitness[i];
}

// order[rank_i] = i for the members whose rank is below T
__global__ void ga_scatter_kernel(int32_t *__restrict__ order, const int32_t *__restrict__ rank, int64_t N, int64_t T) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N && rank[i] < T) order[rank[i]] = (int32_t)i;
}

// The order's workspace: the negated fitness, the shaped values and the ranks des_centered_rank writes, then its own.
struct OrderWs {
    float *keys, *shaped;
    int32_t *rank;
    void *rank_ws;
};
static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
static OrderWs carve_order(void *ws, int64_t N) {
    uint8_t *p = (uint8_t *)(((uintptr_t)ws + 255) & ~(uintptr_t)255);
    OrderWs w;
    w.keys = (float *)p; p += al256((size_t)N * 4);
    w.shaped = (float *)p; p += al256((size_t)N * 4);
    w.rank = (int32_t *)p; p += al256((size_t)N * 4);
    w.rank_ws = p;
    return w;
}

}  // namespace des

extern "C" DES_API int des_ga_rows(float *rows_out_dev, const float *parents_dev, int64_t n_parents, int64_t n_elites,
                                   int64_t P, double sigma, uint64_t seed, uint64_t generation, int64_t member_offset,
                                   int64_t n_local, const int32_t *members_dev, void *stream) {
    using namespace des;
    const char *who = "des_ga_rows";
    DES_REQUIRE(n_local >= 0 && P >= 1 && P <= ((int64_t)1 << 34), "%s: bad size (n_local=%lld, P=%lld)", who,
                (long long)n_local, (long long)P);
    DES_REQUIRE(n_parents >= 1 && n_parents <= INT32_MAX, "%s: n_parents must be in [1, 2^31) (got %lld)", who,
                (long long)n_parents);
    DES_REQUIRE(n_elites >= 0 && n_elites <= n_parents, "%s: n_elites must be in [0, n_parents = %lld] (got %lld)", who,
                (long long)n_parents, (long long)n_elites);
    DES_REQUIRE(members_dev || member_range_ok(member_offset, n_local, 32), "%s: member index must fit 32 bits", who);
    if (n_local == 0) return DES_OK;
    DES_REQUIRE(rows_out_dev && parents_dev, "%s: NULL pointer", who);
    {       // the table is double-buffered: the rows may not overlap the parents they are built from
        const uintptr_t o0 = (uintptr_t)rows_out_dev, o1 = o0 + (uintptr_t)(n_local * P) * sizeof(float);
        const uintptr_t p0 = (uintptr_t)parents_dev, p1 = p0 + (uintptr_t)(n_parents * P) * sizeof(float);
        DES_REQUIRE(o1 <= p0 || p1 <= o0, "%s: rows_out overlaps parents (the table is double-buffered)", who);
    }
    const int threads = 256;
    int64_t blocks = (n_local * ((P + 3) / 4) + threads - 1) / threads;
    if (blocks > 132 * 64) blocks = 132 * 64;      // 132 SMs (H100 SXM), as launch_rows
    ga_rows_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(
        rows_out_dev, parents_dev, (uint32_t)n_parents, (uint32_t)n_elites, n_local, P, (float)sigma,
        make_philox_key(seed), (uint32_t)generation, (uint64_t)member_offset, members_dev);
    DES_LAUNCH_CHECK("ga_rows_kernel");
    return DES_OK;
}

extern "C" DES_API size_t des_ga_order_workspace_bytes(int64_t N) {
    if (N < 2) return 0;
    return 256 + 3 * des::al256((size_t)N * 4) + des_rank_workspace_bytes(N, N);
}

extern "C" DES_API int des_ga_order(int32_t *order_out_dev, const float *fitness_dev, int64_t N, int64_t T,
                                    void *workspace_dev, size_t workspace_bytes, void *stream) {
    using namespace des;
    const char *who = "des_ga_order";
    DES_REQUIRE(N >= 2 && N <= INT32_MAX, "%s: N=%lld, need 2 <= N < 2^31", who, (long long)N);
    DES_REQUIRE(T >= 1 && T <= N, "%s: T must be in [1, N = %lld] (got %lld)", who, (long long)N, (long long)T);
    DES_REQUIRE(order_out_dev && fitness_dev, "%s: NULL pointer", who);
    const size_t need = des_ga_order_workspace_bytes(N);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const OrderWs w = carve_order(workspace_dev, N);
    const unsigned blocks = (unsigned)((N + 255) / 256);
    ga_negate_kernel<<<blocks, 256, 0, st>>>(w.keys, fitness_dev, N);
    DES_LAUNCH_CHECK("ga_negate_kernel");
    const uint8_t *end = (const uint8_t *)workspace_dev + workspace_bytes;
    const int rc = des_centered_rank(w.shaped, w.rank, w.keys, N, 0, N, w.rank_ws, (size_t)(end - (uint8_t *)w.rank_ws),
                                     stream);
    if (rc != DES_OK) return rc;
    ga_scatter_kernel<<<blocks, 256, 0, st>>>(order_out_dev, w.rank, N, T);
    DES_LAUNCH_CHECK("ga_scatter_kernel");
    return DES_OK;
}

extern "C" DES_API size_t des_ns_ga_order_workspace_bytes(int64_t N) {
    if (N < 2) return 0;
    return 256 + 5 * des::al256((size_t)N * 4) + des_ns_shape_workspace_bytes(N);
}

// The negated fitness and novelty, their blend (des_ns_shape: both ranks, then fmaf(w, c_f, fp32(1 - w) * c_n)), the
// ascending rank of that key (ties to the lower index) and des_ga_order's scatter.  The rank of the key and des_ns_shape
// run one after the other on the stream, so they share the tail of the workspace.
extern "C" DES_API int des_ns_ga_order(int32_t *order_out_dev, const float *fitness_dev, const float *novelty_dev,
                                       int64_t N, int64_t T, double reward_weight, void *workspace_dev,
                                       size_t workspace_bytes, void *stream) {
    using namespace des;
    const char *who = "des_ns_ga_order";
    DES_REQUIRE(N >= 2 && N <= ((int64_t)1 << 24), "%s: N=%lld, need 2 <= N <= 2^24 (above, two centered ranks can round "
                "to one fp32 key)", who, (long long)N);
    DES_REQUIRE(T >= 1 && T <= N, "%s: T must be in [1, N = %lld] (got %lld)", who, (long long)N, (long long)T);
    DES_REQUIRE(reward_weight >= 0.0 && reward_weight <= 1.0, "%s: reward_weight must be in [0, 1] (got %g)", who,
                reward_weight);
    DES_REQUIRE(order_out_dev && fitness_dev && novelty_dev, "%s: NULL pointer", who);
    const size_t need = des_ns_ga_order_workspace_bytes(N);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    uint8_t *p = (uint8_t *)(((uintptr_t)workspace_dev + 255) & ~(uintptr_t)255);
    float *neg_f = (float *)p; p += al256((size_t)N * 4);
    float *neg_n = (float *)p; p += al256((size_t)N * 4);
    float *key = (float *)p; p += al256((size_t)N * 4);
    float *shaped = (float *)p; p += al256((size_t)N * 4);
    int32_t *rank = (int32_t *)p; p += al256((size_t)N * 4);
    const size_t tail = (size_t)((const uint8_t *)workspace_dev + workspace_bytes - p);
    const unsigned blocks = (unsigned)((N + 255) / 256);
    ga_negate_kernel<<<blocks, 256, 0, st>>>(neg_f, fitness_dev, N);
    DES_LAUNCH_CHECK("ga_negate_kernel");
    ga_negate_kernel<<<blocks, 256, 0, st>>>(neg_n, novelty_dev, N);
    DES_LAUNCH_CHECK("ga_negate_kernel");
    int rc = des_ns_shape(key, neg_f, neg_n, N, reward_weight, p, tail, stream);
    if (rc != DES_OK) return rc;
    rc = des_centered_rank(shaped, rank, key, N, 0, N, p, tail, stream);
    if (rc != DES_OK) return rc;
    ga_scatter_kernel<<<blocks, 256, 0, st>>>(order_out_dev, rank, N, T);
    DES_LAUNCH_CHECK("ga_scatter_kernel");
    return DES_OK;
}
