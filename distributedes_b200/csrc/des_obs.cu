// Observation normaliser (SURVEY 8f row 1): StaticNormalizer / SharedStats, utils.py:37-106.
//   des_obs_stats_merge          tape statistics -> shared statistics           (tape environment)
//   des_obs_normalize            (o - m)/sqrt(v + 1e-6) of the tape
//   des_obs_parts_reduce         per-member partial sums -> totals               (des_rollout_eval, des_policy_act rows)
//   des_obs_stats_merge_totals   totals (all-reduced over ranks) -> shared statistics
//   des_obs_stats_merge_totals_runs  the same for a batch of runs: one row of totals into one row of statistics per run
// In the reference every worker feeds each observation into online Welford statistics (utils.py:68-73) and, after
// the generation, the master Chan-merges them into the shared statistics (utils.py:85-96); observations are
// normalised with the statistics of the PREVIOUS generations, (o - m)/sqrt(v + 1e-6), raw while n == 0
// (utils.py:48-51).  On the tape environment every member sees the same T observations, so one generation's
// online statistics are the tape's mean / population variance with weight n_feed = members * T.
#include "des_common.cuh"

namespace des {

// stats layout (device, fp32 like the reference's torch tensors): m[d0] | v[d0] | n[1]
// SharedStats.merge, utils.py:85-96: column k of the shared statistics (A) absorbs batch statistics (mb, vb) of weight nB.
// One block; every thread of a live column calls it.
__device__ __forceinline__ void chan_merge(float *__restrict__ stats, int d0, int k, double mb, double vb, double nB) {
    const double nA = (double)stats[2 * d0], n = nA + nB;
    const double mA = (double)stats[k], vA = (double)stats[d0 + k];
    const double delta = mb - mA;
    const double m = mA + delta * nB / n;
    const double v = (vA * nA + vb * nB + delta * delta * nA * nB / n) / n;
    __syncthreads();                      // every thread has read n before thread 0 updates it (single block)
    stats[k] = (float)m;
    stats[d0 + k] = (float)v;
    if (k == 0) stats[2 * d0] = (float)n;
}

__global__ void obs_stats_merge_kernel(float *__restrict__ stats, const float *__restrict__ obs, int T, int d0,
                                       double n_feed) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= d0) return;
    // batch statistics of the tape column k (fp64 two-pass; the reference accumulates them one sample at a time)
    double s = 0.0;
    for (int t = 0; t < T; ++t) s += (double)obs[(int64_t)t * d0 + k];
    const double mb = s / T;
    double q = 0.0;
    for (int t = 0; t < T; ++t) {
        const double d = (double)obs[(int64_t)t * d0 + k] - mb;
        q += d * d;
    }
    chan_merge(stats, d0, k, mb, q / T, n_feed);
}

__global__ void obs_normalize_kernel(float *__restrict__ out, const float *__restrict__ obs, const float *__restrict__ stats,
                                     int T, int d0) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)T * d0) return;
    const int k = (int)(i % d0);
    const float o = obs[i];
    if (stats[2 * d0] == 0.f) {           // utils.py:48-49: no statistics yet -> pass through
        out[i] = o;
        return;
    }
    const float std_ = sqrtf(stats[d0 + k] + 1e-6f);      // utils.py:50
    out[i] = (o - stats[k]) / std_;                        // utils.py:51
}

// Chan-merge the observation totals (all members of all ranks, after an all-reduce of the three sums) into the shared
// statistics.  totals = [sum(d0) | sumsq(d0) | count] in fp64.
__global__ void obs_stats_merge_totals_kernel(float *__restrict__ stats, const double *__restrict__ totals, int d0) {
    const int k = threadIdx.x;
    if (k >= d0) return;
    const double nB = totals[2 * d0];
    if (nB <= 0) return;
    const double mb = totals[k] / nB, vb = fmax(totals[d0 + k] / nB - mb * mb, 0.0);
    chan_merge(stats, d0, k, mb, vb, nB);
}

__global__ void stat_part_reduce_kernel(double *__restrict__ totals, const double *__restrict__ part, int64_t n_local, int width) {
    // one thread per column, fixed order over members: deterministic
    const int c = threadIdx.x;
    if (c >= width) return;
    double s = 0.0;
    for (int64_t i = 0; i < n_local; ++i) s += part[i * width + c];
    totals[c] = s;
}

// one CTA per run: run blockIdx.x's rows in member order, as stat_part_reduce_kernel sums a single population's
__global__ void stat_part_reduce_runs_kernel(double *__restrict__ totals, const double *__restrict__ part, int64_t run_size,
                                             int width) {
    const int c = threadIdx.x;
    if (c >= width) return;
    const double *p = part + (int64_t)blockIdx.x * run_size * width;
    double s = 0.0;
    for (int64_t i = 0; i < run_size; ++i) s += p[i * width + c];
    totals[(int64_t)blockIdx.x * width + c] = s;
}

// one CTA per run, the columns of obs_stats_merge_totals_kernel
__global__ void obs_stats_merge_totals_runs_kernel(float *__restrict__ stats, const double *__restrict__ totals, int d0) {
    const int k = threadIdx.x;
    if (k >= d0) return;
    const int w = 2 * d0 + 1;
    stats += (int64_t)blockIdx.x * w;
    totals += (int64_t)blockIdx.x * w;
    const double nB = totals[2 * d0];
    if (nB <= 0) return;
    const double mb = totals[k] / nB, vb = fmax(totals[d0 + k] / nB - mb * mb, 0.0);
    chan_merge(stats, d0, k, mb, vb, nB);
}

int obs_parts_reduce_runs(double *totals, const double *parts, int64_t n_runs, int64_t run_size, int width, cudaStream_t st) {
    if (n_runs == 0) return DES_OK;
    stat_part_reduce_runs_kernel<<<(unsigned)n_runs, (unsigned)((width + 31) / 32 * 32), 0, st>>>(totals, parts, run_size,
                                                                                                 width);
    DES_LAUNCH_CHECK("stat_part_reduce_runs_kernel");
    return DES_OK;
}

int obs_parts_reduce(double *totals, const double *parts, int64_t n_local, int width, cudaStream_t st) {
    stat_part_reduce_kernel<<<1, (unsigned)((width + 31) / 32 * 32), 0, st>>>(totals, parts, n_local, width);
    DES_LAUNCH_CHECK("stat_part_reduce_kernel");
    return DES_OK;
}

}  // namespace des

extern "C" DES_API int des_obs_stats_merge(float *stats_dev, const float *obs_dev, int32_t tape_len, int32_t state_dim,
                                           double n_feed, void *stream) {
    DES_REQUIRE(stats_dev && obs_dev, "des_obs_stats_merge: NULL pointer");
    DES_REQUIRE(tape_len > 0 && state_dim > 0 && state_dim <= 1024 && n_feed > 0, "des_obs_stats_merge: bad sizes");
    des::obs_stats_merge_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(stats_dev, obs_dev, tape_len, state_dim, n_feed);
    DES_LAUNCH_CHECK("obs_stats_merge_kernel");
    return DES_OK;
}

extern "C" DES_API int des_obs_normalize(float *obs_out_dev, const float *obs_dev, const float *stats_dev, int32_t tape_len,
                                         int32_t state_dim, void *stream) {
    DES_REQUIRE(obs_out_dev && obs_dev && stats_dev, "des_obs_normalize: NULL pointer");
    DES_REQUIRE(tape_len > 0 && state_dim > 0, "des_obs_normalize: bad sizes");
    const int64_t total = (int64_t)tape_len * state_dim;
    des::obs_normalize_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(obs_out_dev, obs_dev, stats_dev,
                                                                                           tape_len, state_dim);
    DES_LAUNCH_CHECK("obs_normalize_kernel");
    return DES_OK;
}

extern "C" DES_API int des_obs_parts_reduce(double *obs_totals_out_dev, const double *parts_dev, int64_t n_local,
                                            int32_t state_dim, void *stream) {
    DES_REQUIRE(state_dim > 0 && state_dim <= 511 && n_local >= 0, "des_obs_parts_reduce: bad arguments");
    DES_REQUIRE(obs_totals_out_dev && (parts_dev || n_local == 0), "des_obs_parts_reduce: NULL pointer");
    return des::obs_parts_reduce(obs_totals_out_dev, parts_dev, n_local, 2 * state_dim + 1, (cudaStream_t)stream);
}

extern "C" DES_API int des_obs_stats_merge_totals(float *stats_dev, const double *obs_totals_dev, int32_t state_dim,
                                                  void *stream) {
    DES_REQUIRE(stats_dev && obs_totals_dev && state_dim > 0 && state_dim <= 1024, "des_obs_stats_merge_totals: bad arguments");
    des::obs_stats_merge_totals_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(stats_dev, obs_totals_dev, state_dim);
    DES_LAUNCH_CHECK("obs_stats_merge_totals_kernel");
    return DES_OK;
}

extern "C" DES_API int des_obs_stats_merge_totals_runs(float *stats_dev, const double *obs_totals_dev, int32_t state_dim,
                                                       int64_t n_runs, void *stream) {
    const char *who = "des_obs_stats_merge_totals_runs";
    DES_REQUIRE(state_dim > 0 && state_dim <= 1024, "%s: state_dim must be in [1, 1024] (got %d)", who, (int)state_dim);
    DES_REQUIRE(n_runs >= 0 && n_runs <= ((int64_t)1 << 28), "%s: need 0 <= n_runs <= 2^28 (got %lld)", who,
                (long long)n_runs);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(stats_dev && obs_totals_dev, "%s: NULL pointer", who);
    des::obs_stats_merge_totals_runs_kernel<<<(unsigned)n_runs, (unsigned)((state_dim + 31) / 32 * 32), 0,
                                              (cudaStream_t)stream>>>(stats_dev, obs_totals_dev, state_dim);
    DES_LAUNCH_CHECK("obs_stats_merge_totals_runs_kernel");
    return DES_OK;
}

extern "C" DES_API int des_obs_parts_reduce_runs(double *obs_totals_out_dev, const double *parts_dev, int64_t n_runs,
                                                 int64_t run_size, int32_t state_dim, void *stream) {
    const char *who = "des_obs_parts_reduce_runs";
    const int rc = des::check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(state_dim > 0 && state_dim <= 511, "%s: state_dim must be in [1, 511] (got %d)", who, (int)state_dim);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(obs_totals_out_dev && parts_dev, "%s: NULL pointer", who);
    return des::obs_parts_reduce_runs(obs_totals_out_dev, parts_dev, n_runs, run_size, 2 * state_dim + 1,
                                      (cudaStream_t)stream);
}
