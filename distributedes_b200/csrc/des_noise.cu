// Debug / parity ops that MATERIALISE the noise (the hot path never does):
//   des_noise_fill   eps[n][P]                    replaces np.random.randn, natural_es.py:29
//   des_nes_perturb  theta'[n][P] = theta+sigma*eps   natural_es.py:28-30
#include "des_common.cuh"

namespace des {

// One thread per (member, quad).  Rows are P floats with arbitrary P, so stores are scalar and guarded.
// mirrored (perturb rows only): member m is theta + (-1)^(m & 1) sigma * eps of counter word m >> 1.
template <bool kPerturb>
__global__ void noise_rows_kernel(float *__restrict__ out, const float *__restrict__ theta, int64_t n_members,
                                  int64_t P, float sigma, PhiloxKey key, uint32_t gen,
                                  uint32_t tag, uint64_t member_offset, int mirrored) {
    const int64_t nq = (P + 3) >> 2;
    const int64_t total = n_members * nq;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = idx / nq;
        const int64_t q = idx - m * nq;
        const uint64_t gm = member_offset + m;
        const float4 z = noise_quad((uint32_t)q, (uint32_t)(mirrored ? gm >> 1 : gm), gen, tag, key);
        const float s = mirrored && (gm & 1u) ? -sigma : sigma;
        const float zz[4] = {z.x, z.y, z.z, z.w};
        float *row = out + m * P;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int64_t j = 4 * q + e;
            if (j < P) row[j] = kPerturb ? __fmaf_rn(s, zz[e], theta[j]) : zz[e];
        }
    }
}

static int launch_rows(bool perturb, float *out, const float *theta, int64_t n, int64_t P, double sigma,
                       uint64_t seed, uint64_t gen, int64_t member_offset, uint32_t tag, bool mirrored, cudaStream_t st) {
    if (n == 0 || P == 0) return DES_OK;
    const int64_t total = n * ((P + 3) / 4);
    const int threads = 256;
    int64_t blocks = (total + threads - 1) / threads;
    if (blocks > 132 * 64) blocks = 132 * 64;      // 132 SMs (H100 SXM)
    const PhiloxKey key = make_philox_key(seed);
    if (perturb)
        noise_rows_kernel<true><<<(unsigned)blocks, threads, 0, st>>>(out, theta, n, P, (float)sigma, key,
                                                                      (uint32_t)gen, tag, (uint64_t)member_offset,
                                                                      mirrored ? 1 : 0);
    else
        noise_rows_kernel<false><<<(unsigned)blocks, threads, 0, st>>>(out, nullptr, n, P, 0.f, key,
                                                                       (uint32_t)gen, tag, (uint64_t)member_offset, 0);
    DES_LAUNCH_CHECK("noise_rows_kernel");
    return DES_OK;
}

}  // namespace des

extern "C" DES_API int des_noise_fill(float *eps_out_dev, int64_t n_members, int64_t P, uint64_t seed, uint64_t generation,
                              int64_t member_offset, uint32_t stream_tag, void *stream) {
    DES_REQUIRE(n_members >= 0 && P >= 0, "des_noise_fill: negative size (n_members=%lld, P=%lld)",
                (long long)n_members, (long long)P);
    DES_REQUIRE(eps_out_dev || n_members * P == 0, "des_noise_fill: eps_out_dev is NULL");
    DES_REQUIRE(member_offset >= 0 && member_offset + n_members <= (int64_t)1 << 32,
                "des_noise_fill: member index must fit 32 bits");
    DES_REQUIRE(P <= ((int64_t)1 << 34), "des_noise_fill: P too large for the 32-bit quad counter");
    return des::launch_rows(false, eps_out_dev, nullptr, n_members, P, 0.0, seed, generation, member_offset,
                            stream_tag, false, (cudaStream_t)stream);
}

namespace des {

static int nes_perturb(const char *who, float *theta_out_dev, const float *theta_dev, int64_t n_members, int64_t P,
                       double sigma, uint64_t seed, uint64_t generation, int64_t member_offset, bool mirrored,
                       cudaStream_t st) {
    DES_REQUIRE(n_members >= 0 && P >= 0, "%s: negative size", who);
    DES_REQUIRE(!mirrored || (member_offset % 2 == 0 && n_members % 2 == 0),
                "%s: a mirrored shard holds whole pairs: member_offset (%lld) and n_members (%lld) must be even", who,
                (long long)member_offset, (long long)n_members);
    DES_REQUIRE((theta_out_dev && theta_dev) || n_members * P == 0, "%s: NULL pointer", who);
    DES_REQUIRE(member_offset >= 0 && member_offset + n_members <= (int64_t)1 << 32, "%s: member index must fit 32 bits", who);
    return launch_rows(true, theta_out_dev, theta_dev, n_members, P, sigma, seed, generation, member_offset, kStreamNesEps,
                       mirrored, st);
}

}  // namespace des

extern "C" DES_API int des_nes_perturb(float *theta_out_dev, const float *theta_dev, int64_t n_members, int64_t P,
                               double sigma, uint64_t seed, uint64_t generation, int64_t member_offset,
                               void *stream) {
    return des::nes_perturb("des_nes_perturb", theta_out_dev, theta_dev, n_members, P, sigma, seed, generation,
                            member_offset, false, (cudaStream_t)stream);
}

extern "C" DES_API int des_nes_perturb_mirrored(float *theta_out_dev, const float *theta_dev, int64_t n_members, int64_t P,
                                                double sigma, uint64_t seed, uint64_t generation, int64_t member_offset,
                                                void *stream) {
    return des::nes_perturb("des_nes_perturb_mirrored", theta_out_dev, theta_dev, n_members, P, sigma, seed, generation,
                            member_offset, true, (cudaStream_t)stream);
}

// ---- observation normaliser (SURVEY 8f row 1): StaticNormalizer / SharedStats, utils.py:37-106 ---------------------
// In the reference every worker feeds each observation into online Welford statistics (utils.py:68-73) and, after
// the generation, the master Chan-merges them into the shared statistics (utils.py:85-96); observations are
// normalised with the statistics of the PREVIOUS generations, (o - m)/sqrt(v + 1e-6), raw while n == 0
// (utils.py:48-51).  On the tape environment every member sees the same T observations, so one generation's
// online statistics are the tape's mean / population variance with weight n_feed = members * T.
namespace des {

// stats layout (device, fp32 like the reference's torch tensors): m[d0] | v[d0] | n[1]
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
    const double vb = q / T;
    // SharedStats.merge, utils.py:85-96 (A = shared stats, B = this generation's online stats)
    const double nA = (double)stats[2 * d0], nB = n_feed, n = nA + nB;
    const double mA = (double)stats[k], vA = (double)stats[d0 + k];
    const double delta = mb - mA;
    const double m = mA + delta * nB / n;
    const double v = (vA * nA + vb * nB + delta * delta * nA * nB / n) / n;
    __syncthreads();                      // every thread has read n before thread 0 updates it (single block)
    stats[k] = (float)m;
    stats[d0 + k] = (float)v;
    if (k == 0) stats[2 * d0] = (float)n;
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
