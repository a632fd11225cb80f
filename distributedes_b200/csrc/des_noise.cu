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
        const float4 z = noise_quad((uint32_t)q, noise_word(gm, mirrored), gen, tag, key);
        const float s = member_sigma(gm, mirrored, sigma);
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
    DES_REQUIRE(des::member_range_ok(member_offset, n_members, 32), "des_noise_fill: member index must fit 32 bits");
    DES_REQUIRE(P <= ((int64_t)1 << 34), "des_noise_fill: P too large for the 32-bit quad counter");
    return des::launch_rows(false, eps_out_dev, nullptr, n_members, P, 0.0, seed, generation, member_offset,
                            stream_tag, false, (cudaStream_t)stream);
}

namespace des {

static int nes_perturb(const char *who, float *theta_out_dev, const float *theta_dev, int64_t n_members, int64_t P,
                       double sigma, uint64_t seed, uint64_t generation, int64_t member_offset, bool mirrored,
                       cudaStream_t st) {
    DES_REQUIRE(n_members >= 0 && P >= 0, "%s: negative size", who);
    if (mirrored && !whole_pairs(member_offset, n_members)) return not_whole_pairs(who, "n_members", member_offset, n_members);
    DES_REQUIRE((theta_out_dev && theta_dev) || n_members * P == 0, "%s: NULL pointer", who);
    DES_REQUIRE(member_range_ok(member_offset, n_members, 32), "%s: member index must fit 32 bits", who);
    return launch_rows(true, theta_out_dev, theta_dev, n_members, P, sigma, seed, generation, member_offset, kStreamNesEps,
                       mirrored, st);
}

// A sweep's rows (des_nes_perturb_sweep): CTA row y takes run y, whose run_size rows are noise_rows_kernel<true>'s rows of
// theta_y with the seed and sigma of its table row, member_offset 0.  The round keys are set up once per thread.
__global__ void perturb_sweep_kernel(float *__restrict__ out, const float *__restrict__ theta, int64_t run_size, int64_t P,
                                     const des_run_hp *__restrict__ hp, uint32_t gen) {
    const int64_t nq = (P + 3) >> 2;
    const int64_t total = run_size * nq;
    const des_run_hp h = hp[blockIdx.y];
    PhiloxKey key;
    philox_round_keys(h.seed, key);
    const float s = (float)h.sigma;                               // the host's conversion of des_nes_perturb's sigma
    out += (int64_t)blockIdx.y * run_size * P;
    theta += (int64_t)blockIdx.y * P;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = idx / nq;
        const int64_t q = idx - m * nq;
        const float4 z = noise_quad((uint32_t)q, (uint32_t)m, gen, kStreamNesEps, key);
        const float zz[4] = {z.x, z.y, z.z, z.w};
        float *row = out + m * P;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int64_t j = 4 * q + e;
            if (j < P) row[j] = __fmaf_rn(s, zz[e], theta[j]);
        }
    }
}

// A sweep's normals (des_noise_fill_sweep): CTA row y takes run y, whose run_size rows are noise_rows_kernel<false>'s rows
// under the seed of its table row, member_offset 0 (CMA-ES's z of every run, stream kStreamCmaZ).
__global__ void noise_sweep_kernel(float *__restrict__ out, int64_t run_size, int64_t P, const des_run_hp *__restrict__ hp,
                                   uint32_t gen, uint32_t tag) {
    const int64_t nq = (P + 3) >> 2;
    const int64_t total = run_size * nq;
    PhiloxKey key;
    philox_round_keys(hp[blockIdx.y].seed, key);
    out += (int64_t)blockIdx.y * run_size * P;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = idx / nq;
        const int64_t q = idx - m * nq;
        const float4 z = noise_quad((uint32_t)q, (uint32_t)m, gen, tag, key);
        const float zz[4] = {z.x, z.y, z.z, z.w};
        float *row = out + m * P;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int64_t j = 4 * q + e;
            if (j < P) row[j] = zz[e];
        }
    }
}

}  // namespace des

extern "C" DES_API int des_noise_fill_sweep(float *z_out_dev, int64_t n_runs, int64_t run_size, int64_t P,
                                            const des_run_hp *hp_dev, uint64_t generation, uint32_t stream_tag,
                                            void *stream) {
    using namespace des;
    const char *who = "des_noise_fill_sweep";
    const int rc = check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(P > 0 && P <= ((int64_t)1 << 34), "%s: bad size P=%lld", who, (long long)P);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(z_out_dev && hp_dev, "%s: NULL pointer", who);
    const int threads = 256;
    const int64_t per_run = (run_size * ((P + 3) / 4) + threads - 1) / threads;
    for (int64_t r0 = 0; r0 < n_runs; r0 += 65535) {            // grid y: up to 65535 runs per launch
        const int64_t nr = n_runs - r0 < 65535 ? n_runs - r0 : 65535;
        const int64_t cap = 132 * 64 / nr > 0 ? 132 * 64 / nr : 1;     // about launch_rows' 132 x 64 CTAs in all
        noise_sweep_kernel<<<dim3((unsigned)(per_run < cap ? per_run : cap), (unsigned)nr), threads, 0,
                             (cudaStream_t)stream>>>(z_out_dev + r0 * run_size * P, run_size, P, hp_dev + r0,
                                                     (uint32_t)generation, stream_tag);
        DES_LAUNCH_CHECK("noise_sweep_kernel");
    }
    return DES_OK;
}

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

extern "C" DES_API int des_nes_perturb_sweep(float *rows_out_dev, const float *theta_dev, int64_t n_runs, int64_t run_size,
                                             int64_t P, const des_run_hp *hp_dev, uint64_t generation, void *stream) {
    using namespace des;
    const char *who = "des_nes_perturb_sweep";
    const int rc = check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(P > 0 && P <= ((int64_t)1 << 34), "%s: bad size P=%lld", who, (long long)P);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(rows_out_dev && theta_dev && hp_dev, "%s: NULL pointer", who);
    const int threads = 256;
    const int64_t per_run = (run_size * ((P + 3) / 4) + threads - 1) / threads;
    for (int64_t r0 = 0; r0 < n_runs; r0 += 65535) {            // grid y: up to 65535 runs per launch
        const int64_t nr = n_runs - r0 < 65535 ? n_runs - r0 : 65535;
        const int64_t cap = 132 * 64 / nr > 0 ? 132 * 64 / nr : 1;     // about launch_rows' 132 x 64 CTAs in all
        perturb_sweep_kernel<<<dim3((unsigned)(per_run < cap ? per_run : cap), (unsigned)nr), threads, 0,
                               (cudaStream_t)stream>>>(rows_out_dev + r0 * run_size * P, theta_dev + r0 * P, run_size, P,
                                                       hp_dev + r0, (uint32_t)generation);
        DES_LAUNCH_CHECK("perturb_sweep_kernel");
    }
    return DES_OK;
}
