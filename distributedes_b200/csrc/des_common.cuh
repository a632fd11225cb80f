// Shared device helpers: Philox4x32-10 counter RNG, Box-Muller, error plumbing.
// Target: sm_90a (H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/des_b200.h"

namespace des {

// ---- error plumbing (host) ---------------------------------------------------------------------
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);

#define DES_REQUIRE(cond, ...)                    \
    do {                                          \
        if (!(cond)) {                            \
            ::des::set_error(__VA_ARGS__);        \
            return DES_ERR_INVALID_ARGUMENT;      \
        }                                         \
    } while (0)

#define DES_CUDA(call)                                            \
    do {                                                          \
        cudaError_t e__ = (call);                                 \
        if (e__ != cudaSuccess) return ::des::cuda_fail(e__, #call); \
    } while (0)

#define DES_LAUNCH_CHECK(name)                                    \
    do {                                                          \
        cudaError_t e__ = cudaGetLastError();                     \
        if (e__ != cudaSuccess) return ::des::cuda_fail(e__, name); \
    } while (0)

// ---- layout of the flat parameter vector (model.py:8-25, 30-32) -----------------------------------
struct Layout {
    int d0, H, A;
    int off_w1, off_b1, off_w2, off_b2, off_w3, off_b3, P;
    __host__ __device__ Layout() {}
    __host__ __device__ Layout(int d0_, int H_, int A_) : d0(d0_), H(H_), A(A_) {
        off_w1 = 0;
        off_b1 = off_w1 + H * d0;
        off_w2 = off_b1 + H;
        off_b2 = off_w2 + H * H;
        off_w3 = off_b2 + H;
        off_b3 = off_w3 + A * H;
        P = off_b3 + A;
    }
};

// ---- Philox4x32-R, R = kPhiloxRounds ---------------------------------------------------------------
// Round 2 moved the noise contract from 10 to 7 rounds: Philox4x32-7 is the smallest round count Salmon et al.
// (SC'11, table 2) report as passing BigCrush; the generator is paid for twice per generation (forward and
// fitness x noise reduction), where the ten-round multiplies were the busiest pipe (profiles/README.md §3).
// oracle/nes_oracle.py, the goldens and include/des_b200.h moved in the same commit.
constexpr int kPhiloxRounds = 7;
constexpr uint32_t kPhiloxM0 = 0xD2511F53u;
constexpr uint32_t kPhiloxM1 = 0xCD9E8D57u;
constexpr uint32_t kPhiloxW0 = 0x9E3779B9u;
constexpr uint32_t kPhiloxW1 = 0xBB67AE85u;
// Counter streams (the fourth counter word): NES perturbations, CMA-ES samples, environment resets, action noise.  The
// host-stepped policy (des_act.cu) draws its action noise exactly as the device rollout (des_envs.cu) does.
constexpr uint32_t kStreamNesEps = 0u;
constexpr uint32_t kStreamCmaZ = 1u;
constexpr uint32_t kStreamEnvReset = 2u;
constexpr uint32_t kStreamActNoise = 3u;
// Stream 4 is the host's episode seed (envs.py).  Stream 5: the genetic algorithm's parent draws (ga_parent).
constexpr uint32_t kStreamGaParent = 5u;
// Member word of the test episodes' resets (test(), natural_es.py:101-110): no member of a population reaches it.
constexpr uint32_t kTestEpisodeMember = 0x40000000u;

// Round keys k + r*W precomputed on the host (kernel-parameter constant bank): the xor takes them as
// constant operands, so the key schedule costs no instructions.
struct PhiloxKey {
    uint32_t k0[kPhiloxRounds], k1[kPhiloxRounds];
    uint32_t one_bits;          // 0x3F800000, as a kernel parameter: see u32_to_one_two(x, one)
};
__host__ inline PhiloxKey make_philox_key(uint64_t seed) {
    PhiloxKey k;
    for (int r = 0; r < kPhiloxRounds; ++r) {
        k.k0[r] = (uint32_t)seed + (uint32_t)r * kPhiloxW0;
        k.k1[r] = (uint32_t)(seed >> 32) + (uint32_t)r * kPhiloxW1;
    }
    k.one_bits = 0x3F800000u;
    return k;
}

__device__ __forceinline__ uint4 philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                               const PhiloxKey &key) {
#pragma unroll
    for (int r = 0; r < kPhiloxRounds; ++r) {
        const uint32_t hi0 = __umulhi(kPhiloxM0, c0), lo0 = kPhiloxM0 * c0;
        const uint32_t hi1 = __umulhi(kPhiloxM1, c2), lo1 = kPhiloxM1 * c2;
        const uint32_t n0 = hi1 ^ c1 ^ key.k0[r];
        const uint32_t n2 = hi0 ^ c3 ^ key.k1[r];
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    }
    return make_uint4(c0, c1, c2, c3);
}

// uint32 -> f = 1 + k*2^-23 in [1,2) from the LOW 23 bits k of the word: one LOP3, no int->float conversion
// (I2F issues on the 16-lane XU pipe that the Box-Muller MUFUs already load).  The uniform is
// u = f - (1 - 2^-24) = (2k+1)*2^-24, on the open interval (0,1).
__device__ __forceinline__ float u32_to_one_two(uint32_t x) {
    return __uint_as_float(0x3F800000u | (x & 0x007FFFFFu));
}

// The same in ONE instruction: with both constants immediate ptxas emits two LOP3 (and, or) — an instruction takes one
// immediate.  With 0x3F800000 in a register (`one`, read from the kernel parameters so that it stays a register operand)
// it is LOP3 d = (x & 0x7FFFFF) | one.  8 issue slots less per octet of deviates in the generator loops.
__device__ __forceinline__ float u32_to_one_two(uint32_t x, uint32_t one) {
    uint32_t r;
    asm("lop3.b32 %0, %1, 0x007FFFFF, %2, 0xEA;" : "=r"(r) : "r"(x), "r"(one));
    return __uint_as_float(r);
}

__device__ __forceinline__ float lg2_approx(float x) {
    float y;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// np.clip(v, -c, c): NaN stays NaN (fminf/fmaxf would return the bound); max/min.NaN cost the same as fmaxf/fminf
__device__ __forceinline__ float clip_keep_nan(float v, float c) {
    float y;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(y) : "f"(v), "f"(-c));
    asm("min.NaN.f32 %0, %0, %1;" : "+f"(y) : "f"(c));
    return y;
}
// fp64 form (the device Pendulum's dynamics): PTX has no max.NaN.f64, so NaN is tested for explicitly
__device__ __forceinline__ double clip_keep_nan(double v, double c) { return isnan(v) ? v : fmin(fmax(v, -c), c); }
__device__ __forceinline__ float sqrt_approx(float x) {
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sin_approx(float x) {
    float y;
    asm("sin.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float cos_approx(float x) {
    float y;
    asm("cos.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// tanh as 1 - 2/(1 + 2^(2x log2 e)): two MUFU + three FP32 ops, abs error ~2e-7 (fp32 rounding level of the
// reference's torch.tanh).  40*H/32 of these per member-step make the libm tanhf a third of the instruction count.
// Shared by the closed-loop policies: rollout_pendulum_kernel (des_envs.cu) and policy_act_kernel (des_act.cu).
__device__ __forceinline__ float tanh_mufu(float x) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 2.8853900817779268f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return __fmaf_rn(-2.0f, r, 1.0f);
}

constexpr float kTwoPiF = 6.283185307179586f;             // fl32(2*pi)
constexpr float kAngOffF = 9.424777586262351f;            // fl32(3*pi - pi*2^-23)

// Box-Muller.  With f1, f2 in [1,2) from the two words:
//   u1  = f1 - (1 - 2^-24)                     (exact)
//   ang = fl32(f2*fl32(2*pi) - fl32(3*pi - pi*2^-23))   one FFMA;  ang ~= 2*pi*u2 - pi in (-pi, pi),
//         where the MUFU sin/cos error bound (2^-21.4 abs) holds
//   z0  = -sqrt(-2 ln u1) * cos(ang),  z1 = -sqrt(-2 ln u1) * sin(ang)       (cos(t+pi) = -cos t)
// oracle/nes_oracle.py restates u1 and ang bit-exactly and evaluates ln/sqrt/sin/cos in fp64.
__device__ __forceinline__ void box_muller(uint32_t xa, uint32_t xb, float &z0, float &z1) {
    const float u1 = u32_to_one_two(xa) - 0.99999994039535522f;
    const float nr = -sqrt_approx(-1.3862943611198906f * lg2_approx(u1));     // -2 ln u = (-2 ln 2) lg2 u
    const float ang = __fmaf_rn(u32_to_one_two(xb), kTwoPiF, -kAngOffF);
    z0 = nr * cos_approx(ang);
    z1 = nr * sin_approx(ang);
}

// Box-Muller in parts, for consumers that fold a scale into the radius: the pair is (nr*c, nr*s) with
// nr = -sqrt(scale2 * -2 ln u1) = -scale*sqrt(-2 ln u1) for scale2 = scale^2 (pass kNeg2Ln2 * scale^2).
constexpr float kNeg2Ln2 = -1.3862943611198906f;
struct BmParts {
    float nr, c, s;
};
__device__ __forceinline__ BmParts box_muller_parts(uint32_t xa, uint32_t xb, float neg2ln2_scale2) {
    BmParts p;
    const float u1 = u32_to_one_two(xa) - 0.99999994039535522f;
    p.nr = -sqrt_approx(neg2ln2_scale2 * lg2_approx(u1));
    const float ang = __fmaf_rn(u32_to_one_two(xb), kTwoPiF, -kAngOffF);
    p.c = cos_approx(ang);
    p.s = sin_approx(ang);
    return p;
}
// hot-loop form: `one` = PhiloxKey::one_bits (identical values)
__device__ __forceinline__ BmParts box_muller_parts(uint32_t xa, uint32_t xb, float neg2ln2_scale2, uint32_t one) {
    BmParts p;
    const float u1 = u32_to_one_two(xa, one) - 0.99999994039535522f;
    p.nr = -sqrt_approx(neg2ln2_scale2 * lg2_approx(u1));
    const float ang = __fmaf_rn(u32_to_one_two(xb, one), kTwoPiF, -kAngOffF);
    p.c = cos_approx(ang);
    p.s = sin_approx(ang);
    return p;
}
// out[e] = base[e] + scale * eps[e] for the four parameters of quad q (scale folded into the radius:
// differs from fma(scale, eps, base) by <= 1 ulp of scale*eps).
__device__ __forceinline__ float4 perturbed_quad(uint32_t q, uint32_t member, uint32_t gen, uint32_t tag,
                                                 const PhiloxKey &key, float neg2ln2_scale2, float4 base) {
    const uint4 x = philox4x32(q, member, gen, tag, key);
    const BmParts a = box_muller_parts(x.x, x.y, neg2ln2_scale2, key.one_bits);
    const BmParts b = box_muller_parts(x.z, x.w, neg2ln2_scale2, key.one_bits);
    return make_float4(__fmaf_rn(a.nr, a.c, base.x), __fmaf_rn(a.nr, a.s, base.y), __fmaf_rn(b.nr, b.c, base.z),
                       __fmaf_rn(b.nr, b.s, base.w));
}

// The four normals of quad q of `member` at `gen`.
__device__ __forceinline__ float4 noise_quad(uint32_t q, uint32_t member, uint32_t gen, uint32_t tag,
                                             const PhiloxKey &key) {
    const uint4 x = philox4x32(q, member, gen, tag, key);
    float4 z;
    box_muller(x.x, x.y, z.x, z.y);
    box_muller(x.z, x.w, z.z, z.w);
    return z;
}

// The genetic algorithm's parent of member m at generation `gen` in a table of n_parents rows (include/des_b200.h,
// "genetic algorithm"): (x * n_parents) >> 32 of the first word x of Philox(0, m, gen, 5).  For members past the elites.
__device__ __forceinline__ uint32_t ga_parent(uint32_t member, uint32_t gen, uint32_t n_parents, const PhiloxKey &key) {
    const uint32_t x = philox4x32(0u, member, gen, kStreamGaParent, key).x;
    return (uint32_t)(((uint64_t)x * n_parents) >> 32);
}

// The generation word of the counters: des_state's generation when the caller passes one (graph replay), else `gen`,
// which is read only then.
__device__ __forceinline__ uint32_t generation_word(const des_state *state, const uint32_t &gen) {
    return state ? (uint32_t)state->generation : gen;
}

// Mirrored sampling: member m perturbs with (-1)^(m & 1) * eps of counter word m >> 1.  fma(-sigma, eps, theta) is exactly
// fp32(theta - sigma*eps), and the even member of a pair has the bits of the plain member m >> 1.  `member` keeps the
// caller's integer type: the shift happens in that width.
template <typename Member>
__device__ __forceinline__ uint32_t noise_word(Member member, bool mirrored) {
    return (uint32_t)(mirrored ? member >> 1 : member);
}
template <typename Member>
__device__ __forceinline__ float member_sigma(Member member, bool mirrored, float sigma) {
    return mirrored && (member & 1u) ? -sigma : sigma;
}

// ---- entry-point checks and launches (host) ------------------------------------------------------------------------
// A shard holds the members [member_offset, member_offset + n).  Their indices fit `bits` bits: 32 for the noise counter
// word, 28 where the action-noise counter packs member*16 + repetition.
inline bool member_range_ok(int64_t member_offset, int64_t n, int bits) {
    return n >= 0 && member_offset >= 0 && member_offset + n <= ((int64_t)1 << bits);
}
// A mirrored shard holds whole pairs (members 2p and 2p + 1).
inline bool whole_pairs(int64_t member_offset, int64_t n) { return member_offset % 2 == 0 && n % 2 == 0; }
// Reports a shard that whole_pairs rejects (`count` names n's argument): DES_ERR_INVALID_ARGUMENT.
int not_whole_pairs(const char *who, const char *count, int64_t member_offset, int64_t n);
// A batch of independent runs (the *_runs entry points): n_runs populations of run_size members each, run r's member i
// the global member r * run_size + i.  Runs stop at the counting rank's population (kRunMaxSize): a larger population
// fills the GPU without batching.  check_runs returns DES_OK or reports a bad batch: n_runs >= 0 and
// min_size <= run_size (DES_ERR_INVALID_ARGUMENT), run_size <= kRunMaxSize (DES_ERR_UNSUPPORTED), and every member
// index below 2^28 (DES_ERR_INVALID_ARGUMENT).
constexpr int64_t kRunMaxSize = 2048;
int check_runs(const char *who, int64_t n_runs, int64_t run_size, int64_t min_size);
// A sweep's per-run table (the *_sweep entry points) as the header lays it out; ctypes mirrors it (_lib.RunHp).
static_assert(sizeof(des_run_hp) == 40 && offsetof(des_run_hp, sigma) == 8 && offsetof(des_run_hp, learning_rate) == 16 &&
              offsetof(des_run_hp, weight_decay) == 24 && offsetof(des_run_hp, action_noise_std) == 32,
              "des_run_hp: 40 bytes, the header's field offsets");
// The round keys of make_philox_key(seed), computed where the seed is: a sweep's kernels read it from their run's table.
__device__ __forceinline__ void philox_round_keys(uint64_t seed, PhiloxKey &k) {
#pragma unroll
    for (int r = 0; r < kPhiloxRounds; ++r) {
        k.k0[r] = (uint32_t)seed + (uint32_t)r * kPhiloxW0;
        k.k1[r] = (uint32_t)(seed >> 32) + (uint32_t)r * kPhiloxW1;
    }
}
// Hidden widths of the closed-loop policy kernels (rollout_pendulum_kernel, policy_act_kernel): H/16 units per lane.
inline bool policy_width_ok(int H) { return H == 16 || H == 32 || H == 64 || H == 96 || H == 128; }

// Opts `kernel` in to `smem` bytes of dynamic shared memory and launches it; the status of both.
template <typename... Params, typename... Args>
int launch_smem(const char *name, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                const Args &...args) {
    DES_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, block, smem, st>>>(args...);
    DES_LAUNCH_CHECK(name);
    return DES_OK;
}

// totals[c] = sum over the n_local rows of parts[n_local][width] (des_obs.cu), in member order
int obs_parts_reduce(double *totals, const double *parts, int64_t n_local, int width, cudaStream_t st);
// totals[r][c] = sum over run r's run_size rows of parts[n_runs * run_size][width], each run exactly as obs_parts_reduce
int obs_parts_reduce_runs(double *totals, const double *parts, int64_t n_runs, int64_t run_size, int width, cudaStream_t st);

// ---- CMA rank-mu (des_cma.cu: fp32 FFMA kernel and the entry point; des_cma_tc.cu: split-fp16 wgmma SYRK) ----------
constexpr int64_t kCmaTcMinN = 2048;     // n >= this runs on the tensor cores, smaller n on the FFMA kernel
// side of the packed upper-triangular tiles (des_cma_packed_elems): 64 up to n = 2048, 128 above
__host__ __device__ constexpr int cma_packed_tile(int64_t n) { return n <= 2048 ? 64 : 128; }
size_t cma_tc_workspace_bytes(int64_t n, int64_t lambda);
int cma_rank_mu_tc(float *out, const float *Y, const float *w, int64_t lambda, int64_t n, int packed, void *workspace,
                   cudaStream_t stream);

}  // namespace des
