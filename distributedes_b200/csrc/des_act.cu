// des_policy_act: one environment step of the population's policies for environments stepped on the HOST — the part of
// Evaluator.single_run (utils.py:126-139) that is not env.step: normalise the observation (utils.py:48-51), forward the
// member's own weights (model.py:34-39), add action noise (utils.py:133), clip (config.action_clip, utils.py:134).  The
// caller steps its environments with the actions, copies the next observations back and launches again: one launch per
// environment step for n_local members x `reps` episodes in lockstep.  No kernel waits on the host.
//
// Numerics are those of rollout_pendulum_kernel (des_envs.cu, DESIGN §4.7), so a Pendulum slot stepped on the host gets
// the action the device rollout computes for the same observation and weights:
//   x      = (o - m) / sqrtf(v + 1e-6f), o itself while n == 0
//   h1[j]  = tanh(fma chain b1[j] + W1[j][0] x[0] + ... + W1[j][d0-1] x[d0-1])
//   h2[j]  = tanh(fma chain b2[j] + sum over k of W2[j][k] h1[k]), k in the rollout kernel's order (pk % 16)*R + pk/16,
//            R = H/16, pk = 0..H-1
//   a[c]   = pairwise sum over the 16 unit groups g of (fma chain over r < R of W3[c][gR + r] h2[gR + r]), + b3[c]
//   a[c]  += std * z, z = normal (c % 4) of the quad Philox(t + (c/4)*2^31, member*16 + rep, generation, stream 3)
//   a[c]   = clip_keep_nan(a[c], clip): np.clip, so a NaN observation or NaN weights give a NaN action
// tanh is tanh_mufu (des_common.cuh).  Dead slots get 0 whatever their observation holds.
//
// One CTA (128 threads) per member: the member's row is staged once per launch into shared memory (coalesced scalar
// loads: P is odd, rows are not 16-byte aligned), then thread (j, g) computes hidden unit j for the episode block g.
// Cost per step: n_local * P * 4 bytes of weights read; compute is reps * 2P flop per member.
#include "des_common.cuh"

namespace des {

constexpr int kActThreads = 128;
constexpr int kActMaxReps = 16;        // the action-noise counter packs member*16 + repetition
constexpr int kActMaxD0 = 32;
constexpr int kActMaxA = 8;

struct ActArgs {
    float *actions;                    // [n_local][reps][A]
    double *stat_part;                 // optional [n_local][2*d0+1]: running sum, sum of squares, count of raw observations
    const float *rows;                 // [n_local][P]
    const float *obs;                  // [n_local][reps][d0] raw
    const uint8_t *alive;              // [n_local][reps]
    const float *obs_stats;            // optional [m | v | n]
    Layout L;
    int reps;
    float clip, act_noise;
    PhiloxKey key;
    uint32_t gen, t;
    uint64_t member_offset;
};

// shared-memory floats of one CTA for hidden width H (the layout is spelled out in policy_act_kernel)
__host__ __device__ inline int act_d0s(int d0) { return d0 | 1; }          // odd row stride: conflict-free column reads
__host__ inline size_t act_smem_floats(int d0, int H, int A) {
    const int d0s = act_d0s(d0);
    return 2 * (size_t)H * kActMaxReps + (size_t)H * d0s + H + (size_t)H * (H + 1) + H + (size_t)A * (H + 1) + 8 +
           (size_t)kActMaxReps * d0s;
}

template <int H>
__global__ void __launch_bounds__(kActThreads) policy_act_kernel(ActArgs a) {
    constexpr int R = H / 16;                                  // units per group in the rollout kernel's order
    constexpr int G = (kActThreads / H) > 0 ? kActThreads / H : 1;   // episode blocks (H = 96: one block, 32 threads idle)
    constexpr int RPT = kActMaxReps / G;                        // episodes per thread
    static_assert(RPT == 16 || RPT == 8 || RPT == 4 || RPT == 2, "episode blocks are float2/float4 vectors");
    extern __shared__ __align__(16) float sm[];
    const Layout L = a.L;
    const int d0 = L.d0, A = L.A, d0s = act_d0s(d0);
    float *h1T = sm;                                   // [H][16]: episode index contiguous (16-byte aligned vectors)
    float *h2T = h1T + H * kActMaxReps;                // [H][16]
    float *W1s = h2T + H * kActMaxReps;                // [H][d0s]
    float *b1s = W1s + H * d0s;                        // [H]
    float *W2s = b1s + H;                              // [H][H+1], row j = unit j's inputs
    float *b2s = W2s + H * (H + 1);                    // [H]
    float *W3s = b2s + H;                              // [A][H+1]
    float *b3s = W3s + A * (H + 1);                    // [8]
    float *xs = b3s + 8;                               // [16][d0s] normalised observations
    const int tid = threadIdx.x;
    const int64_t i = blockIdx.x;
    const uint32_t member = (uint32_t)(a.member_offset + (uint64_t)i);

    // ---- stage the member's weights
    const float *row = a.rows + i * L.P;
    for (int f = tid; f < L.P; f += kActThreads) {
        const float w = __ldg(row + f);
        if (f < L.off_b1) { const int j = f / d0; W1s[j * d0s + (f - j * d0)] = w; }
        else if (f < L.off_w2) b1s[f - L.off_b1] = w;
        else if (f < L.off_b2) { const int j = (f - L.off_w2) / H; W2s[j * (H + 1) + (f - L.off_w2 - j * H)] = w; }
        else if (f < L.off_w3) b2s[f - L.off_b2] = w;
        else if (f < L.off_b3) { const int c = (f - L.off_w3) / H; W3s[c * (H + 1) + (f - L.off_w3 - c * H)] = w; }
        else b3s[f - L.off_b3] = w;
    }
    // ---- normalised observations (utils.py:48-51); dead and absent episodes read zeros
    const bool use_stats = a.obs_stats && a.obs_stats[2 * d0] != 0.f;
    const float *obs = a.obs + i * a.reps * d0;
    const uint8_t *alive = a.alive + i * a.reps;
    for (int e = tid; e < kActMaxReps * d0; e += kActThreads) {
        const int r = e / d0, k = e - r * d0;
        float x = 0.f;
        if (r < a.reps && alive[r]) {
            const float o = obs[r * d0 + k];
            const float nm = use_stats ? a.obs_stats[k] : 0.f;
            const float ns = use_stats ? sqrtf(a.obs_stats[d0 + k] + 1e-6f) : 1.f;
            x = (o - nm) / ns;
        }
        xs[r * d0s + k] = x;
    }
    // ---- observation statistics of the raw observations of alive slots: slots in repetition order, steps in time order
    if (a.stat_part) {
        double *part = a.stat_part + i * (2 * d0 + 1);
        if (tid < d0) {
            double s = part[tid], q = part[d0 + tid];
            for (int r = 0; r < a.reps; ++r) {
                if (!alive[r]) continue;
                const double o = (double)obs[r * d0 + tid];
                s += o;
                q += o * o;
            }
            part[tid] = s;
            part[d0 + tid] = q;
        } else if (tid == d0) {
            int n = 0;
            for (int r = 0; r < a.reps; ++r) n += alive[r] ? 1 : 0;
            part[2 * d0] += (double)n;
        }
    }
    __syncthreads();

    const int j = tid % H, g = tid / H;
    const bool unit = tid < H * G;
    // ---- layer 1: unit j for episodes g*RPT .. g*RPT + RPT - 1
    if (unit) {
        const float *w1 = W1s + j * d0s;
        const float b1 = b1s[j];
#pragma unroll
        for (int e = 0; e < RPT; ++e) {
            const float *x = xs + (g * RPT + e) * d0s;
            float v = b1;
            for (int k = 0; k < d0; ++k) v = __fmaf_rn(w1[k], x[k], v);
            h1T[j * kActMaxReps + g * RPT + e] = tanh_mufu(v);
        }
    }
    __syncthreads();
    // ---- layer 2: RPT accumulators per thread, the inputs in the rollout kernel's order
    if (unit) {
        float acc[RPT];
        const float b2 = b2s[j];
#pragma unroll
        for (int e = 0; e < RPT; ++e) acc[e] = b2;
        const float *w2 = W2s + j * (H + 1);
#pragma unroll 4
        for (int pk = 0; pk < H; ++pk) {
            const int k = (pk % 16) * R + pk / 16;
            const float w = w2[k];
            const float *h = h1T + k * kActMaxReps + g * RPT;
            if constexpr (RPT % 4 == 0) {
#pragma unroll
                for (int e4 = 0; e4 < RPT / 4; ++e4) {
                    const float4 hv = *reinterpret_cast<const float4 *>(h + 4 * e4);
                    acc[4 * e4] = __fmaf_rn(w, hv.x, acc[4 * e4]);
                    acc[4 * e4 + 1] = __fmaf_rn(w, hv.y, acc[4 * e4 + 1]);
                    acc[4 * e4 + 2] = __fmaf_rn(w, hv.z, acc[4 * e4 + 2]);
                    acc[4 * e4 + 3] = __fmaf_rn(w, hv.w, acc[4 * e4 + 3]);
                }
            } else {
                const float2 hv = *reinterpret_cast<const float2 *>(h);
                acc[0] = __fmaf_rn(w, hv.x, acc[0]);
                acc[1] = __fmaf_rn(w, hv.y, acc[1]);
            }
        }
#pragma unroll
        for (int e = 0; e < RPT; ++e) h2T[j * kActMaxReps + g * RPT + e] = tanh_mufu(acc[e]);
    }
    __syncthreads();
    // ---- layer 3, noise, clip: one thread per (episode, action)
    if (tid < a.reps * A) {
        const int r = tid / A, c = tid - r * A;
        float p[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            float s = 0.f;
#pragma unroll
            for (int u = 0; u < R; ++u) s = __fmaf_rn(W3s[c * (H + 1) + q * R + u], h2T[(q * R + u) * kActMaxReps + r], s);
            p[q] = s;
        }
#pragma unroll
        for (int st = 1; st < 16; st <<= 1)            // the rollout kernel's xor butterfly over the 16 unit groups
#pragma unroll
            for (int q = 0; q < 16; q += 2 * st) p[q] += p[q + st];
        float act = p[0] + b3s[c];
        if (a.act_noise != 0.f) {                                            // utils.py:133
            const float4 z = noise_quad(a.t + ((uint32_t)(c >> 2) << 31), member * 16u + (uint32_t)r, a.gen,
                                        kStreamActNoise, a.key);
            const int cc = c & 3;
            const float zc = cc == 0 ? z.x : cc == 1 ? z.y : cc == 2 ? z.z : z.w;
            act = __fmaf_rn(zc, a.act_noise, act);
        }
        act = clip_keep_nan(act, a.clip);                                    // np.clip, utils.py:134
        a.actions[(i * a.reps + r) * A + c] = alive[r] ? act : 0.f;
    }
}

}  // namespace des

extern "C" DES_API int des_policy_act(float *actions_out_dev, double *stat_part_dev, const float *rows_dev, int64_t P,
                                      const float *obs_dev, const uint8_t *alive_dev, const float *obs_stats_dev,
                                      des_dims dims, int32_t repetitions, double clip, double action_noise_std,
                                      uint64_t seed, uint64_t generation, int64_t member_offset, int64_t n_local,
                                      int64_t t, void *stream) {
    using namespace des;
    const char *who = "des_policy_act";
    const int H = dims.hidden, d0 = dims.state_dim, A = dims.action_dim;
    DES_REQUIRE(policy_width_ok(H), "%s: hidden must be 16, 32, 64, 96 or 128 (got %d)", who, H);
    DES_REQUIRE(d0 >= 1 && d0 <= kActMaxD0, "%s: state_dim must be in [1, %d] (got %d)", who, kActMaxD0, d0);
    DES_REQUIRE(A >= 1 && A <= kActMaxA, "%s: action_dim must be in [1, %d] (got %d)", who, kActMaxA, A);
    DES_REQUIRE(repetitions >= 1 && repetitions <= kActMaxReps,
                "%s: repetitions must be in [1, %d] (the action-noise counter is member*16 + repetition; got %d)", who,
                kActMaxReps, repetitions);
    const Layout L(d0, H, A);
    DES_REQUIRE(P == L.P, "%s: rows have P = %lld, the (%d,%d,%d) MLP needs %d", who, (long long)P, d0, H, A, L.P);
    DES_REQUIRE(member_range_ok(member_offset, n_local, 28), "%s: bad member range", who);
    DES_REQUIRE(t >= 0 && t < ((int64_t)1 << 31), "%s: step index must be in [0, 2^31)", who);
    DES_REQUIRE(alive_dev, "%s: NULL alive mask", who);
    if (n_local == 0) return DES_OK;
    DES_REQUIRE(actions_out_dev && rows_dev && obs_dev, "%s: NULL pointer", who);
    ActArgs a;
    a.actions = actions_out_dev; a.stat_part = stat_part_dev;
    a.rows = rows_dev; a.obs = obs_dev; a.alive = alive_dev; a.obs_stats = obs_stats_dev;
    a.L = L; a.reps = repetitions;
    a.clip = (float)clip; a.act_noise = (float)action_noise_std;
    a.key = make_philox_key(seed); a.gen = (uint32_t)generation; a.t = (uint32_t)t;
    a.member_offset = (uint64_t)member_offset;
    const size_t smem = sizeof(float) * act_smem_floats(d0, H, A);
    void (*kernel)(ActArgs);
    switch (H) {
        case 16: kernel = policy_act_kernel<16>; break;
        case 32: kernel = policy_act_kernel<32>; break;
        case 64: kernel = policy_act_kernel<64>; break;
        case 96: kernel = policy_act_kernel<96>; break;
        default: kernel = policy_act_kernel<128>; break;
    }
    return launch_smem("policy_act_kernel", kernel, (unsigned)n_local, kActThreads, smem, (cudaStream_t)stream, a);
}
