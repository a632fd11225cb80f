// The host-stepped policy step (des_act.cu): its argument blocks and policy_act_kernel, shared by the translation
// units that instantiate it.  des_act.cu instantiates the single-population kernels (ActArgs) and des_act_sweep.cu
// the sweep kernels (ActSweepArgs): one unit of its own keeps ptxas's code for the first exactly what it was before
// sweeps existed (instantiated together, policy_act_kernel<64, ActArgs> came out scheduled differently).
#pragma once
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

// The arguments of a sweep (des_policy_act_sweep): row b is member b % run_size of run b / run_size, a standalone
// population under its run's seed with its run's action noise and statistics row.  The key, act_noise and member_offset
// of the ActArgs part are unused: each CTA sets the first two from its run's row of the table hp.
struct ActSweepArgs : ActArgs {
    const des_run_hp *hp;              // [n_runs]
    int run_size;                      // members per run
};

// shared-memory floats of one CTA for hidden width H (the layout is spelled out in policy_act_kernel)
__host__ __device__ inline int act_d0s(int d0) { return d0 | 1; }          // odd row stride: conflict-free column reads
__host__ inline size_t act_smem_floats(int d0, int H, int A) {
    const int d0s = act_d0s(d0);
    return 2 * (size_t)H * kActMaxReps + (size_t)H * d0s + H + (size_t)H * (H + 1) + H + (size_t)A * (H + 1) + 8 +
           (size_t)kActMaxReps * d0s;
}

// The member of row i in the counters: member_offset + i, except in a sweep, where every run is a population of its own.
template <typename Args>
__device__ __forceinline__ uint32_t act_member(const Args &a, int64_t i) {
    if constexpr (std::is_same<Args, ActSweepArgs>::value) return blockIdx.x % (unsigned)a.run_size;
    else return (uint32_t)(a.member_offset + (uint64_t)i);
}

// Args = ActArgs: one population (des_policy_act); Args = ActSweepArgs: a sweep (des_policy_act_sweep), which differs in
// the CTA's member, key, action noise and statistics row only.  Everything else is the same code.
template <int H, typename Args>
__global__ void __launch_bounds__(kActThreads) policy_act_kernel(Args a) {
    if constexpr (std::is_same<Args, ActSweepArgs>::value) {
        const unsigned run = blockIdx.x / (unsigned)a.run_size;
        if (a.obs_stats) a.obs_stats += (size_t)run * (2 * a.L.d0 + 1);
        const des_run_hp hp = a.hp[run];
        philox_round_keys(hp.seed, a.key);                  // make_philox_key's words, as the host makes them
        a.act_noise = (float)hp.action_noise_std;           // the host's conversion of the single call
    }
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
    const uint32_t member = act_member(a, i);

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

// Launches the kernel of width H over n rows (the ActArgs or ActSweepArgs instantiations).
template <typename Args>
static int act_launch(const Args &a, int H, int64_t n, cudaStream_t st) {
    const size_t smem = sizeof(float) * act_smem_floats(a.L.d0, H, a.L.A);
    void (*kernel)(Args);
    switch (H) {
        case 16: kernel = policy_act_kernel<16, Args>; break;
        case 32: kernel = policy_act_kernel<32, Args>; break;
        case 64: kernel = policy_act_kernel<64, Args>; break;
        case 96: kernel = policy_act_kernel<96, Args>; break;
        default: kernel = policy_act_kernel<128, Args>; break;
    }
    return launch_smem("policy_act_kernel", kernel, (unsigned)n, kActThreads, smem, st, a);
}

// act_launch<ActSweepArgs>, defined in des_act_sweep.cu
int act_launch_sweep(const ActSweepArgs &a, int H, int64_t n, cudaStream_t st);

}  // namespace des
