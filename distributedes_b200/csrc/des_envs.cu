// des_rollout_eval: closed-loop rollouts with per-member observations (SURVEY 8f row 3) — the reference's actual
// workload: Evaluator.eval utils.py:116-124 -> single_run utils.py:126-139, once per member per repetition, with the
// environment stepped on the device.  Environment 0 = Pendulum-v0 (the reference's PendulumConfig, config.py:26-31:
// obs 3, action 1, clip +-2, 200-step episodes).
//
// One warp per member steps all of the member's episodes in lockstep (see rollout_pendulum_kernel); the member's
// weights go once into shared memory: theta + sigma*eps generated with the same counter noise as every other kernel
// (NES), or row i of an explicit solutions[n_local][P] matrix (des_rollout_eval_solutions: the solutions CMA-ES's ask()
// returns, cma_es.py:22-29).  Everything after the weights are staged is the same code in both modes.
// Policy arithmetic fp32 (FFMA, MUFU-based tanh), dynamics fp64 (gym keeps its state in float64).
// Algorithmic work per environment step: 2*(3H + H*H + H) flop; no HBM traffic beyond theta (L2 resident).
#include <type_traits>
#include "des_common.cuh"

namespace des {

constexpr int kEnvPendulum = 0;

struct RollArgs {
    float *fitness;                    // [n_local] mean return over the repetitions (higher is better)
    float *ep_ret;                     // optional [n_local][reps] per-episode returns
    double *stat_part;                 // optional [n_local][2*d0+1]: per-member sum, sum of squares, count of RAW observations
    const float *theta;                // NES mode: the member's weights are theta + sigma*eps
    const float *rows;                 // explicit mode: [n_local][P] row-major, the member's weights are row blockIdx.x
    const float *obs_stats;            // optional [m | v | n] (StaticNormalizer offline stats), NULL = identity
    const des_state *state;
    Layout L;
    int reps, horizon;
    float sigma, clip, act_noise;
    PhiloxKey key;
    uint32_t gen;
    uint64_t member_offset;
    uint32_t reset_member_base;        // counter word for the reset stream: member index (or the test-episode index)
    int noiseless;                     // 1: evaluate theta itself (test(), natural_es.py:101-110)
    int mirrored;                      // NES mode: member m perturbs with (-1)^(m & 1) * eps of counter word m >> 1
};

// The arguments of a batch of runs (des_rollout_eval_runs).  A struct of its own, so that the single-population kernels
// keep RollArgs, their parameter block, exactly as it is.
struct RunArgs : RollArgs {
    int run_size;                      // members per run
};

__device__ __forceinline__ double unit_open(uint32_t x) { return ((double)(x & 0x7FFFFFu) + 0.5) * (1.0 / 8388608.0); }

// gym Pendulum-v0 (gym/envs/classic_control/pendulum.py): g = 10, m = l = 1, dt = 0.05, max_speed 8, max_torque 2
struct Pendulum {
    double th, thdot, sn, cs;
    __device__ void reset(uint32_t rep, uint32_t member, uint32_t gen, const PhiloxKey &key) {
        const uint4 x = philox4x32(rep, member, gen, kStreamEnvReset, key);
        th = (2.0 * unit_open(x.x) - 1.0) * 3.141592653589793;        // uniform(-pi, pi)
        thdot = (2.0 * unit_open(x.y) - 1.0) * 1.0;                     // uniform(-1, 1)
    }
    // One fp64 sincos per step serves the observation and the torque term: sin(th + pi) = -sin(th).
    __device__ void observe(float *o) {
        sincos(th, &sn, &cs);
        o[0] = (float)cs;
        o[1] = (float)sn;
        o[2] = (float)thdot;
    }
    __device__ double step(double u) {                                  // returns the reward; observe() came first
        u = clip_keep_nan(u, 2.0);                                       // np.clip: a NaN action makes a NaN state
        const double two_pi = 6.283185307179586, pi = 3.141592653589793;
        const double x = th + pi;
        const double an = (x - two_pi * floor(x * (1.0 / two_pi))) - pi;  // ((th + pi) % 2 pi) - pi, python sign rule
        const double cost = an * an + 0.1 * thdot * thdot + 0.001 * u * u;
        const double nthdot = thdot + (15.0 * sn + 3.0 * u) * 0.05;      // -3g/(2l) sin(th + pi) + 3/(m l^2) u
        th = th + nthdot * 0.05;
        thdot = clip_keep_nan(nthdot, 8.0);
        return -cost;
    }
};

constexpr int kEpPerLane = 5;          // episodes per lane half: 2 halves x 5 = up to 10 repetitions (config.py:8)
constexpr int kHS = 8;                 // row stride of an h1 panel (one panel per episode half): 5 episodes + pad

// One warp (= one CTA) per member; the warp steps all `reps` episodes of its member in lockstep, so the hidden layer is
// a [H x H] x [H x reps] product per step instead of `reps` mat-vecs: lane (rg = lane>>1, eg = lane&1) owns the
// R = H/16 hidden units rg*R.. and the episodes 5*eg..5*eg+4 — an R x 5 register tile fed per k by one LDS of R
// transposed weights and one 5-float broadcast of h1.  The fp64 dynamics of episode 5*eg + rg%5 run in every lane
// (the copies in rg >= 5 are redundant), i.e. once per step for the whole member.
// kRows: the weights are row blockIdx.x of a.rows (no noise is generated); otherwise theta + sigma*eps of the member.
// Args = RunArgs: a batch of independent runs (des_rollout_eval_runs, member_offset 0): CTA b is member b % run_size of
// run b / run_size, global member b, with its run's row of theta and of the statistics.  Everything else is the same code.
template <int R, bool kRows, typename Args>   // H = 16*R; Args: RollArgs or RunArgs
__global__ void __launch_bounds__(32) rollout_pendulum_kernel(Args a) {
    constexpr int H = 16 * R, C = kEpPerLane;
    if constexpr (std::is_same<Args, RunArgs>::value) {
        const unsigned run = blockIdx.x / (unsigned)a.run_size;
        a.theta += (size_t)run * a.L.P;
        if (a.obs_stats) a.obs_stats += (size_t)run * 7;
    }
    extern __shared__ __align__(16) float sm[];
    float *W2T = sm;                     // [k][j] = W2[j][k]
    // h1 panels, one per episode half, rows in the permuted order p(k) = (k % R)*16 + k/R so that the 16 unit groups
    // storing their r-th unit hit consecutive 32-byte rows; the second panel is shifted by 16 bytes: conflict-free STS.128
    float *hT = W2T + H * H;             // [2][p(k)][kHS] (+4 floats)
    float *xs = hT + 2 * H * kHS + 8;    // [10][4] normalised observations
    float *W1s = xs + 40;                // [H][4]
    float *b1s = W1s + H * 4;            // [H]
    float *b2s = b1s + H;
    float *W3s = b2s + H;
    float *b3s = W3s + H;                // [4]
    double *red = reinterpret_cast<double *>(b3s + 4);      // [10][8] per-episode results
    const Layout L = a.L;
    const int lane = threadIdx.x, rg = lane >> 1, eg = lane & 1;
    const uint32_t gen = generation_word(a.state, a.gen);
    const uint32_t member = (uint32_t)(a.member_offset + blockIdx.x);

    // flat parameter j of the member -> its place in shared memory
    auto stage = [&](int j, float w) {
        if (j < L.off_b1) W1s[(j / 3) * 4 + (j % 3)] = w;
        else if (j < L.off_w2) b1s[j - L.off_b1] = w;
        else if (j < L.off_b2) { const int r = (j - L.off_w2) / H; const int k = j - L.off_w2 - r * H; W2T[((k % R) * 16 + k / R) * H + r] = w; }
        else if (j < L.off_w3) b2s[j - L.off_b2] = w;
        else if (j < L.off_b3) W3s[j - L.off_w3] = w;
        else b3s[0] = w;
    };
    if constexpr (kRows) {
        // ---- explicit solution row (cma_es.py:27-28).  P is odd, so rows are not 16-byte aligned: coalesced scalar loads
        const float *row = a.rows + (int64_t)blockIdx.x * L.P;
        for (int j = lane; j < L.P; j += 32) stage(j, __ldg(row + j));
    } else {
        // ---- theta' = theta + sigma*eps for this member -> shared memory (natural_es.py:28-30)
        const uint32_t word = noise_word(member, a.mirrored);
        const float sigma = member_sigma(member, a.mirrored, a.sigma);
        for (int q = lane; q < (L.P + 3) / 4; q += 32) {
            float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!a.noiseless) z = noise_quad((uint32_t)q, word, gen, kStreamNesEps, a.key);
            const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int j = 4 * q + e;
                if (j >= L.P) break;
                stage(j, __fmaf_rn(sigma, zz[e], __ldg(a.theta + j)));
            }
        }
    }
    __syncwarp();
    float w1[R][3], b1[R], b2[R], w3[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int j = rg * R + r;
        w1[r][0] = W1s[j * 4]; w1[r][1] = W1s[j * 4 + 1]; w1[r][2] = W1s[j * 4 + 2];
        b1[r] = b1s[j]; b2[r] = b2s[j]; w3[r] = W3s[j];
    }
    const float b3 = b3s[0];

    // StaticNormalizer (utils.py:48-51): identity while n == 0
    float nm[3] = {0.f, 0.f, 0.f}, ns[3] = {1.f, 1.f, 1.f};
    if (a.obs_stats && a.obs_stats[6] != 0.f) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { nm[k] = a.obs_stats[k]; ns[k] = sqrtf(a.obs_stats[3 + k] + 1e-6f); }
    }
    float *hp = hT + eg * (H * kHS + 4);                  // this lane's h1 panel
    const int csel = rg % C, ep = C * eg + csel;         // the episode whose dynamics this lane carries
    const bool writer = rg < C;                           // one lane per episode publishes
    Pendulum env;
    env.reset((uint32_t)ep, a.reset_member_base + (a.noiseless ? 0u : (uint32_t)blockIdx.x), gen, a.key);
    double total = 0.0, osum[3] = {0, 0, 0}, osq[3] = {0, 0, 0};
    for (int t = 0; t < a.horizon; ++t) {
        {
            float o[3];
            env.observe(o);
#pragma unroll
            for (int k = 0; k < 3; ++k) { osum[k] += (double)o[k]; osq[k] += (double)o[k] * (double)o[k]; }
            if (writer)
                *reinterpret_cast<float4 *>(xs + ep * 4) =
                    make_float4((o[0] - nm[0]) / ns[0], (o[1] - nm[1]) / ns[1], (o[2] - nm[2]) / ns[2], 0.f);
        }
        __syncwarp();
        // layer 1: the lane's R units x 5 episodes -> h1 panel
        {
            float4 x[C];
#pragma unroll
            for (int c = 0; c < C; ++c) x[c] = *reinterpret_cast<const float4 *>(xs + (C * eg + c) * 4);
#pragma unroll
            for (int r = 0; r < R; ++r) {
                float v[C];
#pragma unroll
                for (int c = 0; c < C; ++c)
                    v[c] = tanh_mufu(__fmaf_rn(w1[r][2], x[c].z, __fmaf_rn(w1[r][1], x[c].y, __fmaf_rn(w1[r][0], x[c].x, b1[r]))));
                float *dst = hp + (r * 16 + rg) * kHS;
                *reinterpret_cast<float4 *>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                dst[4] = v[4];
            }
        }
        __syncwarp();
        // layer 2: R x 5 register tile
        float acc[R][C];
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int c = 0; c < C; ++c) acc[r][c] = b2[r];
#pragma unroll 16
        for (int k = 0; k < H; ++k) {
            float w[R];
            static_assert(R == 1 || R % 2 == 0, "W2T row loads cover R units: float4, float2 or one float");
            if constexpr (R % 4 == 0) {
#pragma unroll
                for (int r4 = 0; r4 < R / 4; ++r4) {
                    const float4 ww = *reinterpret_cast<const float4 *>(W2T + k * H + rg * R + 4 * r4);
                    w[4 * r4] = ww.x; w[4 * r4 + 1] = ww.y; w[4 * r4 + 2] = ww.z; w[4 * r4 + 3] = ww.w;
                }
            } else if constexpr (R % 2 == 0) {
#pragma unroll
                for (int r2 = 0; r2 < R / 2; ++r2) {
                    const float2 ww = *reinterpret_cast<const float2 *>(W2T + k * H + rg * R + 2 * r2);
                    w[2 * r2] = ww.x; w[2 * r2 + 1] = ww.y;
                }
            } else {                                                           // R = 1 (H = 16): one unit per lane
                w[0] = W2T[k * H + rg];
            }
            const float4 h4 = *reinterpret_cast<const float4 *>(hp + k * kHS);      // k runs in the permuted order
            const float h5 = hp[k * kHS + 4];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                acc[r][0] = __fmaf_rn(w[r], h4.x, acc[r][0]);
                acc[r][1] = __fmaf_rn(w[r], h4.y, acc[r][1]);
                acc[r][2] = __fmaf_rn(w[r], h4.z, acc[r][2]);
                acc[r][3] = __fmaf_rn(w[r], h4.w, acc[r][3]);
                acc[r][4] = __fmaf_rn(w[r], h5, acc[r][4]);
            }
        }
        // layer 3 (one action per episode): partial over the lane's units, butterfly over the 16 unit groups
        float p[C];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < R; ++r) s = __fmaf_rn(w3[r], tanh_mufu(acc[r][c]), s);
            p[c] = s;
        }
#pragma unroll
        for (int off = 2; off < 32; off <<= 1)
#pragma unroll
            for (int c = 0; c < C; ++c) p[c] += __shfl_xor_sync(0xffffffffu, p[c], off);
        float act = p[0];
#pragma unroll
        for (int c = 1; c < C; ++c) act = (csel == c) ? p[c] : act;
        act += b3;
        if (a.act_noise != 0.f) {                                        // utils.py:133
            const uint4 xr = philox4x32((uint32_t)t, member * 16u + (uint32_t)ep, gen, kStreamActNoise, a.key);
            float z0, z1;
            box_muller(xr.x, xr.y, z0, z1);
            act = __fmaf_rn(z0, a.act_noise, act);
        }
        act = clip_keep_nan(act, a.clip);                                // config.action_clip, utils.py:134
        total += env.step((double)act);                                  // utils.py:135-137
    }
    if (writer) {
        red[ep * 8] = total;
#pragma unroll
        for (int k = 0; k < 3; ++k) { red[ep * 8 + 1 + k] = osum[k]; red[ep * 8 + 4 + k] = osq[k]; }
    }
    __syncwarp();
    if (lane == 0) {
        double s = 0.0;
        for (int r = 0; r < a.reps; ++r) s += red[r * 8];
        a.fitness[blockIdx.x] = (float)(s / a.reps);                     // -cost of utils.py:124
    }
    if (a.ep_ret && lane < a.reps) a.ep_ret[(int64_t)blockIdx.x * a.reps + lane] = (float)red[lane * 8];
    if (a.stat_part) {      // raw observations fed to the normaliser by this member, episodes summed in a fixed order
        if (lane < 6) {
            double s = 0.0;
            for (int r = 0; r < a.reps; ++r) s += red[r * 8 + 1 + lane];
            a.stat_part[(int64_t)blockIdx.x * 7 + lane] = s;
        }
        if (lane == 6) a.stat_part[(int64_t)blockIdx.x * 7 + 6] = (double)a.reps * a.horizon;
    }
}

// Shared by the entry points: argument checks (before any CUDA work), workspace, launch.  rows_mode selects the
// explicit-solution kernels: `weights` is then rows[n_local][P] instead of the theta that sigma*eps perturbs.  run_size > 0
// makes the n_local members a batch of runs of run_size (des_rollout_eval_runs, member_offset 0): `weights` and
// `obs_stats_dev` hold one row per run, and the observation totals are reduced per run.
static int rollout_launch(const char *who, float *fitness_out_dev, float *episode_returns_out_dev,
                          double *obs_totals_out_dev, const float *weights_dev, bool rows_mode,
                          const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions, double sigma,
                          double clip, double action_noise_std, uint64_t seed, uint64_t generation,
                          const des_state *state_dev, int64_t member_offset, int64_t n_local, int noiseless,
                          void *workspace_dev, size_t workspace_bytes, bool mirrored, int64_t run_size, cudaStream_t st) {
    DES_REQUIRE(env == kEnvPendulum, "%s: unknown environment %d (0 = Pendulum-v0)", who, env);
    if (mirrored && !(member_offset >= 0 && n_local >= 0 && whole_pairs(member_offset, n_local)))
        return not_whole_pairs(who, "n_local", member_offset, n_local);
    DES_REQUIRE(!mirrored || !noiseless, "%s: test episodes (noiseless) have no pairs; use des_rollout_eval", who);
    DES_REQUIRE(dims.state_dim == 3 && dims.action_dim == 1, "%s: Pendulum-v0 has state_dim 3, action_dim 1", who);
    DES_REQUIRE(policy_width_ok(dims.hidden), "%s: hidden must be 16 or a multiple of 32, <= 128 (got %d)", who, dims.hidden);
    DES_REQUIRE(repetitions >= 1 && repetitions <= 10, "%s: repetitions must be in [1, 10] (one warp each)", who);
    DES_REQUIRE(dims.tape_len >= 1, "%s: episode length (dims.tape_len) must be >= 1", who);
    DES_REQUIRE(member_range_ok(member_offset, n_local, 28), "%s: bad member range", who);
    if (n_local == 0) return DES_OK;
    DES_REQUIRE(fitness_out_dev && weights_dev, "%s: NULL pointer", who);
    RollArgs a;
    a.fitness = fitness_out_dev; a.ep_ret = episode_returns_out_dev;
    a.theta = rows_mode ? nullptr : weights_dev; a.rows = rows_mode ? weights_dev : nullptr;
    a.obs_stats = obs_stats_dev; a.state = state_dev;
    a.L = Layout(3, dims.hidden, 1);
    a.reps = repetitions; a.horizon = dims.tape_len;
    a.sigma = noiseless ? 0.f : (float)sigma; a.clip = (float)clip; a.act_noise = (float)action_noise_std;
    a.key = make_philox_key(seed); a.gen = (uint32_t)generation;
    a.member_offset = (uint64_t)member_offset;
    a.reset_member_base = noiseless ? kTestEpisodeMember : (uint32_t)member_offset;
    a.noiseless = noiseless ? 1 : 0;
    a.mirrored = mirrored ? 1 : 0;
    a.stat_part = nullptr;
    if (obs_totals_out_dev) {
        const size_t need = (size_t)n_local * 7 * sizeof(double);
        if (!workspace_dev || workspace_bytes < need) {
            set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
            return DES_ERR_WORKSPACE;
        }
        a.stat_part = (double *)workspace_dev;
    }
    const int H = dims.hidden;
    const size_t smem = sizeof(float) * ((size_t)H * H + 2 * (size_t)H * kHS + 8 + 40 + (size_t)H * 4 + 3 * (size_t)H + 4) +
                        sizeof(double) * 80;
    if (run_size > 0) {
        RunArgs ra;
        static_cast<RollArgs &>(ra) = a;
        ra.run_size = (int)run_size;
        void (*runs_kernel)(RunArgs);
        switch (H / 16) {
            case 1: runs_kernel = rollout_pendulum_kernel<1, false, RunArgs>; break;
            case 2: runs_kernel = rollout_pendulum_kernel<2, false, RunArgs>; break;
            case 4: runs_kernel = rollout_pendulum_kernel<4, false, RunArgs>; break;
            case 6: runs_kernel = rollout_pendulum_kernel<6, false, RunArgs>; break;
            default: runs_kernel = rollout_pendulum_kernel<8, false, RunArgs>; break;
        }
        const int rc = launch_smem("rollout_pendulum_kernel", runs_kernel, (unsigned)n_local, 32, smem, st, ra);
        if (rc != DES_OK || !obs_totals_out_dev) return rc;
        return obs_parts_reduce_runs(obs_totals_out_dev, a.stat_part, n_local / run_size, run_size, 7, st);
    }
    void (*kernel)(RollArgs);
    switch (H / 16) {                    // R = H/16 hidden units per lane
        case 1: kernel = rows_mode ? rollout_pendulum_kernel<1, true, RollArgs> : rollout_pendulum_kernel<1, false, RollArgs>; break;
        case 2: kernel = rows_mode ? rollout_pendulum_kernel<2, true, RollArgs> : rollout_pendulum_kernel<2, false, RollArgs>; break;
        case 4: kernel = rows_mode ? rollout_pendulum_kernel<4, true, RollArgs> : rollout_pendulum_kernel<4, false, RollArgs>; break;
        case 6: kernel = rows_mode ? rollout_pendulum_kernel<6, true, RollArgs> : rollout_pendulum_kernel<6, false, RollArgs>; break;
        default: kernel = rows_mode ? rollout_pendulum_kernel<8, true, RollArgs> : rollout_pendulum_kernel<8, false, RollArgs>; break;
    }
    const int rc = launch_smem("rollout_pendulum_kernel", kernel, (unsigned)n_local, 32, smem, st, a);
    if (rc != DES_OK || !obs_totals_out_dev) return rc;
    return obs_parts_reduce(obs_totals_out_dev, a.stat_part, n_local, 7, st);
}

}  // namespace des

extern "C" DES_API int des_rollout_eval(float *fitness_out_dev, float *episode_returns_out_dev,
                                        double *obs_totals_out_dev, const float *theta_dev,
                                        const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions,
                                        double sigma, double clip, double action_noise_std, uint64_t seed,
                                        uint64_t generation, const des_state *state_dev, int64_t member_offset,
                                        int64_t n_local, int noiseless, void *workspace_dev, size_t workspace_bytes,
                                        void *stream) {
    return des::rollout_launch("des_rollout_eval", fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, theta_dev,
                               false, obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed,
                               generation, state_dev, member_offset, n_local, noiseless, workspace_dev, workspace_bytes,
                               false, 0, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_mirrored(float *fitness_out_dev, float *episode_returns_out_dev,
                                                 double *obs_totals_out_dev, const float *theta_dev,
                                                 const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions,
                                                 double sigma, double clip, double action_noise_std, uint64_t seed,
                                                 uint64_t generation, const des_state *state_dev, int64_t member_offset,
                                                 int64_t n_local, int noiseless, void *workspace_dev, size_t workspace_bytes,
                                                 void *stream) {
    return des::rollout_launch("des_rollout_eval_mirrored", fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev,
                               theta_dev, false, obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed,
                               generation, state_dev, member_offset, n_local, noiseless, workspace_dev, workspace_bytes,
                               true, 0, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_solutions(float *fitness_out_dev, float *episode_returns_out_dev,
                                                  double *obs_totals_out_dev, const float *solutions_dev,
                                                  const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions,
                                                  double clip, double action_noise_std, uint64_t seed,
                                                  uint64_t generation, int64_t member_offset, int64_t n_local,
                                                  void *workspace_dev, size_t workspace_bytes, void *stream) {
    return des::rollout_launch("des_rollout_eval_solutions", fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev,
                               solutions_dev, true, obs_stats_dev, env, dims, repetitions, 0.0, clip, action_noise_std,
                               seed, generation, nullptr, member_offset, n_local, 0, workspace_dev, workspace_bytes,
                               false, 0, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_runs(float *fitness_out_dev, float *episode_returns_out_dev,
                                             double *obs_totals_out_dev, const float *theta_dev, const float *obs_stats_dev,
                                             int env, des_dims dims, int32_t repetitions, double sigma, double clip,
                                             double action_noise_std, uint64_t seed, uint64_t generation,
                                             const des_state *state_dev, int64_t n_runs, int64_t run_size, int noiseless,
                                             void *workspace_dev, size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_runs";
    const int rc = des::check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(!noiseless || run_size == 1, "%s: test episodes (noiseless) evaluate one theta per run: run_size must be 1 "
                "(got %lld)", who, (long long)run_size);
    return des::rollout_launch(who, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, theta_dev, false,
                               obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed, generation,
                               state_dev, 0, n_runs * run_size, noiseless, workspace_dev, workspace_bytes, false, run_size,
                               (cudaStream_t)stream);
}
