// The closed-loop Pendulum rollout kernel and its launcher rollout_kernels (des_envs.cu), in a header for the units that
// instantiate them.  Each unit compiles the kernels of its own entry points:
//   des_envs.cu            RollArgs, RunArgs, SweepArgs   des_rollout_eval[_mirrored|_solutions|_runs|_sweep]
//   des_envs_sweep.cu      SweepArgs in row mode          des_rollout_eval_solutions_sweep
//   des_envs_record.cu     RecordArgs                     des_rollout_record[_solutions]
//   des_envs_ga.cu         GaArgs                         des_rollout_eval_ga
//   des_envs_ga_sweep.cu   GaSweepArgs                    des_rollout_eval_ga_sweep
//   des_envs_bc.cu         BcArgs                         des_rollout_eval_bc
//   des_envs_bc_sweep.cu   BcSweepArgs                    des_rollout_eval_bc_sweep
//   des_envs_ga_bc.cu      GaBcArgs                       des_rollout_eval_ga_bc
// The split keeps ptxas's code for des_envs.cu's kernels what it was before the others existed: instantiated together
// with the row-mode sweep kernels, rollout_pendulum_kernel<8, true, RollArgs> came out scheduled differently.
#pragma once
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

// The arguments of a sweep (des_rollout_eval_sweep): a batch of runs whose seed, sigma and action noise are run r's row
// of the device table hp.  The key, sigma and act_noise of the RollArgs part are unused: each CTA sets them from its row.
struct SweepArgs : RunArgs {
    const des_run_hp *hp;              // [n_runs]
};

// The arguments of a recording (des_rollout_record[_solutions]): an evaluation that also writes, for each member i, each
// episode e < reps and each step t < horizon, the step's row of four trajectories [n_local][reps][horizon][...].  Each
// pointer may be NULL (not written).
struct RecordArgs : RollArgs {
    double *states;                    // [..][2] gym's self.state before the step: (th unwrapped, thdot)
    float *obs;                        // [..][3] the raw observation the policy was given (what stat_part sums)
    float *actions;                    // [..][1] the action passed to env.step: after noise and the clip, before the +-2
    double *rewards;                   // [..]    the reward Pendulum::step returned
};

// The arguments of a genetic-algorithm generation (des_rollout_eval_ga): member m's weights are row m of the parents
// table for m < n_elites, else fmaf(sigma, eps_m, parents[ga_parent(m)]) (include/des_b200.h, "genetic algorithm").
// theta is unused.
struct GaArgs : RollArgs {
    const float *parents;              // [n_parents][P]
    int n_parents, n_elites;
};

// The arguments of a genetic-algorithm sweep (des_rollout_eval_ga_sweep): a sweep (SweepArgs: the run's seed, sigma and
// action noise from its hp row) whose CTA builds its member as a GaArgs kernel does, from its run's table of the buffer
// parents [n_runs][table_rows][P] and the counts of its des_ga_run row, clamped so that no table read leaves the buffer.
// The CTA sets parents, n_parents and n_elites itself; theta is unused.
struct GaSweepArgs : SweepArgs {
    const float *parents;              // [n_runs][table_rows][P], then the CTA's run's table
    int n_parents, n_elites;
    const des_ga_run *ga;              // [n_runs]
    int table_rows;                    // >= 1
};

// The arguments of an evaluation that also writes each member's behaviour characterisation (des_rollout_eval_bc): the
// raw observation after the last step of each of its episodes, averaged over the repetitions (fp64 sum in episode
// order, stored as fp32).
struct BcArgs : RollArgs {
    float *bc_out;                     // [n_local][d0]
};

// The arguments of a sweep evaluation that also writes each member's behaviour (des_rollout_eval_bc_sweep): a sweep
// (SweepArgs: the run's seed, sigma and action noise from its hp row) whose CTA writes its behaviour as a BcArgs kernel
// does, at row blockIdx.x of bc_out [n_runs * run_size][d0].
struct BcSweepArgs : SweepArgs {
    float *bc_out;                     // [n_runs * run_size][d0]
};

// The arguments of a genetic-algorithm generation that also writes each member's behaviour (des_rollout_eval_ga_bc): a
// GaArgs generation whose CTA writes its behaviour as a BcArgs kernel does, at row blockIdx.x of bc_out.  It derives from
// neither RunArgs nor SweepArgs, so the member is blockIdx.x and no run block applies.
struct GaBcArgs : GaArgs {
    float *bc_out;                     // [n_local][d0]
};

// The Args whose members are built from a parents table (the genetic algorithm's fill stage).  Named one by one, not by
// base class, so that a new Args joins no other Args' code paths.
template <typename Args>
constexpr bool kGaFill = std::is_same<Args, GaArgs>::value || std::is_same<Args, GaSweepArgs>::value ||
                         std::is_same<Args, GaBcArgs>::value;

// The Args of a behaviour-writing evaluation (after the step loop).
template <typename Args>
constexpr bool kBc = std::is_same<Args, BcArgs>::value || std::is_same<Args, BcSweepArgs>::value ||
                     std::is_same<Args, GaBcArgs>::value;

// The CTA's member within its population: member_offset + member_slot(a) is the member in the counters.  blockIdx.x,
// except in a sweep, where every run is a population of its own.
template <typename Args>
__device__ __forceinline__ unsigned member_slot(const Args &a) {
    if constexpr (std::is_base_of<SweepArgs, Args>::value) return blockIdx.x % (unsigned)a.run_size;
    else return blockIdx.x;
}

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
// Args = SweepArgs: a sweep (des_rollout_eval_sweep): as RunArgs, but CTA b is member b % run_size of a standalone
// population under its run's seed, with the run's sigma and action noise; the round keys are set up from that seed.
// kRows with SweepArgs (des_rollout_eval_solutions_sweep): CTA b evaluates row b of a.rows as member b % run_size of its
// run, under the run's seed and action noise.
// Args = RecordArgs (des_rollout_record[_solutions]): RollArgs, and the lane that publishes episode ep (< reps) writes
// each step's state, observation, action and reward; the ones of the episodes past reps, stepped all the same, are not.
// Args = GaArgs (des_rollout_eval_ga, kRows false): the member's weights are built from its row of the parents table:
// an elite's row as it is, any other member's parent row plus sigma*eps of the member, through the same stage().
// Args = GaSweepArgs (des_rollout_eval_ga_sweep, kRows false): a sweep CTA that fills as GaArgs does, from its run's
// table and counts.
// Args = BcArgs (des_rollout_eval_bc, kRows false): RollArgs, and after the last step each episode's publishing lane
// observes its state once more; lane 0 writes the member's mean of those raw observations.
// Args = BcSweepArgs (des_rollout_eval_bc_sweep, kRows false): a sweep CTA that writes its behaviour as BcArgs does.
// Args = GaBcArgs (des_rollout_eval_ga_bc, kRows false): fills as GaArgs does and writes its behaviour as BcArgs does.
template <int R, bool kRows, typename Args>   // H = 16*R; Args: RollArgs, RunArgs, SweepArgs, RecordArgs, GaArgs, GaSweepArgs,
                                              // BcArgs, BcSweepArgs or GaBcArgs
__global__ void __launch_bounds__(32) rollout_pendulum_kernel(Args a) {
    constexpr int H = 16 * R, C = kEpPerLane;
    if constexpr (std::is_base_of<RunArgs, Args>::value) {
        const unsigned run = blockIdx.x / (unsigned)a.run_size;
        if constexpr (!kRows && !kGaFill<Args>) a.theta += (size_t)run * a.L.P;   // NULL otherwise
        if (a.obs_stats) a.obs_stats += (size_t)run * 7;
        if constexpr (std::is_base_of<SweepArgs, Args>::value) {
            const des_run_hp hp = a.hp[run];
            philox_round_keys(hp.seed, a.key);                  // make_philox_key's words, as the host makes them
            a.sigma = a.noiseless ? 0.f : (float)hp.sigma;      // the host's conversions of the single call
            a.act_noise = (float)hp.action_noise_std;
        }
        if constexpr (std::is_same<Args, GaSweepArgs>::value) {
            // the run's table and counts, clamped to the buffer: n_parents in [1, table_rows], n_elites in [0, n_parents]
            const des_ga_run g = a.ga[run];
            a.n_parents = min(max(g.n_parents, 1), a.table_rows);
            a.n_elites = min(max(g.n_elites, 0), a.n_parents);
            a.parents += (size_t)run * (size_t)a.table_rows * a.L.P;
        }
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
    const uint32_t member = (uint32_t)(a.member_offset + member_slot(a));

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
    } else if constexpr (kGaFill<Args>) {
        // ---- an elite's parent row as it is, any other member's parent row + sigma*eps (P is odd: scalar loads)
        if (member < (uint32_t)a.n_elites) {
            const float *row = a.parents + (int64_t)member * L.P;
            for (int j = lane; j < L.P; j += 32) stage(j, __ldg(row + j));
        } else {
            const float *row = a.parents + (int64_t)ga_parent(member, gen, (uint32_t)a.n_parents, a.key) * L.P;
            for (int q = lane; q < (L.P + 3) / 4; q += 32) {
                const float4 z = noise_quad((uint32_t)q, member, gen, kStreamNesEps, a.key);
                const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int j = 4 * q + e;
                    if (j >= L.P) break;
                    stage(j, __fmaf_rn(a.sigma, zz[e], __ldg(row + j)));
                }
            }
        }
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
    env.reset((uint32_t)ep, a.reset_member_base + (a.noiseless ? 0u : (uint32_t)member_slot(a)), gen, a.key);
    double total = 0.0, osum[3] = {0, 0, 0}, osq[3] = {0, 0, 0};
    constexpr bool kRecord = std::is_same<Args, RecordArgs>::value;
    // a recording's row of episode ep at step t, ((member * reps + ep) * horizon + t), and whether this lane writes it;
    // the kernels of the evaluations compile none of it
    auto row_at = [&](int t) { return ((int64_t)blockIdx.x * a.reps + ep) * a.horizon + t; };
    for (int t = 0; t < a.horizon; ++t) {
        {
            float o[3];
            env.observe(o);                                              // leaves th and thdot as they were
            if constexpr (kRecord) {
                const int64_t at = row_at(t);
                if (writer && ep < a.reps && a.states) { a.states[2 * at] = env.th; a.states[2 * at + 1] = env.thdot; }
                if (writer && ep < a.reps && a.obs) { a.obs[3 * at] = o[0]; a.obs[3 * at + 1] = o[1]; a.obs[3 * at + 2] = o[2]; }
            }
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
        if constexpr (kRecord) {
            const double reward = env.step((double)act);
            total += reward;
            const int64_t at = row_at(t);
            if (writer && ep < a.reps && a.actions) a.actions[at] = act;
            if (writer && ep < a.reps && a.rewards) a.rewards[at] = reward;
        } else {
            total += env.step((double)act);                              // utils.py:135-137
        }
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
    if constexpr (kBc<Args>) {
        // the behaviour: the raw observation after the last step, in the reduction area once every read above is done.
        // Observed here, after the step loop, so that the loop is the evaluation's own code and schedule
        float bc[3];
        env.observe(bc);
        __syncwarp();
        if (writer) {
#pragma unroll
            for (int k = 0; k < 3; ++k) red[ep * 8 + 1 + k] = (double)bc[k];
        }
        __syncwarp();
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                double s = 0.0;
                for (int r = 0; r < a.reps; ++r) s += red[r * 8 + 1 + k];
                a.bc_out[(int64_t)blockIdx.x * 3 + k] = (float)(s / a.reps);
            }
        }
    }
}

// Launches rollout_pendulum_kernel<H / 16, kRows, Args> over `blocks` CTAs of one warp.  Not inline, so that the
// extern template declarations below keep des_envs.cu from compiling the kernels another unit instantiates.
template <bool kRows, typename Args>
int rollout_kernels(const Args &a, int H, unsigned blocks, size_t smem, cudaStream_t st) {
    void (*kernel)(Args);
    switch (H / 16) {                    // R = H/16 hidden units per lane
        case 1: kernel = rollout_pendulum_kernel<1, kRows, Args>; break;
        case 2: kernel = rollout_pendulum_kernel<2, kRows, Args>; break;
        case 4: kernel = rollout_pendulum_kernel<4, kRows, Args>; break;
        case 6: kernel = rollout_pendulum_kernel<6, kRows, Args>; break;
        default: kernel = rollout_pendulum_kernel<8, kRows, Args>; break;
    }
    return launch_smem("rollout_pendulum_kernel", kernel, blocks, 32, smem, st, a);
}

// The instantiations of the other units (see the top of this file); des_envs.cu instantiates the rest.
extern template int rollout_kernels<true, SweepArgs>(const SweepArgs &, int, unsigned, size_t, cudaStream_t);
extern template int rollout_kernels<false, RecordArgs>(const RecordArgs &, int, unsigned, size_t, cudaStream_t);
extern template int rollout_kernels<true, RecordArgs>(const RecordArgs &, int, unsigned, size_t, cudaStream_t);
extern template int rollout_kernels<false, GaArgs>(const GaArgs &, int, unsigned, size_t, cudaStream_t);
extern template int rollout_kernels<false, GaSweepArgs>(const GaSweepArgs &, int, unsigned, size_t, cudaStream_t);
extern template int rollout_kernels<false, BcArgs>(const BcArgs &, int, unsigned, size_t, cudaStream_t);
extern template int rollout_kernels<false, BcSweepArgs>(const BcSweepArgs &, int, unsigned, size_t, cudaStream_t);
extern template int rollout_kernels<false, GaBcArgs>(const GaBcArgs &, int, unsigned, size_t, cudaStream_t);

}  // namespace des
