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
#include "des_act.cuh"

namespace des {

// Shared by des_policy_act and des_policy_act_sweep: argument checks (before any CUDA work), then the launch over n_local
// rows.  A table hp_dev makes the rows a sweep of runs of run_size (member_offset 0, seed and action noise per run).
static int policy_act(const char *who, float *actions_out_dev, double *stat_part_dev, const float *rows_dev, int64_t P,
                      const float *obs_dev, const uint8_t *alive_dev, const float *obs_stats_dev, des_dims dims,
                      int32_t repetitions, double clip, double action_noise_std, uint64_t seed, uint64_t generation,
                      int64_t member_offset, int64_t n_local, int64_t t, const des_run_hp *hp_dev, int64_t run_size,
                      cudaStream_t st) {
    const int H = dims.hidden, d0 = dims.state_dim, A = dims.action_dim;
    DES_REQUIRE(policy_width_ok(H), "%s: hidden must be 16, 32, 64, 96 or 128 (got %d)", who, H);
    DES_REQUIRE(d0 >= 1 && d0 <= kActMaxD0, "%s: state_dim must be in [1, %d] (got %d)", who, kActMaxD0, d0);
    DES_REQUIRE(A >= 1 && A <= kActMaxA, "%s: action_dim must be in [1, %d] (got %d)", who, kActMaxA, A);
    DES_REQUIRE(repetitions >= 1 && repetitions <= kActMaxReps,
                "%s: repetitions must be in [1, %d] (the action-noise counter is member*16 + repetition; got %d)", who,
                kActMaxReps, repetitions);
    const Layout L(d0, H, A);
    DES_REQUIRE(P == L.P, "%s: rows have P = %lld, the (%d,%d,%d) MLP needs %d", who, (long long)P, d0, H, A, L.P);
    DES_REQUIRE(member_range_ok(member_offset, hp_dev ? run_size : n_local, 28), "%s: bad member range", who);
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
    if (!hp_dev) return act_launch(a, H, n_local, st);
    ActSweepArgs sa;
    static_cast<ActArgs &>(sa) = a;
    sa.hp = hp_dev;
    sa.run_size = (int)run_size;
    return act_launch_sweep(sa, H, n_local, st);
}

}  // namespace des

extern "C" DES_API int des_policy_act(float *actions_out_dev, double *stat_part_dev, const float *rows_dev, int64_t P,
                                      const float *obs_dev, const uint8_t *alive_dev, const float *obs_stats_dev,
                                      des_dims dims, int32_t repetitions, double clip, double action_noise_std,
                                      uint64_t seed, uint64_t generation, int64_t member_offset, int64_t n_local,
                                      int64_t t, void *stream) {
    return des::policy_act("des_policy_act", actions_out_dev, stat_part_dev, rows_dev, P, obs_dev, alive_dev,
                           obs_stats_dev, dims, repetitions, clip, action_noise_std, seed, generation, member_offset,
                           n_local, t, nullptr, 0, (cudaStream_t)stream);
}

extern "C" DES_API int des_policy_act_sweep(float *actions_out_dev, double *stat_part_dev, const float *rows_dev, int64_t P,
                                            const float *obs_dev, const uint8_t *alive_dev, const float *obs_stats_dev,
                                            des_dims dims, int32_t repetitions, double clip, const des_run_hp *hp_dev,
                                            uint64_t generation, int64_t n_runs, int64_t run_size, int64_t t,
                                            void *stream) {
    const char *who = "des_policy_act_sweep";
    const int rc = des::check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(n_runs == 0 || hp_dev, "%s: NULL pointer", who);
    return des::policy_act(who, actions_out_dev, stat_part_dev, rows_dev, P, obs_dev, alive_dev, obs_stats_dev, dims,
                           repetitions, clip, 0.0, 0, generation, 0, n_runs * run_size, t, hp_dev, run_size,
                           (cudaStream_t)stream);
}
