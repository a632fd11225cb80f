// des_rollout_eval: closed-loop rollouts with per-member observations (SURVEY 8f row 3) — the reference's actual
// workload: Evaluator.eval utils.py:116-124 -> single_run utils.py:126-139, once per member per repetition, with the
// environment stepped on the device.  Environment 0 = Pendulum-v0 (the reference's PendulumConfig, config.py:26-31:
// obs 3, action 1, clip +-2, 200-step episodes).
//
// One warp per member steps all of the member's episodes in lockstep (see rollout_pendulum_kernel, des_envs.cuh); the member's
// weights go once into shared memory: theta + sigma*eps generated with the same counter noise as every other kernel
// (NES), or row i of an explicit solutions[n_local][P] matrix (des_rollout_eval_solutions: the solutions CMA-ES's ask()
// returns, cma_es.py:22-29).  Everything after the weights are staged is the same code in both modes.
// Policy arithmetic fp32 (FFMA, MUFU-based tanh), dynamics fp64 (gym keeps its state in float64).
// Algorithmic work per environment step: 2*(3H + H*H + H) flop; no HBM traffic beyond theta (L2 resident).
#include "des_envs.cuh"

namespace des {

// Shared by the entry points, after their own checks: the argument checks (before any CUDA work), the RollArgs part of
// `a`, the workspace, the launch of rollout_pendulum_kernel<H / 16, kRows, Args> and the observation totals.  The entry
// point fills the rest of `a`, and Args decides the rest of the evaluation.  kRows makes `weights` explicit rows[n_local][P]
// instead of the theta that sigma*eps perturbs, and kGaFill<Args> makes it the genetic algorithm's parents table
// (des_rollout_eval_ga[_sweep|_bc]).  A recording (RecordArgs, des_rollout_record[_solutions]) has the element counts of
// its four trajectories checked, and a behaviour-writing evaluation (kBc<Args>) its behaviour output.  A batch of runs
// (Args derived from RunArgs: des_rollout_eval_runs, member_offset 0) has one row per run in `weights` and
// `obs_stats_dev`, and its observation totals are reduced per run; a sweep (Args derived from SweepArgs) takes seed, sigma
// and action_noise_std from each run's row of the table a.hp instead.
template <bool kRows, typename Args>
static int rollout_eval(const char *who, Args a, float *fitness_out_dev, float *episode_returns_out_dev,
                        double *obs_totals_out_dev, const float *weights_dev, const float *obs_stats_dev, int env,
                        des_dims dims, int32_t repetitions, double sigma, double clip, double action_noise_std,
                        uint64_t seed, uint64_t generation, const des_state *state_dev, int64_t member_offset,
                        int64_t n_local, int noiseless, void *workspace_dev, size_t workspace_bytes, bool mirrored,
                        cudaStream_t st) {
    DES_REQUIRE(env == kEnvPendulum, "%s: unknown environment %d (0 = Pendulum-v0)", who, env);
    if (mirrored && !(member_offset >= 0 && n_local >= 0 && whole_pairs(member_offset, n_local)))
        return not_whole_pairs(who, "n_local", member_offset, n_local);
    DES_REQUIRE(!mirrored || !noiseless, "%s: test episodes (noiseless) have no pairs; use des_rollout_eval", who);
    DES_REQUIRE(dims.state_dim == 3 && dims.action_dim == 1, "%s: Pendulum-v0 has state_dim 3, action_dim 1", who);
    DES_REQUIRE(policy_width_ok(dims.hidden), "%s: hidden must be 16 or a multiple of 32, <= 128 (got %d)", who, dims.hidden);
    DES_REQUIRE(repetitions >= 1 && repetitions <= 10, "%s: repetitions must be in [1, 10] (one warp each)", who);
    DES_REQUIRE(dims.tape_len >= 1, "%s: episode length (dims.tape_len) must be >= 1", who);
    DES_REQUIRE(member_range_ok(member_offset, n_local, 28), "%s: bad member range", who);
    if constexpr (std::is_same<Args, RecordArgs>::value) {
        // each trajectory's element count n_local * reps * horizon * width within int64
        const void *traj[4] = {a.states, a.obs, a.actions, a.rewards};
        const int width[4] = {2, 3, 1, 1};
        for (int k = 0; k < 4; ++k)
            DES_REQUIRE(!traj[k] || n_local == 0 || dims.tape_len <= INT64_MAX / (n_local * repetitions * width[k]),
                        "%s: trajectories of %lld members x %d episodes x %d steps exceed int64 elements", who,
                        (long long)n_local, repetitions, dims.tape_len);
    }
    if (n_local == 0) return DES_OK;
    bool bc_ok = true;
    if constexpr (kBc<Args>) bc_ok = a.bc_out != nullptr;
    DES_REQUIRE(fitness_out_dev && weights_dev && bc_ok, "%s: NULL pointer", who);
    a.fitness = fitness_out_dev; a.ep_ret = episode_returns_out_dev;
    a.theta = kRows || kGaFill<Args> ? nullptr : weights_dev; a.rows = kRows ? weights_dev : nullptr;
    if constexpr (kGaFill<Args>) a.parents = weights_dev;
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
    const int rc = rollout_kernels<kRows>(a, H, (unsigned)n_local, smem, st);
    if (rc != DES_OK || !obs_totals_out_dev) return rc;
    if constexpr (std::is_base_of<RunArgs, Args>::value)
        return obs_parts_reduce_runs(obs_totals_out_dev, a.stat_part, n_local / a.run_size, a.run_size, 7, st);
    else
        return obs_parts_reduce(obs_totals_out_dev, a.stat_part, n_local, 7, st);
}

// A batch of n_runs runs of run_size members (des_rollout_eval_runs, _sweep, _bc_sweep, _solutions_sweep): its checks,
// made before the evaluation's, and the run block of `a`.  A sweep (Args derived from SweepArgs) needs its table hp_dev.
template <typename Args>
static int batch_args(const char *who, Args &a, int64_t n_runs, int64_t run_size, int noiseless, const des_run_hp *hp_dev) {
    const int rc = check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(!noiseless || run_size == 1, "%s: test episodes (noiseless) evaluate one theta per run: run_size must be 1 "
                "(got %lld)", who, (long long)run_size);
    a.run_size = (int)run_size;
    if constexpr (std::is_base_of<SweepArgs, Args>::value) {
        DES_REQUIRE(n_runs == 0 || hp_dev, "%s: NULL pointer", who);
        a.hp = hp_dev;
    }
    return DES_OK;
}

// The counts of a genetic-algorithm generation's parents table (des_rollout_eval_ga, _ga_bc): their checks, made before
// the evaluation's, and `a`'s counts.
static int ga_counts(const char *who, GaArgs &a, int64_t n_parents, int64_t n_elites) {
    DES_REQUIRE(n_parents >= 1 && n_parents <= INT32_MAX, "%s: n_parents must be in [1, 2^31) (got %lld)", who,
                (long long)n_parents);
    DES_REQUIRE(n_elites >= 0 && n_elites <= n_parents, "%s: n_elites must be in [0, n_parents = %lld] (got %lld)", who,
                (long long)n_parents, (long long)n_elites);
    a.n_parents = (int)n_parents; a.n_elites = (int)n_elites;
    return DES_OK;
}

}  // namespace des

extern "C" DES_API int des_rollout_eval(float *fitness_out_dev, float *episode_returns_out_dev,
                                        double *obs_totals_out_dev, const float *theta_dev,
                                        const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions,
                                        double sigma, double clip, double action_noise_std, uint64_t seed,
                                        uint64_t generation, const des_state *state_dev, int64_t member_offset,
                                        int64_t n_local, int noiseless, void *workspace_dev, size_t workspace_bytes,
                                        void *stream) {
    return des::rollout_eval<false>("des_rollout_eval", des::RollArgs(), fitness_out_dev, episode_returns_out_dev,
                                    obs_totals_out_dev, theta_dev, obs_stats_dev, env, dims, repetitions, sigma, clip,
                                    action_noise_std, seed, generation, state_dev, member_offset, n_local, noiseless,
                                    workspace_dev, workspace_bytes, false, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_bc(float *fitness_out_dev, float *episode_returns_out_dev,
                                           double *obs_totals_out_dev, const float *theta_dev, const float *obs_stats_dev,
                                           int env, des_dims dims, int32_t repetitions, double sigma, double clip,
                                           double action_noise_std, uint64_t seed, uint64_t generation,
                                           const des_state *state_dev, int64_t member_offset, int64_t n_local,
                                           int noiseless, float *bc_out_dev, void *workspace_dev, size_t workspace_bytes,
                                           void *stream) {
    des::BcArgs bc;
    bc.bc_out = bc_out_dev;
    return des::rollout_eval<false>("des_rollout_eval_bc", bc, fitness_out_dev, episode_returns_out_dev,
                                    obs_totals_out_dev, theta_dev, obs_stats_dev, env, dims, repetitions, sigma, clip,
                                    action_noise_std, seed, generation, state_dev, member_offset, n_local, noiseless,
                                    workspace_dev, workspace_bytes, false, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_ga(float *fitness_out_dev, float *episode_returns_out_dev,
                                           double *obs_totals_out_dev, const float *parents_dev, int64_t n_parents,
                                           int64_t n_elites, const float *obs_stats_dev, int env, des_dims dims,
                                           int32_t repetitions, double sigma, double clip, double action_noise_std,
                                           uint64_t seed, uint64_t generation, const des_state *state_dev,
                                           int64_t member_offset, int64_t n_local, int noiseless, void *workspace_dev,
                                           size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_ga";
    DES_REQUIRE(!noiseless, "%s: test episodes (noiseless) evaluate one row; use des_rollout_eval on it", who);
    des::GaArgs ga;
    const int rc = des::ga_counts(who, ga, n_parents, n_elites);
    if (rc != DES_OK) return rc;
    return des::rollout_eval<false>(who, ga, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, parents_dev,
                                    obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed, generation,
                                    state_dev, member_offset, n_local, 0, workspace_dev, workspace_bytes, false,
                                    (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_ga_bc(float *fitness_out_dev, float *episode_returns_out_dev,
                                              double *obs_totals_out_dev, const float *parents_dev, int64_t n_parents,
                                              int64_t n_elites, const float *obs_stats_dev, int env, des_dims dims,
                                              int32_t repetitions, double sigma, double clip, double action_noise_std,
                                              uint64_t seed, uint64_t generation, const des_state *state_dev,
                                              int64_t member_offset, int64_t n_local, int noiseless, float *bc_out_dev,
                                              void *workspace_dev, size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_ga_bc";
    DES_REQUIRE(!noiseless, "%s: test episodes (noiseless) evaluate one row; use des_rollout_eval_bc on it", who);
    des::GaBcArgs ga;
    const int rc = des::ga_counts(who, ga, n_parents, n_elites);
    if (rc != DES_OK) return rc;
    ga.bc_out = bc_out_dev;
    return des::rollout_eval<false>(who, ga, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, parents_dev,
                                    obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed, generation,
                                    state_dev, member_offset, n_local, 0, workspace_dev, workspace_bytes, false,
                                    (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_ga_sweep(float *fitness_out_dev, float *episode_returns_out_dev,
                                                 double *obs_totals_out_dev, const float *parents_dev,
                                                 const des_ga_run *ga_dev, int64_t table_rows, const float *obs_stats_dev,
                                                 int env, des_dims dims, int32_t repetitions, double clip,
                                                 const des_run_hp *hp_dev, uint64_t generation, const des_state *state_dev,
                                                 int64_t n_runs, int64_t run_size, void *workspace_dev,
                                                 size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_ga_sweep";
    const int rc = des::check_runs(who, n_runs, run_size, 2);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(table_rows >= 1 && table_rows <= run_size, "%s: table_rows must be in [1, run_size = %lld] (got %lld)", who,
                (long long)run_size, (long long)table_rows);
    DES_REQUIRE(n_runs == 0 || (hp_dev && ga_dev), "%s: NULL pointer", who);
    des::GaSweepArgs ga;
    ga.run_size = (int)run_size; ga.hp = hp_dev;
    ga.ga = ga_dev; ga.table_rows = (int)table_rows;
    ga.n_parents = 1; ga.n_elites = 0;                  // each CTA sets its run's
    return des::rollout_eval<false>(who, ga, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, parents_dev,
                                    obs_stats_dev, env, dims, repetitions, 0.0, clip, 0.0, 0, generation, state_dev, 0,
                                    n_runs * run_size, 0, workspace_dev, workspace_bytes, false, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_mirrored(float *fitness_out_dev, float *episode_returns_out_dev,
                                                 double *obs_totals_out_dev, const float *theta_dev,
                                                 const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions,
                                                 double sigma, double clip, double action_noise_std, uint64_t seed,
                                                 uint64_t generation, const des_state *state_dev, int64_t member_offset,
                                                 int64_t n_local, int noiseless, void *workspace_dev, size_t workspace_bytes,
                                                 void *stream) {
    return des::rollout_eval<false>("des_rollout_eval_mirrored", des::RollArgs(), fitness_out_dev, episode_returns_out_dev,
                                    obs_totals_out_dev, theta_dev, obs_stats_dev, env, dims, repetitions, sigma, clip,
                                    action_noise_std, seed, generation, state_dev, member_offset, n_local, noiseless,
                                    workspace_dev, workspace_bytes, true, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_solutions(float *fitness_out_dev, float *episode_returns_out_dev,
                                                  double *obs_totals_out_dev, const float *solutions_dev,
                                                  const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions,
                                                  double clip, double action_noise_std, uint64_t seed,
                                                  uint64_t generation, int64_t member_offset, int64_t n_local,
                                                  void *workspace_dev, size_t workspace_bytes, void *stream) {
    return des::rollout_eval<true>("des_rollout_eval_solutions", des::RollArgs(), fitness_out_dev, episode_returns_out_dev,
                                   obs_totals_out_dev, solutions_dev, obs_stats_dev, env, dims, repetitions, 0.0, clip,
                                   action_noise_std, seed, generation, nullptr, member_offset, n_local, 0, workspace_dev,
                                   workspace_bytes, false, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_runs(float *fitness_out_dev, float *episode_returns_out_dev,
                                             double *obs_totals_out_dev, const float *theta_dev, const float *obs_stats_dev,
                                             int env, des_dims dims, int32_t repetitions, double sigma, double clip,
                                             double action_noise_std, uint64_t seed, uint64_t generation,
                                             const des_state *state_dev, int64_t n_runs, int64_t run_size, int noiseless,
                                             void *workspace_dev, size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_runs";
    des::RunArgs a;
    const int rc = des::batch_args(who, a, n_runs, run_size, noiseless, nullptr);
    if (rc != DES_OK) return rc;
    return des::rollout_eval<false>(who, a, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, theta_dev,
                                    obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed, generation,
                                    state_dev, 0, n_runs * run_size, noiseless, workspace_dev, workspace_bytes, false,
                                    (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_sweep(float *fitness_out_dev, float *episode_returns_out_dev,
                                              double *obs_totals_out_dev, const float *theta_dev, const float *obs_stats_dev,
                                              int env, des_dims dims, int32_t repetitions, double clip,
                                              const des_run_hp *hp_dev, uint64_t generation, const des_state *state_dev,
                                              int64_t n_runs, int64_t run_size, int noiseless, void *workspace_dev,
                                              size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_sweep";
    des::SweepArgs a;
    const int rc = des::batch_args(who, a, n_runs, run_size, noiseless, hp_dev);
    if (rc != DES_OK) return rc;
    return des::rollout_eval<false>(who, a, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, theta_dev,
                                    obs_stats_dev, env, dims, repetitions, 0.0, clip, 0.0, 0, generation, state_dev, 0,
                                    n_runs * run_size, noiseless, workspace_dev, workspace_bytes, false,
                                    (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_bc_sweep(float *fitness_out_dev, float *episode_returns_out_dev,
                                                 double *obs_totals_out_dev, const float *theta_dev,
                                                 const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions,
                                                 double clip, const des_run_hp *hp_dev, uint64_t generation,
                                                 const des_state *state_dev, int64_t n_runs, int64_t run_size,
                                                 int noiseless, float *bc_out_dev, void *workspace_dev,
                                                 size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_bc_sweep";
    des::BcSweepArgs bc;
    const int rc = des::batch_args(who, bc, n_runs, run_size, noiseless, hp_dev);
    if (rc != DES_OK) return rc;
    bc.bc_out = bc_out_dev;
    return des::rollout_eval<false>(who, bc, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, theta_dev,
                                    obs_stats_dev, env, dims, repetitions, 0.0, clip, 0.0, 0, generation, state_dev, 0,
                                    n_runs * run_size, noiseless, workspace_dev, workspace_bytes, false,
                                    (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_solutions_sweep(float *fitness_out_dev, float *episode_returns_out_dev,
                                                        double *obs_totals_out_dev, const float *rows_dev,
                                                        const float *obs_stats_dev, int env, des_dims dims,
                                                        int32_t repetitions, double clip, const des_run_hp *hp_dev,
                                                        uint64_t generation, int64_t n_runs, int64_t run_size,
                                                        void *workspace_dev, size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_solutions_sweep";
    des::SweepArgs a;
    const int rc = des::batch_args(who, a, n_runs, run_size, 0, hp_dev);
    if (rc != DES_OK) return rc;
    return des::rollout_eval<true>(who, a, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, rows_dev,
                                   obs_stats_dev, env, dims, repetitions, 0.0, clip, 0.0, 0, generation, nullptr, 0,
                                   n_runs * run_size, 0, workspace_dev, workspace_bytes, false, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_record(float *fitness_out_dev, float *episode_returns_out_dev,
                                          double *obs_totals_out_dev, const float *theta_dev, const float *obs_stats_dev,
                                          int env, des_dims dims, int32_t repetitions, double sigma, double clip,
                                          double action_noise_std, uint64_t seed, uint64_t generation,
                                          const des_state *state_dev, int64_t member_offset, int64_t n_local, int noiseless,
                                          int mirrored, double *states_out_dev, float *obs_out_dev, float *actions_out_dev,
                                          double *rewards_out_dev, void *workspace_dev, size_t workspace_bytes,
                                          void *stream) {
    des::RecordArgs rec;
    rec.states = states_out_dev; rec.obs = obs_out_dev; rec.actions = actions_out_dev; rec.rewards = rewards_out_dev;
    return des::rollout_eval<false>("des_rollout_record", rec, fitness_out_dev, episode_returns_out_dev,
                                    obs_totals_out_dev, theta_dev, obs_stats_dev, env, dims, repetitions, sigma, clip,
                                    action_noise_std, seed, generation, state_dev, member_offset, n_local, noiseless,
                                    workspace_dev, workspace_bytes, mirrored != 0, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_record_solutions(float *fitness_out_dev, float *episode_returns_out_dev,
                                                    double *obs_totals_out_dev, const float *solutions_dev,
                                                    const float *obs_stats_dev, int env, des_dims dims,
                                                    int32_t repetitions, double clip, double action_noise_std,
                                                    uint64_t seed, uint64_t generation, int64_t member_offset,
                                                    int64_t n_local, double *states_out_dev, float *obs_out_dev,
                                                    float *actions_out_dev, double *rewards_out_dev, void *workspace_dev,
                                                    size_t workspace_bytes, void *stream) {
    des::RecordArgs rec;
    rec.states = states_out_dev; rec.obs = obs_out_dev; rec.actions = actions_out_dev; rec.rewards = rewards_out_dev;
    return des::rollout_eval<true>("des_rollout_record_solutions", rec, fitness_out_dev, episode_returns_out_dev,
                                   obs_totals_out_dev, solutions_dev, obs_stats_dev, env, dims, repetitions, 0.0, clip,
                                   action_noise_std, seed, generation, nullptr, member_offset, n_local, 0, workspace_dev,
                                   workspace_bytes, false, (cudaStream_t)stream);
}
