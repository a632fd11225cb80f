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

// Shared by the entry points: argument checks (before any CUDA work), workspace, launch.  rows_mode selects the
// explicit-solution kernels: `weights` is then rows[n_local][P] instead of the theta that sigma*eps perturbs.  run_size > 0
// makes the n_local members a batch of runs of run_size (des_rollout_eval_runs, member_offset 0): `weights` and
// `obs_stats_dev` hold one row per run, and the observation totals are reduced per run.  A table hp_dev makes that batch a
// sweep (des_rollout_eval_sweep, or des_rollout_eval_solutions_sweep in rows_mode): seed, sigma and action_noise_std are
// then each run's row of the table.  A non-NULL `record` makes the launch a recording (des_rollout_record[_solutions]): its
// four trajectory pointers, each optional, are written beside the evaluation's outputs by the RecordArgs kernels.  A
// non-NULL `ga` makes it a genetic-algorithm generation (des_rollout_eval_ga): `weights` is then its parents table.  A
// non-NULL `ga_sweep` with a table hp_dev makes the sweep one of genetic-algorithm runs (des_rollout_eval_ga_sweep):
// `weights` is then the buffer of every run's parents table.  A non-NULL `bc` makes it an evaluation that also writes
// each member's behaviour characterisation (des_rollout_eval_bc), and a non-NULL `bc_sweep` with a table hp_dev a sweep
// that does (des_rollout_eval_bc_sweep).  A non-NULL `ga_bc` makes it a genetic-algorithm generation that also writes each
// member's behaviour (des_rollout_eval_ga_bc): `weights` is then its parents table.
static int rollout_launch(const char *who, float *fitness_out_dev, float *episode_returns_out_dev,
                          double *obs_totals_out_dev, const float *weights_dev, bool rows_mode,
                          const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions, double sigma,
                          double clip, double action_noise_std, uint64_t seed, uint64_t generation,
                          const des_state *state_dev, int64_t member_offset, int64_t n_local, int noiseless,
                          void *workspace_dev, size_t workspace_bytes, bool mirrored, int64_t run_size,
                          const des_run_hp *hp_dev, const RecordArgs *record, cudaStream_t st,
                          const GaArgs *ga = nullptr, const GaSweepArgs *ga_sweep = nullptr,
                          const BcArgs *bc = nullptr, const BcSweepArgs *bc_sweep = nullptr,
                          const GaBcArgs *ga_bc = nullptr) {
    DES_REQUIRE(env == kEnvPendulum, "%s: unknown environment %d (0 = Pendulum-v0)", who, env);
    if (mirrored && !(member_offset >= 0 && n_local >= 0 && whole_pairs(member_offset, n_local)))
        return not_whole_pairs(who, "n_local", member_offset, n_local);
    DES_REQUIRE(!mirrored || !noiseless, "%s: test episodes (noiseless) have no pairs; use des_rollout_eval", who);
    DES_REQUIRE(dims.state_dim == 3 && dims.action_dim == 1, "%s: Pendulum-v0 has state_dim 3, action_dim 1", who);
    DES_REQUIRE(policy_width_ok(dims.hidden), "%s: hidden must be 16 or a multiple of 32, <= 128 (got %d)", who, dims.hidden);
    DES_REQUIRE(repetitions >= 1 && repetitions <= 10, "%s: repetitions must be in [1, 10] (one warp each)", who);
    DES_REQUIRE(dims.tape_len >= 1, "%s: episode length (dims.tape_len) must be >= 1", who);
    DES_REQUIRE(member_range_ok(member_offset, n_local, 28), "%s: bad member range", who);
    if (record) {           // each trajectory's element count n_local * reps * horizon * width within int64
        const void *traj[4] = {record->states, record->obs, record->actions, record->rewards};
        const int width[4] = {2, 3, 1, 1};
        for (int k = 0; k < 4; ++k)
            DES_REQUIRE(!traj[k] || n_local == 0 || dims.tape_len <= INT64_MAX / (n_local * repetitions * width[k]),
                        "%s: trajectories of %lld members x %d episodes x %d steps exceed int64 elements", who,
                        (long long)n_local, repetitions, dims.tape_len);
    }
    if (n_local == 0) return DES_OK;
    DES_REQUIRE(fitness_out_dev && weights_dev && (!bc || bc->bc_out) && (!bc_sweep || bc_sweep->bc_out) &&
                (!ga_bc || ga_bc->bc_out), "%s: NULL pointer", who);
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
    if (record) {
        RecordArgs ra = *record;
        static_cast<RollArgs &>(ra) = a;
        const int rc = rollout_record_launch(ra, H, rows_mode, (unsigned)n_local, smem, st);
        if (rc != DES_OK || !obs_totals_out_dev) return rc;
        return obs_parts_reduce(obs_totals_out_dev, a.stat_part, n_local, 7, st);
    }
    if (bc) {
        BcArgs b = *bc;
        static_cast<RollArgs &>(b) = a;
        const int rc = rollout_bc_launch(b, H, (unsigned)n_local, smem, st);
        if (rc != DES_OK || !obs_totals_out_dev) return rc;
        return obs_parts_reduce(obs_totals_out_dev, a.stat_part, n_local, 7, st);
    }
    if (ga_bc) {
        GaBcArgs g = *ga_bc;
        static_cast<RollArgs &>(g) = a;
        g.theta = nullptr;
        g.parents = weights_dev;
        const int rc = rollout_ga_bc_launch(g, H, (unsigned)n_local, smem, st);
        if (rc != DES_OK || !obs_totals_out_dev) return rc;
        return obs_parts_reduce(obs_totals_out_dev, a.stat_part, n_local, 7, st);
    }
    if (ga) {
        GaArgs g = *ga;
        static_cast<RollArgs &>(g) = a;
        g.theta = nullptr;
        g.parents = weights_dev;
        const int rc = rollout_ga_launch(g, H, (unsigned)n_local, smem, st);
        if (rc != DES_OK || !obs_totals_out_dev) return rc;
        return obs_parts_reduce(obs_totals_out_dev, a.stat_part, n_local, 7, st);
    }
    if (run_size > 0) {
        RunArgs ra;
        static_cast<RollArgs &>(ra) = a;
        ra.run_size = (int)run_size;
        if (hp_dev) {
            SweepArgs sa;
            static_cast<RunArgs &>(sa) = ra;
            sa.hp = hp_dev;
            if (ga_sweep) {
                GaSweepArgs g = *ga_sweep;
                static_cast<SweepArgs &>(g) = sa;
                g.theta = nullptr;
                g.parents = weights_dev;
                const int rc = rollout_ga_sweep_launch(g, H, (unsigned)n_local, smem, st);
                if (rc != DES_OK || !obs_totals_out_dev) return rc;
                return obs_parts_reduce_runs(obs_totals_out_dev, a.stat_part, n_local / run_size, run_size, 7, st);
            }
            if (bc_sweep) {
                BcSweepArgs b = *bc_sweep;
                static_cast<SweepArgs &>(b) = sa;
                const int rc = rollout_bc_sweep_launch(b, H, (unsigned)n_local, smem, st);
                if (rc != DES_OK || !obs_totals_out_dev) return rc;
                return obs_parts_reduce_runs(obs_totals_out_dev, a.stat_part, n_local / run_size, run_size, 7, st);
            }
            void (*sweep_kernel)(SweepArgs);
            switch (H / 16) {
                case 1: sweep_kernel = rollout_pendulum_kernel<1, false, SweepArgs>; break;
                case 2: sweep_kernel = rollout_pendulum_kernel<2, false, SweepArgs>; break;
                case 4: sweep_kernel = rollout_pendulum_kernel<4, false, SweepArgs>; break;
                case 6: sweep_kernel = rollout_pendulum_kernel<6, false, SweepArgs>; break;
                default: sweep_kernel = rollout_pendulum_kernel<8, false, SweepArgs>; break;
            }
            const int rc = rows_mode ? rollout_rows_sweep_launch(sa, H, (unsigned)n_local, smem, st)
                                     : launch_smem("rollout_pendulum_kernel", sweep_kernel, (unsigned)n_local, 32, smem, st, sa);
            if (rc != DES_OK || !obs_totals_out_dev) return rc;
            return obs_parts_reduce_runs(obs_totals_out_dev, a.stat_part, n_local / run_size, run_size, 7, st);
        }
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
                               false, 0, nullptr, nullptr, (cudaStream_t)stream);
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
    return des::rollout_launch("des_rollout_eval_bc", fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev,
                               theta_dev, false, obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed,
                               generation, state_dev, member_offset, n_local, noiseless, workspace_dev, workspace_bytes,
                               false, 0, nullptr, nullptr, (cudaStream_t)stream, nullptr, nullptr, &bc);
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
    DES_REQUIRE(n_parents >= 1 && n_parents <= INT32_MAX, "%s: n_parents must be in [1, 2^31) (got %lld)", who,
                (long long)n_parents);
    DES_REQUIRE(n_elites >= 0 && n_elites <= n_parents, "%s: n_elites must be in [0, n_parents = %lld] (got %lld)", who,
                (long long)n_parents, (long long)n_elites);
    des::GaArgs ga;
    ga.n_parents = (int)n_parents; ga.n_elites = (int)n_elites;
    return des::rollout_launch(who, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, parents_dev, false,
                               obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed, generation,
                               state_dev, member_offset, n_local, 0, workspace_dev, workspace_bytes, false, 0, nullptr,
                               nullptr, (cudaStream_t)stream, &ga);
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
    DES_REQUIRE(n_parents >= 1 && n_parents <= INT32_MAX, "%s: n_parents must be in [1, 2^31) (got %lld)", who,
                (long long)n_parents);
    DES_REQUIRE(n_elites >= 0 && n_elites <= n_parents, "%s: n_elites must be in [0, n_parents = %lld] (got %lld)", who,
                (long long)n_parents, (long long)n_elites);
    des::GaBcArgs ga;
    ga.n_parents = (int)n_parents; ga.n_elites = (int)n_elites;
    ga.bc_out = bc_out_dev;
    return des::rollout_launch(who, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, parents_dev, false,
                               obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed, generation,
                               state_dev, member_offset, n_local, 0, workspace_dev, workspace_bytes, false, 0, nullptr,
                               nullptr, (cudaStream_t)stream, nullptr, nullptr, nullptr, nullptr, &ga);
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
    ga.ga = ga_dev; ga.table_rows = (int)table_rows;
    ga.n_parents = 1; ga.n_elites = 0;                  // each CTA sets its run's
    return des::rollout_launch(who, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, parents_dev, false,
                               obs_stats_dev, env, dims, repetitions, 0.0, clip, 0.0, 0, generation, state_dev, 0,
                               n_runs * run_size, 0, workspace_dev, workspace_bytes, false, run_size, hp_dev, nullptr,
                               (cudaStream_t)stream, nullptr, &ga);
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
                               true, 0, nullptr, nullptr, (cudaStream_t)stream);
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
                               false, 0, nullptr, nullptr, (cudaStream_t)stream);
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
                               nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_sweep(float *fitness_out_dev, float *episode_returns_out_dev,
                                              double *obs_totals_out_dev, const float *theta_dev, const float *obs_stats_dev,
                                              int env, des_dims dims, int32_t repetitions, double clip,
                                              const des_run_hp *hp_dev, uint64_t generation, const des_state *state_dev,
                                              int64_t n_runs, int64_t run_size, int noiseless, void *workspace_dev,
                                              size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_sweep";
    const int rc = des::check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(!noiseless || run_size == 1, "%s: test episodes (noiseless) evaluate one theta per run: run_size must be 1 "
                "(got %lld)", who, (long long)run_size);
    DES_REQUIRE(n_runs == 0 || hp_dev, "%s: NULL pointer", who);
    return des::rollout_launch(who, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, theta_dev, false,
                               obs_stats_dev, env, dims, repetitions, 0.0, clip, 0.0, 0, generation, state_dev, 0,
                               n_runs * run_size, noiseless, workspace_dev, workspace_bytes, false, run_size, hp_dev,
                               nullptr, (cudaStream_t)stream);
}

extern "C" DES_API int des_rollout_eval_bc_sweep(float *fitness_out_dev, float *episode_returns_out_dev,
                                                 double *obs_totals_out_dev, const float *theta_dev,
                                                 const float *obs_stats_dev, int env, des_dims dims, int32_t repetitions,
                                                 double clip, const des_run_hp *hp_dev, uint64_t generation,
                                                 const des_state *state_dev, int64_t n_runs, int64_t run_size,
                                                 int noiseless, float *bc_out_dev, void *workspace_dev,
                                                 size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_bc_sweep";
    const int rc = des::check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(!noiseless || run_size == 1, "%s: test episodes (noiseless) evaluate one theta per run: run_size must be 1 "
                "(got %lld)", who, (long long)run_size);
    DES_REQUIRE(n_runs == 0 || hp_dev, "%s: NULL pointer", who);
    des::BcSweepArgs bc;
    bc.bc_out = bc_out_dev;
    return des::rollout_launch(who, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, theta_dev, false,
                               obs_stats_dev, env, dims, repetitions, 0.0, clip, 0.0, 0, generation, state_dev, 0,
                               n_runs * run_size, noiseless, workspace_dev, workspace_bytes, false, run_size, hp_dev,
                               nullptr, (cudaStream_t)stream, nullptr, nullptr, nullptr, &bc);
}

extern "C" DES_API int des_rollout_eval_solutions_sweep(float *fitness_out_dev, float *episode_returns_out_dev,
                                                        double *obs_totals_out_dev, const float *rows_dev,
                                                        const float *obs_stats_dev, int env, des_dims dims,
                                                        int32_t repetitions, double clip, const des_run_hp *hp_dev,
                                                        uint64_t generation, int64_t n_runs, int64_t run_size,
                                                        void *workspace_dev, size_t workspace_bytes, void *stream) {
    const char *who = "des_rollout_eval_solutions_sweep";
    const int rc = des::check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(n_runs == 0 || hp_dev, "%s: NULL pointer", who);
    return des::rollout_launch(who, fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, rows_dev, true,
                               obs_stats_dev, env, dims, repetitions, 0.0, clip, 0.0, 0, generation, nullptr, 0,
                               n_runs * run_size, 0, workspace_dev, workspace_bytes, false, run_size, hp_dev,
                               nullptr, (cudaStream_t)stream);
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
    return des::rollout_launch("des_rollout_record", fitness_out_dev, episode_returns_out_dev, obs_totals_out_dev, theta_dev,
                               false, obs_stats_dev, env, dims, repetitions, sigma, clip, action_noise_std, seed,
                               generation, state_dev, member_offset, n_local, noiseless, workspace_dev, workspace_bytes,
                               mirrored != 0, 0, nullptr, &rec, (cudaStream_t)stream);
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
    return des::rollout_launch("des_rollout_record_solutions", fitness_out_dev, episode_returns_out_dev,
                               obs_totals_out_dev, solutions_dev, true, obs_stats_dev, env, dims, repetitions, 0.0, clip,
                               action_noise_std, seed, generation, nullptr, member_offset, n_local, 0, workspace_dev,
                               workspace_bytes, false, 0, nullptr, &rec, (cudaStream_t)stream);
}
