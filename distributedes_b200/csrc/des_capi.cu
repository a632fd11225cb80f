// C-ABI glue: error reporting, argument validation for des_nes_eval, and the host-buffer session
// (des_session_*) — the call a reference-side binding makes (see include/des_b200.h, INTEGRATION.md).
#include <stdarg.h>
#include <string.h>
#include <new>
#include "des_common.cuh"

namespace des {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what) {
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? DES_ERR_NO_DEVICE : DES_ERR_CUDA;
}

int not_whole_pairs(const char *who, const char *count, int64_t member_offset, int64_t n) {
    set_error("%s: a mirrored shard holds whole pairs: member_offset (%lld) and %s (%lld) must be even", who,
              (long long)member_offset, count, (long long)n);
    return DES_ERR_INVALID_ARGUMENT;
}

int eval_ffma_launch(float *fitness, const float *theta, const float *obs, const float *target, des_dims dims,
                     double sigma, double clip, uint64_t seed, uint64_t generation, const des_state *state,
                     int64_t member_offset, int64_t n_local, const float *solutions, bool mirrored, cudaStream_t st);
int eval_tc_launch(float *fitness, const float *theta, const float *obs, const float *target, des_dims dims,
                   double sigma, double clip, uint64_t seed, uint64_t generation, const des_state *state,
                   int64_t member_offset, int64_t n_local, int precision, void *workspace, size_t workspace_bytes,
                   bool mirrored, cudaStream_t st);
size_t eval_tc_workspace_bytes(des_dims dims, int precision);

}  // namespace des

extern "C" DES_API const char *des_last_error(void) { return des::g_err; }
extern "C" DES_API const char *des_version(void) { return "distributedes_b200 0.1 (sm_90a)"; }

extern "C" DES_API int des_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" DES_API size_t des_nes_eval_workspace_bytes(des_dims dims, int precision) {
    if (precision == DES_FWD_F16 || precision == DES_FWD_F16X3) return des::eval_tc_workspace_bytes(dims, precision);
    return 0;
}

extern "C" DES_API int64_t des_param_count(int32_t d0, int32_t H, int32_t A) {
    if (d0 <= 0 || H <= 0 || A <= 0) return -1;
    return (int64_t)d0 * H + H + (int64_t)H * H + H + (int64_t)H * A + A;
}

extern "C" DES_API int des_pop_eval(float *fitness_out_dev, const float *solutions_dev, const float *obs_dev,
                                    const float *target_dev, des_dims dims, double clip, int64_t n_solutions, void *stream) {
    using namespace des;
    DES_REQUIRE(dims.state_dim > 0 && dims.hidden > 0 && dims.action_dim > 0 && dims.tape_len > 0,
                "des_pop_eval: bad dims (d0=%d H=%d A=%d T=%d)", dims.state_dim, dims.hidden, dims.action_dim, dims.tape_len);
    DES_REQUIRE(n_solutions >= 0 && n_solutions < ((int64_t)1 << 31), "des_pop_eval: bad n_solutions");
    DES_REQUIRE(clip >= 0.0, "des_pop_eval: clip must be >= 0");
    if (n_solutions == 0) return DES_OK;
    DES_REQUIRE(fitness_out_dev && solutions_dev && obs_dev && target_dev, "des_pop_eval: NULL pointer");
    return eval_ffma_launch(fitness_out_dev, solutions_dev, obs_dev, target_dev, dims, 0.0, clip, 0, 0, nullptr, 0, n_solutions,
                            solutions_dev, false, (cudaStream_t)stream);
}

namespace des {

// Shared by des_nes_eval and des_nes_eval_mirrored: argument checks (before any CUDA work), then the precision's launcher.
static int nes_eval(const char *who, float *fitness_out_dev, const float *theta_dev, const float *obs_dev,
                    const float *target_dev, des_dims dims, double sigma, double clip, uint64_t seed, uint64_t generation,
                    const des_state *state_dev, int64_t member_offset, int64_t n_local, int precision, void *workspace_dev,
                    size_t workspace_bytes, bool mirrored, cudaStream_t st) {
    DES_REQUIRE(dims.state_dim > 0 && dims.hidden > 0 && dims.action_dim > 0 && dims.tape_len > 0,
                "%s: bad dims (d0=%d H=%d A=%d T=%d)", who, dims.state_dim, dims.hidden, dims.action_dim, dims.tape_len);
    DES_REQUIRE(des_param_count(dims.state_dim, dims.hidden, dims.action_dim) < ((int64_t)1 << 31),
                "%s: parameter count exceeds 2^31", who);
    DES_REQUIRE(n_local >= 0 && n_local < ((int64_t)1 << 31), "%s: bad n_local=%lld", who, (long long)n_local);
    DES_REQUIRE(member_range_ok(member_offset, n_local, 32), "%s: member index must fit 32 bits", who);
    if (mirrored && !whole_pairs(member_offset, n_local)) return not_whole_pairs(who, "n_local", member_offset, n_local);
    DES_REQUIRE(clip >= 0.0, "%s: clip must be >= 0", who);
    if (n_local == 0) return DES_OK;
    DES_REQUIRE(fitness_out_dev && theta_dev && obs_dev && target_dev, "%s: NULL pointer", who);
    switch (precision) {
        case DES_FWD_FP32:
            return eval_ffma_launch(fitness_out_dev, theta_dev, obs_dev, target_dev, dims, sigma, clip, seed, generation,
                                    state_dev, member_offset, n_local, nullptr, mirrored, st);
        case DES_FWD_F16:
        case DES_FWD_F16X3:
            return eval_tc_launch(fitness_out_dev, theta_dev, obs_dev, target_dev, dims, sigma, clip, seed, generation,
                                  state_dev, member_offset, n_local, precision, workspace_dev, workspace_bytes, mirrored, st);
        default:
            set_error("%s: unknown precision %d", who, precision);
            return DES_ERR_INVALID_ARGUMENT;
    }
}

}  // namespace des

extern "C" DES_API int des_nes_eval(float *fitness_out_dev, const float *theta_dev, const float *obs_dev, const float *target_dev,
                            des_dims dims, double sigma, double clip, uint64_t seed, uint64_t generation,
                            const des_state *state_dev, int64_t member_offset, int64_t n_local, int precision,
                            void *workspace_dev, size_t workspace_bytes, void *stream) {
    return des::nes_eval("des_nes_eval", fitness_out_dev, theta_dev, obs_dev, target_dev, dims, sigma, clip, seed,
                         generation, state_dev, member_offset, n_local, precision, workspace_dev, workspace_bytes, false,
                         (cudaStream_t)stream);
}

extern "C" DES_API int des_nes_eval_mirrored(float *fitness_out_dev, const float *theta_dev, const float *obs_dev,
                                             const float *target_dev, des_dims dims, double sigma, double clip,
                                             uint64_t seed, uint64_t generation, const des_state *state_dev,
                                             int64_t member_offset, int64_t n_local, int precision, void *workspace_dev,
                                             size_t workspace_bytes, void *stream) {
    return des::nes_eval("des_nes_eval_mirrored", fitness_out_dev, theta_dev, obs_dev, target_dev, dims, sigma, clip,
                         seed, generation, state_dev, member_offset, n_local, precision, workspace_dev, workspace_bytes,
                         true, (cudaStream_t)stream);
}

// ---- host-buffer session --------------------------------------------------------------------------------
struct des_session {
    int device;
    des_dims dims;
    int64_t N, member_offset, n_local, P;
    des_opt opt;
    double clip;
    uint64_t seed;
    int precision;
    cudaStream_t stream;
    float *theta, *obs, *target, *fitness_all, *shaped, *partial, *update;
    double *adam_m, *adam_v;
    des_state *state;
    void *rank_ws, *grad_ws, *eval_ws;
    size_t rank_ws_bytes, grad_ws_bytes, eval_ws_bytes;
};

static void session_free(des_session *s) {
    if (!s) return;
    cudaSetDevice(s->device);
    void *ptrs[] = {s->theta, s->obs, s->target, s->fitness_all, s->shaped, s->partial, s->update,
                    s->adam_m, s->adam_v, s->state, s->rank_ws, s->grad_ws, s->eval_ws};
    for (void *p : ptrs)
        if (p) cudaFree(p);
    if (s->stream) cudaStreamDestroy(s->stream);
    delete s;
}

#define DES_S_CUDA(call)                                   \
    do {                                                   \
        cudaError_t e__ = (call);                          \
        if (e__ != cudaSuccess) {                          \
            int rc__ = ::des::cuda_fail(e__, #call);       \
            session_free(s);                               \
            return rc__;                                   \
        }                                                  \
    } while (0)

extern "C" DES_API int des_session_create(des_session **out, int device, des_dims dims, int64_t N, int64_t member_offset,
                                  int64_t n_local, des_opt opt, double clip, uint64_t seed, int precision,
                                  const float *theta0_host) {
    using namespace des;
    DES_REQUIRE(out, "des_session_create: out is NULL");
    *out = nullptr;
    const int64_t P = des_param_count(dims.state_dim, dims.hidden, dims.action_dim);
    DES_REQUIRE(P > 0 && dims.tape_len > 0, "des_session_create: bad dims");
    DES_REQUIRE(N >= 2 && member_offset >= 0 && n_local >= 0 && member_offset + n_local <= N,
                "des_session_create: bad population split (N=%lld offset=%lld n_local=%lld)", (long long)N,
                (long long)member_offset, (long long)n_local);
    DES_REQUIRE(theta0_host, "des_session_create: theta0_host is NULL");
    DES_REQUIRE(opt.sigma > 0, "des_session_create: sigma must be > 0");
    int ndev = des_device_count();
    if (ndev <= 0) {
        set_error("des_session_create: no CUDA device (there is no CPU fallback)");
        return DES_ERR_NO_DEVICE;
    }
    DES_REQUIRE(device >= 0 && device < ndev, "des_session_create: device %d out of range [0,%d)", device, ndev);
    des_session *s = new (std::nothrow) des_session();
    DES_REQUIRE(s, "des_session_create: out of host memory");
    memset(s, 0, sizeof(*s));
    s->device = device; s->dims = dims; s->N = N; s->member_offset = member_offset; s->n_local = n_local; s->P = P;
    s->opt = opt; s->clip = clip; s->seed = seed; s->precision = precision;
    DES_S_CUDA(cudaSetDevice(device));
    DES_S_CUDA(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    const int T = dims.tape_len;
    DES_S_CUDA(cudaMalloc(&s->theta, P * sizeof(float)));
    DES_S_CUDA(cudaMalloc(&s->obs, (size_t)T * dims.state_dim * sizeof(float)));
    DES_S_CUDA(cudaMalloc(&s->target, (size_t)T * dims.action_dim * sizeof(float)));
    DES_S_CUDA(cudaMalloc(&s->fitness_all, N * sizeof(float)));
    DES_S_CUDA(cudaMalloc(&s->shaped, (n_local > 0 ? n_local : 1) * sizeof(float)));
    DES_S_CUDA(cudaMalloc(&s->partial, P * sizeof(float)));
    DES_S_CUDA(cudaMalloc(&s->update, P * sizeof(float)));
    DES_S_CUDA(cudaMalloc(&s->adam_m, P * sizeof(double)));
    DES_S_CUDA(cudaMalloc(&s->adam_v, P * sizeof(double)));
    DES_S_CUDA(cudaMalloc(&s->state, sizeof(des_state)));
    s->rank_ws_bytes = des_rank_workspace_bytes(N, n_local) + 16;
    s->grad_ws_bytes = des_grad_workspace_bytes(n_local, P) + 16;
    DES_S_CUDA(cudaMalloc(&s->rank_ws, s->rank_ws_bytes));
    DES_S_CUDA(cudaMalloc(&s->grad_ws, s->grad_ws_bytes));
    s->eval_ws_bytes = des_nes_eval_workspace_bytes(dims, precision);
    if (s->eval_ws_bytes) DES_S_CUDA(cudaMalloc(&s->eval_ws, s->eval_ws_bytes));
    DES_S_CUDA(cudaMemsetAsync(s->adam_m, 0, P * sizeof(double), s->stream));
    DES_S_CUDA(cudaMemsetAsync(s->adam_v, 0, P * sizeof(double), s->stream));
    DES_S_CUDA(cudaMemsetAsync(s->fitness_all, 0, N * sizeof(float), s->stream));
    DES_S_CUDA(cudaMemcpyAsync(s->theta, theta0_host, P * sizeof(float), cudaMemcpyHostToDevice, s->stream));
    int rc = des_state_init(s->state, 0, s->stream);
    if (rc != DES_OK) { session_free(s); return rc; }
    DES_S_CUDA(cudaStreamSynchronize(s->stream));
    *out = s;
    return DES_OK;
}

extern "C" DES_API void des_session_destroy(des_session *s) { session_free(s); }

#define DES_SESSION(s)                                                   \
    DES_REQUIRE((s) != nullptr, "%s: session is NULL", __func__);         \
    DES_CUDA(cudaSetDevice((s)->device))

extern "C" DES_API int des_session_upload_tape(des_session *s, const float *obs_host, const float *target_host) {
    DES_SESSION(s);
    DES_REQUIRE(obs_host && target_host, "des_session_upload_tape: NULL pointer");
    const int T = s->dims.tape_len;
    DES_CUDA(cudaMemcpyAsync(s->obs, obs_host, (size_t)T * s->dims.state_dim * sizeof(float), cudaMemcpyHostToDevice, s->stream));
    DES_CUDA(cudaMemcpyAsync(s->target, target_host, (size_t)T * s->dims.action_dim * sizeof(float), cudaMemcpyHostToDevice, s->stream));
    return DES_OK;
}

extern "C" DES_API int des_session_eval(des_session *s) {
    DES_SESSION(s);
    if (s->n_local < s->N) DES_CUDA(cudaMemsetAsync(s->fitness_all, 0, s->N * sizeof(float), s->stream));
    return des_nes_eval(s->fitness_all + s->member_offset, s->theta, s->obs, s->target, s->dims, s->opt.sigma, s->clip,
                        s->seed, 0, s->state, s->member_offset, s->n_local, s->precision, s->eval_ws, s->eval_ws_bytes,
                        s->stream);
}

extern "C" DES_API int des_session_rank_and_grad(des_session *s) {
    DES_SESSION(s);
    int rc = des_centered_rank(s->shaped, nullptr, s->fitness_all, s->N, s->member_offset, s->n_local, s->rank_ws,
                               s->rank_ws_bytes, s->stream);
    if (rc != DES_OK) return rc;
    return des_nes_grad_partial(s->partial, s->shaped, s->n_local, s->P, s->seed, 0, s->state, s->member_offset,
                                s->grad_ws, s->grad_ws_bytes, s->stream);
}

extern "C" DES_API int des_session_apply(des_session *s) {
    DES_SESSION(s);
    int rc = des_nes_apply(s->theta, s->adam_m, s->adam_v, s->update, nullptr, s->partial, s->P, s->N, s->opt, s->state,
                           s->stream);
    if (rc != DES_OK) return rc;
    return des_state_advance(s->state, s->opt.beta1, s->opt.beta2, s->stream);
}

extern "C" DES_API int des_session_generation_host(des_session *s, const float *obs_host, const float *target_host,
                                           const float *theta_in_host, float *fitness_out_host, float *update_out_host,
                                           float *theta_out_host) {
    DES_SESSION(s);
    DES_REQUIRE(s->n_local == s->N && s->member_offset == 0,
                "des_session_generation_host: session holds a shard (%lld of %lld members); drive the phases and the "
                "two collectives explicitly", (long long)s->n_local, (long long)s->N);
    int rc;
    if (obs_host || target_host) {
        rc = des_session_upload_tape(s, obs_host, target_host);
        if (rc != DES_OK) return rc;
    }
    if (theta_in_host)
        DES_CUDA(cudaMemcpyAsync(s->theta, theta_in_host, s->P * sizeof(float), cudaMemcpyHostToDevice, s->stream));
    if ((rc = des_session_eval(s)) != DES_OK) return rc;
    if ((rc = des_session_rank_and_grad(s)) != DES_OK) return rc;
    if ((rc = des_session_apply(s)) != DES_OK) return rc;
    if (fitness_out_host)
        DES_CUDA(cudaMemcpyAsync(fitness_out_host, s->fitness_all, s->N * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
    if (update_out_host)
        DES_CUDA(cudaMemcpyAsync(update_out_host, s->update, s->P * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
    if (theta_out_host)
        DES_CUDA(cudaMemcpyAsync(theta_out_host, s->theta, s->P * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
    DES_CUDA(cudaStreamSynchronize(s->stream));
    return DES_OK;
}

extern "C" DES_API float *des_session_fitness_all_dev(des_session *s) { return s ? s->fitness_all : nullptr; }
extern "C" DES_API float *des_session_partial_dev(des_session *s) { return s ? s->partial : nullptr; }
extern "C" DES_API float *des_session_theta_dev(des_session *s) { return s ? s->theta : nullptr; }
extern "C" DES_API void *des_session_stream(des_session *s) { return s ? (void *)s->stream : nullptr; }
extern "C" DES_API int des_session_sync(des_session *s) {
    DES_SESSION(s);
    DES_CUDA(cudaStreamSynchronize(s->stream));
    return DES_OK;
}
