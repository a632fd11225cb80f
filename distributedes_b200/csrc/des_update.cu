// Fitness x noise reduction and the parameter update.
//
//   des_nes_grad_partial   partial[j] = sum_{i in shard} s_i * eps_ij        natural_es.py:91 (per shard)
//   des_nes_apply          g = (sum/N)/sigma; g -= wd*g; Adam; theta += lr*fp32(step)   natural_es.py:92-96,
//                                                                                utils.py:159-166
//   des_state_init/advance generation / Adam-step counters kept on the device (graph replay)
//
// The reduction never reads eps from memory: every thread owns one quad of parameters (4 consecutive j)
// and a contiguous slice of members, regenerates the quad's four normals per member from the counter
// RNG and FMAs them with the member's shaped fitness.  Work = one Philox4x32-7 + two Box-Muller per
// 4 products: the kernel is ALU/MUFU bound, HBM traffic is O(n_local + C*P).
// Under the materialised-noise contract of SURVEY §8d it stands for reading 4*n_local*P bytes.
#include "des_common.cuh"

namespace des {

#ifndef DES_GRAD_THREADS
#define DES_GRAD_THREADS 128
#endif
constexpr int kGradThreads = DES_GRAD_THREADS;
// members per trip of the inner loop: 1: 3.01 ms, 2: 2.92, 4: 2.78, 8: 2.78 (pop 65 536, P = 73 220; 32 registers throughout)
#ifndef DES_GRAD_UNROLL
#define DES_GRAD_UNROLL 4
#endif
constexpr int kGradUnroll = DES_GRAD_UNROLL;

struct GradPlan {
    int64_t nq;        // quads = ceil(P/4)
    int64_t Ppad;      // 4*nq
    int chunks;        // member slices (grid.y)
    int64_t per_chunk; // members per slice
};

__host__ inline GradPlan grad_plan(int64_t n_local, int64_t P) {
    GradPlan p;
    p.nq = (P + 3) / 4;
    p.Ppad = 4 * p.nq;
    const int64_t bx = (p.nq + kGradThreads - 1) / kGradThreads;
    // ~16 resident CTAs of 128 threads per SM, a few waves; keep slices >= 32 members so that the
    // per-thread fp32 running sum stays short (<= 1024 terms) and the setup cost is amortised.
    int64_t want = (132 * 16 * 2 + bx - 1) / bx;     // 132 SMs (H100 SXM)
    int64_t max_chunks = (n_local + 31) / 32;
    int64_t min_chunks = (n_local + 1023) / 1024;
    if (want > max_chunks) want = max_chunks;
    if (want < min_chunks) want = min_chunks;
    if (want < 1) want = 1;
    if (want > 65535) want = 65535;
    p.per_chunk = (n_local + want - 1) / want;
    p.chunks = (int)((n_local + p.per_chunk - 1) / p.per_chunk);
    if (p.chunks < 1) p.chunks = 1;
    return p;
}

// Quad q of slice blockIdx.y of a shard: ws[blockIdx.y][4q..4q+3] = sum over the slice's members i of s_i * eps_i.
// kMirror: i runs over the n_local pairs of a mirrored shard, member_offset is the pair index of its first pair, and
// pair i contributes (s_2i - s_2i+1) * eps_i: sum_m s_m eps_m with eps_2i+1 = -eps_2i, half the normals to regenerate.
// member_offset is taken by reference: passed by value, ptxas scheduled grad_chunk_kernel<false, true>'s loop differently
// from the kernel it was before this body moved here.
template <bool kMirror>
__device__ __forceinline__ void grad_chunk(float *__restrict__ ws, const float *__restrict__ shaped, int64_t n_local,
                                           int64_t q, int64_t Ppad, int64_t per_chunk, const PhiloxKey &key, uint32_t gen,
                                           const uint64_t &member_offset) {   // a reference: see below
    const int64_t i0 = (int64_t)blockIdx.y * per_chunk;
    const int64_t i1 = min(n_local, i0 + per_chunk);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll kGradUnroll
    for (int64_t i = i0; i < i1; ++i) {
        // warp-uniform broadcast loads
        const float s = kMirror ? __fsub_rn(__ldg(shaped + 2 * i), __ldg(shaped + 2 * i + 1)) : __ldg(shaped + i);
        const uint4 x = philox4x32((uint32_t)q, (uint32_t)(member_offset + i), gen, kStreamNesEps, key);
        const BmParts a = box_muller_parts(x.x, x.y, kNeg2Ln2, key.one_bits);
        const BmParts b = box_muller_parts(x.z, x.w, kNeg2Ln2, key.one_bits);
        const float as = a.nr * s, bs = b.nr * s;                 // s_i * radius: one multiply per pair
        acc.x = __fmaf_rn(as, a.c, acc.x);
        acc.y = __fmaf_rn(as, a.s, acc.y);
        acc.z = __fmaf_rn(bs, b.c, acc.z);
        acc.w = __fmaf_rn(bs, b.s, acc.w);
    }
    *reinterpret_cast<float4 *>(ws + (int64_t)blockIdx.y * Ppad + 4 * q) = acc;
}

// kRuns: CTA row z takes run z of a batch (des_nes_grad_partial_runs), a shard of n_local members at member_offset +
// z * n_local whose gridDim.y slices have their own rows of ws.
template <bool kMirror, bool kRuns>
__global__ void __launch_bounds__(kGradThreads) grad_chunk_kernel(float *__restrict__ ws, const float *__restrict__ shaped,
                                                                   int64_t n_local, int64_t nq, int64_t Ppad,
                                                                   int64_t per_chunk, PhiloxKey key,
                                                                   uint32_t gen_arg, const des_state *state,
                                                                   uint64_t member_offset) {
    const int64_t q = (int64_t)blockIdx.x * kGradThreads + threadIdx.x;
    if (q >= nq) return;
    if constexpr (kRuns) {
        ws += (int64_t)blockIdx.z * gridDim.y * Ppad;
        shaped += (int64_t)blockIdx.z * n_local;
        member_offset += (uint64_t)blockIdx.z * n_local;
    }
    const uint32_t gen = generation_word(state, gen_arg);
    grad_chunk<kMirror>(ws, shaped, n_local, q, Ppad, per_chunk, key, gen, member_offset);
}

// A sweep (des_nes_grad_partial_sweep): CTA row z takes run z, a standalone shard of n_local members (member_offset 0)
// under its own seed hp[z].seed, with grad_chunk_kernel<false, true>'s ws rows.  The round keys live in registers, set
// up from the seed; `one` is PhiloxKey::one_bits, a parameter so that it stays a register operand.
__global__ void __launch_bounds__(kGradThreads) grad_chunk_sweep_kernel(float *__restrict__ ws,
                                                                         const float *__restrict__ shaped, int64_t n_local,
                                                                         int64_t nq, int64_t Ppad, int64_t per_chunk,
                                                                         const des_run_hp *__restrict__ hp, uint32_t one,
                                                                         uint32_t gen_arg, const des_state *state) {
    const int64_t q = (int64_t)blockIdx.x * kGradThreads + threadIdx.x;
    if (q >= nq) return;
    ws += (int64_t)blockIdx.z * gridDim.y * Ppad;
    shaped += (int64_t)blockIdx.z * n_local;
    PhiloxKey key;
    philox_round_keys(hp[blockIdx.z].seed, key);
    key.one_bits = one;
    grad_chunk<false>(ws, shaped, n_local, q, Ppad, per_chunk, key, generation_word(state, gen_arg), 0);
}

// partial[j] = fp32( sum_c ws[c][j] ) with the cross-chunk sum in fp64, fixed order (deterministic): a CTA of 32 x 8
// threads takes 32 columns; row y adds chunks y, y+8, ... in order, then row 0 adds the eight row sums in order.
// (One thread per column walking all chunks serially took 13 us at P = 6020 / 128 chunks: 24 CTAs of dependent loads.)
constexpr int kReduceRows = 8;
__device__ __forceinline__ void grad_reduce(float *__restrict__ partial, const float *__restrict__ ws, int64_t P,
                                            int64_t Ppad, int chunks) {
    __shared__ double rows[kReduceRows][33];
    const int x = threadIdx.x, y = threadIdx.y;
    const int64_t j = (int64_t)blockIdx.x * 32 + x;
    double s = 0.0;
    if (j < P)
        for (int c = y; c < chunks; c += kReduceRows) s += (double)__ldg(ws + (int64_t)c * Ppad + j);
    rows[y][x] = s;
    __syncthreads();
    if (y == 0 && j < P) {
        double t = rows[0][x];
#pragma unroll
        for (int r = 1; r < kReduceRows; ++r) t += rows[r][x];
        partial[j] = (float)t;
    }
}

__global__ void __launch_bounds__(32 * kReduceRows) grad_reduce_kernel(float *__restrict__ partial, const float *__restrict__ ws,
                                                                       int64_t P, int64_t Ppad, int chunks) {
    grad_reduce(partial, ws, P, Ppad, chunks);
}

// run r: partial[r][P] from its `chunks` rows of ws; runs along y, strided past 65535
__global__ void __launch_bounds__(32 * kReduceRows) grad_reduce_runs_kernel(float *__restrict__ partial,
                                                                            const float *__restrict__ ws, int64_t n_runs,
                                                                            int64_t P, int64_t Ppad, int chunks) {
    for (int64_t r = blockIdx.y; r < n_runs; r += gridDim.y) {
        grad_reduce(partial + r * P, ws + r * chunks * Ppad, P, Ppad, chunks);
        __syncthreads();                 // the shared row sums are reused by the next run
    }
}

// parameter j of one population
__device__ __forceinline__ void apply_at(int64_t j, float *__restrict__ theta, double *__restrict__ am,
                                         double *__restrict__ av, float *__restrict__ update_out,
                                         double *__restrict__ grad_out, const float *__restrict__ partial, int64_t N,
                                         const des_opt &o, const des_state *__restrict__ state) {
    // utils.py:160-161: beta_t *= beta happens before use, so this step uses beta^(t+1)
    const double b1t = state->beta1_t * o.beta1;
    const double b2t = state->beta2_t * o.beta2;
    // natural_es.py:92: np.mean(gradient, 0) / sigma
    double g = ((double)partial[j] / (double)N) / o.sigma;
    if (grad_out) grad_out[j] = g;
    g -= o.weight_decay * g;                                   // natural_es.py:93
    const double m = o.beta1 * am[j] + (1.0 - o.beta1) * g;   // utils.py:162
    const double v = o.beta2 * av[j] + (1.0 - o.beta2) * (g * g);
    am[j] = m;
    av[j] = v;
    const double m_ = m / (1.0 - b1t);                          // utils.py:164-165
    const double v_ = v / (1.0 - b2t);
    const double step = m_ / (sqrt(v_) + o.epsilon);            // utils.py:166
    const float step32 = (float)step;                           // natural_es.py:95 torch.FloatTensor(gradient)
    const float upd = __fmul_rn((float)o.learning_rate, step32);   // :96 lr * gradient (fp32 tensor op)
    if (update_out) update_out[j] = upd;
    theta[j] = __fadd_rn(theta[j], upd);                        // :96 param.add_
}

__global__ void apply_kernel(float *__restrict__ theta, double *__restrict__ am, double *__restrict__ av,
                             float *__restrict__ update_out, double *__restrict__ grad_out,
                             const float *__restrict__ partial, int64_t P, double inv_n_unused, int64_t N, des_opt o,
                             const des_state *__restrict__ state) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= P) return;
    apply_at(j, theta, am, av, update_out, grad_out, partial, N, o, state);
}

// run r's rows of every [n_runs][P] argument; runs along y, strided past 65535
__global__ void apply_runs_kernel(float *__restrict__ theta, double *__restrict__ am, double *__restrict__ av,
                                  float *__restrict__ update_out, double *__restrict__ grad_out,
                                  const float *__restrict__ partial, int64_t P, int64_t n_runs, int64_t N, des_opt o,
                                  const des_state *__restrict__ state) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= P) return;
    for (int64_t r = blockIdx.y; r < n_runs; r += gridDim.y) {
        const int64_t o_r = r * P;
        apply_at(j, theta + o_r, am + o_r, av + o_r, update_out ? update_out + o_r : nullptr,
                 grad_out ? grad_out + o_r : nullptr, partial + o_r, N, o, state);
    }
}

// run r's rows of every [n_runs][P] argument, with the optimiser of run r's row of the table and the shared beta / epsilon
__global__ void apply_sweep_kernel(float *__restrict__ theta, double *__restrict__ am, double *__restrict__ av,
                                   float *__restrict__ update_out, double *__restrict__ grad_out,
                                   const float *__restrict__ partial, int64_t P, int64_t n_runs, int64_t N,
                                   const des_run_hp *__restrict__ hp, double beta1, double beta2, double epsilon,
                                   const des_state *__restrict__ state) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= P) return;
    for (int64_t r = blockIdx.y; r < n_runs; r += gridDim.y) {
        const int64_t o_r = r * P;
        const des_opt o = {hp[r].sigma, hp[r].learning_rate, hp[r].weight_decay, beta1, beta2, epsilon};
        apply_at(j, theta + o_r, am + o_r, av + o_r, update_out ? update_out + o_r : nullptr,
                 grad_out ? grad_out + o_r : nullptr, partial + o_r, N, o, state);
    }
}

__global__ void state_init_kernel(des_state *st, uint64_t generation) {
    st->generation = generation;
    st->adam_t = 0;
    st->beta1_t = 1.0;
    st->beta2_t = 1.0;
}

__global__ void state_advance_kernel(des_state *st, double beta1, double beta2) {
    st->generation += 1;
    st->adam_t += 1;
    st->beta1_t *= beta1;   // utils.py:160
    st->beta2_t *= beta2;   // utils.py:161
}

}  // namespace des

extern "C" DES_API size_t des_grad_workspace_bytes(int64_t n_local, int64_t P) {
    if (n_local <= 0 || P <= 0) return 0;
    const des::GradPlan p = des::grad_plan(n_local, P);
    return (size_t)p.chunks * (size_t)p.Ppad * sizeof(float);
}

namespace des {

// Shared by both entry points.  Mirrored shards are planned by pairs: the slices of the plain plan of n_local members,
// each holding half as many pairs, so the mirrored call never needs more slices (nor workspace) than the plain one.
static int grad_partial(const char *who, float *partial_out_dev, const float *shaped_local_dev, int64_t n_local, int64_t P,
                        uint64_t seed, uint64_t generation, const des_state *state_dev, int64_t member_offset,
                        void *workspace_dev, size_t workspace_bytes, bool mirrored, cudaStream_t st) {
    DES_REQUIRE(n_local >= 0 && P > 0, "%s: bad sizes n_local=%lld P=%lld", who, (long long)n_local, (long long)P);
    DES_REQUIRE(partial_out_dev, "%s: partial_out_dev is NULL", who);
    DES_REQUIRE(member_range_ok(member_offset, n_local, 32), "%s: member index must fit 32 bits", who);
    if (mirrored && !whole_pairs(member_offset, n_local)) return not_whole_pairs(who, "n_local", member_offset, n_local);
    if (n_local == 0) {
        DES_CUDA(cudaMemsetAsync(partial_out_dev, 0, (size_t)P * sizeof(float), st));
        return DES_OK;
    }
    DES_REQUIRE(shaped_local_dev, "%s: shaped_local_dev is NULL", who);
    const GradPlan p = grad_plan(n_local, P);
    const size_t need = (size_t)p.chunks * (size_t)p.Ppad * sizeof(float);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    DES_REQUIRE(((uintptr_t)workspace_dev & 15) == 0, "%s: workspace must be 16-byte aligned", who);
    float *ws = (float *)workspace_dev;
    const unsigned bx = (unsigned)((p.nq + kGradThreads - 1) / kGradThreads);
    const PhiloxKey key = make_philox_key(seed);
    int chunks = p.chunks;
    if (mirrored) {
        const int64_t pairs = n_local / 2, per_chunk = (p.per_chunk + 1) / 2;
        chunks = (int)((pairs + per_chunk - 1) / per_chunk);     // <= p.chunks
        grad_chunk_kernel<true, false><<<dim3(bx, (unsigned)chunks), kGradThreads, 0, st>>>(
            ws, shaped_local_dev, pairs, p.nq, p.Ppad, per_chunk, key, (uint32_t)generation, state_dev,
            (uint64_t)member_offset / 2);
    } else {
        grad_chunk_kernel<false, false><<<dim3(bx, (unsigned)chunks), kGradThreads, 0, st>>>(
            ws, shaped_local_dev, n_local, p.nq, p.Ppad, p.per_chunk, key, (uint32_t)generation, state_dev,
            (uint64_t)member_offset);
    }
    DES_LAUNCH_CHECK("grad_chunk_kernel");
    grad_reduce_kernel<<<(unsigned)((P + 31) / 32), dim3(32, kReduceRows), 0, st>>>(partial_out_dev, ws, P, p.Ppad, chunks);
    DES_LAUNCH_CHECK("grad_reduce_kernel");
    return DES_OK;
}

}  // namespace des

extern "C" DES_API int des_nes_grad_partial(float *partial_out_dev, const float *shaped_local_dev, int64_t n_local, int64_t P,
                                    uint64_t seed, uint64_t generation, const des_state *state_dev,
                                    int64_t member_offset, void *workspace_dev, size_t workspace_bytes, void *stream) {
    return des::grad_partial("des_nes_grad_partial", partial_out_dev, shaped_local_dev, n_local, P, seed, generation,
                             state_dev, member_offset, workspace_dev, workspace_bytes, false, (cudaStream_t)stream);
}

extern "C" DES_API int des_nes_grad_partial_mirrored(float *partial_out_dev, const float *shaped_local_dev, int64_t n_local,
                                                     int64_t P, uint64_t seed, uint64_t generation,
                                                     const des_state *state_dev, int64_t member_offset, void *workspace_dev,
                                                     size_t workspace_bytes, void *stream) {
    return des::grad_partial("des_nes_grad_partial_mirrored", partial_out_dev, shaped_local_dev, n_local, P, seed,
                             generation, state_dev, member_offset, workspace_dev, workspace_bytes, true,
                             (cudaStream_t)stream);
}

extern "C" DES_API int des_nes_apply(float *theta_dev, double *adam_m_dev, double *adam_v_dev, float *update_out_dev,
                             double *grad_out_dev, const float *partial_sum_dev, int64_t P, int64_t N, des_opt opt,
                             const des_state *state_dev, void *stream) {
    using namespace des;
    DES_REQUIRE(P > 0 && N >= 1, "des_nes_apply: bad sizes P=%lld N=%lld", (long long)P, (long long)N);
    DES_REQUIRE(theta_dev && adam_m_dev && adam_v_dev && partial_sum_dev && state_dev, "des_nes_apply: NULL pointer");
    DES_REQUIRE(opt.sigma > 0.0, "des_nes_apply: sigma must be > 0 (natural_es.py:92 divides by it)");
    apply_kernel<<<(unsigned)((P + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        theta_dev, adam_m_dev, adam_v_dev, update_out_dev, grad_out_dev, partial_sum_dev, P, 0.0, N, opt, state_dev);
    DES_LAUNCH_CHECK("apply_kernel");
    return DES_OK;
}

extern "C" DES_API int des_state_init(des_state *state_dev, uint64_t generation, void *stream) {
    DES_REQUIRE(state_dev, "des_state_init: state_dev is NULL");
    des::state_init_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state_dev, generation);
    DES_LAUNCH_CHECK("state_init_kernel");
    return DES_OK;
}

extern "C" DES_API int des_state_advance(des_state *state_dev, double beta1, double beta2, void *stream) {
    DES_REQUIRE(state_dev, "des_state_advance: state_dev is NULL");
    des::state_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state_dev, beta1, beta2);
    DES_LAUNCH_CHECK("state_advance_kernel");
    return DES_OK;
}

extern "C" DES_API size_t des_grad_runs_workspace_bytes(int64_t n_runs, int64_t run_size, int64_t P) {
    if (n_runs <= 0 || run_size <= 0 || P <= 0 || run_size > des::kRunMaxSize || n_runs > ((int64_t)1 << 28) / run_size)
        return 0;
    return (size_t)n_runs * des_grad_workspace_bytes(run_size, P);
}

extern "C" DES_API int des_nes_grad_partial_runs(float *partial_out_dev, const float *shaped_dev, int64_t n_runs,
                                                 int64_t run_size, int64_t P, uint64_t seed, uint64_t generation,
                                                 const des_state *state_dev, void *workspace_dev, size_t workspace_bytes,
                                                 void *stream) {
    using namespace des;
    const char *who = "des_nes_grad_partial_runs";
    const int rc = check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(P > 0, "%s: bad size P=%lld", who, (long long)P);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(partial_out_dev && shaped_dev, "%s: NULL pointer", who);
    const GradPlan p = grad_plan(run_size, P);           // each run sliced as a shard of run_size members
    const size_t need = des_grad_runs_workspace_bytes(n_runs, run_size, P);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    DES_REQUIRE(((uintptr_t)workspace_dev & 15) == 0, "%s: workspace must be 16-byte aligned", who);
    cudaStream_t st = (cudaStream_t)stream;
    float *ws = (float *)workspace_dev;
    const unsigned bx = (unsigned)((p.nq + kGradThreads - 1) / kGradThreads);
    const PhiloxKey key = make_philox_key(seed);
    for (int64_t r0 = 0; r0 < n_runs; r0 += 65535) {            // grid z: up to 65535 runs per launch
        const int64_t nr = n_runs - r0 < 65535 ? n_runs - r0 : 65535;
        grad_chunk_kernel<false, true><<<dim3(bx, (unsigned)p.chunks, (unsigned)nr), kGradThreads, 0, st>>>(
            ws + r0 * p.chunks * p.Ppad, shaped_dev + r0 * run_size, run_size, p.nq, p.Ppad, p.per_chunk, key,
            (uint32_t)generation, state_dev, (uint64_t)(r0 * run_size));
        DES_LAUNCH_CHECK("grad_chunk_kernel");
    }
    const unsigned bz = (unsigned)(n_runs < 65535 ? n_runs : 65535);
    grad_reduce_runs_kernel<<<dim3((unsigned)((P + 31) / 32), bz), dim3(32, kReduceRows), 0, st>>>(partial_out_dev, ws,
                                                                                                 n_runs, P, p.Ppad, p.chunks);
    DES_LAUNCH_CHECK("grad_reduce_runs_kernel");
    return DES_OK;
}

extern "C" DES_API int des_nes_apply_runs(float *theta_dev, double *adam_m_dev, double *adam_v_dev, float *update_out_dev,
                                          double *grad_out_dev, const float *partial_sum_dev, int64_t P, int64_t n_runs,
                                          int64_t run_size, des_opt opt, const des_state *state_dev, void *stream) {
    using namespace des;
    const char *who = "des_nes_apply_runs";
    const int rc = check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(P > 0, "%s: bad size P=%lld", who, (long long)P);
    DES_REQUIRE(opt.sigma > 0.0, "%s: sigma must be > 0 (natural_es.py:92 divides by it)", who);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(theta_dev && adam_m_dev && adam_v_dev && partial_sum_dev && state_dev, "%s: NULL pointer", who);
    const unsigned by = (unsigned)(n_runs < 65535 ? n_runs : 65535);
    apply_runs_kernel<<<dim3((unsigned)((P + 255) / 256), by), 256, 0, (cudaStream_t)stream>>>(
        theta_dev, adam_m_dev, adam_v_dev, update_out_dev, grad_out_dev, partial_sum_dev, P, n_runs, run_size, opt,
        state_dev);
    DES_LAUNCH_CHECK("apply_runs_kernel");
    return DES_OK;
}

extern "C" DES_API int des_nes_grad_partial_sweep(float *partial_out_dev, const float *shaped_dev, int64_t n_runs,
                                                  int64_t run_size, int64_t P, const des_run_hp *hp_dev, uint64_t generation,
                                                  const des_state *state_dev, void *workspace_dev, size_t workspace_bytes,
                                                  void *stream) {
    using namespace des;
    const char *who = "des_nes_grad_partial_sweep";
    const int rc = check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(P > 0, "%s: bad size P=%lld", who, (long long)P);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(partial_out_dev && shaped_dev && hp_dev, "%s: NULL pointer", who);
    const GradPlan p = grad_plan(run_size, P);           // each run sliced as a shard of run_size members
    const size_t need = des_grad_runs_workspace_bytes(n_runs, run_size, P);
    if (!workspace_dev || workspace_bytes < need) {
        set_error("%s: workspace %zu B < required %zu B", who, workspace_bytes, need);
        return DES_ERR_WORKSPACE;
    }
    DES_REQUIRE(((uintptr_t)workspace_dev & 15) == 0, "%s: workspace must be 16-byte aligned", who);
    cudaStream_t st = (cudaStream_t)stream;
    float *ws = (float *)workspace_dev;
    const unsigned bx = (unsigned)((p.nq + kGradThreads - 1) / kGradThreads);
    const uint32_t one = make_philox_key(0).one_bits;
    for (int64_t r0 = 0; r0 < n_runs; r0 += 65535) {            // grid z: up to 65535 runs per launch
        const int64_t nr = n_runs - r0 < 65535 ? n_runs - r0 : 65535;
        grad_chunk_sweep_kernel<<<dim3(bx, (unsigned)p.chunks, (unsigned)nr), kGradThreads, 0, st>>>(
            ws + r0 * p.chunks * p.Ppad, shaped_dev + r0 * run_size, run_size, p.nq, p.Ppad, p.per_chunk, hp_dev + r0, one,
            (uint32_t)generation, state_dev);
        DES_LAUNCH_CHECK("grad_chunk_sweep_kernel");
    }
    const unsigned bz = (unsigned)(n_runs < 65535 ? n_runs : 65535);
    grad_reduce_runs_kernel<<<dim3((unsigned)((P + 31) / 32), bz), dim3(32, kReduceRows), 0, st>>>(partial_out_dev, ws,
                                                                                                 n_runs, P, p.Ppad, p.chunks);
    DES_LAUNCH_CHECK("grad_reduce_runs_kernel");
    return DES_OK;
}

extern "C" DES_API int des_nes_apply_sweep(float *theta_dev, double *adam_m_dev, double *adam_v_dev, float *update_out_dev,
                                           double *grad_out_dev, const float *partial_sum_dev, int64_t P, int64_t n_runs,
                                           int64_t run_size, const des_run_hp *hp_dev, double beta1, double beta2,
                                           double epsilon, const des_state *state_dev, void *stream) {
    using namespace des;
    const char *who = "des_nes_apply_sweep";
    const int rc = check_runs(who, n_runs, run_size, 1);
    if (rc != DES_OK) return rc;
    DES_REQUIRE(P > 0, "%s: bad size P=%lld", who, (long long)P);
    if (n_runs == 0) return DES_OK;
    DES_REQUIRE(theta_dev && adam_m_dev && adam_v_dev && partial_sum_dev && hp_dev && state_dev, "%s: NULL pointer", who);
    const unsigned by = (unsigned)(n_runs < 65535 ? n_runs : 65535);
    apply_sweep_kernel<<<dim3((unsigned)((P + 255) / 256), by), 256, 0, (cudaStream_t)stream>>>(
        theta_dev, adam_m_dev, adam_v_dev, update_out_dev, grad_out_dev, partial_sum_dev, P, n_runs, run_size, hp_dev,
        beta1, beta2, epsilon, state_dev);
    DES_LAUNCH_CHECK("apply_sweep_kernel");
    return DES_OK;
}
