// des_nes_eval, precision DES_FWD_FP32: fused sample + perturb + forward + fitness on CUDA cores.
//
// One CTA per population member (Worker.run natural_es.py:27-32 for that member):
//   for each tile of 64 observations of the tape
//     layer 1..3 of StandardFCNet.forward (model.py:34-39), output features in chunks of 32 rows;
//     the chunk's perturbed weights  fp32(theta + sigma*eps)  (natural_es.py:28-30) are generated
//     straight into shared memory from the counter RNG — theta' never exists in HBM;
//     fitness += -|| clip(a_t) - a*_t ||^2   (utils.py:134-137 over the tape env)
// fp32 FFMA everywhere, accurate tanhf: this is the parity-grade path and supports any (d0, H, A, T).
// Bound: CUDA-core FMA issue (2*T*(d0*H+H*H+H*A) flop per member) + RNG regeneration per obs tile.
#include "des_common.cuh"

namespace des {

constexpr int kTileT = 64;    // observations per tile
constexpr int kRows = 32;     // weight rows (output features) staged per chunk
constexpr int kThreads = 256; // 8 warps; warp w owns observations [8w, 8w+8) of the tile
constexpr int kObsPerWarp = kTileT / (kThreads / 32);

struct EvalArgs {
    float *fitness;
    const float *theta, *obs, *target;
    const float *solutions;   // FROM_MATRIX: [n_local][P] explicit weight vectors (cma_es.py:63-64 ships solutions), else NULL
    const des_state *state;
    Layout L;
    int T;
    int S;            // shared row stride in floats ((S/4) odd -> conflict-free float4 rows)
    float sigma, clip;
    PhiloxKey key;
    uint32_t gen;
    uint64_t member_offset;
    int mirrored;     // member m perturbs with (-1)^(m & 1) * eps of counter word m >> 1
};

__device__ __forceinline__ int round_up4(int x) { return (x + 3) & ~3; }

// Generate theta'[off, off+cnt) into dst laid out as rows of K (row stride S); zero the K..Kp pad.
// FROM_MATRIX: copy the member's explicit solution instead of perturbing theta.
template <bool FROM_MATRIX>
__device__ __forceinline__ void gen_rows(float *__restrict__ dst, const float *__restrict__ theta, int off, int R,
                                         int K, int Kp, int S, float sigma, uint32_t member, uint32_t gen,
                                         const PhiloxKey &key) {
    const int cnt = R * K;
    if (FROM_MATRIX) {
        for (int i = threadIdx.x; i < cnt; i += kThreads) dst[(i / K) * S + (i % K)] = __ldg(theta + off + i);
    } else {
    const int qa = off >> 2, qb = (off + cnt - 1) >> 2;
    for (int q = qa + (int)threadIdx.x; q <= qb; q += kThreads) {
        const float4 z = noise_quad((uint32_t)q, member, gen, kStreamNesEps, key);
        const float zz[4] = {z.x, z.y, z.z, z.w};
        int local = 4 * q - off;
        int r = (local >= 0) ? local / K : 0;
        int k = (local >= 0) ? local - r * K : 0;
#pragma unroll
        for (int e = 0; e < 4; ++e, ++local) {
            if (local >= 0 && local < cnt) {
                dst[r * S + k] = __fmaf_rn(sigma, zz[e], __ldg(theta + off + local));
                if (++k == K) { k = 0; ++r; }
            }
        }
    }
    }
    if (Kp > K) {
        const int pad = Kp - K;
        for (int i = threadIdx.x; i < kRows * pad; i += kThreads) dst[(i / pad) * S + K + (i % pad)] = 0.f;
    }
    // rows R..kRows-1 are never read with a live lane (guarded by n < Nout) but must stay finite
    for (int i = R * Kp + threadIdx.x; i < kRows * Kp; i += kThreads) dst[(i / Kp) * S + (i % Kp)] = 0.f;
}

template <bool FROM_MATRIX>
__global__ void __launch_bounds__(kThreads) eval_ffma_kernel(EvalArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int S = a.S;
    float *actA = smem;                     // [kTileT][S]
    float *actB = actA + kTileT * S;        // [kTileT][S]
    float *Ws = actB + kTileT * S;          // [kRows][S]
    float *bias = Ws + kRows * S;           // [kRows]
    __shared__ double warp_sums[kThreads / 32];

    const Layout L = a.L;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t gen = generation_word(a.state, a.gen);
    const uint64_t gm = a.member_offset + blockIdx.x;
    const uint32_t member = noise_word(gm, a.mirrored);
    const float sigma = member_sigma(gm, a.mirrored, a.sigma);
    const float *wsrc = FROM_MATRIX ? a.solutions + (int64_t)blockIdx.x * L.P : a.theta;
    double fit = 0.0;                       // meaningful in thread 0 only

    for (int t0 = 0; t0 < a.T; t0 += kTileT) {
        // observations -> actA (zero padded rows/cols)
        const int K0p = round_up4(L.d0);
        for (int i = threadIdx.x; i < kTileT * K0p; i += kThreads) {
            const int t = i / K0p, k = i - t * K0p;
            actA[t * S + k] = (t0 + t < a.T && k < L.d0) ? __ldg(a.obs + (int64_t)(t0 + t) * L.d0 + k) : 0.f;
        }
        float sq = 0.f;
        float *in = actA, *out = actB;
#pragma unroll 1
        for (int layer = 0; layer < 3; ++layer) {
            const int K = layer == 0 ? L.d0 : L.H;
            const int Kp = round_up4(K);
            const int Nout = layer == 2 ? L.A : L.H;
            const int off_w = layer == 0 ? L.off_w1 : (layer == 1 ? L.off_w2 : L.off_w3);
            const int off_b = layer == 0 ? L.off_b1 : (layer == 1 ? L.off_b2 : L.off_b3);
            const int Np = round_up4(Nout);
#pragma unroll 1
            for (int n0 = 0; n0 < Np; n0 += kRows) {
                const int R = min(kRows, Nout - n0);
                __syncthreads();            // previous chunk's readers of Ws/bias (and obs load) done
                if (R > 0) {
                    gen_rows<FROM_MATRIX>(Ws, wsrc, off_w + n0 * K, R, K, Kp, S, sigma, member, gen, a.key);
                    // biases of the chunk: off_b + n0 .. + R
                    const int ob = off_b + n0;
                    if (FROM_MATRIX) {
                        for (int i = threadIdx.x; i < R; i += kThreads) bias[i] = __ldg(wsrc + ob + i);
                    } else {
                        const int qa = ob >> 2, qb = (ob + R - 1) >> 2;
                        for (int q = qa + (int)threadIdx.x; q <= qb; q += kThreads) {
                            const float4 z = noise_quad((uint32_t)q, member, gen, kStreamNesEps, a.key);
                            const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const int local = 4 * q + e - ob;
                                if (local >= 0 && local < R)
                                    bias[local] = __fmaf_rn(sigma, zz[e], __ldg(a.theta + ob + local));
                            }
                        }
                    }
                }
                __syncthreads();
                float acc[kObsPerWarp];
#pragma unroll
                for (int t = 0; t < kObsPerWarp; ++t) acc[t] = 0.f;
                const float *wrow = Ws + lane * S;
                const float *arow = in + (warp * kObsPerWarp) * S;
                for (int k = 0; k < Kp; k += 4) {
                    const float4 w = *reinterpret_cast<const float4 *>(wrow + k);
#pragma unroll
                    for (int t = 0; t < kObsPerWarp; ++t) {
                        const float4 x = *reinterpret_cast<const float4 *>(arow + t * S + k);
                        acc[t] = __fmaf_rn(x.x, w.x, acc[t]);
                        acc[t] = __fmaf_rn(x.y, w.y, acc[t]);
                        acc[t] = __fmaf_rn(x.z, w.z, acc[t]);
                        acc[t] = __fmaf_rn(x.w, w.w, acc[t]);
                    }
                }
                const int n = n0 + lane;
                if (layer < 2) {
                    if (n < Np) {
                        const float b = (n < Nout) ? bias[lane] : 0.f;
#pragma unroll
                        for (int t = 0; t < kObsPerWarp; ++t)
                            out[(warp * kObsPerWarp + t) * S + n] = (n < Nout) ? tanhf(acc[t] + b) : 0.f;
                    }
                } else if (n < Nout) {
                    const float b = bias[lane];
#pragma unroll
                    for (int t = 0; t < kObsPerWarp; ++t) {
                        const int tt = t0 + warp * kObsPerWarp + t;
                        if (tt < a.T) {
                            float v = acc[t] + b;
                            v = clip_keep_nan(v, a.clip);          // np.clip, config.py:29,37
                            const float d = v - __ldg(a.target + (int64_t)tt * L.A + n);
                            sq = __fmaf_rn(d, d, sq);
                        }
                    }
                }
            }
            float *tmp = in; in = out; out = tmp;
        }
        // deterministic block reduction of the tile's squared error
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
        __syncthreads();                    // warp_sums free; all chunk work of this tile done
        if (lane == 0) warp_sums[warp] = (double)sq;
        __syncthreads();
        if (threadIdx.x == 0) {
#pragma unroll
            for (int w = 0; w < kThreads / 32; ++w) fit += warp_sums[w];
        }
    }
    if (threadIdx.x == 0) a.fitness[blockIdx.x] = (float)(-fit);
}

int eval_ffma_launch(float *fitness, const float *theta, const float *obs, const float *target, des_dims dims,
                     double sigma, double clip, uint64_t seed, uint64_t generation, const des_state *state,
                     int64_t member_offset, int64_t n_local, const float *solutions, bool mirrored, cudaStream_t st) {
    EvalArgs a;
    a.solutions = solutions;
    a.mirrored = mirrored ? 1 : 0;
    a.fitness = fitness; a.theta = theta; a.obs = obs; a.target = target; a.state = state;
    a.L = Layout(dims.state_dim, dims.hidden, dims.action_dim);
    a.T = dims.tape_len;
    int kmax = dims.hidden > dims.state_dim ? dims.hidden : dims.state_dim;
    int S = ((kmax + 3) & ~3) + 4;
    if (((S >> 2) & 1) == 0) S += 4;
    a.S = S;
    a.sigma = (float)sigma; a.clip = (float)clip;
    a.key = make_philox_key(seed); a.gen = (uint32_t)generation;
    a.member_offset = (uint64_t)member_offset;
    const size_t smem = sizeof(float) * ((size_t)(2 * kTileT + kRows) * S + kRows);
    if (smem > 227 * 1024) {
        set_error("des_nes_eval(FP32): hidden/state_dim %d needs %zu B shared memory (> 227 KB)", kmax, smem);
        return DES_ERR_UNSUPPORTED;
    }
    return launch_smem("eval_ffma_kernel", solutions ? eval_ffma_kernel<true> : eval_ffma_kernel<false>, (unsigned)n_local,
                       kThreads, smem, st, a);
}

}  // namespace des
