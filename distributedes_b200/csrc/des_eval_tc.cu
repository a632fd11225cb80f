// des_nes_eval, precision DES_FWD_F16 / DES_FWD_F16X3: fused sample + perturb + forward + fitness with the two
// hidden-layer GEMMs on Hopper tensor cores (wgmma).
//
// One persistent CTA per SM (or one 2-CTA cluster per two SMs, see below) walks its members (Worker.run
// natural_es.py:27-32 per member).  A CTA has two consumer warpgroups; each owns 64 observation rows of a 128-row
// tile (one "pass" over the tape is one such tile).  For a member, StandardFCNet.forward (model.py:34-39) is
//
//   D1 = X  W1'^T            wgmma m64n64k16, A = X (fp16 registers, loaded once per pass), B = W1' (shared memory)
//   H1 = tanh(D1 + b1')      in registers; packed to fp16 the accumulator IS the A operand of layer 2 (des_tc.cuh)
//   D2 = H1 W2'^T            wgmma, A = H1 (registers), B = W2' in 64-feature chunks (two-stage shared-memory ring)
//   H2 = tanh(D2 + b2')      epilogue, registers only
//   a  = H2 W3'^T + b3'      A <= 8 outputs: exact fp32 FFMA in the same epilogue (no third MMA)
//   fitness += -|| clip(a) - a* ||^2                                              (utils.py:134-137)
//
// W' = fp32(theta + sigma*eps) (natural_es.py:28-30) is never stored in HBM: two producer warpgroups regenerate eps
// from the counter RNG and write fp16 operand tiles straight into the 128B-swizzled K-major layout wgmma reads.
// Warp specialisation (512 threads, setmaxnreg: producers 56 registers, consumers 200; 40 / 216 for f16x3, H = 256, NA = 8):
//   producers  per member: b1 | b2 | W3' | b3 into one of two small-array buffers, W1' into its single buffer once
//              every consumer of the cluster has run the previous member's layer 1, then the W2' chunks of every
//              pass into the ring.  They run ahead across member boundaries, bounded only by the buffers.
//   consumers  layer 1, the layer-2 chunks, the epilogues and the fitness reduction; they never generate weights.
// Every buffer has full / empty mbarriers, and all synchronisation is CTA-scope (no GPU-scope fence, no L1
// invalidation in the loop).  The producers store into their own CTA only, each runs fence.proxy.async.shared::cta,
// and they meet on a named barrier; then one thread arrives on the full barrier.  Empty takes one arrival per consumer
// warp of the cluster, right after the wgmma_wait of the MMAs that read the buffer, so a W2' stage is refilled while
// the consumers run its epilogue.  Stage and phase come from one running chunk counter that both roles advance alike.
// The two consumer warpgroups are not kept in step: fitness partials are double-buffered by member parity and the last
// consumer warp to finish a member adds them in warp order.
//
// Clusters: when the tape has an even number of 128-row tiles, two CTAs of a cluster share a member.  Each evaluates
// its own tiles and generates HALF of every weight tile into its own shared memory; the thread that arrives on its
// full barrier (arrive.expect_tx for the peer's half) pushes that half to the peer with cp.async.bulk (4 KB per 8 KB
// atom of a W2' chunk, H/2 rows per W1' plane), which completes on the peer's full barrier.  Consumers release a
// buffer on both CTAs' empty barriers (a plain remote mbarrier.arrive).  The flagship shape (T = 256) is then one pass
// per CTA.  Other shapes loop over passes; with the optional workspace the W2' chunks generated in pass 0 are
// mirrored to global memory (L2-resident) and copied back in the later passes, without it they are regenerated (same
// bytes either way).
//
// Mirrored sampling (des_nes_eval_mirrored): eval_tc_mirrored_kernel is the same body with the producers' kMirror flag
// set (member m perturbs with (-1)^(m & 1) * eps of counter word m >> 1); eval_tc_kernel compiles to the plain code.
//
// Precision modes
//   F16    operands rounded to fp16 (11 significant bits, as TF32), fp32 accumulate, MUFU tanh.approx.
//   F16X3  every operand split x = hi + lo (fp16 each, ~22 bits); D += A_hi B_hi + A_lo B_hi + A_hi B_lo;
//          tanh as 1 - 2/(1 + 2^(2x log2 e)).  ~fp32 accuracy at 3 MMAs per k-step.
#include "des_common.cuh"
#include "des_tc.cuh"

namespace des {

using namespace tc;

constexpr int kK1 = 32;        // layer-1 K (state_dim zero-padded): 2 k-steps of 16
constexpr int kMaxA = 8;
// Roles: warpgroups 0-1 generate the perturbed weights (one producer warpgroup cannot keep up: a Philox +
// Box-Muller chain per thread at one warp per scheduler is latency bound), warpgroups 2-3 run the MMAs and epilogues.
constexpr int kProdWGs = 2;
constexpr int kProdThreads = 128 * kProdWGs;
constexpr int kTcThreads = kProdThreads + 256;
constexpr int kConsWarps = 8;
// register budgets: the launch gives every thread 65536 / 512 = 128; the producers hand theirs to the consumers.  The
// producers get 56 (measured on the headline shape: 40 make the kernel 1.2 ms slower, 48 are no faster than 56);
// only f16x3 at H = 256 with 8 action sums needs more than 200 consumer registers (128 of them layer-1 activations)
// and gets 256 x 40 + 256 x 216 = 65536.
template <int H, bool X3, int NA>
__host__ __device__ constexpr uint32_t prod_regs() { return (H == 256 && X3 && NA == 8) ? 40u : 56u; }
template <int H, bool X3, int NA>
__host__ __device__ constexpr uint32_t cons_regs() { return (((65536u / kTcThreads) & ~7u) * kTcThreads - kProdThreads * prod_regs<H, X3, NA>()) / 256u & ~7u; }
static_assert(cons_regs<256, true, 4>() == 200 && cons_regs<256, true, 8>() == 216, "register split");

// Phase trace (build with -DDES_EVAL_TRACE, scripts/trace_eval.py): every thread charges the clock64() time since its
// previous mark to the phase it has just finished; lane 0 of every warp of CTAs 0 and 1 prints its totals at the end.
// Without the macro the marks compile to nothing.
#ifdef DES_EVAL_TRACE
enum { TR_WAIT, TR_MMA, TR_SYNC, TR_EPI, TR_GEN, TR_OTHER, TR_N };
#define DES_TRACE_INIT uint32_t tr_[TR_N] = {}; long long tr_t = clock64(), tr_0 = tr_t;
#define DES_TRACE(k) do { const long long t_ = clock64(); tr_[k] += (uint32_t)(t_ - tr_t); tr_t = t_; } while (0)
#define DES_TRACE_PRINT(role, members)                                                                                \
    if (blockIdx.x < 2 && lane == 0)                                                                                  \
        printf("DES_TRACE cta=%d warp=%d role=%s members=%d wait=%u mma=%u sync=%u epi=%u gen=%u other=%u total=%u\n", \
               (int)blockIdx.x, warp, role, members, tr_[TR_WAIT], tr_[TR_MMA], tr_[TR_SYNC], tr_[TR_EPI], tr_[TR_GEN],  \
               tr_[TR_OTHER], (uint32_t)(clock64() - tr_0))
#else
#define DES_TRACE_INIT
#define DES_TRACE(k)
#define DES_TRACE_PRINT(role, members)
#endif

template <int H, bool X3>
struct TcCfg {
    static constexpr int NCH = H / 64;                        // 64-feature output chunks per layer
    static constexpr int KAT = H / 64;                        // 64-wide k atoms of layer 2
    static constexpr int KS2 = H / 16;                        // k16 steps of layer 2
    static constexpr int PLANES = X3 ? 2 : 1;                 // hi [, lo]
    static constexpr int CHUNK_BYTES = PLANES * KAT * 8192;   // W2' rows [64c, 64c + 64), every k: hi atoms | lo atoms
    static constexpr int W1_BYTES = PLANES * H * 128;         // W1' rows of 128 B (k < 32 used): hi | lo
    static constexpr int SMALL_FLOATS = 2 * H + kMaxA * H + kMaxA;   // b1, b2, W3' [8][H], b3[8]
    // mbarriers: W2' stage s full / empty, W1' full / empty, small-array buffer b empty
    enum { BAR_W2_FULL = 0, BAR_W2_EMPTY = 2, BAR_W1_FULL = 4, BAR_W1_EMPTY = 5, BAR_SMALL_EMPTY = 6, NBARS = 8 };
    // W2' ring [2][CHUNK_BYTES] | W1' | small [2][SMALL_FLOATS] | fitness partials [2][8] | arrival counters [2] | mbarriers
    static constexpr size_t OFF_W1 = 2 * (size_t)CHUNK_BYTES;
    static constexpr size_t OFF_SMALL = OFF_W1 + W1_BYTES;
    static constexpr size_t OFF_FIT = OFF_SMALL + 2 * (size_t)SMALL_FLOATS * sizeof(float);
    static constexpr size_t OFF_CNT = OFF_FIT + 2 * kConsWarps * sizeof(float);
    static constexpr size_t OFF_BAR = (OFF_CNT + 2 * sizeof(uint32_t) + 7) & ~(size_t)7;
    static constexpr size_t SMEM = 1024 + OFF_BAR + NBARS * sizeof(uint64_t);
    static_assert(SMEM <= 227 * 1024, "eval_tc_kernel: shared memory over the 227 KB per-block limit");
    static_assert(SMALL_FLOATS * sizeof(float) % 16 == 0, "small-array buffers must stay float4 aligned");
};

struct TcArgs {
    float *fitness;
    const float *theta, *obs, *target;
    const des_state *state;
    Layout L;
    int T, n_pass;
    float sigma, clip, neg2ln2_sigma2;
    PhiloxKey key;
    uint32_t gen;
    uint64_t member_offset;
    int64_t n_local;
    uint8_t *cache;        // optional per-CTA image of one member's W2' chunks (multi-pass shapes), else NULL
};

// one perturbed parameter at arbitrary flat index j (slow path: whole quad per element)
__device__ __forceinline__ float perturbed1(const float *__restrict__ theta, int j, float sigma, uint32_t member,
                                            uint32_t gen, const PhiloxKey &key) {
    const float4 z = noise_quad((uint32_t)(j >> 2), member, gen, kStreamNesEps, key);
    const int e = j & 3;
    const float zz = e == 0 ? z.x : (e == 1 ? z.y : (e == 2 ? z.z : z.w));
    return __fmaf_rn(sigma, zz, __ldg(theta + j));
}

// perturbed_quad of the NES stream; mirrored (kMirror): sgn = -1 for the odd member of a pair.  sigma is folded into the
// radius through sigma^2, which loses its sign, so the radius itself is negated: fma(-r, c, theta) is exactly
// fp32(theta - sigma*eps), and sgn = +1 gives the bits of the plain member.
template <bool kMirror>
__device__ __forceinline__ float4 member_quad(uint32_t q, uint32_t member, uint32_t gen, const PhiloxKey &key,
                                              float neg2ln2_sigma2, float4 base, float sgn) {
    if (!kMirror) return perturbed_quad(q, member, gen, kStreamNesEps, key, neg2ln2_sigma2, base);
    const uint4 x = philox4x32(q, member, gen, kStreamNesEps, key);
    const BmParts a = box_muller_parts(x.x, x.y, neg2ln2_sigma2, key.one_bits);
    const BmParts b = box_muller_parts(x.z, x.w, neg2ln2_sigma2, key.one_bits);
    const float ra = a.nr * sgn, rb = b.nr * sgn;
    return make_float4(__fmaf_rn(ra, a.c, base.x), __fmaf_rn(ra, a.s, base.y), __fmaf_rn(rb, b.c, base.z),
                       __fmaf_rn(rb, b.s, base.w));
}

template <bool X3>
__device__ __forceinline__ void octet(const float (&w)[8], uint4 &hi, uint4 &lo) {
    if (X3) {
        split_h2(w[0], w[1], hi.x, lo.x); split_h2(w[2], w[3], hi.y, lo.y);
        split_h2(w[4], w[5], hi.z, lo.z); split_h2(w[6], w[7], hi.w, lo.w);
    } else {
        hi = make_uint4(pack_h2(w[0], w[1]), pack_h2(w[2], w[3]), pack_h2(w[4], w[5]), pack_h2(w[6], w[7]));
        lo = hi;
    }
}

// A operand of the two layer-1 k-steps for rows ra, ra + 8 of the observation tape (zero beyond state_dim)
template <bool X3>
__device__ __forceinline__ void load_x(uint32_t (&xh)[2][4], uint32_t (&xl)[2][4], const float *__restrict__ obs, int d0,
                                       int ra, int lane) {
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int row = ra + (i & 1) * 8, k = ks * 16 + (i >> 1) * 8 + (lane & 3) * 2;
            const float v0 = k < d0 ? __ldg(obs + (int64_t)row * d0 + k) : 0.f;
            const float v1 = k + 1 < d0 ? __ldg(obs + (int64_t)row * d0 + k + 1) : 0.f;
            if (X3) split_h2(v0, v1, xh[ks][i], xl[ks][i]);
            else xh[ks][i] = pack_h2(v0, v1);
        }
    }
}

// NA: compile-time bound on the action count (4 or 8) that sizes the per-thread action sums.  kMirror: mirrored
// sampling, member m perturbs with (-1)^(m & 1) * eps of counter word m >> 1 (producers only; the consumers are the same)
template <int H, bool X3, int CL, int NA, bool kMirror>
__device__ __forceinline__ void eval_tc_body(const TcArgs &a) {
    using C = TcCfg<H, X3>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *w2buf = smem;                                                  // [2][CHUNK_BYTES]
    uint8_t *w1 = smem + C::OFF_W1;                                         // [W1_BYTES]
    float *small_buf = reinterpret_cast<float *>(smem + C::OFF_SMALL);      // [2][SMALL_FLOATS]
    float *fit_part = reinterpret_cast<float *>(smem + C::OFF_FIT);         // [2][kConsWarps]
    uint32_t *fit_cnt = reinterpret_cast<uint32_t *>(smem + C::OFF_CNT);    // [2]
    const uint32_t bars = smem_u32(smem + C::OFF_BAR);
    auto bar = [&](int k) { return bars + 8u * (uint32_t)k; };

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t rank = CL == 2 ? cluster_ctarank() : 0u;
    const Layout L = a.L;
    const uint32_t gen = generation_word(a.state, a.gen);
    const int64_t first = blockIdx.x / CL, stride = gridDim.x / CL;

    // A CTA's half of a weight tile in a cluster: rows [32 rank, 32 rank + 32) of every 8 KB atom of a W2' chunk, rows
    // [H/2 rank, H/2 rank + H/2) of each W1' plane.  Its producers store it locally; one thread then pushes it to the
    // peer with one bulk copy per atom (per plane for W1'), which completes on the peer's full barrier.
    constexpr uint32_t kW2Copy = (64 / CL) * 128, kW2Copies = C::PLANES * C::KAT;
    constexpr uint32_t kW1Copy = (H / CL) * 128, kW1Copies = C::PLANES;
    static_assert(CL * kW2Copies * kW2Copy == C::CHUNK_BYTES && CL * kW1Copies * kW1Copy == C::W1_BYTES,
                  "the two halves must make up the whole tile, or a full barrier never completes");
    static_assert(kW2Copy % 16 == 0 && kW1Copy % 16 == 0, "bulk copies move multiples of 16 bytes");
    static_assert(kW2Copies * kW2Copy < (1u << 20) && kW1Copies * kW1Copy < (1u << 20), "mbarrier tx-count range");

    // full: one arrival, by the elected producer thread after its CTA's producers have stored their half, plus in a
    // cluster the bytes of the peer's half (complete_tx of its bulk copies); empty: one arrival per consumer warp of the
    // cluster (each reads its own CTA's copy, which both producers fill); small arrays are per CTA
    if (tid == 0) {
        for (int s = 0; s < 2; ++s) {
            mbar_init(bar(C::BAR_W2_FULL + s), 1);
            mbar_init(bar(C::BAR_W2_EMPTY + s), kConsWarps * CL);
            mbar_init(bar(C::BAR_SMALL_EMPTY + s), kTcThreads - kProdThreads);
        }
        mbar_init(bar(C::BAR_W1_FULL), 1);
        mbar_init(bar(C::BAR_W1_EMPTY), kConsWarps * CL);
        fit_cnt[0] = fit_cnt[1] = 0u;
        fence_barrier_init();
    }
    // distributed shared memory and the peer's barriers may only be used once every CTA of the cluster runs and has
    // initialised them (fence_barrier_init publishes the initialisation); the CTA barrier orders fit_cnt
    if (CL == 2) cluster_sync_relaxed();
    __syncthreads();
    // consumers: one arrival on empty barrier k of every CTA of the cluster, once this warp's MMAs have read the buffer
    const uint32_t peer_bars = CL == 2 ? map_cluster(bars, rank ^ 1u) : 0u;
    auto release_all = [&](int k) {
        mbar_arrive(bar(k));
        if (CL == 2) mbar_arrive_remote(peer_bars + 8u * (uint32_t)k);
    };

    if (warp < 4 * kProdWGs) {
        // ================= producer warpgroups: perturbed weights for the consumers, running ahead across members
        setmaxnreg_dec<prod_regs<H, X3, NA>()>();
        DES_TRACE_INIT
        const int ptid = tid;
        uint8_t *const cache = (a.cache && a.n_pass > 1) ? a.cache + (size_t)blockIdx.x * C::NCH * C::CHUNK_BYTES : nullptr;
        // a 16-byte chunk of an operand tile (hi plane at `off`, lo plane `lo_off` further) into this CTA
        auto put = [&](uint8_t *base, uint32_t off, uint32_t lo_off, const uint4 &hi, const uint4 &lo) {
            *reinterpret_cast<uint4 *>(base + off) = hi;
            if (X3) *reinterpret_cast<uint4 *>(base + lo_off + off) = lo;
        };
        // this CTA's half of a tile at `base` is stored (ncopy pieces of `bytes`, `step` apart, this CTA's at
        // + rank * bytes): make it visible to wgmma and the bulk copy, then one thread arrives on the local full barrier
        // k, expecting the peer's half, and pushes this CTA's half into the peer, completing on the peer's barrier k
        auto publish = [&](int k, uint32_t base, uint32_t bytes, uint32_t ncopy, uint32_t step) {
            fence_proxy_async_cta();
            named_bar_sync(1, kProdThreads);
            if (ptid == 0) {
                if (CL == 2) {
                    mbar_expect_tx(bar(k), ncopy * bytes);
                    const uint32_t peer_bar = map_cluster(bar(k), rank ^ 1u);
                    for (uint32_t j = 0; j < ncopy; ++j) {
                        const uint32_t src = base + j * step + rank * bytes;
                        bulk_copy_to_peer(map_cluster(src, rank ^ 1u), src, bytes, peer_bar);
                    }
                } else {
                    mbar_arrive(bar(k));
                }
            }
        };
        // this CTA's share of W2' chunk c (rows [64c, 64c + 64)) into stage `buf`; pass > 0 copies the cached image back
        constexpr int kOct = H / 8;                               // octets per row
        constexpr int kRows = 64 / CL;                            // rows of a chunk generated here
        auto gen_chunk = [&](uint32_t member, float sgn, int c, int pass, int buf) {
            uint8_t *dst = w2buf + buf * C::CHUNK_BYTES;
            uint8_t *mirror = cache ? cache + (size_t)c * C::CHUNK_BYTES : nullptr;
            for (int idx = ptid; idx < kRows * kOct; idx += kProdThreads) {
                const int rr = (int)rank * kRows + idx / kOct, o = idx % kOct;
                const uint32_t off = (uint32_t)((o >> 3) * 8192 + rr * 128 + (((o & 7) ^ (rr & 7)) << 4));
                uint4 hi, lo;
                if (mirror && pass > 0) {
                    hi = *reinterpret_cast<const uint4 *>(mirror + off);
                    if (X3) lo = *reinterpret_cast<const uint4 *>(mirror + C::KAT * 8192 + off);
                    else lo = hi;
                } else {
                    const int j0 = L.off_w2 + (c * 64 + rr) * H + o * 8;
                    const float4 p0 = member_quad<kMirror>((uint32_t)(j0 >> 2), member, gen, a.key, a.neg2ln2_sigma2,
                                                           __ldg(reinterpret_cast<const float4 *>(a.theta + j0)), sgn);
                    const float4 p1 = member_quad<kMirror>((uint32_t)(j0 >> 2) + 1, member, gen, a.key, a.neg2ln2_sigma2,
                                                           __ldg(reinterpret_cast<const float4 *>(a.theta + j0 + 4)), sgn);
                    const float w[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
                    octet<X3>(w, hi, lo);
                    if (mirror) {       // the same thread reads exactly these bytes back in the later passes
                        *reinterpret_cast<uint4 *>(mirror + off) = hi;
                        if (X3) *reinterpret_cast<uint4 *>(mirror + C::KAT * 8192 + off) = lo;
                    }
                }
                put(dst, off, C::KAT * 8192, hi, lo);
            }
        };

        uint32_t q = 0;                                           // running W2' chunk counter, as in the consumers
        int i = 0;
        for (int64_t m = first; m < a.n_local; m += stride, ++i) {
            // the counter word of the noise and, mirrored, the sign of the pair member
            const uint32_t member = noise_word(a.member_offset + (uint64_t)m, kMirror);
            const float sgn = member_sigma(a.member_offset + (uint64_t)m, kMirror, 1.0f);
            // ---- small fp32 arrays (whole, in every CTA) into buffer i & 1: b1 | b2 | W3[8][H] | b3[8]
            float *small = small_buf + (i & 1) * C::SMALL_FLOATS;
            if (i >= 2) mbar_wait(bar(C::BAR_SMALL_EMPTY + (i & 1)), ((i >> 1) - 1) & 1);
            DES_TRACE(TR_WAIT);
            for (int k = ptid; k < H / 4; k += kProdThreads) {
                const float4 v1 = member_quad<kMirror>((uint32_t)((L.off_b1 >> 2) + k), member, gen, a.key, a.neg2ln2_sigma2,
                                                       __ldg(reinterpret_cast<const float4 *>(a.theta + L.off_b1) + k), sgn);
                const float4 v2 = member_quad<kMirror>((uint32_t)((L.off_b2 >> 2) + k), member, gen, a.key, a.neg2ln2_sigma2,
                                                       __ldg(reinterpret_cast<const float4 *>(a.theta + L.off_b2) + k), sgn);
                // the f16x3 epilogue evaluates tanh(v + b) as 1 - 2/(1 + 2^(v*c + b*c)), c = 2 log2 e: store b*c
                const float bsc = X3 ? kTwoLog2e : 1.0f;
                reinterpret_cast<float4 *>(small)[k] = make_float4(v1.x * bsc, v1.y * bsc, v1.z * bsc, v1.w * bsc);
                reinterpret_cast<float4 *>(small + H)[k] = make_float4(v2.x * bsc, v2.y * bsc, v2.z * bsc, v2.w * bsc);
            }
            for (int k = ptid; k < L.A * H / 4; k += kProdThreads)             // W3' [q][n] row-major: aligned quads
                reinterpret_cast<float4 *>(small + 2 * H)[k] =
                    member_quad<kMirror>((uint32_t)((L.off_w3 >> 2) + k), member, gen, a.key, a.neg2ln2_sigma2,
                                         __ldg(reinterpret_cast<const float4 *>(a.theta + L.off_w3) + k), sgn);
            for (int k = L.A * H + ptid; k < H * kMaxA; k += kProdThreads) small[2 * H + k] = 0.f;   // unused action rows
            if (ptid < kMaxA)
                small[2 * H + kMaxA * H + ptid] = ptid < L.A ? perturbed1(a.theta, L.off_b3 + ptid, sgn * a.sigma, member, gen, a.key) : 0.f;
            // ---- W1' (this CTA's half of the rows in a cluster), once every consumer has run member i-1's layer 1
            DES_TRACE(TR_GEN);
            if (i >= 1) mbar_wait(bar(C::BAR_W1_EMPTY), (i - 1) & 1);
            DES_TRACE(TR_WAIT);
            for (int idx = ptid; idx < (H / CL) * 4; idx += kProdThreads) {
                const int n = (int)rank * (H / CL) + (idx >> 2), c8 = idx & 3;
                float w[8];
                if ((L.d0 & 3) == 0) {                                        // row starts are quad aligned
#pragma unroll
                    for (int hq = 0; hq < 2; ++hq) {
                        const int k = c8 * 8 + hq * 4;
                        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (k < L.d0) {
                            const int j = L.off_w1 + n * L.d0 + k;
                            v = member_quad<kMirror>((uint32_t)(j >> 2), member, gen, a.key, a.neg2ln2_sigma2,
                                                     __ldg(reinterpret_cast<const float4 *>(a.theta + j)), sgn);
                        }
                        w[4 * hq] = v.x; w[4 * hq + 1] = v.y; w[4 * hq + 2] = v.z; w[4 * hq + 3] = v.w;
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        const int k = c8 * 8 + e;
                        w[e] = (k < L.d0) ? perturbed1(a.theta, L.off_w1 + n * L.d0 + k, sgn * a.sigma, member, gen, a.key) : 0.f;
                    }
                }
                uint4 hi, lo;
                octet<X3>(w, hi, lo);
                put(w1, (uint32_t)(n * 128 + ((c8 ^ (n & 7)) << 4)), H * 128, hi, lo);
            }
            DES_TRACE(TR_GEN);
            publish(C::BAR_W1_FULL, smem_u32(w1), kW1Copy, kW1Copies, H * 128);   // and the small arrays
            DES_TRACE(TR_SYNC);
            // ---- W2' chunks of every pass through the two-stage ring
            for (int pass = 0; pass < a.n_pass; ++pass) {
                for (int c = 0; c < C::NCH; ++c, ++q) {
                    const int s = (int)(q & 1u);
                    if (q >= 2) mbar_wait(bar(C::BAR_W2_EMPTY + s), ((q >> 1) - 1) & 1u);
                    DES_TRACE(TR_WAIT);
                    gen_chunk(member, sgn, c, pass, s);
                    DES_TRACE(TR_GEN);
                    publish(C::BAR_W2_FULL + s, smem_u32(w2buf + s * C::CHUNK_BYTES), kW2Copy, kW2Copies, 8192);
                    DES_TRACE(TR_SYNC);
                }
            }
        }
        // A CTA leaves only when its peer can no longer arrive on its barriers or copy into its shared memory: once
        // every consumer warp of the cluster has released W1' and the last two W2' stages.  Those releases follow the
        // consumers' full waits, so every bulk copy of either CTA has landed too.
        if (CL == 2) {
            for (uint32_t t = q > 2u ? q - 2u : 0u; t < q; ++t) mbar_wait(bar(C::BAR_W2_EMPTY + (int)(t & 1u)), (t >> 1) & 1u);
            if (i >= 1) mbar_wait(bar(C::BAR_W1_EMPTY), (i - 1) & 1);
        }
        DES_TRACE_PRINT("producer", i);
    } else {
        // ================= consumer warpgroups cw = 0, 1: rows [64 cw, 64 cw + 64) of the pass's tile
        setmaxnreg_inc<cons_regs<H, X3, NA>()>();
        DES_TRACE_INIT
        const int cwarp = warp - 4 * kProdWGs, cw = cwarp >> 2;
        const int r_in_tile = cw * 64 + (cwarp & 3) * 16 + (lane >> 2);   // this thread: rows ra and ra + 8
        const int cq = (lane & 3) * 2;                            // column pair inside every 8-column block
        uint32_t q = 0;
        int i = 0;
        for (int64_t m = first; m < a.n_local; m += stride, ++i) {
            const float *small = small_buf + (i & 1) * C::SMALL_FLOATS;
            const float *b1 = small, *b2 = small + H, *w3 = small + 2 * H, *b3 = small + 2 * H + kMaxA * H;
            mbar_wait(bar(C::BAR_W1_FULL), (uint32_t)i & 1u);
            DES_TRACE(TR_WAIT);

            float sq = 0.f;
            for (int pass = 0; pass < a.n_pass; ++pass) {
                const int tile = pass * CL + (int)rank;
                const int ra = tile * 128 + r_in_tile;
                // ---------------- layer 1: H1 = tanh(X W1'^T + b1), kept as the fp16 A operand of layer 2
                uint32_t h1h[C::KS2][4], h1l[X3 ? C::KS2 : 1][4];
                {
                    uint32_t xh[2][4], xl[2][4];
                    load_x<X3>(xh, xl, a.obs, L.d0, ra, lane);
                    DES_TRACE(TR_OTHER);
#pragma unroll
                    for (int c = 0; c < C::NCH; ++c) {
                        float d[32];
#pragma unroll
                        for (int k = 0; k < 32; ++k) d[k] = 0.f;
                        wgmma_fence();
#pragma unroll
                        for (int ks = 0; ks < 2; ++ks) {
                            const uint32_t bh = smem_u32(w1) + c * 8192 + ks * 32;
                            wgmma_rs_n64(d, xh[ks], smem_desc_sw128(bh), ks > 0);
                            if (X3) {
                                wgmma_rs_n64(d, xl[ks], smem_desc_sw128(bh), 1);                   // X_lo W_hi
                                wgmma_rs_n64(d, xh[ks], smem_desc_sw128(bh + H * 128), 1);         // X_hi W_lo
                            }
                        }
                        wgmma_commit();
                        wgmma_wait<0>();
                        fence_regs(d);
                        DES_TRACE(TR_MMA);
                        // the last layer-1 MMA of the member has read W1': the producer may write the next member's
                        if (c == C::NCH - 1 && pass == a.n_pass - 1 && lane == 0) release_all(C::BAR_W1_EMPTY);
                        DES_TRACE(TR_SYNC);
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float2 b = *reinterpret_cast<const float2 *>(b1 + c * 64 + j * 8 + cq);
                            const int s = c * 4 + (j >> 1), e = (j & 1) * 2;
#pragma unroll
                            for (int r = 0; r < 2; ++r) {
                                const float v0 = d[4 * j + 2 * r], v1 = d[4 * j + 2 * r + 1];
                                if (X3) split_h2(tanh_acc_b(v0, b.x), tanh_acc_b(v1, b.y), h1h[s][e + r], h1l[s][e + r]);
                                else h1h[s][e + r] = pack_h2(tanh_fast(v0 + b.x), tanh_fast(v1 + b.y));
                            }
                        }
                        DES_TRACE(TR_EPI);
                    }
                }
                // ---------------- layer 2 + 3: per 64-feature chunk, H2 = tanh(H1 W2'^T + b2); a += H2 W3'^T
                float act[NA][2];
#pragma unroll
                for (int k = 0; k < NA; ++k) act[k][0] = act[k][1] = 0.f;
                for (int c = 0; c < C::NCH; ++c, ++q) {
                    const int st = (int)(q & 1u);
                    mbar_wait(bar(C::BAR_W2_FULL + st), (q >> 1) & 1u);
                    DES_TRACE(TR_WAIT);
                    const uint32_t bbase = smem_u32(w2buf + st * C::CHUNK_BYTES);
                    float d[32];
#pragma unroll
                    for (int k = 0; k < 32; ++k) d[k] = 0.f;
                    wgmma_fence();
#pragma unroll
                    for (int s = 0; s < C::KS2; ++s) {
                        const uint32_t bh = bbase + (s >> 2) * 8192 + (s & 3) * 32;
                        wgmma_rs_n64(d, h1h[s], smem_desc_sw128(bh), s > 0);
                        if (X3) {
                            wgmma_rs_n64(d, h1l[s], smem_desc_sw128(bh), 1);                          // H1_lo W_hi
                            wgmma_rs_n64(d, h1h[s], smem_desc_sw128(bh + C::KAT * 8192), 1);          // H1_hi W_lo
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    fence_regs(d);
                    DES_TRACE(TR_MMA);
                    // every MMA of this warp that read the stage has completed: the producer may refill it during the epilogue
                    if (lane == 0) release_all(C::BAR_W2_EMPTY + st);
                    DES_TRACE(TR_SYNC);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int n = c * 64 + j * 8 + cq;
                        const float2 b = *reinterpret_cast<const float2 *>(b2 + n);
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            float h0, h1;
                            if (X3) {          // b2 holds b * 2log2(e)
                                h0 = tanh_acc_b(d[4 * j + 2 * r], b.x);
                                h1 = tanh_acc_b(d[4 * j + 2 * r + 1], b.y);
                            } else {
                                h0 = tanh_fast(d[4 * j + 2 * r] + b.x);
                                h1 = tanh_fast(d[4 * j + 2 * r + 1] + b.y);
                            }
                            // layer 3 (model.py:38) in fp32: W3' row-major [q][n]
#pragma unroll
                            for (int k = 0; k < NA; ++k) {
                                if (k < L.A) {
                                    const float2 w = *reinterpret_cast<const float2 *>(w3 + k * H + n);
                                    act[k][r] = __fmaf_rn(h1, w.y, __fmaf_rn(h0, w.x, act[k][r]));
                                }
                            }
                        }
                    }
                    DES_TRACE(TR_EPI);
                }
                // ---- the four lanes of a quad hold the action sums over disjoint columns of the same two rows
#pragma unroll
                for (int k = 0; k < NA; ++k) {
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        act[k][r] += __shfl_xor_sync(0xffffffffu, act[k][r], 1);
                        act[k][r] += __shfl_xor_sync(0xffffffffu, act[k][r], 2);
                    }
                }
                if ((lane & 3) == 0) {
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int t = ra + 8 * r;
#pragma unroll
                        for (int k = 0; k < NA; ++k) {
                            if (k < L.A) {
                                float v = act[k][r] + b3[k];
                                v = clip_keep_nan(v, a.clip);
                                const float dd = v - __ldg(a.target + (int64_t)t * L.A + k);
                                sq = __fmaf_rn(dd, dd, sq);
                            }
                        }
                    }
                }
            }
            // ---- member done: reduce squared error over all rows (fixed order -> deterministic)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
            if (lane == 0) {
                // the two consumer warpgroups need not be on the same member: partials and counter are double-buffered
                // by member parity, and the last consumer warp to arrive adds the partials in warp order
                float *part = fit_part + (i & 1) * kConsWarps;
                part[cwarp] = sq;
                __threadfence_block();
                if (atomicAdd(fit_cnt + (i & 1), 1u) == kConsWarps - 1) {
                    __threadfence_block();
                    double f = 0.0;
                    for (int w = 0; w < kConsWarps; ++w) f += (double)reinterpret_cast<volatile float *>(part)[w];
                    fit_cnt[i & 1] = 0u;
                    // a cluster adds its two halves into the (pre-zeroed) output: two commutative fp32 adds -> deterministic
                    if (CL == 2) atomicAdd(a.fitness + m, (float)(-f));
                    else a.fitness[m] = (float)(-f);
                }
            }
            // every thread's reads of this member's small arrays (and its fitness bookkeeping) are done
            mbar_arrive(bar(C::BAR_SMALL_EMPTY + (i & 1)));
            DES_TRACE(TR_OTHER);
        }
        DES_TRACE_PRINT("consumer", i);
    }
}

template <int H, bool X3, int CL, int NA>
__global__ void __launch_bounds__(kTcThreads, 1) eval_tc_kernel(TcArgs a) { eval_tc_body<H, X3, CL, NA, false>(a); }

template <int H, bool X3, int CL, int NA>
__global__ void __launch_bounds__(kTcThreads, 1) eval_tc_mirrored_kernel(TcArgs a) { eval_tc_body<H, X3, CL, NA, true>(a); }

template <int H, bool X3, int CL, int NA, bool kMirror>
static int launch_tc(TcArgs &a, cudaStream_t st) {
    using C = TcCfg<H, X3>;
    const auto kernel = kMirror ? eval_tc_mirrored_kernel<H, X3, CL, NA> : eval_tc_kernel<H, X3, CL, NA>;
    a.n_pass = a.T / 128 / CL;
    int dev = 0, sms = 132;
    DES_CUDA(cudaGetDevice(&dev));
    DES_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (CL == 2) {
        DES_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
        // each cluster accumulates its two halves into the output with atomicAdd: zero it first
        DES_CUDA(cudaMemsetAsync(a.fitness, 0, (size_t)a.n_local * sizeof(float), st));
        const int64_t clusters = a.n_local < sms / 2 ? a.n_local : sms / 2;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(2 * clusters));
        cfg.blockDim = dim3(kTcThreads);
        cfg.dynamicSmemBytes = C::SMEM;
        cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 2;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        DES_CUDA(cudaLaunchKernelEx(&cfg, kernel, a));
        DES_LAUNCH_CHECK("eval_tc_kernel");
        return DES_OK;
    }
    const int64_t grid = a.n_local < sms ? a.n_local : sms;
    return launch_smem("eval_tc_kernel", kernel, (unsigned)grid, kTcThreads, C::SMEM, st, a);
}

template <int H, bool X3, bool kMirror>
static int launch_tc_m(TcArgs &a, cudaStream_t st) {
    const bool even = (a.T / 128) % 2 == 0;
    if (a.L.A <= 4) return even ? launch_tc<H, X3, 2, 4, kMirror>(a, st) : launch_tc<H, X3, 1, 4, kMirror>(a, st);
    return even ? launch_tc<H, X3, 2, kMaxA, kMirror>(a, st) : launch_tc<H, X3, 1, kMaxA, kMirror>(a, st);
}

template <int H, bool X3>
static int launch_tc_h(TcArgs &a, bool mirrored, cudaStream_t st) {
    return mirrored ? launch_tc_m<H, X3, true>(a, st) : launch_tc_m<H, X3, false>(a, st);
}

static int tc_passes(int T) { const int tiles = T / 128; return tiles % 2 == 0 ? tiles / 2 : tiles; }

size_t eval_tc_workspace_bytes(des_dims dims, int precision) {
    const int H = dims.hidden;
    if (!(H == 64 || H == 128 || H == 256) || dims.tape_len % 128 != 0 || tc_passes(dims.tape_len) <= 1) return 0;
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
        cudaGetLastError();
        sms = 132;
    }
    // one image of a member's W2' chunks per CTA: H/64 chunks of (hi [+ lo]) 64 x H fp16
    return (size_t)sms * (size_t)H * H * 2 * (precision == DES_FWD_F16X3 ? 2 : 1);
}

int eval_tc_launch(float *fitness, const float *theta, const float *obs, const float *target, des_dims dims,
                   double sigma, double clip, uint64_t seed, uint64_t generation, const des_state *state,
                   int64_t member_offset, int64_t n_local, int precision, void *workspace, size_t workspace_bytes,
                   bool mirrored, cudaStream_t st) {
    const int H = dims.hidden;
    if (!(H == 64 || H == 128 || H == 256) || dims.state_dim > kK1 || dims.action_dim > kMaxA || dims.tape_len % 128 != 0) {
        set_error("des_nes_eval(tensor): needs hidden in {64,128,256}, state_dim <= %d, action_dim <= %d, tape_len %% 128 == 0 "
                  "(got d0=%d H=%d A=%d T=%d); use DES_FWD_FP32 for other shapes", kK1, kMaxA, dims.state_dim, H,
                  dims.action_dim, dims.tape_len);
        return DES_ERR_UNSUPPORTED;
    }
    if (((uintptr_t)theta & 15) != 0) {
        set_error("des_nes_eval(tensor): theta_dev must be 16-byte aligned");
        return DES_ERR_INVALID_ARGUMENT;
    }
    TcArgs a;
    a.fitness = fitness; a.theta = theta; a.obs = obs; a.target = target; a.state = state;
    a.L = Layout(dims.state_dim, H, dims.action_dim);
    a.T = dims.tape_len;
    a.sigma = (float)sigma; a.clip = (float)clip;
    a.neg2ln2_sigma2 = kNeg2Ln2 * (float)sigma * (float)sigma;
    a.key = make_philox_key(seed); a.gen = (uint32_t)generation;
    a.member_offset = (uint64_t)member_offset; a.n_local = n_local;
    const bool x3 = precision == DES_FWD_F16X3;
    const size_t need = eval_tc_workspace_bytes(dims, precision);
    a.cache = (need > 0 && workspace && workspace_bytes >= need && ((uintptr_t)workspace & 15) == 0) ? (uint8_t *)workspace : nullptr;
    switch (H) {
        case 64: return x3 ? launch_tc_h<64, true>(a, mirrored, st) : launch_tc_h<64, false>(a, mirrored, st);
        case 128: return x3 ? launch_tc_h<128, true>(a, mirrored, st) : launch_tc_h<128, false>(a, mirrored, st);
        default: return x3 ? launch_tc_h<256, true>(a, mirrored, st) : launch_tc_h<256, false>(a, mirrored, st);
    }
}

}  // namespace des
