// One quad of one member row of a genetic-algorithm generation (include/des_b200.h, "genetic algorithm"), in a header for
// the units that materialise rows: des_ga.cu (des_ga_rows) and des_ga_sweep.cu (des_ga_rows_sweep).
#pragma once
#include "des_common.cuh"

namespace des {

// row[4q .. 4q+3] (those below P) of member m of the generation whose table is parents[n_parents][P] with n_elites
// elites: an elite's parent row as it is, any other member's parent row plus sigma*eps of the member.
__device__ __forceinline__ void ga_row_quad(float *row, const float *parents, uint32_t n_parents, uint32_t n_elites,
                                            int64_t P, int64_t q, float sigma, const PhiloxKey &key,
                                            uint32_t gen, uint32_t m) {
    if (m < n_elites) {
        const float *src = parents + (int64_t)m * P;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int64_t j = 4 * q + e;
            if (j < P) row[j] = src[j];
        }
    } else {
        const float *src = parents + (int64_t)ga_parent(m, gen, n_parents, key) * P;
        const float4 z = noise_quad((uint32_t)q, m, gen, kStreamNesEps, key);
        const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int64_t j = 4 * q + e;
            if (j < P) row[j] = __fmaf_rn(sigma, zz[e], src[j]);
        }
    }
}

}  // namespace des
