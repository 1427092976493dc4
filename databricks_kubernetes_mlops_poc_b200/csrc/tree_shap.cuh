/*
 * tree_shap.cuh -- K5: exact path-dependent TreeSHAP per request field (Lundberg et al., arXiv:1802.03888, Algorithm 2)
 * over a path table (forest_paths.h), the merged-path form of GPUTreeShap (Mitchell et al., PeerJ CS 2022).
 *
 * Work split.  A CTA of B2F_SHAP_WARPS warps owns one tile of 32 rows (lane = row) and one contiguous range of paths
 * (blockIdx.y of gridDim.y ranges); each warp walks an equal share of that range.  Every lane of a warp is on the same
 * path, so path records and elements are warp-uniform broadcast loads (L1 / L2), and the path length is a uniform branch.
 * The host picks the number of ranges from n (b2f_api.cu launch_explain): a large batch has one range and one CTA per row
 * tile, a small one spreads its paths over enough ranges to fill every SM, so a single row is not walked by one warp.
 *
 * Per (row, path): the one-fraction of each merged element is the prediction kernels' test on the imputed row word (NaN
 * -> float32 median, float32 compare, category code), EXTEND runs over the elements in registers (pw[MAXL] doubles, fully
 * unrolled per length bucket MAXL = 9 / 16 / 24 so that compile-time indices keep pw out of local memory), then each element
 * is unwound in closed form.  Float64 throughout; no division: 1 / zero_fraction comes from the table and the
 * (i+1)/(l+1), (l-i)/(l+1), (l+1)/(i+1), (l+1)/(l-i) factors from c_shap_tab.
 *
 * Sums.  Each warp adds its paths' contributions, in path order, into its own phi[field][lane] float64 slice of shared
 * memory; the CTA then adds its warps' slices in warp order.  With one range that is the result (divided by denom, as the
 * prediction kernels divide the tree sum); with several, each CTA writes its partial to scratch ([range][row][field],
 * ranges * n * fields doubles, bounded by launch_explain) and k_tree_shap_finish adds the ranges in range order.  No
 * atomics: the same batch gives bit-identical results on every run.
 */
#ifndef B2F_TREE_SHAP_CUH
#define B2F_TREE_SHAP_CUH
#include <stdint.h>

#include "forest_paths.h"

#define B2F_SHAP_WARPS 8
#define B2F_SHAP_THREADS (32 * B2F_SHAP_WARPS)
#define B2F_SHAP_TAB_L 24

struct SParams {
    const b2f_path *paths;
    const b2f_path_elem *elems;
    int n_paths;
    int n_cat, n_num;
    double denom;
    float impute[24];
};

/* [0] (i+1)/(l+1)  [1] (l-i)/(l+1)  [2] (l+1)/(i+1)  [3] (l+1)/(l-i)  (0 where undefined); written by b2f_model_attach_explainer */
__constant__ double c_shap_tab[4][B2F_SHAP_TAB_L][B2F_SHAP_TAB_L];

__host__ __device__ inline int shap_smem_bytes(int n_fields) { return 24 * 32 * 4 + B2F_SHAP_WARPS * n_fields * 32 * 8; }

/* imputed row word f of row `row`, as the prediction kernels see it */
template <bool PACKED>
__device__ __forceinline__ uint32_t shap_row_word(const SParams &p, const uint32_t *__restrict__ rows, long long row, int f) {
    uint32_t v;
    if constexpr (PACKED) {
        /* words 0..1: nine 7-bit fields (code + 1, 0 = unknown); words 2..15: the numerics */
        const uint32_t *r = rows + row * B2F_PACKED_ROW_WORDS;
        if (f < p.n_cat) {
            const unsigned long long bits = ((unsigned long long)__ldg(r + 1) << 32) | __ldg(r);
            v = (uint32_t)((bits >> (7 * f)) & 0x7fu) - 1u;
        } else {
            v = __ldg(r + 2 + (f - p.n_cat));
        }
    } else {
        v = __ldg(rows + row * B2F_ROW_WORDS + f);
    }
    if (f >= p.n_cat && isnan(__uint_as_float(v))) v = __float_as_uint(p.impute[f]);
    return v;
}

/* xs[f * 32 + c] = imputed word f of the tile's row row0 + c (0 past n), for f < F; all threads of the CTA */
template <bool PACKED>
__device__ __forceinline__ void shap_stage_tile(const SParams &p, const uint32_t *__restrict__ rows, long long n, long long row0, int F, uint32_t *xs) {
    for (int i = threadIdx.x; i < 32 * F; i += B2F_SHAP_THREADS) {
        const long long row = row0 + (i & 31);
        xs[i] = row < n ? shap_row_word<PACKED>(p, rows, row, i >> 5) : 0u;
    }
}

/* a[j] for a run-time j < N, reading a at compile-time indices only (so a stays in registers) */
template <int N>
__device__ __forceinline__ double shap_pick(const double (&a)[N], int j) {
    double v = a[0];
#pragma unroll
    for (int k = 1; k < N; ++k)
        if (k == j) v = a[k];
    return v;
}

/* does this lane's row follow the path at element e?  -> also the element's field and zero-fraction pair */
__device__ __forceinline__ bool shap_follows(const b2f_path_elem *e, const uint32_t *xs, int lane, uint32_t &field, double &z, double &iz) {
    const uint4 q0 = __ldg(reinterpret_cast<const uint4 *>(e));
    const uint4 q1 = __ldg(reinterpret_cast<const uint4 *>(e) + 1);
    const double2 q2 = __ldg(reinterpret_cast<const double2 *>(e) + 2);
    field = q0.x;
    z = q2.x;
    iz = q2.y;
    const uint32_t x = xs[field * 32 + lane];
    if (q0.y & B2F_PE_CAT) {
        const int code = (int)x;
        const uint32_t bit = (code >= -1 && code <= 126) ? (uint32_t)(code + 1) : 0u;
        const uint32_t w = bit < 64 ? (bit < 32 ? q1.x : q1.y) : (bit < 96 ? q1.z : q1.w);
        return (w >> (bit & 31u)) & 1u;
    }
    const float xf = __uint_as_float(x);
    const bool above = !(xf < __uint_as_float(q0.z)); /* geu: x >= lo or unordered */
    const bool below = !(q0.y & B2F_PE_HAS_HI) || xf < __uint_as_float(q0.w);
    return above && below;
}

/* EXTEND over the len elements E[0..len) of one path (E[0] the bias) for this lane's row: pw[0..len) the path's polynomial,
 * pw[len..MAXL) = 0, and ones bit k set when the row follows element k (bit 0 always).  Returns pw[len - 1]. */
template <int MAXL>
__device__ __forceinline__ double shap_extend(const b2f_path_elem *E, int len, const uint32_t *xs, int lane, double (&pw)[MAXL], uint32_t &ones) {
    ones = 1u;
    pw[0] = 1.0;
#pragma unroll
    for (int l = 1; l < MAXL; ++l) {
        pw[l] = 0.0;
        if (l < len) {
            uint32_t field;
            double z, iz;
            const bool o = shap_follows(E + l, xs, lane, field, z, iz);
            ones |= (uint32_t)o << l;
#pragma unroll
            for (int i = l - 1; i >= 0; --i) {
                const double pi = pw[i];
                if (o) pw[i + 1] = fma(pi, c_shap_tab[0][l][i], pw[i + 1]);
                pw[i] = z * pi * c_shap_tab[1][l][i];
            }
        }
    }
    return shap_pick(pw, len - 1);
}

/* The closed-form UNWIND of one element out of the polynomial pw[0..d] (d < N, last = pw[d]): the sum of the unwound
 * polynomial's d entries.  o: the row follows the element, z / iz: its zero fraction and reciprocal.  STORE: w[0..N-1)
 * also receives the unwound entries (0 from d on), the polynomial of the path without the element. */
template <bool STORE, int N>
__device__ __forceinline__ double shap_unwound_sum(const double (&pw)[N], int d, double last, bool o, double z, double iz, double *w = nullptr) {
    double tot = 0.0;
    if (o) {
        double nxt = last;
#pragma unroll
        for (int i = N - 2; i >= 0; --i) {
            if constexpr (STORE) w[i] = 0.0;
            if (i < d) {
                const double tmp = nxt * c_shap_tab[2][d][i];
                if constexpr (STORE) w[i] = tmp;
                tot += tmp;
                nxt = pw[i] - tmp * z * c_shap_tab[1][d][i];
            }
        }
    } else {
#pragma unroll
        for (int i = N - 2; i >= 0; --i) {
            if constexpr (STORE) w[i] = 0.0;
            if (i < d) {
                const double tmp = pw[i] * iz * c_shap_tab[3][d][i];
                if constexpr (STORE) w[i] = tmp;
                tot += tmp;
            }
        }
    }
    return tot;
}

/* one path for this warp's 32 rows: EXTEND, then the closed-form UNWIND sum per element, added into my[field][lane] */
template <int MAXL>
__device__ __forceinline__ void shap_path(const SParams &p, int q, const uint32_t *xs, double *my, int lane) {
    /* a 24-byte record is 8-byte aligned only: {first, len} and the leaf are two 8-byte loads */
    const uint2 rec = __ldg(reinterpret_cast<const uint2 *>(p.paths + q));
    const double leaf = __ldg(&p.paths[q].leaf);
    const int len = (int)rec.y;
    const b2f_path_elem *E = p.elems + rec.x;
    double pw[MAXL];
    uint32_t ones;
    const double last = shap_extend(E, len, xs, lane, pw, ones);
    const int d = len - 1;
    for (int k = 1; k < len; ++k) {
        const double2 zz = __ldg(reinterpret_cast<const double2 *>(E + k) + 2);
        const uint32_t field = __ldg(&E[k].field);
        const bool o = (ones >> k) & 1u;
        const double tot = shap_unwound_sum<false>(pw, d, last, o, zz.x, zz.y);
        my[field * 32 + lane] += tot * ((o ? 1.0 : 0.0) - zz.x) * leaf;
    }
}

/* grid (row tiles, path ranges); dynamic shared memory shap_smem_bytes(F).  One range: out[row][field] = phi; several:
 * partials[range][row][field] = the range's sum (k_tree_shap_finish completes them) */
template <int MAXL, bool PACKED>
__global__ void __launch_bounds__(B2F_SHAP_THREADS, 2)
    k_tree_shap(const __grid_constant__ SParams p, const uint32_t *__restrict__ rows, long long n, double *__restrict__ out,
                double *__restrict__ partials) {
    extern __shared__ __align__(16) uint8_t shap_smem[];
    const int F = p.n_cat + p.n_num;
    uint32_t *xs = reinterpret_cast<uint32_t *>(shap_smem);         /* [24][32] imputed row words of the tile */
    double *acc = reinterpret_cast<double *>(shap_smem + 24 * 32 * 4); /* [warps][F][32] */
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = (long long)blockIdx.x * 32;
    shap_stage_tile<PACKED>(p, rows, n, row0, F, xs);
    double *my = acc + (size_t)warp * F * 32;
    for (int f = 0; f < F; ++f) my[f * 32 + lane] = 0.0;
    __syncthreads();

    const long long P = p.n_paths, R = gridDim.y, r = blockIdx.y;
    const long long c_lo = P * r / R, c_hi = P * (r + 1) / R;
    const int w_lo = (int)(c_lo + (c_hi - c_lo) * warp / B2F_SHAP_WARPS);
    const int w_hi = (int)(c_lo + (c_hi - c_lo) * (warp + 1) / B2F_SHAP_WARPS);
    for (int q = w_lo; q < w_hi; ++q) shap_path<MAXL>(p, q, xs, my, lane);
    __syncthreads();

    for (int i = threadIdx.x; i < 32 * F; i += B2F_SHAP_THREADS) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < B2F_SHAP_WARPS; ++w) s += acc[(size_t)w * F * 32 + i];
        const long long row = row0 + (i & 31);
        if (row >= n) continue;
        const int f = i >> 5;
        if (R == 1)
            out[row * F + f] = s / p.denom;
        else
            partials[((size_t)r * (size_t)n + (size_t)row) * F + f] = s;
    }
}

/* phi = (sum over ranges, in range order) / denom */
__global__ void __launch_bounds__(256) k_tree_shap_finish(const double *__restrict__ partials, int ranges, long long n_values, double denom,
                                                         double *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_values; i += (long long)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int r = 0; r < ranges; ++r) s += partials[(size_t)r * (size_t)n_values + (size_t)i];
        out[i] = s / denom;
    }
}
#endif
