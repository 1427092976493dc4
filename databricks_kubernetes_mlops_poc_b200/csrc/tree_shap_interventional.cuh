/*
 * tree_shap_interventional.cuh -- K5c: exact interventional TreeSHAP against a background set (Lundberg et al., Nat. Mach.
 * Intell. 2020, arXiv:1905.04610; what shap's TreeExplainer computes when given a dataset) over the same path table as K5
 * (forest_paths.h), request fields as players: phi(x) is the mean over background rows z of the Shapley values of the game
 * v_z(S) = f(x_S, z_rest).  With a one-row background that is baseline Shapley.
 *
 * Per path of d merged elements and pair (x, z): Fx / Fz are the elements x / z satisfies (the prediction kernels' test on
 * the imputed row word, as K5), as a mask with bit k for element k and bit 0 (the bias) always set.  The hybrid row reaches
 * the leaf iff every element is satisfied by x or by z; the path's game is then 1[A in S, S and B disjoint] with
 * A = Fx \ Fz, B = Fz \ Fx, a = |A|, b = |B|: each field of A gets +leaf W[a][b], each of B -leaf W[b][a], with
 * W[x][y] = (x-1)! y! / (x+y)! (W[0][.] = 0), every other field 0.  phi = sum over paths and background rows / (denom |Z|).
 *
 * Background table (b2f_model_attach_background, once per background).  Only Fz matters, so each path keeps its distinct
 * masks and how many background rows have each, in mask order (paths of up to B2F_BG_HIST_LEN field elements: a
 * shared-memory histogram), or one entry of count 1 per background row, in row order (longer paths: forests deeper than
 * 12).  For a given Fx an entry m counts iff m covers every element x fails; B is then exactly those elements, the same for
 * every entry of the path, and A = Fx \ m.
 *   table: offsets[n_paths + 1] int64 (path p's entries are [offsets[p], offsets[p + 1])), then entries uint2 {mask, count}
 *
 * Kernel.  K5's grid (32-row tiles x path ranges, one lane per row, warp-uniform path data), tile staging, per-warp
 * accumulator, epilogue and finishing kernel.  Per path: Fx, then the path's entries as broadcast loads; the per-element sums
 * stay in registers (unrolled to MAXL) and reach my[field][lane] once per path.  W is a table in shared memory: lanes index
 * it by different (a, b), which the constant cache would serialise.  Float64, no atomics, a fixed order: the same batch
 * gives bit-identical results on every run.
 */
#ifndef B2F_TREE_SHAP_INTERVENTIONAL_CUH
#define B2F_TREE_SHAP_INTERVENTIONAL_CUH
#include "tree_shap.cuh"

#define B2F_BG_HIST_LEN 12 /* paths of up to 12 field elements: a histogram of 4 096 counters */

struct VParams {
    SParams s;                /* the path table, with s.denom = its denom * background rows */
    const long long *offsets; /* [n_paths + 1] */
    const uint2 *entries;     /* {mask, count} */
};

__host__ __device__ inline int interv_smem_bytes(int n_fields) { return shap_smem_bytes(n_fields) + B2F_SHAP_TAB_L * B2F_SHAP_TAB_L * 8; }

/* wt[x * 24 + y] = W[x][y] = (x-1)! y! / (x+y)! = 1 / (x C(x+y, y)), W[0][y] = 0: exact integers, one rounding */
__device__ __forceinline__ void interv_weights(double *wt) {
    for (int i = threadIdx.x; i < B2F_SHAP_TAB_L * B2F_SHAP_TAB_L; i += B2F_SHAP_THREADS) {
        const int x = i / B2F_SHAP_TAB_L, y = i % B2F_SHAP_TAB_L;
        unsigned long long c = 1; /* C(x + j, j) */
        for (int j = 1; j <= y; ++j) c = c * (unsigned long long)(x + j) / (unsigned long long)j;
        wt[i] = x == 0 ? 0.0 : 1.0 / ((double)x * (double)c);
    }
}

/* one path for this warp's 32 rows: Fx, the sums over the path's background entries, added into my[field][lane] */
template <int MAXL>
__device__ __forceinline__ void interv_path(const VParams &v, int q, const uint32_t *xs, const double *wt, double *my, int lane) {
    const SParams &p = v.s;
    const uint2 rec = __ldg(reinterpret_cast<const uint2 *>(p.paths + q));
    const double leaf = __ldg(&p.paths[q].leaf);
    const int len = (int)rec.y;
    const b2f_path_elem *E = p.elems + rec.x;
    uint32_t fx = 1u;
#pragma unroll
    for (int l = 1; l < MAXL; ++l)
        if (l < len) {
            uint32_t field;
            double z, iz;
            fx |= (uint32_t)shap_follows(E + l, xs, lane, field, z, iz) << l;
        }
    const uint32_t need = ((1u << len) - 1u) & ~fx; /* B of every entry that counts */
    const int b = __popc(need);
    double sa[MAXL]; /* sa[k]: sum of count * W[a][b] over the entries with element k in A */
#pragma unroll
    for (int k = 0; k < MAXL; ++k) sa[k] = 0.0;
    double sb = 0.0; /* sum of count * W[b][a] over the entries that count */
    const long long e_hi = __ldg(v.offsets + q + 1);
    for (long long j = __ldg(v.offsets + q); j < e_hi; ++j) {
        const uint2 e = __ldg(v.entries + j);
        if ((e.x & need) != need) continue;
        const uint32_t am = fx & ~e.x;
        const int a = __popc(am);
        const double c = (double)e.y;
        sb += c * wt[b * B2F_SHAP_TAB_L + a];
        const double w = c * wt[a * B2F_SHAP_TAB_L + b];
#pragma unroll
        for (int k = 1; k < MAXL; ++k)
            if ((am >> k) & 1u) sa[k] += w;
    }
#pragma unroll
    for (int k = 1; k < MAXL; ++k)
        if (k < len) {
            const uint32_t field = __ldg(&E[k].field);
            my[field * 32 + lane] += (((fx >> k) & 1u) ? sa[k] : -sb) * leaf;
        }
}

/* grid (row tiles, path ranges); dynamic shared memory interv_smem_bytes(F).  Outputs as k_tree_shap's, divided by v.s.denom */
template <int MAXL, bool PACKED>
__global__ void __launch_bounds__(B2F_SHAP_THREADS, 2)
    k_tree_shap_interventional(const __grid_constant__ VParams v, const uint32_t *__restrict__ rows, long long n, double *__restrict__ out,
                               double *__restrict__ partials) {
    extern __shared__ __align__(16) uint8_t interv_smem[];
    const SParams &p = v.s;
    const int F = p.n_cat + p.n_num;
    uint32_t *xs = reinterpret_cast<uint32_t *>(interv_smem);         /* [24][32] imputed row words of the tile */
    double *acc = reinterpret_cast<double *>(interv_smem + 24 * 32 * 4); /* [warps][F][32] */
    double *wt = acc + B2F_SHAP_WARPS * F * 32;                         /* [24][24] */
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = (long long)blockIdx.x * 32;
    shap_stage_tile<PACKED>(p, rows, n, row0, F, xs);
    interv_weights(wt);
    double *my = acc + (size_t)warp * F * 32;
    for (int f = 0; f < F; ++f) my[f * 32 + lane] = 0.0;
    __syncthreads();

    const long long P = p.n_paths, R = gridDim.y, r = blockIdx.y;
    const long long c_lo = P * r / R, c_hi = P * (r + 1) / R;
    const int w_lo = (int)(c_lo + (c_hi - c_lo) * warp / B2F_SHAP_WARPS);
    const int w_hi = (int)(c_lo + (c_hi - c_lo) * (warp + 1) / B2F_SHAP_WARPS);
    for (int q = w_lo; q < w_hi; ++q) interv_path<MAXL>(v, q, xs, wt, my, lane);
    __syncthreads();

    for (int i = threadIdx.x; i < 32 * F; i += B2F_SHAP_THREADS) { /* k_tree_shap's epilogue */
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

/* ------------------------------------------------------------------ building the background table */

/* words[tile][F][32] = the imputed words of background rows tile * 32 + lane (0 past n): K5's staged tile, in global memory */
template <bool PACKED>
__global__ void __launch_bounds__(B2F_SHAP_THREADS) k_background_words(const __grid_constant__ SParams p, const uint32_t *__restrict__ rows,
                                                                       long long n, uint32_t *__restrict__ words) {
    const int F = p.n_cat + p.n_num;
    shap_stage_tile<PACKED>(p, rows, n, (long long)blockIdx.x * 32, F, words + (size_t)blockIdx.x * F * 32);
}

/* One CTA per path (grid-stride).  Counting pass (!FILL): counts[p] = the path's entries.  Fill pass: the entries from
 * v.offsets[p], and moved[p] = leaf * (background rows reaching the leaf / n - prod of its zero fractions): the path's share
 * of base_value's move from the path-dependent expectation to the background mean. */
template <bool FILL>
__global__ void __launch_bounds__(B2F_SHAP_THREADS) k_background_table(const __grid_constant__ VParams v, const uint32_t *__restrict__ words,
                                                                       long long n, long long *__restrict__ counts, uint2 *__restrict__ entries,
                                                                       double *__restrict__ moved) {
    __shared__ uint32_t hist[1 << B2F_BG_HIST_LEN];
    __shared__ int warp_nz[B2F_SHAP_WARPS];
    __shared__ unsigned int reach_rows;
    const SParams &p = v.s;
    const int F = p.n_cat + p.n_num, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int q = blockIdx.x; q < p.n_paths; q += gridDim.x) {
        const uint2 rec = __ldg(reinterpret_cast<const uint2 *>(p.paths + q));
        const int len = (int)rec.y;
        const b2f_path_elem *E = p.elems + rec.x;
        const uint32_t full = (1u << len) - 1u;
        const bool histogram = len - 1 <= B2F_BG_HIST_LEN;
        const int bins = histogram ? 1 << (len - 1) : 0; /* bin = mask >> 1 */
        for (int i = threadIdx.x; i < bins; i += B2F_SHAP_THREADS) hist[i] = 0;
        if (threadIdx.x == 0) reach_rows = 0;
        __syncthreads();
        for (long long r = threadIdx.x; r < n; r += B2F_SHAP_THREADS) {
            const uint32_t *xs = words + (size_t)(r >> 5) * F * 32; /* lane == r & 31 */
            uint32_t m = 1u;
            for (int k = 1; k < len; ++k) {
                uint32_t field;
                double z, iz;
                m |= (uint32_t)shap_follows(E + k, xs, lane, field, z, iz) << k;
            }
            if (histogram) {
                atomicAdd(&hist[m >> 1], 1u);
            } else {
                if (m == full) atomicAdd(&reach_rows, 1u);
                if (FILL) entries[v.offsets[q] + r] = make_uint2(m, 1u);
            }
        }
        __syncthreads();
        long long total = n;
        if (histogram) { /* the non-empty bins in mask order: each thread a contiguous run, an exclusive scan over threads */
            const int per = (bins + B2F_SHAP_THREADS - 1) / B2F_SHAP_THREADS, b0 = min(bins, (int)threadIdx.x * per), b1 = min(bins, b0 + per);
            int mine = 0;
            for (int i = b0; i < b1; ++i) mine += hist[i] != 0u;
            int inc = mine;
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            if (lane == 31) warp_nz[warp] = inc;
            __syncthreads();
            long long before = inc - mine;
            total = 0;
            for (int w = 0; w < B2F_SHAP_WARPS; ++w) {
                if (w < warp) before += warp_nz[w];
                total += warp_nz[w];
            }
            if (FILL) {
                uint2 *dst = entries + v.offsets[q] + before;
                for (int i = b0; i < b1; ++i)
                    if (hist[i]) *dst++ = make_uint2(((uint32_t)i << 1) | 1u, hist[i]);
            }
        }
        if (threadIdx.x == 0) {
            if (!FILL) {
                counts[q] = total;
            } else {
                const unsigned int reach = histogram ? hist[bins - 1] : reach_rows;
                double pz = 1.0;
                for (int k = 1; k < len; ++k) pz *= __ldg(&E[k].zero_fraction);
                moved[q] = __ldg(&p.paths[q].leaf) * ((double)reach / (double)n - pz);
            }
        }
        __syncthreads(); /* hist, warp_nz and reach_rows serve the next path */
    }
}
#endif
