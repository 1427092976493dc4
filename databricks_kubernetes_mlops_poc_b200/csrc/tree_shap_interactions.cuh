/*
 * tree_shap_interactions.cuh -- K5b: exact path-dependent TreeSHAP interaction values per pair of request fields
 * (Lundberg et al., arXiv:1802.03888 §4, the Shapley interaction index) over the same path table as K5 (forest_paths.h).
 *
 * Per path of d merged elements the game is a product game and fields off the path are null players, so the pair term of
 * two elements a != b is  leaf (o_a - z_a)(o_b - z_b) / 2 * sum_{S in P\{a,b}} |S|!(d-2-|S|)!/(d-1)! prod_S o prod_rest z:
 * UNWIND a out of the EXTEND polynomial pw (the w[] below, also giving phi_a as K5 does), then K5's closed-form unwound sum
 * of b over w[].  Each unordered pair is computed once, by the owner of its lower field, and stored for both orders: every
 * matrix is exactly symmetric.  Float64 throughout, no division (c_shap_tab and inv_zero_fraction, as K5).
 *
 * Work split.  A CTA of B2F_SHAP_WARPS warps owns one tile of 32 rows (lane = row) and one contiguous range of paths.  Its
 * shared accumulator holds the upper triangle plus diagonal of the F x F matrix per row ([F(F+1)/2][32] doubles, 70 656 B
 * for F = 23), too large for K5's accumulator per warp.  Instead each warp owns a fixed set of fields (IParams::own, chosen
 * on the host to balance the pair work): the owner of field a alone writes slot (a, a) -- phi_a during the walk -- and the
 * slots (a, b), b > a.  Every warp walks every path of the range in order, skips a path that holds none of its fields (a
 * warp-uniform test), and otherwise runs EXTEND and conditions on its own elements.  So no atomics and no barrier per path.
 *
 * Epilogue (one range): after one __syncthreads the diagonal becomes phi_a - sum_{b != a} Phi_ab (b ascending), then the
 * triangle is expanded to the row-major F x F matrix / denom with consecutive threads storing consecutive doubles.  Several
 * ranges: each CTA writes its raw triangle to partials[range][row][F(F+1)/2] and k_tree_shap_interactions_finish adds the
 * ranges in range order before the same epilogue.  The same batch gives bit-identical results on every run.
 */
#ifndef B2F_TREE_SHAP_INTERACTIONS_CUH
#define B2F_TREE_SHAP_INTERACTIONS_CUH
#include "tree_shap.cuh"

struct IParams {
    SParams s;
    uint32_t own[B2F_SHAP_WARPS]; /* bit f: this warp owns field f */
};

__host__ __device__ inline int inter_slots(int F) { return F * (F + 1) / 2; }
/* slot of (a, b), a <= b: row a of the upper triangle */
__host__ __device__ inline int inter_slot(int F, int a, int b) { return a * F - a * (a - 1) / 2 + (b - a); }
__host__ __device__ inline int inter_smem_bytes(int n_fields) { return 24 * 32 * 4 + inter_slots(n_fields) * 32 * 8; }

/* t[slot * LD + col]: slot (a, a) holds phi_a on entry and Phi_aa = phi_a - sum_{b != a} Phi_ab on return.  Reads only
 * off-diagonal slots, so threads of different a may run it at once. */
template <int LD>
__device__ __forceinline__ void inter_diagonal(double *t, int F, int a, int col) {
    double s = t[inter_slot(F, a, a) * LD + col];
    for (int b = 0; b < F; ++b)
        if (b != a) s -= t[inter_slot(F, b < a ? b : a, b < a ? a : b) * LD + col];
    t[inter_slot(F, a, a) * LD + col] = s;
}

/* one path for this warp's 32 rows: EXTEND, then per own element a: UNWIND a (phi_a) and the unwound sum of every element
 * b of a higher field (Phi_ab), added into acc[slot][lane] */
template <int MAXL>
__device__ __forceinline__ void inter_path(const IParams &ip, uint32_t own, int q, const uint32_t *xs, double *acc, int lane) {
    const SParams &p = ip.s;
    const int F = p.n_cat + p.n_num;
    const uint2 rec = __ldg(reinterpret_cast<const uint2 *>(p.paths + q));
    const int len = (int)rec.y;
    const b2f_path_elem *E = p.elems + rec.x;
    uint32_t held = 0;
    for (int k = 1; k < len; ++k) held |= 1u << __ldg(&E[k].field);
    if (!(held & own)) return;
    const double leaf = __ldg(&p.paths[q].leaf);
    double pw[MAXL];
    uint32_t ones;
    const double last = shap_extend(E, len, xs, lane, pw, ones);
    const int d = len - 1;
    for (int ka = 1; ka < len; ++ka) {
        const uint32_t fa = __ldg(&E[ka].field);
        if (!((own >> fa) & 1u)) continue;
        const double2 za = __ldg(reinterpret_cast<const double2 *>(E + ka) + 2);
        const bool oa = (ones >> ka) & 1u;
        double w[MAXL - 1]; /* pw with a unwound (d entries) */
        const double tot = shap_unwound_sum<true>(pw, d, last, oa, za.x, za.y, w);
        const double ga = ((oa ? 1.0 : 0.0) - za.x) * leaf;
        acc[inter_slot(F, (int)fa, (int)fa) * 32 + lane] += tot * ga;
        const double ha = 0.5 * ga;
        const int e = d - 1; /* w holds e + 1 entries */
        const double wlast = shap_pick(w, e);
        for (int kb = 1; kb < len; ++kb) {
            const uint32_t fb = __ldg(&E[kb].field);
            if (fb <= fa) continue; /* the pair belongs to the owner of the lower field; fa itself is met once */
            const double2 zb = __ldg(reinterpret_cast<const double2 *>(E + kb) + 2);
            const bool ob = (ones >> kb) & 1u;
            const double t = shap_unwound_sum<false>(w, e, wlast, ob, zb.x, zb.y);
            acc[inter_slot(F, (int)fa, (int)fb) * 32 + lane] += t * ha * ((ob ? 1.0 : 0.0) - zb.x);
        }
    }
}

/* CTAs per SM the register budget is cut for: three fit the 9-element bucket in 80 registers without spills.  The 16-element
 * bucket still spills at 128 (two CTAs), so the longer buckets take one CTA per SM and no spills (ptxas report in DESIGN.md K5b) */
template <int MAXL>
struct InterBlocks {
    static constexpr int value = MAXL <= 9 ? 3 : 1;
};

/* grid (row tiles, path ranges); dynamic shared memory inter_smem_bytes(F).  One range: out[row][a][b] = Phi_ab; several:
 * partials[range][row][slot] = the range's raw triangle (k_tree_shap_interactions_finish completes them) */
template <int MAXL, bool PACKED>
__global__ void __launch_bounds__(B2F_SHAP_THREADS, InterBlocks<MAXL>::value)
    k_tree_shap_interactions(const __grid_constant__ IParams ip, const uint32_t *__restrict__ rows, long long n, double *__restrict__ out,
                             double *__restrict__ partials) {
    extern __shared__ __align__(16) uint8_t inter_smem[];
    const SParams &p = ip.s;
    const int F = p.n_cat + p.n_num, T = inter_slots(F);
    uint32_t *xs = reinterpret_cast<uint32_t *>(inter_smem);           /* [24][32] imputed row words of the tile */
    double *acc = reinterpret_cast<double *>(inter_smem + 24 * 32 * 4); /* [T][32] */
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = (long long)blockIdx.x * 32;
    shap_stage_tile<PACKED>(p, rows, n, row0, F, xs);
    for (int i = threadIdx.x; i < 32 * T; i += B2F_SHAP_THREADS) acc[i] = 0.0;
    __syncthreads();

    const long long P = p.n_paths, R = gridDim.y, r = blockIdx.y;
    const int c_lo = (int)(P * r / R), c_hi = (int)(P * (r + 1) / R);
    const uint32_t own = ip.own[warp];
    if (own)
        for (int q = c_lo; q < c_hi; ++q) inter_path<MAXL>(ip, own, q, xs, acc, lane);
    __syncthreads();

    const long long rows_here = n - row0 < 32 ? n - row0 : 32;
    if (R > 1) {
        for (int i = threadIdx.x; i < 32 * T; i += B2F_SHAP_THREADS) {
            const int s = i / 32, c = i & 31;
            if (c < rows_here) partials[((size_t)r * (size_t)n + (size_t)(row0 + c)) * T + s] = acc[s * 32 + c];
        }
        return;
    }
    for (int i = threadIdx.x; i < 32 * F; i += B2F_SHAP_THREADS) inter_diagonal<32>(acc, F, i >> 5, i & 31);
    __syncthreads();
    const int FF = F * F;
    double *o = out + row0 * FF;
    for (long long i = threadIdx.x; i < rows_here * FF; i += B2F_SHAP_THREADS) {
        const int c = (int)(i / FF), ab = (int)(i - (long long)c * FF), a = ab / F, b = ab - a * F;
        o[i] = acc[inter_slot(F, a < b ? a : b, a < b ? b : a) * 32 + c] / p.denom;
    }
}

/* one CTA per row: its triangle = sum over ranges in range order, then the diagonal, then out[row] = the F x F matrix / denom;
 * dynamic shared memory T doubles */
__global__ void __launch_bounds__(256) k_tree_shap_interactions_finish(const double *__restrict__ partials, int ranges, long long n, int F,
                                                                      double denom, double *__restrict__ out) {
    extern __shared__ __align__(16) uint8_t inter_fin_smem[];
    double *t = reinterpret_cast<double *>(inter_fin_smem);
    const int T = inter_slots(F);
    for (long long row = blockIdx.x; row < n; row += gridDim.x) {
        for (int s = threadIdx.x; s < T; s += blockDim.x) {
            double v = 0.0;
            for (int r = 0; r < ranges; ++r) v += partials[((size_t)r * (size_t)n + (size_t)row) * T + s];
            t[s] = v;
        }
        __syncthreads();
        for (int a = threadIdx.x; a < F; a += blockDim.x) inter_diagonal<1>(t, F, a, 0);
        __syncthreads();
        for (int ab = threadIdx.x; ab < F * F; ab += blockDim.x) {
            const int a = ab / F, b = ab - a * F;
            out[row * F * F + ab] = t[inter_slot(F, a < b ? a : b, a < b ? b : a)] / denom;
        }
        __syncthreads();
    }
}
#endif
