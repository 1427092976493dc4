/*
 * counterfactual.cuh -- K7: nearest single-field counterfactuals (sm_90a).
 *
 * For a row x and a probed numeric row word w with the forest's sorted distinct split values t'_0 < ... < t'_{m-1}
 * (forest_rank.h forest_split_values), the float32 line falls into m + 1 pieces, piece k = [t'_{k-1}, t'_k) with
 * t'_{-1} = -inf and t'_m = +inf.  Every value of a piece walks every tree the same way (x <= thr <=> x < t'), so the row
 * scores the same anywhere in it.  The row's own piece is j = #{t' <= x} (x as scored: NaN imputed; an unordered x takes
 * every second child, so it counts as beyond every split value).  The decision of a piece is p1 > cutoff.  Per (row,
 * probed word) the kernels find the nearest piece below and above j whose decision differs from piece j's:
 *     upper = t'_{k-1}          for the least k > j that flips  (the smallest float32 above x that flips)
 *     lower = nextdown(t'_k)    for the greatest k < j that flips (the largest float32 below x that flips)
 *
 * k_counterfactual scores every piece of every probed word with K6's mask walk (partial_dependence.cuh pd_mask_walk, the
 * same device function): thread = row, warp = 32-row tile, CTA = B2F_PD_WARPS tiles x one segment (blockIdx.y) of up to
 * 32 consecutive pieces of one word.  A piece's point is its representative, t'_{k-1} (nextdown(t'_0) for piece 0), read
 * from the model's split-value table in HBM.  Each thread finds its own j by binary search in the same table.  The
 * epilogue turns the 32 accumulators into p1 with aggregate() -- the tile kernel's order, so each p1 is bit for bit the
 * tile kernel's score of the row with the word set to the representative -- and writes one 32-byte CfCand per (row,
 * segment) to scratch; no curve leaves the kernel.  The row's decision need not be known there: a segment wholly below
 * (above) j records, for each decision, its greatest (least) piece of that decision; the segment holding j records p1_j
 * and its own nearest flips on both sides.
 *
 * k_counterfactual_finish (thread = row, blockIdx.y = probed word) starts from the segment holding j, takes the
 * decision p1_j > cutoff, and walks the word's other segments outwards, in fixed order, to the first one holding a piece
 * of the other decision.  No atomics: results are bit-identical from run to run and a row's results depend on nothing
 * but the row, the forest, the words and the cutoff.
 */
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "partial_dependence.cuh"

#define B2F_CF_MAX_WORDS 23 /* probed words per call */
#define B2F_CF_TAB_HEAD 48  /* uint32 words ahead of the split values in the device table: offset[24], count[24] */

/* one (row, segment) candidate.  Segment below j: (k[c], p[c]) = its greatest piece of decision c (k = -1: none).
 * Segment above j: its least piece of decision c.  Segment holding j: k[0] / k[1] = its greatest flip below j / least flip
 * above j, with their p1 in p[0] / p[1], and p[2] = p1_j. */
struct CfCand {
    double p[3];
    int32_t k[2];
};

struct CfParams {
    PdParams pd;         /* the forest (segs, grid and points unused) */
    const uint32_t *tab; /* device split-value table: offset[24], count[24] per row word, then the float32 values */
    double cutoff;
    int32_t n_words;     /* probed words of the call */
    int32_t seg_base;    /* segment of blockIdx.y = 0 (a call's segments may take several launches) */
    uint32_t word[B2F_CF_MAX_WORDS];
    uint32_t seg0[B2F_CF_MAX_WORDS + 1]; /* first segment of each probed word; seg0[n_words] = the call's segment count */
};

/* j = #{t' <= x}, an unordered x past every t' (take_second sends it to the second child at every split) */
__device__ __forceinline__ int cf_piece(const float *v, int count, float x) {
    int lo = 0, hi = count;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (x < v[mid])
            hi = mid;
        else
            lo = mid + 1;
    }
    return lo;
}

template <bool PACKED>
__global__ void __launch_bounds__(B2F_PD_WARPS * 32)
    k_counterfactual(const __grid_constant__ CfParams p, const uint32_t *__restrict__ rows, long long n, CfCand *__restrict__ cand) {
    __shared__ uint32_t xs[B2F_PD_WARPS][B2F_ROW_WORDS][32];
    __shared__ unsigned long long stk[B2F_PD_STACK][B2F_PD_WARPS * 32];
    __shared__ uint32_t gv[B2F_PD_SEG];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int seg = p.seg_base + (int)blockIdx.y;
    int f = 0;
    while (f + 1 < p.n_words && (int)p.seg0[f + 1] <= seg) ++f;
    const uint32_t word = p.word[f];
    const int first = (seg - (int)p.seg0[f]) * B2F_PD_SEG; /* the segment's first piece */
    const int m = (int)__ldg(p.tab + B2F_ROW_WORDS + word);
    const float *v = reinterpret_cast<const float *>(p.tab + B2F_CF_TAB_HEAD) + __ldg(p.tab + word);
    const int count = min(B2F_PD_SEG, m + 1 - first);
    if (threadIdx.x < B2F_PD_SEG) {
        uint32_t g = 0u;
        if ((int)threadIdx.x < count) {
            const int k = first + (int)threadIdx.x;
            /* piece 0 of a word no node splits on: any value scores the same; 0 */
            g = __float_as_uint(k == 0 ? (m > 0 ? nextafterf(__ldg(v), -INFINITY) : 0.0f) : __ldg(v + k - 1));
        }
        gv[threadIdx.x] = g;
    }
    const long long row = ((long long)blockIdx.x * B2F_PD_WARPS + warp) * 32 + lane;
    const bool live = row < n;
    pd_stage_row<PACKED>(p.pd, rows, row, live, xs[warp], lane);
    __syncthreads();
    if (!live) return; /* no block-wide barrier below */

    const uint32_t full = count >= 32 ? 0xffffffffu : ((1u << count) - 1u);
    double acc[B2F_PD_SEG];
#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) acc[k] = p.pd.agg_mode == B2F_AGG_GBDT_LOGISTIC ? p.pd.init_raw : 0.0;
    pd_mask_walk(p.pd, word, full, gv, xs[warp], lane, stk, acc);

    const int j = cf_piece(v, m, __uint_as_float(xs[warp][word][lane]));
    int kb[2] = {-1, -1}, ka[2] = {-1, -1}; /* greatest piece below j / least piece above j, per decision */
    double pb[2] = {0.0, 0.0}, pa[2] = {0.0, 0.0}, pj = 0.0;
#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) {
        if (k < count) {
            double p1;
            int lab;
            aggregate(p.pd.agg_mode, p.pd.agg_mode == B2F_AGG_GBDT_LOGISTIC ? 0.0 : p.pd.init_raw, p.pd.denom, p.pd.threshold, acc[k], p1, lab);
            const int K = first + k, d = p1 > p.cutoff ? 1 : 0;
            if (K < j) {
                kb[d] = K, pb[d] = p1;
            } else if (K > j) {
                if (ka[d] < 0) ka[d] = K, pa[d] = p1;
            } else {
                pj = p1;
            }
        }
    }
    CfCand c;
    if (j >= first && j < first + count) {
        const int o = pj > p.cutoff ? 0 : 1; /* the other decision */
        c.p[0] = pb[o], c.k[0] = kb[o];
        c.p[1] = pa[o], c.k[1] = ka[o];
        c.p[2] = pj;
    } else if (j >= first + count) {
        c.p[0] = pb[0], c.p[1] = pb[1], c.k[0] = kb[0], c.k[1] = kb[1], c.p[2] = 0.0;
    } else {
        c.p[0] = pa[0], c.p[1] = pa[1], c.k[0] = ka[0], c.k[1] = ka[1], c.p[2] = 0.0;
    }
    cand[(long long)seg * n + row] = c; /* [segment][row]: a warp's 32 records are contiguous */
}

/* out: b2f_counterfactual records (include/b2f.h), row r's probe f at byte r * out_stride + f * 32; proba (may be NULL):
 * row r's p1 at byte r * proba_stride */
template <bool PACKED>
__global__ void __launch_bounds__(128)
    k_counterfactual_finish(const __grid_constant__ CfParams p, const uint32_t *__restrict__ rows, long long n, const CfCand *__restrict__ cand,
                            uint8_t *__restrict__ out, long long out_stride, uint8_t *__restrict__ proba, long long proba_stride) {
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int f = (int)blockIdx.y;
    if (row >= n) return;
    const uint32_t word = p.word[f];
    uint32_t xb = PACKED ? __ldg(rows + row * B2F_PACKED_ROW_WORDS + 2 + (word - (uint32_t)p.pd.n_cat)) : __ldg(rows + row * B2F_ROW_WORDS + word);
    if (isnan(__uint_as_float(xb))) xb = __float_as_uint(p.pd.impute[word]);
    const float x = __uint_as_float(xb);
    const int m = (int)__ldg(p.tab + B2F_ROW_WORDS + word);
    const float *v = reinterpret_cast<const float *>(p.tab + B2F_CF_TAB_HEAD) + __ldg(p.tab + word);
    const int j = cf_piece(v, m, x);
    const int s0 = (int)p.seg0[f], s1 = (int)p.seg0[f + 1], sj = s0 + j / B2F_PD_SEG;
    const CfCand c = cand[(long long)sj * n + row];
    const int o = c.p[2] > p.cutoff ? 0 : 1; /* the other decision */
    int klo = c.k[0], khi = c.k[1];
    double plo = c.p[0], phi = c.p[1];
    for (int s = sj - 1; s >= s0 && klo < 0; --s) {
        const CfCand b = cand[(long long)s * n + row];
        klo = b.k[o], plo = b.p[o];
    }
    for (int s = sj + 1; s < s1 && khi < 0; ++s) {
        const CfCand b = cand[(long long)s * n + row];
        khi = b.k[o], phi = b.p[o];
    }
    double *r = reinterpret_cast<double *>(out + row * out_stride + (long long)f * 32);
    r[0] = klo >= 0 ? plo : __longlong_as_double(0x7ff8000000000000ll);
    r[1] = khi >= 0 ? phi : __longlong_as_double(0x7ff8000000000000ll);
    float *rf = reinterpret_cast<float *>(r + 2);
    rf[0] = klo >= 0 ? nextafterf(__ldg(v + klo), -INFINITY) : __int_as_float(0x7fc00000);
    rf[1] = khi >= 0 ? __ldg(v + khi - 1) : __int_as_float(0x7fc00000);
    rf[2] = x;
    reinterpret_cast<int32_t *>(rf)[3] = 0;
    if (f == 0 && proba) *reinterpret_cast<double *>(proba + row * proba_stride) = c.p[2];
}
