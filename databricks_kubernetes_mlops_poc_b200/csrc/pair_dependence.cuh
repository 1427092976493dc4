/*
 * pair_dependence.cuh -- K10: two-way partial dependence, and its mean over rows on the device (sm_90a).
 *
 * For every row i and every point (u, v) of a probed pair of request fields (a, b), the kernel returns the prediction of
 * row i with row word a replaced by u and row word b by v -- sklearn's two-way `partial_dependence(..., [a, b],
 * method="brute")` `individual` curves.  It is K6's mask walk over two probed words (partial_dependence.cuh pd_mask_walk
 * with TWO = true): each (row, tree, segment of up to 32 points) is one walk with an explicit stack of (node, point
 * mask) that
 *
 *   split on word a       : splits the mask on take_second(u_k)
 *   split on word b       : splits the mask on take_second(v_k)
 *   split on another word : follows the row
 *   leaf                  : adds the payload to every point in the mask
 *
 * Every fork pushes the second child of a node on the current path, so the stack still needs one entry per level (forests
 * deeper than B2F_PD_STACK levels are refused by the host).  A one-way probe puts B2F_PP_NO_WORD in b's place: no node
 * splits on it, and the walk is K6's.
 *
 * k_pair_dependence<PACKED, MEAN>: K6's geometry -- thread = row, warp = 32-row tile, CTA = B2F_PD_WARPS tiles x one
 * segment (blockIdx.y) -- and K6's row staging and imputation.  Every point is a tree-order sum from the GBDT init value,
 * then aggregate(): bit for bit the tile kernel's score of the substituted row.
 *   MEAN = false: out[row][point], as K6.
 *   MEAN = true : the CTA's rows are reduced per point in a fixed order -- a shuffle tree within each warp, then the warps
 *                 in order -- into one partial per (CTA, point), partial[blockIdx.x][point - point0];
 *                 k_pair_dependence_finish sums a point's partials in CTA order and divides by n.
 * No atomics: a point's value depends on nothing but the rows, the forest and its two words, so results are bit-identical
 * from run to run and do not depend on how points are grouped into segments, launches or calls.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "partial_dependence.cuh"

#define B2F_PP_NO_WORD 0xffffffffu /* second word of a one-way probe: no node splits on it */

/* one segment: up to B2F_PD_SEG points of the pair (word_a, word_b) */
struct PpSeg {
    uint32_t word_a;
    uint32_t word_b; /* or B2F_PP_NO_WORD */
    uint32_t count;  /* 1..B2F_PD_SEG */
    uint32_t off;    /* first point: its column in an output row, and its index in the point table (2 words per point) */
};

/* p.grid: the call's point table, (a word, b word) per point, numerics imputed; p.points: doubles per output row (MEAN =
 * false).  segs: this launch's segments (blockIdx.y).  MEAN = false: out[row * p.points + point]; MEAN = true:
 * out[blockIdx.x * group_points + point - point0], the CTA's partial sums of the launch's group of points. */
template <bool PACKED, bool MEAN>
__global__ void __launch_bounds__(B2F_PD_WARPS * 32)
    k_pair_dependence(const __grid_constant__ PdParams p, const PpSeg *__restrict__ segs, const uint32_t *__restrict__ rows, long long n,
                      double *__restrict__ out, int point0, int group_points) {
    __shared__ uint32_t xs[B2F_PD_WARPS][B2F_ROW_WORDS][32];
    __shared__ unsigned long long stk[B2F_PD_STACK][B2F_PD_WARPS * 32];
    __shared__ uint32_t gv[2][B2F_PD_SEG];
    __shared__ double red[MEAN ? B2F_PD_WARPS : 1][MEAN ? B2F_PD_SEG : 1];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const PpSeg sg = segs[blockIdx.y];
    if (threadIdx.x < 2 * B2F_PD_SEG) {
        const int k = threadIdx.x >> 1;
        gv[threadIdx.x & 1][k] = k < (int)sg.count ? p.grid[2 * ((size_t)sg.off + k) + (threadIdx.x & 1)] : 0u;
    }
    const long long row = ((long long)blockIdx.x * B2F_PD_WARPS + warp) * 32 + lane;
    const bool live = row < n;
    pd_stage_row<PACKED>(p, rows, row, live, xs[warp], lane);
    __syncthreads();
    if (!MEAN && !live) return; /* no block-wide barrier below without MEAN */

    const uint32_t full = sg.count >= 32 ? 0xffffffffu : ((1u << sg.count) - 1u);
    double acc[B2F_PD_SEG];
#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) acc[k] = p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? p.init_raw : 0.0;
    if (live) pd_mask_walk<1, true>(p, sg.word_a, full, gv[0], xs[warp], lane, stk, acc, sg.word_b, gv[1]);

#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) {
        double p1 = 0.0;
        if (live && k < (int)sg.count) {
            int lab;
            /* the GBDT init value is already in acc (added first, as sklearn does) */
            aggregate(p.agg_mode, p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? 0.0 : p.init_raw, p.denom, p.threshold, acc[k], p1, lab);
        }
        if constexpr (MEAN) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) p1 += __shfl_down_sync(0xffffffffu, p1, o);
            if (lane == 0) red[warp][k] = p1;
        } else {
            if (k < (int)sg.count) out[row * (long long)p.points + sg.off + k] = p1;
        }
    }
    if constexpr (MEAN) {
        __syncthreads();
        if (threadIdx.x < sg.count) {
            double s = red[0][threadIdx.x];
#pragma unroll
            for (int w = 1; w < B2F_PD_WARPS; ++w) s += red[w][threadIdx.x];
            out[(long long)blockIdx.x * group_points + (sg.off - (uint32_t)point0) + threadIdx.x] = s;
        }
    }
}

/* thread = point of the group: the mean over n rows of its n_cta partial sums, added in CTA order */
__global__ void __launch_bounds__(256)
    k_pair_dependence_finish(const double *__restrict__ partial, int n_cta, int group_points, long long n, double *__restrict__ out) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= group_points) return;
    double s = partial[q];
    for (int c = 1; c < n_cta; ++c) s += partial[(long long)c * group_points + q];
    out[q] = s / (double)n;
}
