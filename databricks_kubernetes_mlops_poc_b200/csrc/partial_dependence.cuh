/*
 * partial_dependence.cuh -- K6: one-way partial dependence and ICE curves (sm_90a).
 *
 * For every row i and every grid point g of a probed request field, the kernel returns the prediction of row i with that
 * field's row word replaced by the grid point's encoded word -- sklearn's `partial_dependence(..., method="brute")`
 * `individual` curves.  No point gets a walk of its own: each (row, tree, segment of up to 32 grid points) is one walk
 * that forks only at splits on the probed word, with an explicit stack of (node, point mask), so every node is visited at
 * most once per (row, tree, segment).
 *
 *   split on another word : follow the row, as the predict kernels do (in-kernel median imputation, take_second)
 *   split on the probed word: split the mask -- the points for which take_second holds go to the second child
 *   leaf                  : add the payload to every point in the mask
 *
 * Geometry: thread = row, warp = 32-row tile, CTA = B2F_PD_WARPS tiles x one segment (blockIdx.y).  The forest is read
 * from the blob in HBM (forest_blob.h), which stays in L2/L1: every lane of a warp walks the same tree.  The tile's rows
 * sit transposed in shared memory (xs[word][lane], as k_forest_predict_tile), the segment's grid words in a 32-word
 * broadcast table, the walk stacks in shared memory ([depth][thread], conflict-free).  The 32 float64 accumulators of a
 * thread are registers: a leaf adds to them with 32 predicated adds, which costs less than looping over the mask's bits
 * for the one to three leaves a walk usually reaches.
 *
 * Arithmetic: every point's payloads are added in tree order, from the GBDT init value (or 0), then aggregate() -- the
 * tile kernel's order -- so a point equals, bit for bit, k_forest_predict_tile on the row with the word replaced.  No
 * atomics; a row's outputs depend on nothing but the row, the forest and the grid.
 *
 * The mask walk is pd_mask_walk, which K7 (counterfactual.cuh) calls as well.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "forest_predict.cuh"

#define B2F_PD_SEG 32      /* grid points per walk: one 32-bit mask */
#define B2F_PD_WARPS 4     /* row tiles per CTA */
#define B2F_PD_STACK 32    /* walk stack entries per thread: deepest tree the kernel takes */

/* one segment of a probe's grid: up to B2F_PD_SEG points of row word `word` */
struct PdSeg {
    uint32_t word;
    uint32_t count;   /* 1..B2F_PD_SEG */
    uint32_t off;     /* first point: its column in an output row, and its index in PdParams::grid */
    uint32_t pad;
};

struct PdParams {
    const uint8_t *chunks;   /* device: the forest blob's first chunk */
    const PdSeg *segs;       /* device: blockIdx.y -> segment */
    const uint32_t *grid;    /* device: every point's word, in output order; numerics already imputed */
    int32_t n_groups;
    int32_t agg_mode;
    int32_t n_cat;
    int32_t n_num;
    int32_t points; /* doubles per output row: the call's total grid points */
    int32_t pad;
    double init_raw;
    double denom;
    double threshold;
    float impute[24];
    uint32_t g_off[B2F_MAX_GROUPS];   /* chunk byte offset of each tree group */
    uint32_t g_slots[B2F_MAX_GROUPS]; /* node slots per tree: the leaf area follows */
    uint32_t g_trees[B2F_MAX_GROUPS]; /* real trees of the group */
};

/* Stage this lane's row into xw[word][lane] (its warp's tile): decode, impute the numerics, sentinel above the fields
 * (k_forest_predict_tile's staging).  A dead lane stages sentinels.  k_partial_dependence keeps its own inline copy of
 * these lines: through this function its SASS would change (same work, another instruction schedule). */
template <bool PACKED>
__device__ __forceinline__ void pd_stage_row(const PdParams &p, const uint32_t *__restrict__ rows, long long row, bool live,
                                             uint32_t (*xw)[32], int lane) {
    uint32_t w[B2F_ROW_WORDS];
#pragma unroll
    for (int k = 0; k < B2F_ROW_WORDS; ++k) w[k] = B2F_SENTINEL_BITS;
    if (live) {
        if constexpr (PACKED) {
            const uint4 *src = reinterpret_cast<const uint4 *>(rows + row * B2F_PACKED_ROW_WORDS);
            uint32_t q[B2F_PACKED_ROW_WORDS];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint4 v = __ldg(src + k);
                q[4 * k + 0] = v.x, q[4 * k + 1] = v.y, q[4 * k + 2] = v.z, q[4 * k + 3] = v.w;
            }
            const unsigned long long codes = (((unsigned long long)q[1]) << 32) | q[0];
#pragma unroll
            for (int k = 0; k < 9; ++k) w[k] = ((uint32_t)(codes >> (7 * k)) & 0x7fu) - 1u;
#pragma unroll
            for (int k = 0; k < 14; ++k) w[9 + k] = q[2 + k];
        } else {
            const uint4 *src = reinterpret_cast<const uint4 *>(rows + row * B2F_ROW_WORDS);
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const uint4 v = __ldg(src + k);
                w[4 * k + 0] = v.x, w[4 * k + 1] = v.y, w[4 * k + 2] = v.z, w[4 * k + 3] = v.w;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < B2F_ROW_WORDS; ++k) {
        uint32_t v = w[k];
        if (k >= p.n_cat && k < p.n_cat + p.n_num && isnan(__uint_as_float(v))) v = __float_as_uint(p.impute[k]);
        if (k >= (int)B2F_SENTINEL_WORD) v = B2F_SENTINEL_BITS;
        xw[k][lane] = v;
    }
}

/* The mask walk: acc[k] += every leaf payload that point k of a segment reaches, tree by tree in tree order.  One walk per
 * (row, tree) forks only at splits on row word `word`, with gv[k * PSTRIDE] (shared) the word point k puts there and `full`
 * the mask of the segment's points; xw = the warp's staged rows; stk = the block's walk stacks, column threadIdx.x this
 * thread's.  PSTRIDE = 1: one point table for the block (K6, K7); K8 passes its thread's column of a per-thread table. */
template <int PSTRIDE = 1>
__device__ __forceinline__ void pd_mask_walk(const PdParams &p, uint32_t word, uint32_t full, const uint32_t *gv, const uint32_t (*xw)[32],
                                             int lane, unsigned long long (*stk)[B2F_PD_WARPS * 32], double (&acc)[B2F_PD_SEG]) {
    for (int g = 0; g < p.n_groups; ++g) {
        const uint8_t *chunk = p.chunks + p.g_off[g];
        const size_t leaf_area = (size_t)p.g_slots[g] * B2F_NODE_STRIDE;
        const int n_trees = (int)p.g_trees[g];
        for (int l = 0; l < n_trees; ++l) { /* tree 32 g + l: tree order */
            const uint8_t *nodes = chunk + l * 8;
            uint32_t node = 0, mask = full;
            int sp = 0;
            while (true) {
                const uint2 tm = __ldg(reinterpret_cast<const uint2 *>(nodes + (size_t)node * B2F_NODE_STRIDE));
                const uint32_t first = tm.y & B2F_META_SLOT_MASK;
                if (first == node) { /* a leaf is the only node that is its own first child */
                    const double v = __ldg(reinterpret_cast<const double *>(nodes + leaf_area + (size_t)tm.x * B2F_NODE_STRIDE));
#pragma unroll
                    for (int k = 0; k < B2F_PD_SEG; ++k)
                        if ((mask >> k) & 1u) acc[k] += v;
                    if (sp == 0) break;
                    const unsigned long long e = stk[--sp][threadIdx.x];
                    node = (uint32_t)e;
                    mask = (uint32_t)(e >> 32);
                    continue;
                }
                const uint32_t feat = tm.y >> B2F_META_FEAT_SHIFT;
                if (feat == word) {
                    uint32_t sec = 0;
#pragma unroll
                    for (int k = 0; k < B2F_PD_SEG; ++k) sec |= (take_second(gv[k * PSTRIDE], tm.x, tm.y) ? 1u : 0u) << k;
                    const uint32_t m2 = mask & sec, m1 = mask & ~sec;
                    if (m1 && m2) { /* fork: the second child waits on the stack */
                        stk[sp++][threadIdx.x] = ((unsigned long long)m2 << 32) | (first + 1u);
                        node = first;
                        mask = m1;
                    } else {
                        node = first + (m2 ? 1u : 0u);
                    }
                } else {
                    node = first + (take_second(xw[feat][lane], tm.x, tm.y) ? 1u : 0u);
                }
            }
        }
    }
}

template <bool PACKED>
__global__ void __launch_bounds__(B2F_PD_WARPS * 32)
    k_partial_dependence(const __grid_constant__ PdParams p, const uint32_t *__restrict__ rows, long long n, double *__restrict__ out) {
    __shared__ uint32_t xs[B2F_PD_WARPS][B2F_ROW_WORDS][32];
    __shared__ unsigned long long stk[B2F_PD_STACK][B2F_PD_WARPS * 32];
    __shared__ uint32_t gv[B2F_PD_SEG];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const PdSeg sg = p.segs[blockIdx.y];
    if (threadIdx.x < B2F_PD_SEG) gv[threadIdx.x] = threadIdx.x < sg.count ? p.grid[sg.off + threadIdx.x] : 0u;
    const long long row = ((long long)blockIdx.x * B2F_PD_WARPS + warp) * 32 + lane;
    const bool live = row < n;
    /* stage this lane's row: decode, impute, sentinel above the fields (k_forest_predict_tile's staging) */
    {
        uint32_t w[B2F_ROW_WORDS];
#pragma unroll
        for (int k = 0; k < B2F_ROW_WORDS; ++k) w[k] = B2F_SENTINEL_BITS;
        if (live) {
            if constexpr (PACKED) {
                const uint4 *src = reinterpret_cast<const uint4 *>(rows + row * B2F_PACKED_ROW_WORDS);
                uint32_t q[B2F_PACKED_ROW_WORDS];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint4 v = __ldg(src + k);
                    q[4 * k + 0] = v.x, q[4 * k + 1] = v.y, q[4 * k + 2] = v.z, q[4 * k + 3] = v.w;
                }
                const unsigned long long codes = (((unsigned long long)q[1]) << 32) | q[0];
#pragma unroll
                for (int k = 0; k < 9; ++k) w[k] = ((uint32_t)(codes >> (7 * k)) & 0x7fu) - 1u;
#pragma unroll
                for (int k = 0; k < 14; ++k) w[9 + k] = q[2 + k];
            } else {
                const uint4 *src = reinterpret_cast<const uint4 *>(rows + row * B2F_ROW_WORDS);
#pragma unroll
                for (int k = 0; k < 6; ++k) {
                    const uint4 v = __ldg(src + k);
                    w[4 * k + 0] = v.x, w[4 * k + 1] = v.y, w[4 * k + 2] = v.z, w[4 * k + 3] = v.w;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < B2F_ROW_WORDS; ++k) {
            uint32_t v = w[k];
            if (k >= p.n_cat && k < p.n_cat + p.n_num && isnan(__uint_as_float(v))) v = __float_as_uint(p.impute[k]);
            if (k >= (int)B2F_SENTINEL_WORD) v = B2F_SENTINEL_BITS;
            xs[warp][k][lane] = v;
        }
    }
    __syncthreads();
    if (!live) return; /* no block-wide barrier below */

    const uint32_t full = sg.count >= 32 ? 0xffffffffu : ((1u << sg.count) - 1u);
    double acc[B2F_PD_SEG];
#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) acc[k] = p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? p.init_raw : 0.0;
    pd_mask_walk(p, sg.word, full, gv, xs[warp], lane, stk, acc);

    double *o = out + row * (long long)p.points + sg.off;
#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) {
        if (k < (int)sg.count) {
            double p1;
            int lab;
            /* the GBDT init value is already in acc (added first, as sklearn does) */
            aggregate(p.agg_mode, p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? 0.0 : p.init_raw, p.denom, p.threshold, acc[k], p1, lab);
            o[k] = p1;
        }
    }
}
