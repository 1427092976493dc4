/*
 * ale.cuh -- K12: accumulated local effects of numeric request fields, summed per bin on the device (sm_90a).
 *
 * For every row i and every probed numeric field j whose value x_ij is present, the row is scored twice: with the field
 * set to the lower edge z_{k-1} and to the upper edge z_k of its own bin k = clamp(#{z < x_ij}, 1, K).  The kernel returns,
 * per (field, bin), the sum of f(upper) - f(lower) over the bin's rows and the number of those rows.
 *
 * One walk per (row, tree, segment of up to B2F_ALE_SEG_PROBES fields) carries all 2 x (fields) points of the row at once;
 * point 2j is field j's lower edge, point 2j + 1 its upper edge, and each point substitutes its own word:
 *
 *   split on a probed word s (field j) : points of other fields go with the row (take_second(x_s)), point 2j by
 *                                        take_second(lower_j), point 2j + 1 by take_second(upper_j); the mask forks
 *   split on another word               : every point follows the row
 *   leaf                                : add the payload to every point in the mask
 *
 * Every fork still pushes the second child of a node on the current path, so the stack needs one entry per level (forests
 * deeper than B2F_PD_STACK are refused by the host).  Each point's payloads are added in tree order from the GBDT init
 * value, then aggregate(): bit for bit the tile kernel's score of the substituted row.  A row whose field is missing
 * (NaN before imputation) leaves that field's two points out of its mask; its other missing numerics are imputed.
 *
 * k_ale<PACKED>: K6's geometry -- thread = row, warp = 32-row tile, CTA = B2F_PD_WARPS tiles x one segment (blockIdx.y)
 * -- and K6's row staging (pd_stage_row).  Shared memory: the staged rows, the walk stacks, and each row's bin per field
 * (as the index of its lower edge in the call's edge table).  Before the walk the stack area holds the segment's edges for
 * the bin search (binary search over float32 edges); after it, each row's delta per field (NaN: the row takes no part).
 *
 * Reduction order (no atomics): a CTA's partial of (field, bin) is the sum of its rows' deltas in that bin in row order,
 * from 0.0; k_ale_finish adds a bin's CTA partials in CTA order to a running sum from 0.0 (launches over pieces of the
 * rows continue the same sum).  A bin's result depends only on the rows, the forest and that field's edges: not on the
 * device, the run, the piece size or the other fields of the call.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "partial_dependence.cuh"

#define B2F_ALE_SEG_PROBES 16 /* fields per walk: two points each, one 32-bit mask */

/* one probed field of a segment: row word, first edge in the call's edge table, bins K, first bin in the call's output */
struct AleProbe {
    uint32_t word;
    uint32_t eoff;
    uint32_t bins;
    uint32_t boff;
};

/* one segment: up to B2F_ALE_SEG_PROBES fields in ascending word order (field j of a probed word w is the number of
 * probed words below w), their words as a bit mask, and the segment's bins */
struct AleSeg {
    uint32_t count;
    uint32_t words; /* bit w: row word w is probed here */
    uint32_t bins;  /* sum of the fields' bins */
    uint32_t pad;
    AleProbe p[B2F_ALE_SEG_PROBES];
};

/* the multi-word mask walk: acc[k] += every leaf payload point k reaches, tree by tree in tree order.  probed: bit w set
 * for each probed row word w, ascending (the field of word w is popc(probed below w)); full: the points this row takes
 * part with; lower[j] = the index in `edges` of field j's lower edge for this thread's row (its upper edge follows it).  The edges
 * are read from global memory (L1-resident): per-thread edge words in shared memory would not fit beside the stacks. */
__device__ __forceinline__ void ale_mask_walk(const PdParams &p, uint32_t probed, uint32_t full, const uint16_t (*lower)[B2F_PD_WARPS * 32],
                                              const float *__restrict__ edges, const uint32_t (*xw)[32], int lane,
                                              unsigned long long (*stk)[B2F_PD_WARPS * 32], double (&acc)[B2F_PD_SEG]) {
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
                const bool row_second = take_second(xw[feat][lane], tm.x, tm.y);
                if ((probed >> feat) & 1u) {
                    const int j = __popc(probed & ((1u << feat) - 1u));
                    const uint32_t e = lower[j][threadIdx.x];
                    const uint32_t own = 3u << (2 * j);
                    const uint32_t sec = (row_second ? ~own : 0u) | (take_second(__float_as_uint(__ldg(edges + e)), tm.x, tm.y) ? 1u << (2 * j) : 0u) |
                                         (take_second(__float_as_uint(__ldg(edges + e + 1)), tm.x, tm.y) ? 2u << (2 * j) : 0u);
                    const uint32_t m2 = mask & sec, m1 = mask & ~sec;
                    if (m1 && m2) { /* fork: the second child waits on the stack */
                        stk[sp++][threadIdx.x] = ((unsigned long long)m2 << 32) | (first + 1u);
                        node = first;
                        mask = m1;
                    } else {
                        node = first + (m2 ? 1u : 0u);
                    }
                } else {
                    node = first + (row_second ? 1u : 0u);
                }
            }
        }
    }
}

/* segs: the call's segments (blockIdx.y); edges: the call's float32 edges; rows: this piece's n rows.  psum / pcnt:
 * [blockIdx.x][total_bins] partials of this piece's CTAs; a CTA writes the bins of its segment only. */
template <bool PACKED>
__global__ void __launch_bounds__(B2F_PD_WARPS * 32)
    k_ale(const __grid_constant__ PdParams p, const AleSeg *__restrict__ segs, const float *__restrict__ edges, const uint32_t *__restrict__ rows,
          long long n, int total_bins, double *__restrict__ psum, uint32_t *__restrict__ pcnt) {
    constexpr int T = B2F_PD_WARPS * 32;
    constexpr int J = B2F_ALE_SEG_PROBES;
    __shared__ uint32_t xs[B2F_PD_WARPS][B2F_ROW_WORDS][32];
    __shared__ unsigned long long stk[B2F_PD_STACK][T]; /* edges before the walk, deltas after it */
    __shared__ uint16_t lower[J][T]; /* index of the row's lower edge per field: 48 KB in all */
    static_assert(J * (B2F_PD_MAX_POINTS + 1) * sizeof(float) <= sizeof(stk), "a segment's edges fit the stack area");
    static_assert(J * T * sizeof(double) <= sizeof(stk), "a segment's deltas fit the stack area");

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const AleSeg &sg = segs[blockIdx.y];
    const int count = (int)sg.count;
    float *ze = reinterpret_cast<float *>(&stk[0][0]); /* field j's edges at ze[j * (B2F_PD_MAX_POINTS + 1) ..] */
    for (int j = 0; j < count; ++j) {
        const AleProbe pr = sg.p[j];
        for (int e = threadIdx.x; e <= (int)pr.bins; e += T) ze[j * (B2F_PD_MAX_POINTS + 1) + e] = __ldg(edges + pr.eoff + e);
    }
    __syncthreads();

    const long long row = ((long long)blockIdx.x * B2F_PD_WARPS + warp) * 32 + lane;
    const bool live = row < n;
    pd_stage_row<PACKED>(p, rows, row, live, xs[warp], lane);

    /* each field's bin from the raw word (NaN: missing, no part), by binary search over the edges */
    uint32_t full = 0u;
#pragma unroll
    for (int j = 0; j < J; ++j) {
        uint32_t b = 0;
        if (j < count && live) {
            const AleProbe pr = sg.p[j];
            const uint32_t raw = PACKED ? __ldg(rows + row * B2F_PACKED_ROW_WORDS + pr.word - 7u) : __ldg(rows + row * B2F_ROW_WORDS + pr.word);
            const float x = __uint_as_float(raw);
            if (!isnan(x)) {
                const float *z = ze + j * (B2F_PD_MAX_POINTS + 1);
                int lo = 0, hi = (int)pr.bins + 1; /* first index with z >= x, in [0, K + 1] */
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (z[mid] < x) lo = mid + 1;
                    else hi = mid;
                }
                b = (uint32_t)(min(max(lo, 1), (int)pr.bins) - 1);
                full |= 3u << (2 * j);
            }
            lower[j][threadIdx.x] = (uint16_t)(pr.eoff + b);
        }
    }
    __syncthreads(); /* the stack area is free */

    double acc[B2F_PD_SEG];
#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) acc[k] = p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? p.init_raw : 0.0;
    if (full) ale_mask_walk(p, sg.words, full, lower, edges, xs[warp], lane, stk, acc);
    __syncthreads(); /* every walk is done with the stacks */

    double *delta = reinterpret_cast<double *>(&stk[0][0]); /* delta[j * T + thread] */
#pragma unroll
    for (int j = 0; j < J; ++j) {
        if (j < count) {
            double d = __longlong_as_double(0x7ff8000000000000ll); /* NaN: no part */
            if ((full >> (2 * j)) & 1u) {
                double lo, hi;
                int lab;
                /* the GBDT init value is already in acc (added first, as sklearn does) */
                aggregate(p.agg_mode, p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? 0.0 : p.init_raw, p.denom, p.threshold, acc[2 * j], lo, lab);
                aggregate(p.agg_mode, p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? 0.0 : p.init_raw, p.denom, p.threshold, acc[2 * j + 1], hi, lab);
                d = hi - lo;
            }
            delta[j * T + threadIdx.x] = d;
        }
    }
    __syncthreads();

    /* thread q of the segment's bins: its rows' deltas in row order */
    for (int q = threadIdx.x; q < (int)sg.bins; q += T) {
        int j = 0, b = q;
        while (b >= (int)sg.p[j].bins) b -= (int)sg.p[j++].bins;
        double s = 0.0;
        uint32_t c = 0;
        const uint32_t e = sg.p[j].eoff + (uint32_t)b;
        for (int r = 0; r < T; ++r) {
            const double d = delta[j * T + r];
            if (lower[j][r] == e && !isnan(d)) {
                s += d;
                ++c;
            }
        }
        const long long o = (long long)blockIdx.x * total_bins + sg.p[j].boff + b;
        psum[o] = s;
        pcnt[o] = c;
    }
}

/* thread = bin: its n_cta partials added in CTA order to the running sum (from 0 when first) */
__global__ void __launch_bounds__(256)
    k_ale_finish(const double *__restrict__ psum, const uint32_t *__restrict__ pcnt, int n_cta, int total_bins, int first, double *__restrict__ sums,
                 long long *__restrict__ counts) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= total_bins) return;
    double s = first ? 0.0 : sums[q];
    long long c = first ? 0 : counts[q];
    for (int k = 0; k < n_cta; ++k) {
        s += psum[(long long)k * total_bins + q];
        c += pcnt[(long long)k * total_bins + q];
    }
    sums[q] = s;
    counts[q] = c;
}
