/*
 * permutation_importance.cuh -- K8: permutation importance against labelled rows (sm_90a).
 *
 * sklearn's permutation_importance shuffles one column at a time, rescores every row and reports the drop in a metric.
 * Row i with field f taken from row sigma_r(i) differs from row i in one row word, so all repeats r of a (row, tree,
 * field) are one mask walk that forks only at splits on that word -- the what-if kernels' pd_mask_walk
 * (partial_dependence.cuh), except that the points differ per lane: lane t's point k is word f of row sigma_{r0+k}(t's
 * row), gathered from the device copy of every row (pd_mask_walk<T> reads column threadIdx.x of a per-thread point table).
 *
 * k_permutation_scores: thread = row, warp = 32-row tile, CTA = B2F_PD_WARPS tiles x one segment (blockIdx.y) = one
 * probed word and up to 32 consecutive repeats.  The baseline is a segment with no probed word (one point: the row as it
 * is).  The tile's rows sit transposed in shared memory (xs[word][lane]), the points as pv[k][thread] (conflict-free),
 * the walk stack as stk[depth][thread]; all three are dynamic shared memory, the stack sized to the forest's depth.
 * Each point is a tree-order sum from the GBDT init value, then aggregate(): bit for bit the tile kernel's score of the
 * substituted row.  The epilogue writes one ranking key and one flags byte per (point, row), [point][row]:
 *     key   RandomForest: the bits of P(class 1) (never negative, so the bits order as the values)
 *           GBDT: the order-preserving image of the raw margin (sklearn's roc_auc ranks a GBDT by decision_function,
 *           and the logistic can merge distinct margins)
 *     flags bit 0 = the predicted label, bit 1 = the row's true label
 *
 * k_permutation_metrics (block = point): confusion counts, and the log-loss and Brier sums, each thread over rows
 * t, t + 256, ... then a fixed-order tree reduction; p1 is recomputed from the key with aggregate()'s formula.
 * k_permutation_auc (block = point) reads the point's (key, flags) sorted by key (cub::DeviceSegmentedRadixSort) and
 * adds, per tie group, pos * (C(a) + C(b)) into auc_u2, where C(j) = the negatives before sorted position j and [a, b)
 * is the group: 2 * pos * neg_before + pos * neg_in_group, the Mann-Whitney statistic with ties counted 1/2, doubled.
 * Each thread owns a contiguous run of positions and handles the groups that start in it, walking past its run's end
 * to finish the last one.  Integers are order-free and the float sums are in a fixed order: a call is bit-identical
 * from run to run, and a point's results depend on nothing but its rows, labels, permutation and the forest.
 */
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "partial_dependence.cuh"

#define B2F_PI_NO_WORD 0xffffffffu /* segment word of the baseline: no node splits on it */
#define B2F_PI_METRIC_THREADS 256

/* one segment: up to B2F_PD_SEG consecutive repeats of one probed word, or the baseline */
struct PiSeg {
    uint32_t word;  /* row word, or B2F_PI_NO_WORD */
    uint32_t r0;    /* first repeat */
    uint32_t count; /* 1..B2F_PD_SEG */
    uint32_t point; /* the segment's first point within the launch's group */
};

/* per (point) device results, written by the metric kernels (layout = struct b2f_perm_score) */
struct PiScore {
    long long tp, fp, tn, fn;
    double log_loss_sum, brier_sum;
    unsigned long long auc_u2;
    unsigned long long reserved;
};

__device__ __forceinline__ unsigned long long pi_margin_key(double raw) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(raw);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double pi_key_margin(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

/* word `word` of row `row` as the kernels score it: decoded from the packed form, NaN numerics imputed */
template <bool PACKED>
__device__ __forceinline__ uint32_t pi_row_word(const PdParams &p, const uint32_t *__restrict__ rows, long long row, uint32_t word) {
    uint32_t v;
    if constexpr (PACKED) {
        if ((int)word < p.n_cat) {
            const unsigned long long codes = (((unsigned long long)__ldg(rows + row * B2F_PACKED_ROW_WORDS + 1)) << 32) | __ldg(rows + row * B2F_PACKED_ROW_WORDS);
            v = ((uint32_t)(codes >> (7 * word)) & 0x7fu) - 1u;
        } else {
            v = __ldg(rows + row * B2F_PACKED_ROW_WORDS + 2 + (word - (uint32_t)p.n_cat));
        }
    } else {
        v = __ldg(rows + row * B2F_ROW_WORDS + word);
    }
    if ((int)word >= p.n_cat && (int)word < p.n_cat + p.n_num && isnan(__uint_as_float(v))) v = __float_as_uint(p.impute[word]);
    return v;
}

/* dynamic shared memory of k_permutation_scores for a forest of depth `depth`: a walk holds at most one stack entry per
 * split level of its path */
static inline size_t pi_smem_bytes(int depth) {
    return (size_t)B2F_PD_WARPS * B2F_ROW_WORDS * 32 * 4 + (size_t)B2F_PD_SEG * B2F_PD_WARPS * 32 * 4 + (size_t)(depth + 1) * B2F_PD_WARPS * 32 * 8;
}

/* rows: every row of the call; labels: one 0/1 byte per row; perm: sigma_r at perm + r * n; key / flags: [point][row] of
 * the launch's group */
template <bool PACKED>
__global__ void __launch_bounds__(B2F_PD_WARPS * 32)
    k_permutation_scores(const __grid_constant__ PdParams p, const PiSeg *__restrict__ segs, const uint32_t *__restrict__ rows,
                         const uint8_t *__restrict__ labels, const int32_t *__restrict__ perm, long long n,
                         unsigned long long *__restrict__ key, uint8_t *__restrict__ flags) {
    extern __shared__ __align__(16) unsigned char pi_smem[];
    constexpr int T = B2F_PD_WARPS * 32;
    /* layout: xs [B2F_PD_WARPS][24][32] | pv [B2F_PD_SEG][T] | stk [depth][T] */
    uint32_t(*xs)[B2F_ROW_WORDS][32] = reinterpret_cast<uint32_t(*)[B2F_ROW_WORDS][32]>(pi_smem);
    uint32_t *pv = reinterpret_cast<uint32_t *>(pi_smem + (size_t)B2F_PD_WARPS * B2F_ROW_WORDS * 32 * 4);
    unsigned long long(*stk)[T] = reinterpret_cast<unsigned long long(*)[T]>(pi_smem + (size_t)B2F_PD_WARPS * B2F_ROW_WORDS * 32 * 4 + (size_t)B2F_PD_SEG * T * 4);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const PiSeg sg = segs[blockIdx.y];
    const long long row = ((long long)blockIdx.x * B2F_PD_WARPS + warp) * 32 + lane;
    const bool live = row < n;
    pd_stage_row<PACKED>(p, rows, row, live, xs[warp], lane);
    if (live && sg.word != B2F_PI_NO_WORD) {
        for (int k = 0; k < (int)sg.count; ++k) {
            const long long src = __ldg(perm + (long long)(sg.r0 + k) * n + row);
            pv[k * T + threadIdx.x] = pi_row_word<PACKED>(p, rows, src, sg.word);
        }
    }
    __syncthreads();
    if (!live) return; /* no block-wide barrier below */

    const uint32_t full = sg.count >= 32 ? 0xffffffffu : ((1u << sg.count) - 1u);
    double acc[B2F_PD_SEG];
#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) acc[k] = p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? p.init_raw : 0.0;
    pd_mask_walk<T>(p, sg.word, full, pv + threadIdx.x, xs[warp], lane, stk, acc);

    const uint8_t y = (uint8_t)(__ldg(labels + row) << 1);
#pragma unroll
    for (int k = 0; k < B2F_PD_SEG; ++k) {
        if (k < (int)sg.count) {
            double p1;
            int lab;
            /* the GBDT init value is already in acc (added first, as sklearn does) */
            const bool gbdt = p.agg_mode == B2F_AGG_GBDT_LOGISTIC;
            aggregate(p.agg_mode, gbdt ? 0.0 : p.init_raw, p.denom, p.threshold, acc[k], p1, lab);
            const long long at = (long long)(sg.point + k) * n + row; /* [point][row]: a warp's 32 entries are contiguous */
            key[at] = gbdt ? pi_margin_key(0.0 + acc[k]) : (unsigned long long)__double_as_longlong(p1);
            flags[at] = y | (uint8_t)lab;
        }
    }
}

template <typename V>
__device__ __forceinline__ V pi_block_sum(V v, V *sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int s = B2F_PI_METRIC_THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
        __syncthreads();
    }
    const V r = sh[0];
    __syncthreads();
    return r;
}

/* block = point of the group: confusion counts and the two loss sums into out[point] (auc_u2 by k_permutation_auc) */
__global__ void __launch_bounds__(B2F_PI_METRIC_THREADS)
    k_permutation_metrics(const __grid_constant__ PdParams p, const unsigned long long *__restrict__ key, const uint8_t *__restrict__ flags,
                          long long n, PiScore *__restrict__ out) {
    __shared__ double shd[B2F_PI_METRIC_THREADS];
    __shared__ long long shl[B2F_PI_METRIC_THREADS];
    const long long base = (long long)blockIdx.x * n;
    long long tn = 0, fp = 0, fn = 0, tp = 0;
    double ll = 0.0, br = 0.0;
    const double eps = 2.220446049250313e-16; /* float64 machine epsilon: sklearn's log_loss clip */
    for (long long i = threadIdx.x; i < n; i += B2F_PI_METRIC_THREADS) {
        const unsigned long long k = key[base + i];
        const int f = flags[base + i], y = f >> 1;
        tn += f == 0, fp += f == 1, fn += f == 2, tp += f == 3; /* f = 2 y + label */
        double p1;
        if (p.agg_mode == B2F_AGG_GBDT_LOGISTIC) {
            p1 = 1.0 / (1.0 + exp(-pi_key_margin(k))); /* aggregate()'s expit of the same margin */
        } else {
            p1 = __longlong_as_double((long long)k);
        }
        const double q = y ? p1 : 1.0 - p1;
        ll -= log(fmin(fmax(q, eps), 1.0 - eps));
        const double d = (double)y - p1;
        br += d * d;
    }
    PiScore s;
    s.tn = pi_block_sum(tn, shl);
    s.fp = pi_block_sum(fp, shl);
    s.fn = pi_block_sum(fn, shl);
    s.tp = pi_block_sum(tp, shl);
    s.log_loss_sum = pi_block_sum(ll, shd);
    s.brier_sum = pi_block_sum(br, shd);
    if (threadIdx.x == 0) {
        PiScore &o = out[blockIdx.x];
        o.tp = s.tp, o.fp = s.fp, o.tn = s.tn, o.fn = s.fn;
        o.log_loss_sum = s.log_loss_sum, o.brier_sum = s.brier_sum;
        o.reserved = 0;
    }
}

/* block = point of the group; key / flags sorted by key within each point */
__global__ void __launch_bounds__(B2F_PI_METRIC_THREADS)
    k_permutation_auc(const unsigned long long *__restrict__ key, const uint8_t *__restrict__ flags, long long n, PiScore *__restrict__ out) {
    __shared__ unsigned long long sh[B2F_PI_METRIC_THREADS];
    const unsigned long long *kk = key + (long long)blockIdx.x * n;
    const uint8_t *ff = flags + (long long)blockIdx.x * n;
    const long long per = (n + B2F_PI_METRIC_THREADS - 1) / B2F_PI_METRIC_THREADS;
    const long long lo = min(n, per * (long long)threadIdx.x), hi = min(n, lo + per);
    unsigned long long neg = 0;
    for (long long j = lo; j < hi; ++j) neg += (ff[j] >> 1) ^ 1;
    /* exclusive prefix of the runs' negatives, in thread order */
    sh[threadIdx.x] = neg;
    __syncthreads();
    for (int o = 1; o < B2F_PI_METRIC_THREADS; o <<= 1) {
        const unsigned long long v = (int)threadIdx.x >= o ? sh[threadIdx.x - o] : 0ull;
        __syncthreads();
        sh[threadIdx.x] += v;
        __syncthreads();
    }
    unsigned long long cneg = sh[threadIdx.x] - neg; /* C(lo) */
    __syncthreads();
    unsigned long long u2 = 0;
    long long j = lo;
    if (j > 0 && j < hi) { /* skip the tail of a group that started in an earlier run */
        const unsigned long long prev = kk[j - 1];
        while (j < hi && kk[j] == prev) cneg += (ff[j++] >> 1) ^ 1;
    }
    while (j < hi) { /* groups starting in [lo, hi) */
        const unsigned long long k0 = kk[j];
        const unsigned long long ca = cneg;
        unsigned long long pos = 0;
        for (; j < n && kk[j] == k0; ++j) {
            const unsigned y = ff[j] >> 1;
            pos += y;
            cneg += y ^ 1;
        }
        u2 += pos * (ca + cneg);
    }
    const unsigned long long total = pi_block_sum(u2, sh);
    if (threadIdx.x == 0) out[blockIdx.x].auc_u2 = total;
}
