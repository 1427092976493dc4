/*
 * forest_decide.cuh -- the decision of a row whose float64 tree sum lies inside its rounding band, shared by the predict
 * kernels (warp, split, tile, rank).
 *
 * Every kernel adds a row's leaf payloads in its own order (lane partials and a butterfly, tree order, group order, warp
 * partials), so two kernels -- which the engine picks by batch size -- can round the same row's sum to different sides of
 * a decision threshold.  A row whose sum lies within the rounding band of the threshold is rare, and only its label (or
 * outlier flag) is re-decided here, off the hot loop and without touching its score:
 *   RF      : the label is the exact sign of sum p1 - T/2 (sklearn's argmax of the exact means, a tie to class 0): the
 *             payloads are re-read by one thread in tree order and added into a fixed-point integer accumulator, which
 *             is exact and order-independent;
 *   IFOREST : the flag is sklearn's: the payloads (sklearn's per-tree terms, flatten.py) are added in tree order, as
 *             sklearn does, and compared with the path-length bound the host derived from numpy's own formula.
 * One thread re-walks the row from global memory: the blob layout for 96-byte / 64-byte rows, the rank layout for ranked
 * rows.
 */
#pragma once
/* included by forest_predict.cuh once KParams and take_second are defined */

/* |margin| <= band: a float64 sum of T payloads in [0, 1] is within T^2 eps / 2 of the exact one in any order, so 4 T^2 eps
 * of 2 s - T holds every row whose label could depend on the order.  Isolation forest: the sum of T positive payloads is
 * within T eps s of the tree-order one; B2F_MAX_GROUPS * 32 bounds T. */
__device__ __forceinline__ bool decide_exactly(int agg_mode, double s, double denom, double threshold) {
    const double eps = 2.220446049250313e-16;
    if (agg_mode == B2F_AGG_RF_MEAN) return fabs(2.0 * s - denom) <= 4.0 * denom * denom * eps;
    if (agg_mode == B2F_AGG_IFOREST) return fabs(s - threshold) <= 4.0 * (B2F_MAX_GROUPS * 32) * eps * s;
    return false;
}

/* Exact sum of non-negative finite doubles: bit k of the 1152-bit integer weighs 2^(k - 1088), so every double in
 * [2^-1074, 2^63] lands on whole bits. */
#define B2F_XSUM_LIMBS 18
struct ExactSum {
    unsigned long long l[B2F_XSUM_LIMBS];
    __device__ void clear() {
        for (int k = 0; k < B2F_XSUM_LIMBS; ++k) l[k] = 0ull;
    }
    __device__ void add(double x) {
        const unsigned long long b = (unsigned long long)__double_as_longlong(x);
        const int ex = (int)((b >> 52) & 0x7ff);
        if (x <= 0.0) return; /* RF payloads are in [0, 1]: zero adds nothing */
        const unsigned long long m = ex ? ((b & 0xFFFFFFFFFFFFFull) | (1ull << 52)) : (b & 0xFFFFFFFFFFFFFull);
        const int pos = (ex ? ex - 1075 : -1074) + 1088;
        const int k = pos >> 6, sh = pos & 63;
        const unsigned long long lo = m << sh, hi = sh ? (m >> (64 - sh)) : 0ull;
        unsigned long long c = 0ull;
        for (int j = k; j < B2F_XSUM_LIMBS; ++j) {
            const unsigned long long a = j == k ? lo : (j == k + 1 ? hi : 0ull);
            const unsigned long long s = l[j] + a;
            const unsigned long long s2 = s + c;
            c = (unsigned long long)(s < a) + (unsigned long long)(s2 < s);
            l[j] = s2;
            if (j > k && !c) break;
        }
    }
    /* -1, 0, 1 */
    __device__ int compare(const ExactSum &o) const {
        for (int k = B2F_XSUM_LIMBS - 1; k >= 0; --k)
            if (l[k] != o.l[k]) return l[k] > o.l[k] ? 1 : -1;
        return 0;
    }
};

/* RF label / isolation-forest flag from the payloads, offered in tree order by `walk(f)` */
template <typename Walk>
__device__ __noinline__ int decide_from_payloads(int agg_mode, double denom, double threshold, Walk walk) {
    if (agg_mode == B2F_AGG_RF_MEAN) {
        ExactSum acc, half;
        acc.clear();
        half.clear();
        walk([&](double x) { acc.add(x); });
        half.add(0.5 * denom);
        return acc.compare(half) > 0;
    }
    double s = 0.0;
    walk([&](double x) { s += x; });
    return s <= threshold;
}

/* one row word of a 96-byte or packed 64-byte row, NaN numerics imputed (what the kernels' row staging produces) */
template <bool PACKED>
__device__ __forceinline__ uint32_t blob_row_word(const KParams &p, const uint32_t *rows, long long row, uint32_t w) {
    if (w >= B2F_SENTINEL_WORD) return B2F_SENTINEL_BITS;
    uint32_t v;
    if constexpr (PACKED) {
        const uint32_t *q = rows + row * B2F_PACKED_ROW_WORDS;
        if (w < 9) {
            const unsigned long long codes = (((unsigned long long)__ldg(q + 1)) << 32) | __ldg(q);
            v = ((uint32_t)(codes >> (7 * w)) & 0x7fu) - 1u;
        } else {
            v = __ldg(q + 2 + (w - 9));
        }
    } else {
        v = __ldg(rows + row * B2F_ROW_WORDS + w);
    }
    if ((int)w >= p.n_cat && (int)w < p.n_cat + p.n_num && isnan(__uint_as_float(v))) v = __float_as_uint(p.impute[w]);
    return v;
}

/* the decision of one row of a 96-byte / 64-byte batch, walking the blob in global memory tree by tree */
template <bool PACKED>
__device__ __noinline__ int decide_row_blob(const KParams &p, const uint32_t *rows, long long row) {
    return decide_from_payloads(p.agg_mode, p.denom, p.threshold, [&](auto add) {
        for (int g = 0; g < p.n_groups; ++g) {
            const KGroup gd = p.g[g];
            const uint8_t *nodes = p.chunks + gd.chunk_off;
            const uint8_t *leaves = nodes + (size_t)gd.n_slots * B2F_NODE_STRIDE;
            for (uint32_t lane = 0; lane < 32; ++lane) {
                uint32_t slot = 0;
                for (uint32_t d = 0; d < gd.depth; ++d) {
                    const uint2 tm = __ldg(reinterpret_cast<const uint2 *>(nodes + (size_t)slot * B2F_NODE_STRIDE + lane * 8u));
                    const uint32_t x = blob_row_word<PACKED>(p, rows, row, tm.y >> B2F_META_FEAT_SHIFT);
                    slot = (tm.y & B2F_META_SLOT_MASK) + (take_second(x, tm.x, tm.y) ? 1u : 0u);
                }
                const uint32_t leaf = __ldg(reinterpret_cast<const uint32_t *>(nodes + (size_t)slot * B2F_NODE_STRIDE + lane * 8u));
                add(__ldg(reinterpret_cast<const double *>(leaves + (size_t)leaf * B2F_NODE_STRIDE + lane * 8u)));
            }
        }
    });
}
