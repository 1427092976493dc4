/*
 * drift_stats.cuh -- K3: batch drift scores on the GPU (SURVEY.md section 8a row a7, 8f rank 2).
 *
 * Replaces `self.drift.predict(df[self.all_features].values)` (reference databricks/src/02-register-model.ipynb:338;
 * detector built at :224-229 as alibi-detect TabularDrift(x_ref, p_val=0.05, categories_per_feature={0..8: None})):
 * per request, one p-value per feature of the batch against the 30 000-row reference table --
 *   categorical: chi-squared test on the 2 x K table of reference / batch category counts (scipy chi2_contingency:
 *                Pearson statistic, Yates correction when dof == 1, p = Q(dof/2, stat/2));
 *   numeric    : two-sided two-sample Kolmogorov-Smirnov test, EXACT p-value (scipy ks_2samp(method="exact")).
 * The reference re-sorts and re-counts its 30 000 reference rows on every request and then runs scipy's
 * O(m * window) lattice-path recursion on one core; here the reference columns live pre-sorted in HBM and
 *
 *   k_drift_count   one thread per (feature, batch element): two binary searches of the element in the sorted
 *                   reference column (a = #ref < x, b = #ref <= x) -> two histograms over reference positions;
 *                   categorical elements -> a histogram over category codes.
 *   k_drift_finish  one CTA per feature.
 *     numeric : (1) prefix sums of the two histograms give #batch <= r_j and #batch < r_j at every reference point;
 *               the K-S numerator  max_t |n*#{ref<=t} - m*#{batch<=t}|  is attained at a reference point or at the
 *               left limit of one (both ECDFs are right-continuous steps), so it is an exact INTEGER;
 *               (2) the exact p-value: the probability that a lattice path (0,0)->(m,n) leaves the band
 *               |ng*i - mg*j| < h (Hodges 1958; the 1-p recursion of Viehmann 2021 that scipy's
 *               _compute_outer_prob_inside_method runs column by column).  Cell (i,j) needs (i-1,j) and (i,j-1):
 *               the CTA sweeps ANTI-DIAGONALS t = i + j, all in-band cells of a diagonal in parallel (one per
 *               thread, values exchanged through a shared-memory ring indexed by j mod L), m + n steps instead
 *               of m * window.
 *     categorical: one thread forms the chi-squared statistic and the regularised upper incomplete gamma function.
 *
 * Everything is float64 / int64; results match scipy to ~1e-13 relative (the recursion multiplies by a correctly
 * rounded 1/t where scipy divides by t).
 */
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#define B2F_DRIFT_THREADS 1024
#define B2F_DRIFT_RING_MAX 4096 /* slots of the anti-diagonal ring (2 x 32 KB of shared memory) */
#define B2F_DRIFT_MAX_CATS 512  /* categories per feature, reference + new ones of the batch */

struct DriftParams {
    int64_t n_ref;            /* reference rows m0 */
    int64_t n;                /* batch rows */
    int32_t n_num, n_cat;
    const double *ref_sorted; /* [n_num][n_ref] ascending */
    const double *x;          /* [n_num][n]  batch numerics, column-major */
    const int32_t *codes;     /* [n_cat][n]  batch category codes, -1 = not a reference category */
    uint32_t *hist_a;         /* [n_num][n_ref + 1]  #batch elements with (#ref <  x) == k */
    uint32_t *hist_b;         /* [n_num][n_ref + 1]  #batch elements with (#ref <= x) == k */
    uint32_t *nan_count;      /* [n_num] */
    uint32_t *cat_hist;       /* [sum cat_sizes] batch counts per reference category */
    const int32_t *cat_off;   /* [n_cat + 1] offsets into cat_hist / ref_counts */
    const int64_t *ref_counts; /* [sum cat_sizes] */
    const int32_t *new_off;   /* [n_cat + 1] offsets into new_counts (categories of the batch absent from the reference) */
    const int64_t *new_counts;
    double *p_val;            /* [n_cat + n_num]  categorical features first */
    double *stat;             /* chi-squared statistic / K-S D */
    int32_t *flags;           /* 0 ok; 1 = exact K-S not applicable (scipy switches to the asymptotic formula); 2 = NaN input */
    double *row_scratch;      /* [n_num][2][B2F_DRIFT_ROW_STRIDE(n_ref)]: the two rows of the row-scan form of the exact p-value (NULL: sweep only) */
    int32_t rowscan_max_n;    /* batches of 2 .. this many rows take the row scan through the global scratch (0 = never) */
    int32_t rowscan_smem_max_n; /* batches of 2 .. this many rows take the shared-memory row scan when their band fits (0 = never) */
    int32_t rowscan_cap;      /* doubles of dynamic shared memory available to it */
    double *wide_scratch;     /* [n_num][2][wide_ring]: the sweep's two ring buffers when the band is wider than B2F_DRIFT_RING_MAX */
    int64_t wide_ring;        /* slots per buffer there: the widest ring this batch size can need (0: none allocated) */
};

/* ------------------------------------------------------------------ k_drift_count */
__global__ void __launch_bounds__(256) k_drift_count(DriftParams p) {
    const int64_t per = p.n;
    const int64_t total = per * (p.n_num + p.n_cat);
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int f = (int)(idx / per);
        const int64_t e = idx - (int64_t)f * per;
        if (f < p.n_num) {
            const double x = p.x[(int64_t)f * per + e];
            if (x != x) {
                atomicAdd(&p.nan_count[f], 1u);
                continue;
            }
            const double *r = p.ref_sorted + (int64_t)f * p.n_ref;
            int64_t lo = 0, hi = p.n_ref; /* a = first index with r[idx] >= x  == #ref < x */
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if (__ldg(&r[mid]) < x) lo = mid + 1; else hi = mid;
            }
            const int64_t a = lo;
            hi = p.n_ref;                 /* b = first index with r[idx] > x  == #ref <= x */
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if (__ldg(&r[mid]) <= x) lo = mid + 1; else hi = mid;
            }
            atomicAdd(&p.hist_a[(int64_t)f * (p.n_ref + 1) + a], 1u);
            atomicAdd(&p.hist_b[(int64_t)f * (p.n_ref + 1) + lo], 1u);
        } else {
            const int c = f - p.n_num;
            const int32_t code = p.codes[(int64_t)c * per + e];
            const int32_t size = p.cat_off[c + 1] - p.cat_off[c];
            if (code >= 0 && code < size) atomicAdd(&p.cat_hist[p.cat_off[c] + code], 1u);
        }
    }
}

/* ------------------------------------------------------------------ chi-squared tail: Q(a, x) = Gamma(a, x) / Gamma(a) */
__device__ inline double gamma_q(double a, double x) {
    if (!(x > 0.0)) return 1.0;
    if (x < a + 1.0) { /* series for P(a, x), Q = 1 - P */
        double ap = a, sum = 1.0 / a, del = sum;
        for (int it = 0; it < 100000; ++it) {
            ap += 1.0;
            del *= x / ap;
            sum += del;
            if (fabs(del) < fabs(sum) * 1e-17) break;
        }
        return 1.0 - sum * exp(-x + a * log(x) - lgamma(a));
    }
    /* modified Lentz continued fraction for Q(a, x) */
    const double tiny = 1e-300;
    double b = x + 1.0 - a, c = 1.0 / tiny, d = 1.0 / b, hcf = d;
    for (int it = 1; it < 100000; ++it) {
        const double an = -(double)it * ((double)it - a);
        b += 2.0;
        d = an * d + b;
        if (fabs(d) < tiny) d = tiny;
        c = b + an / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        const double del = d * c;
        hcf *= del;
        if (fabs(del - 1.0) < 1e-16) break;
    }
    return exp(-x + a * log(x) - lgamma(a)) * hcf;
}

/* scipy.stats.chi2_contingency on the 2 x K table (reference row, batch row): K = reference categories + new ones */
__device__ inline void chi2_feature(const DriftParams &p, int c, double &stat, double &pv) {
    const int k_ref = p.cat_off[c + 1] - p.cat_off[c];
    const int k_new = p.new_off ? p.new_off[c + 1] - p.new_off[c] : 0;
    const int K = k_ref + k_new;
    double row0 = 0.0, row1 = 0.0;
    for (int k = 0; k < K; ++k) {
        row0 += k < k_ref ? (double)p.ref_counts[p.cat_off[c] + k] : 0.0;
        row1 += k < k_ref ? (double)p.cat_hist[p.cat_off[c] + k] : (double)p.new_counts[p.new_off[c] + k - k_ref];
    }
    if (K < 2) { /* dof == 0 */
        stat = 0.0;
        pv = 1.0;
        return;
    }
    const double tot = row0 + row1;
    const bool yates = K == 2;
    double s = 0.0;
    for (int k = 0; k < K; ++k) {
        const double o0 = k < k_ref ? (double)p.ref_counts[p.cat_off[c] + k] : 0.0;
        const double o1 = k < k_ref ? (double)p.cat_hist[p.cat_off[c] + k] : (double)p.new_counts[p.new_off[c] + k - k_ref];
        const double col = o0 + o1;
        const double e0 = row0 * col / tot, e1 = row1 * col / tot;
        double d0 = o0 - e0, d1 = o1 - e1;
        if (yates) { /* observed moves towards expected by min(0.5, |diff|) */
            d0 = d0 > 0 ? d0 - fmin(0.5, d0) : d0 + fmin(0.5, -d0);
            d1 = d1 > 0 ? d1 - fmin(0.5, d1) : d1 + fmin(0.5, -d1);
        }
        s += d0 * d0 / e0 + d1 * d1 / e1;
    }
    stat = s;
    pv = gamma_q(0.5 * (double)(K - 1), 0.5 * s);
}

/* ------------------------------------------------------------------ k_drift_finish */
__device__ inline int64_t gcd64(int64_t a, int64_t b) {
    while (b) {
        const int64_t t = a % b;
        a = b;
        b = t;
    }
    return a;
}

/* ---- the anti-diagonal sweep ----------------------------------------------------------------------------------
 * P(i,j) = 1 outside the band |ng*i - mg*j| < h or off the lattice, 0 on the first column inside the band, else
 * (P(i-1,j)*i + P(i,j-1)*j) / (i+j).  Diagonal t = i + j holds at most 2h/(ng+mg) + 1 in-band cells, consecutive in j.
 * A ring of `ring` slots (power of two >= that + 3) covers j in [j_lo(t) - 1, j_lo(t) - 1 + ring), slot = j mod ring,
 * where j_lo(t) is the first in-band j of the diagonal; the lowest covered cell is always outside the band (value 1),
 * so when j_lo advances and a slot jumps from j to j + ring the value it leaves behind is exactly the value (1) its
 * new cell's upper neighbour has.  Per step a slot therefore needs its own previous value ("up", a register) and
 * the previous value of slot - 1 ("left": a shuffle inside a warp, shared memory across warps).
 * All bookkeeping is incremental adds (dev = ng*i - mg*j grows by ng per step, a 32-bit counter tracks j_lo); the
 * only floating-point work on the dependent chain is one FMA and one multiply by 1/t.  1/t comes from a per-warp batch:
 * every 32 steps lane l divides once, 1/(t0 + l), and steps fetch their reciprocal with a shuffle. */
struct SweepConst {
    int64_t m, n, mg, ng, den, h, T;
    int ring;
};
/* Slot bookkeeping lives in float64: every quantity is an integer below 2^53 (exact), a float64 add / compare is one
 * instruction where the int64 form is two or three, and i and j are needed as float64 by the recurrence anyway. */
struct SweepF {
    double n, m, h, ng, ringd, den_ring;
};
struct SlotState {
    double dev; /* ng*i - mg*j of the slot's current cell */
    double i, j;
    double v;   /* value of the slot's cell on the previous diagonal */
    int32_t jj; /* j as an integer, for the "lowest covered j" test */
};

__device__ __forceinline__ SweepF sweep_f(const SweepConst &c) {
    SweepF f;
    f.n = (double)c.n;
    f.m = (double)c.m;
    f.h = (double)c.h;
    f.ng = (double)c.ng;
    f.ringd = (double)c.ring;
    f.den_ring = (double)(c.den * (int64_t)c.ring);
    return f;
}
__device__ __forceinline__ void slot_init(SlotState &st, int s, int64_t js0, const SweepConst &c) {
    const int32_t j = (int32_t)js0 + ((s - (int32_t)js0) & (c.ring - 1));
    st.jj = j;
    st.j = (double)j;
    st.i = -(double)j; /* t = 0 */
    st.dev = -(double)(c.den * (int64_t)j);
    st.v = 1.0;
}
__device__ __forceinline__ double slot_eval(const SlotState &st, double left, double rt, const SweepF &f) {
    const bool off = (st.j < 0.0) | (st.j > f.n) | (st.i < 0.0) | (st.i > f.m) | (fabs(st.dev) >= f.h);
    /* blend instead of a chain of selects: the scale (1/t, or 0 off the band / on the first column) and the offset
     * (1 off the band) do not depend on the neighbours, so only two FMAs sit on the dependent chain */
    const double scale = (off | (st.i == 0.0)) ? 0.0 : rt;
    const double offset = off ? 1.0 : 0.0;
    return fma(fma(left, st.j, st.v * st.i), scale, offset);
}
__device__ __forceinline__ void slot_advance(SlotState &st, bool adv, int32_t js_new, int ring, const SweepF &f) {
    st.i += 1.0;
    st.dev += f.ng;
    if (adv && st.jj < js_new) { /* this slot held the lowest covered j: it now covers j + ring */
        st.jj += ring;
        st.j += f.ringd;
        st.i -= f.ringd;
        st.dev -= f.den_ring;
    }
}

/* ring == 32: one warp, one slot per lane, no shared memory */
__device__ __forceinline__ double sweep_warp(const SweepConst &c, int lane) {
    int64_t j_lo = -(c.h / c.den) - 1;
    while (c.den * j_lo <= -c.h) ++j_lo;
    int32_t edge = (int32_t)(-c.h - c.den * j_lo); /* ng*t - h - den*j_lo, in [-den, 0): den < 2^28 */
    int32_t js = (int32_t)j_lo - 1;
    const int32_t ng = (int32_t)c.ng, den = (int32_t)c.den, T = (int32_t)c.T;
    const SweepF f = sweep_f(c);
    SlotState st;
    slot_init(st, lane, js, c);
    double r_mine = 0.0;
    for (int32_t t = 0; t <= T; ++t) {
        if ((t & 31) == 0) {
            const double tl = (double)(t + lane);
            r_mine = tl > 0.0 ? 1.0 / tl : 0.0;
        }
        const double rt = __shfl_sync(0xffffffffu, r_mine, t & 31);
        const double left = __shfl_sync(0xffffffffu, st.v, (lane + 31) & 31);
        st.v = slot_eval(st, left, rt, f);
        edge += ng;
        const bool adv = edge >= 0;
        if (adv) {
            edge -= den;
            ++js;
        }
        slot_advance(st, adv, js, 32, f);
    }
    return __shfl_sync(0xffffffffu, st.v, (int)(c.n & 31));
}

/* ring >= 64: `active` = min(ring, blockDim) threads, NS = ring / active slots each (slot = tid + k*active);
 * "left" values travel through a double-buffered shared-memory ring, one named barrier per diagonal */
template <int NS>
__device__ __forceinline__ double sweep_block(const SweepConst &c, int tid, int active, double *buf0, double *buf1) {
    const int mask = c.ring - 1;
    int64_t j_lo = -(c.h / c.den) - 1;
    while (c.den * j_lo <= -c.h) ++j_lo;
    int32_t edge = (int32_t)(-c.h - c.den * j_lo);
    int32_t js = (int32_t)j_lo - 1;
    const int32_t ng = (int32_t)c.ng, den = (int32_t)c.den, T = (int32_t)c.T;
    const SweepF f = sweep_f(c);
    SlotState st[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) {
        slot_init(st[k], tid + k * active, js, c);
        buf0[tid + k * active] = 1.0;
    }
    asm volatile("bar.sync 1, %0;" ::"r"(active) : "memory");
    double *prev = buf0, *cur = buf1;
    const int lane = tid & 31;
    double r_mine = 0.0;
    for (int32_t t = 0; t <= T; ++t) {
        if ((t & 31) == 0) {
            const double tl = (double)(t + lane);
            r_mine = tl > 0.0 ? 1.0 / tl : 0.0;
        }
        const double rt = __shfl_sync(0xffffffffu, r_mine, t & 31);
        edge += ng;
        const bool adv = edge >= 0;
        if (adv) {
            edge -= den;
            ++js;
        }
#pragma unroll
        for (int k = 0; k < NS; ++k) {
            const int s = tid + k * active;
            const double left = prev[(s - 1) & mask];
            st[k].v = slot_eval(st[k], left, rt, f);
            cur[s] = st[k].v;
            slot_advance(st[k], adv, js, c.ring, f);
        }
        asm volatile("bar.sync 1, %0;" ::"r"(active) : "memory");
        double *tmp = prev;
        prev = cur;
        cur = tmp;
    }
    return prev[(int)(c.n & mask)]; /* written before the last barrier */
}

/* ring > B2F_DRIFT_RING_MAX (large samples, D far from 0): the same sweep with its two ring buffers in a per-feature global
 * scratch (L2; __syncthreads orders global memory inside the CTA) and no per-slot registers -- a thread owns ring / 1024 slots,
 * so each slot's cell is recomputed every step from the diagonal's lowest covered j (the closed forms SlotState tracks
 * incrementally: j = js + ((s - js) mod ring), i = t - j).  All threads of the CTA. */
__device__ double sweep_wide(const SweepConst &c, int tid, int nt, double *buf0, double *buf1) {
    const int64_t mask = c.ring - 1;
    int64_t j_lo = -(c.h / c.den) - 1;
    while (c.den * j_lo <= -c.h) ++j_lo;
    int64_t edge = -c.h - c.den * j_lo;
    int64_t js = j_lo - 1;
    const SweepF f = sweep_f(c);
    for (int s = tid; s < c.ring; s += nt) __stcg(buf0 + s, 1.0);
    __syncthreads();
    double *prev = buf0, *cur = buf1;
    for (int64_t t = 0; t <= c.T; ++t) {
        const double rt = t > 0 ? 1.0 / (double)t : 0.0;
        for (int s0 = tid; s0 < c.ring; s0 += 4 * nt) { /* four slots' loads in flight before their stores */
            double up[4], left[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int s = s0 + k * nt;
                up[k] = s < c.ring ? __ldcg(prev + s) : 0.0;
                left[k] = s < c.ring ? __ldcg(prev + ((s - 1) & mask)) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int s = s0 + k * nt;
                if (s < c.ring) {
                    const int64_t j = js + ((s - js) & mask);
                    SlotState st;
                    st.j = (double)j;
                    st.i = (double)(t - j);
                    st.dev = (double)(c.ng * (t - j) - c.mg * j);
                    st.v = up[k];
                    __stcg(cur + s, slot_eval(st, left[k], rt, f));
                }
            }
        }
        edge += c.ng;
        if (edge >= 0) {
            edge -= c.den;
            ++js;
        }
        __syncthreads();
        double *tmp = prev;
        prev = cur;
        cur = tmp;
    }
    return __ldcg(prev + (c.n & mask));
}

/* ---- the row-scan form (request-sized batches) ---------------------------------------------------------------------
 * W(i,j) = number of lattice paths (0,0)->(i,j) that have left the band.  Multiplying the recursion above through by
 * C(i+j, j) removes the divisions:  inside the band  W(i,j) = W(i-1,j) + W(i,j-1),  outside  W(i,j) = C(i+j, j).
 * The in-band cells of row j are the interval lo_j <= i <= hi_j (it moves right with j), so row j is ONE prefix sum over i
 * of row j-1 -- extended on its right by the binomials of the cells that row j-1 had outside the band -- seeded with the
 * binomial of the cell left of the band:  n block-wide prefix sums of <= m elements instead of m + n dependent steps
 * (n = the batch size: 16 rows against 30 000 reference points is 16 scans, not 30 016 steps).
 * Rows live in a global scratch (L2), element i at (i mod CH) * NT + i / CH so that thread t owns the CH consecutive
 * columns [t CH, (t+1) CH) and every load / store of a pass is coalesced; row j is scaled by 2^-E_j, E_j the exponent of
 * its largest binomial, so nothing overflows.  Sums run in a fixed order (deterministic).  p = W(m,n) / C(m+n, n). */
/* Limits measured with tools/drift_time.py against 30 000 reference rows on an H100 80GB HBM3 (700 W), device ms per request:
 * global-scratch row scan 1.11 at 48 rows vs the sweep's 1.76; shared-memory row scan 1.31 at 320 rows, 2.38 at 512 vs the
 * sweep's 2.15 / 2.17 -- the crossover lies between 320 and 512 rows. */
#define B2F_DRIFT_ROWSCAN_MAX 48       /* global-scratch form: two dependent L2 trips per row, the sweep is faster beyond */
#define B2F_DRIFT_ROWSCAN_SMEM_MAX 448  /* shared-memory form: cost grows per row, the sweep's is flat in n */
#define B2F_DRIFT_ROWSCAN_SMEM_LIMIT 1024 /* what B2F_DRIFT_ROWSCAN_SMEM may raise it to (32 factors per lane in the binomial products) */
#define B2F_DRIFT_ROWSCAN_CAP 28672     /* doubles of the shared-memory row ring (224 KB of the 227 KB a CTA may have) */
/* doubles per scratch row: the transposed layout (i mod CH) * NT + i / CH spans CH * NT >= m + 1 slots */
#define B2F_DRIFT_ROW_STRIDE(m) ((((int64_t)(m) + 1 + B2F_DRIFT_THREADS - 1) / B2F_DRIFT_THREADS) * B2F_DRIFT_THREADS)

struct BinomME {
    double mant; /* in [1, 2^400) */
    int ex;      /* value = mant * 2^ex */
};
/* C(t, k) = prod_{r=1..k} (t - k + r) / r as numerator / denominator products with exponent tracking (no division in the loop) */
__device__ inline BinomME binom_me(int64_t t, int k) {
    double num = 1.0, den = 1.0;
    int ex = 0;
    for (int r = 1; r <= k; ++r) {
        num *= (double)(t - k + r);
        den *= (double)r;
        if (num > 0x1p400) {
            num *= 0x1p-400;
            ex += 400;
        }
        if (den > 0x1p400) {
            den *= 0x1p-400;
            ex -= 400;
        }
    }
    BinomME b;
    b.mant = num / den;
    b.ex = ex;
    return b;
}
__device__ inline double binom_scaled(int64_t t, int k, int e) {
    const BinomME b = binom_me(t, k);
    return ldexp(b.mant, b.ex - e);
}
__device__ inline int binom_exponent(int64_t t, int k) {
    const BinomME b = binom_me(t, k);
    int fe;
    frexp(b.mant, &fe);
    return b.ex + fe;
}
__device__ inline int64_t floor_div(int64_t a, int64_t b) { /* b > 0 */
    int64_t q = a / b;
    if ((a % b != 0) && (a < 0)) --q;
    return q;
}

/* all B2F_DRIFT_THREADS threads of the CTA; buf0 / buf1: B2F_DRIFT_ROW_STRIDE(m) doubles each.  Returns the p-value on thread 0. */
__device__ double rows_scan(const SweepConst &c, double *buf0, double *buf1, int tid, int nt) {
    __shared__ double s_warp[32];
    __shared__ double s_seed;
    __shared__ int s_e;
    const int64_t m = c.m, mg = c.mg, ng = c.ng, h = c.h;
    const int n = (int)c.n;
    const int64_t CH = (m + 1 + nt - 1) / nt;
    const int64_t i0 = (int64_t)tid * CH, i1 = min(i0 + CH, m + 1);
    auto pos = [&](int64_t i) { return (i % CH) * nt + i / CH; };
    const int lane = tid & 31, warp = tid >> 5;

    /* row 0: inside the band no path has left it */
    for (int64_t i = i0; i < i1; ++i) __stcg(buf0 + pos(i), 0.0);
    int64_t hi_p = min(-floor_div(-(h), ng) - 1, m); /* last i with ng*i < h */
    int e_p = 1;                                      /* exponent of C(hi_0, 0) = 1 */
    double *prev = buf0, *cur = buf1;
    __syncthreads();
    for (int j = 1; j <= n; ++j) {
        const int64_t lo = max(floor_div(mg * j - h, ng) + 1, (int64_t)0);
        const int64_t hi = min(-floor_div(-(mg * j + h), ng) - 1, m);
        /* the row's scale and seed (two threads in different warps), and the cells the previous row had outside the band */
        if (tid == 0) s_e = binom_exponent(hi + j, j);
        if (tid == 32) {
            const BinomME b = lo >= 1 ? binom_me(lo - 1 + j, j) : BinomME{0.0, 0};
            s_seed = b.mant;
            s_warp[0] = (double)b.ex; /* applied after the barrier, when the row's exponent is known */
        }
        for (int64_t i = hi_p + 1 + tid; i <= hi; i += nt) __stcg(prev + pos(i), binom_scaled(i + j - 1, j - 1, e_p));
        __syncthreads();
        const int e = s_e;
        const double seed = ldexp(s_seed, (int)s_warp[0] - e);
        const double scale = ldexp(1.0, e_p - e);
        __syncthreads(); /* s_warp is reused by the scan */
        /* pass A: this thread's partial sum.  The row lives in L2: loads go out eight at a time (independent, so their
         * latencies overlap) before the dependent adds consume them */
        const int64_t a0 = max(i0, lo), a1 = min(i1, hi + 1);
        double local = 0.0;
        for (int64_t b = a0; b < a1; b += 8) {
            double v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = (b + q < a1) ? __ldcg(prev + pos(b + q)) : 0.0;
#pragma unroll
            for (int q = 0; q < 8; ++q) local += v[q] * scale;
        }
        /* exclusive block scan of the partials, fixed order */
        double incl = local;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            double w = lane < (nt >> 5) ? s_warp[lane] : 0.0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const double v = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += v;
            }
            s_warp[lane] = w; /* inclusive over warps */
        }
        __syncthreads();
        double run = seed + (warp > 0 ? s_warp[warp - 1] : 0.0) + (incl - local);
        /* pass B: the row's values */
        for (int64_t b = a0; b < a1; b += 8) {
            double v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = (b + q < a1) ? __ldcg(prev + pos(b + q)) : 0.0;
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (b + q < a1) {
                    run += v[q] * scale;
                    __stcg(cur + pos(b + q), run);
                }
        }
        double *t = prev;
        prev = cur;
        cur = t;
        hi_p = hi;
        e_p = e;
        __syncthreads();
    }
    if (tid == 0) return __ldcg(prev + pos(m)) / binom_scaled(m + n, n, e_p);
    return 0.0;
}

/* ---- the row-scan with the row RESIDENT IN SHARED MEMORY ---------------------------------------------------------------
 * The global-scratch form above pays two dependent trips to L2 per row (it loses to the sweep beyond
 * B2F_DRIFT_ROWSCAN_MAX rows).  A row only ever needs its in-band cells [lo_j, hi_j], at most 2h/ng + 1 of them, and the interval only moves
 * right: cell i lives in slot i mod cap of a shared-memory ring of `cap` doubles (cap >= the widest row, checked by the caller),
 * updated IN PLACE.  Thread t owns the L consecutive cells lo_j + tL .. (L odd: the float64 accesses of a half-warp then fall
 * into 16 different bank pairs), adds them up, the block scans the 1024 partial sums (two shuffle scans, fixed order), and a
 * second pass writes the running sums.  The binomials a row needs -- its scale, its seed, and the cells the previous row had
 * outside the band -- are products of up to j factors; they are computed by GROUPS of G lanes (G = 1, 8 or 32 by j), each lane
 * a strided share of the factors, combined by a butterfly of multiplies on (mantissa, exponent) pairs: warp 0 the scale, warp 1
 * the seed, warps 2.. the cells, all at the same time. */
/* frexp / ldexp for the values that occur here (positive, normal): two integer operations instead of the library routines */
__device__ __forceinline__ double frexp_pos(double x, int &e) {
    int hi = __double2hiint(x);
    e = ((hi >> 20) & 0x7ff) - 1022;
    hi = (hi & 0x800fffff) | 0x3fe00000;
    return __hiloint2double(hi, __double2loint(x)); /* in [0.5, 1) */
}
__device__ __forceinline__ double ldexp_fast(double x, int d) {
    if (d > -1000 && d < 1000) return x * __hiloint2double((d + 1023) << 20, 0); /* exact: x is normal and stays normal */
    return ldexp(x, d);
}

/* C(t, k) by a group of G lanes, lane gl multiplying the factors r = 1 + gl, 1 + gl + G, ...  Callers keep k <= 32 G, so a lane
 * multiplies at most 32 factors below 2^31: no overflow check inside the loop. */
template <int G>
__device__ __forceinline__ BinomME binom_me_group(int64_t t, int k, int gl) {
    double num = 1.0, den = 1.0;
    int ex = 0;
    const double base = (double)(t - k), kd = (double)k;
    for (double r = (double)(1 + gl); r <= kd; r += (double)G) {
        num *= base + r;
        den *= r;
    }
    int fe;
    double mant = frexp_pos(num / den, fe); /* in [0.5, 1) */
    ex += fe;
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) { /* a * b == b * a bit for bit: every lane of the group ends with the same pair */
        const double m2 = __shfl_xor_sync(0xffffffffu, mant, o);
        const int e2 = __shfl_xor_sync(0xffffffffu, ex, o);
        int f2;
        mant = frexp_pos(mant * m2, f2);
        ex += e2 + f2;
    }
    BinomME b;
    b.mant = mant;
    b.ex = ex;
    return b;
}

/* cells first .. first + cnt - 1 of the previous row (outside its band): C(i + k, k) * 2^-e_p, by groups of G lanes of warps 2..;
 * slot0 = ring slot of cell `first` */
template <int G>
__device__ __forceinline__ void rows_extend(double *ring, uint32_t cap, int64_t first, uint32_t slot0, int64_t cnt, int k, int e_p, int tid, int nt) {
    const int groups = (nt - 64) / G;         /* warps 0 and 1 are busy with the scale and the seed */
    const int gid = (tid - 64) / G, gl = (tid - 64) % G;
    for (int64_t base = 0; base < cnt; base += groups) { /* trip count uniform over the block: the shuffles need whole warps */
        const int64_t q = base + gid;
        const bool live = q < cnt;
        const int64_t i = first + (live ? q : 0);
        const BinomME b = binom_me_group<G>(i + k, live ? k : 0, gl);
        if (live && gl == 0) {
            uint32_t sl = slot0 + (uint32_t)q; /* slot0 < cap, q < cap */
            if (sl >= cap) sl -= cap;
            ring[sl] = ldexp_fast(b.mant, b.ex - e_p);
        }
    }
}

__device__ double rows_scan_smem(const SweepConst &c, double *ring, int cap_i, int tid, int nt) {
    __shared__ double s_warp[32];
    __shared__ double s_seed_m;
    __shared__ int s_seed_e, s_e;
    const int64_t m = c.m, mg = c.mg, ng = c.ng, h = c.h;
    const int n = (int)c.n;
    const uint32_t cap = (uint32_t)cap_i;
    const int lane = tid & 31, warp = tid >> 5;

    /* band limits without a division per row: lo_j = floor((mg j - h) / ng) + 1, hi_j = floor((mg j + h - 1) / ng), kept as
     * quotient + remainder and advanced by (mg div ng, mg mod ng) */
    const int64_t dq = mg / ng, dr = mg % ng;
    int64_t qa = floor_div(-h, ng), ra = -h - qa * ng;
    int64_t qb = floor_div(h - 1, ng), rb = h - 1 - qb * ng;

    int64_t lo_p = 0, hi_p = min(qb, m); /* row 0: cells 0 .. hi_0, inside the band no path has left it */
    uint32_t lo_slot = 0;                /* ring slot of cell lo_p */
    for (int64_t i = tid; i <= hi_p; i += nt) ring[(uint32_t)i % cap] = 0.0;
    int e_p = 1;
    __syncthreads();
    for (int j = 1; j <= n; ++j) {
        qa += dq, ra += dr;
        if (ra >= ng) ra -= ng, ++qa;
        qb += dq, rb += dr;
        if (rb >= ng) rb -= ng, ++qb;
        const int64_t lo = max(qa + 1, (int64_t)0), hi = min(qb, m);
        /* the cells of the previous row this row reads and that row never computed (they were outside its band): from
         * max(hi_p + 1, lo) -- when the band jumps past the previous one, the cells below lo are not needed, and writing them
         * could wrap onto slots of cells that are */
        lo_slot = (uint32_t)(((uint64_t)lo_slot + (uint64_t)(lo - lo_p)) % cap);
        const int64_t first = max(hi_p + 1, lo);
        uint32_t first_slot = lo_slot + (uint32_t)(first - lo); /* first - lo <= w <= cap */
        if (first_slot >= cap) first_slot -= cap;
        if (warp == 0) {
            const BinomME b = binom_me_group<32>(hi + j, j, lane);
            if (lane == 0) s_e = b.ex;
        } else if (warp == 1) {
            const BinomME b = binom_me_group<32>(lo - 1 + j, lo >= 1 ? j : 0, lane);
            if (lane == 0) {
                s_seed_m = lo >= 1 ? b.mant : 0.0;
                s_seed_e = b.ex;
            }
        } else {
            const int k = j - 1;
            if (k <= 32) rows_extend<1>(ring, cap, first, first_slot, hi - first + 1, k, e_p, tid, nt);
            else if (k <= 256) rows_extend<8>(ring, cap, first, first_slot, hi - first + 1, k, e_p, tid, nt);
            else rows_extend<32>(ring, cap, first, first_slot, hi - first + 1, k, e_p, tid, nt);
        }
        __syncthreads();
        const int e = s_e;
        const double seed = s_seed_m == 0.0 ? 0.0 : ldexp_fast(s_seed_m, s_seed_e - e);
        const double scale = ldexp_fast(1.0, e_p - e);
        const int64_t w = hi - lo + 1;
        const uint32_t L = (((uint32_t)max(w, (int64_t)1) + (uint32_t)nt - 1u) / (uint32_t)nt) | 1u; /* w <= cap */
        const int64_t a0 = lo + (int64_t)((uint32_t)tid * L), a1 = min(a0 + (int64_t)L, hi + 1);
        const int cnt = a1 > a0 ? (int)(a1 - a0) : 0;
        uint32_t s0 = lo_slot + (uint32_t)tid * L; /* tid L < w + 2 nt <= 2 cap */
        if (s0 >= cap) s0 -= cap;
        if (s0 >= cap) s0 -= cap;
        double local = 0.0;
        {
            uint32_t sl = s0;
            for (int q = 0; q < cnt; ++q) {
                local += ring[sl] * scale;
                if (++sl == cap) sl = 0;
            }
        }
        double incl = local;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            double wv = lane < (nt >> 5) ? s_warp[lane] : 0.0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const double v = __shfl_up_sync(0xffffffffu, wv, o);
                if (lane >= o) wv += v;
            }
            s_warp[lane] = wv;
        }
        __syncthreads();
        double run = seed + (warp > 0 ? s_warp[warp - 1] : 0.0) + (incl - local);
        {
            uint32_t sl = s0;
            for (int q = 0; q < cnt; ++q) {
                run += ring[sl] * scale;
                ring[sl] = run;
                if (++sl == cap) sl = 0;
            }
        }
        lo_p = lo;
        hi_p = hi;
        e_p = e;
        __syncthreads();
    }
    if (tid == 0) return ring[(lo_slot + (uint32_t)(m - lo_p)) % cap] / binom_scaled(m + n, n, e_p);
    return 0.0;
}

/* Where the row scans are exact.  Row j is held scaled by 2^-E_j (E_j: the exponent of its largest binomial, 2^E_j <= 2 C(hi_j + j, j)),
 * so what a cell holds below 2^-1074 of that scale -- a seed C(lo - 1 + j, j) far left of the band, a scaled-down cell -- is lost:
 * at most 8 * 2^-1074 * 2^E_j per cell and row, w + 2 cells a row (w = hi - lo + 1 <= 2h/ng + 1).  A loss at (i, j) reaches (m, n)
 * along at most C(m - i + n - j, n - j) paths, and C(hi + j, j) C(m - lo + 1 + n - j, n - j) <= C(m + n + w, n) (Vandermonde), so
 * relative to C(m + n, n) the error of p is at most  n (w + 2) 2^(4 - 1074) prod_k (m + w + k) / (m + k)
 *                                                  <= n (w + 2) 2^(4 - 1074) ((m + w + 1) / (m + 1))^n.
 * A row-scan p-value is kept when it exceeds that bound by 2^40 (relative error <= 1e-12); below (p = 3.4e-183 at n = 1024 against
 * 30 000 rows, D = 0.45, where the row scan gives half of the true p) the sweep recomputes it. */
__device__ inline bool rows_scan_trusted(double pv, int64_t m, int64_t n, int64_t w) {
    const double lg = log2((double)n * (double)(w + 2)) + (4.0 - 1074.0 + 40.0) + (double)n * log2((double)(m + w + 1) / (double)(m + 1));
    return pv >= exp2(lg);
}

extern __shared__ unsigned char drift_smem[];

__global__ void __launch_bounds__(B2F_DRIFT_THREADS) k_drift_finish(DriftParams p) {
    const int f = blockIdx.x;
    const int tid = threadIdx.x, nt = blockDim.x;
    if (f >= p.n_num) { /* categorical feature: a few hundred flops, one thread */
        if (tid == 0) {
            const int c = f - p.n_num;
            double s, pv;
            chi2_feature(p, c, s, pv);
            p.stat[c] = s;
            p.p_val[c] = pv;
            p.flags[c] = 0;
        }
        return;
    }
    const int out = p.n_cat + f;
    __shared__ uint32_t s_wa[32], s_wb[32];
    __shared__ unsigned long long s_num;

    /* ---- (1) K-S numerator: max over reference points of |n*(#ref <= r) - m0*(#batch <= r)| and the left limits.
     *      Running counts over the m0 + 1 histogram bins: warp w owns a contiguous segment, lanes read consecutive bins
     *      (coalesced), pass 1 adds the segment up, one barrier, pass 2 walks it again 32 bins at a time with shuffle scans.
     *      (Giving each THREAD a contiguous run of 30 bins instead makes every load of a warp touch 32 different lines, and
     *      leaves the 1024 partial sums to be scanned by one thread.) */
    const int64_t m0 = p.n_ref, n0 = p.n;
    const uint32_t *ha = p.hist_a + (int64_t)f * (m0 + 1);
    const uint32_t *hb = p.hist_b + (int64_t)f * (m0 + 1);
    const double *r = p.ref_sorted + (int64_t)f * m0;
    {
        const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
        const int64_t total = m0 + 1;
        const int64_t seg = ((total + nwarps - 1) / nwarps + 31) / 32 * 32;
        const int64_t w0 = min((int64_t)warp * seg, total), w1 = min(w0 + seg, total);
        uint32_t sa = 0, sb = 0; /* counts of batch elements: below 2^31 */
        for (int64_t j = w0 + lane; j < w1; j += 32) {
            sa += ha[j];
            sb += hb[j];
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        if (lane == 0) {
            s_wa[warp] = sa;
            s_wb[warp] = sb;
        }
        if (tid == 0) s_num = 0ull;
        __syncthreads();
        uint32_t ca = 0, cb = 0; /* bins before this warp's segment */
        for (int k = 0; k < warp; ++k) {
            ca += s_wa[k];
            cb += s_wb[k];
        }
        int64_t best = 0;
        for (int64_t b = w0; b < w1; b += 32) {
            const int64_t j = b + lane;
            const bool in = j < w1;
            uint32_t ia = in ? ha[j] : 0u, ib = in ? hb[j] : 0u;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t ua = __shfl_up_sync(0xffffffffu, ia, o), ub = __shfl_up_sync(0xffffffffu, ib, o);
                if (lane >= o) {
                    ia += ua;
                    ib += ub;
                }
            }
            if (in && j < m0) {
                const int64_t cle = (int64_t)(ca + ia); /* #batch <= r_j:  x <= r_j  <=>  (#ref <  x) <= j */
                const int64_t clt = (int64_t)(cb + ib); /* #batch <  r_j:  x <  r_j  <=>  (#ref <= x) <= j */
                const double rj = r[j];
                const bool first = j == 0 || r[j - 1] != rj;     /* #ref <  r_j == j     */
                const bool last = j == m0 - 1 || r[j + 1] != rj; /* #ref <= r_j == j + 1 */
                if (last) {
                    int64_t v = (j + 1) * n0 - cle * m0;
                    if (v < 0) v = -v;
                    best = max(best, v);
                }
                if (first) {
                    int64_t v = j * n0 - clt * m0;
                    if (v < 0) v = -v;
                    best = max(best, v);
                }
            }
            ca += __shfl_sync(0xffffffffu, ia, 31);
            cb += __shfl_sync(0xffffffffu, ib, 31);
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) best = max(best, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)best, o));
        if (lane == 0) atomicMax(&s_num, (unsigned long long)best);
    }
    __syncthreads();
    const int64_t num = (int64_t)s_num;
    const double dstat = (double)num / ((double)m0 * (double)n0);

    /* ---- (2) exact two-sided p-value */
    const int64_t g = gcd64(m0, n0);
    const int64_t m = max(m0, n0), n = min(m0, n0); /* the recursion wants m >= n */
    const int64_t mg = m / g, ng = n / g;
    const int64_t h = num / g; /* == round(D * lcm(m, n)) */
    int flag = 0;
    if (p.nan_count[f] != 0) flag = 2;
    else if ((double)(m0 / g) >= 2147483647.0 / (double)(n0 / g)) flag = 1; /* scipy: lcm too big -> asymptotic formula */
    /* widest anti-diagonal of the band: in-band j satisfy |ng*t - (ng+mg)*j| < h */
    const int64_t width = (2 * h) / (ng + mg) + 2;
    int64_t ring_need = 32;
    while (ring_need < width + 3) ring_need <<= 1;
    /* wider than the shared-memory ring: D * mn/(m+n) > ~2045.  p is not necessarily negligible there (1.6e-264 at
     * m = n = 30 000, D = 0.142; ~1e-7 at m = n = 10^6, D = 0.004): the sweep then runs through the global scratch */
    const bool too_wide = ring_need > B2F_DRIFT_RING_MAX;
    const int ring = (int)min(ring_need, (int64_t)B2F_DRIFT_RING_MAX);
    if (tid == 0) {
        p.stat[out] = dstat;
        p.flags[out] = flag;
        if (flag == 2) p.p_val[out] = nan("");
        else if (flag == 1) p.p_val[out] = -1.0; /* caller applies kstwo.sf(D, round(m*n/(m+n))) */
        else if (h == 0) p.p_val[out] = 1.0;
    }
    if (flag != 0 || h == 0) return;
    if (n == 1) {
        /* single-row request (the common one): the m + 1 lattice paths -- one up-step after k right-steps, k = 0..m --
         * are equally likely, and a path stays strictly inside |i - m*j| < h iff m - h < k < h: no sweep needed */
        if (tid == 0) {
            const int64_t lo = max(m - h + 1, (int64_t)0), hi = min(h - 1, m);
            const int64_t inside = hi >= lo ? hi - lo + 1 : 0;
            p.p_val[out] = (double)(m + 1 - inside) / (double)(m + 1);
        }
        return;
    }

    SweepConst c;
    c.m = m;
    c.n = n;
    c.mg = mg;
    c.ng = ng;
    c.den = ng + mg;
    c.h = h;
    c.T = m + n;
    c.ring = too_wide ? (int)ring_need : ring;
    double res;
    const bool smem_rows = n >= 2 && n <= (int64_t)p.rowscan_smem_max_n && m == m0 && m >= 1024 && (2 * h) / ng + 2 <= (int64_t)p.rowscan_cap;
    if (smem_rows || (p.row_scratch && n >= 2 && n <= (int64_t)p.rowscan_max_n && m == m0 && m >= 1024)) {
        __shared__ int s_keep;
        if (smem_rows) {
            /* request-sized batch, band narrow enough for the row to stay in shared memory: n in-place prefix sums */
            res = rows_scan_smem(c, reinterpret_cast<double *>(drift_smem), p.rowscan_cap, tid, nt);
        } else {
            /* request-sized batch against the big reference table: n prefix sums instead of m + n dependent steps */
            double *rows2 = p.row_scratch + (int64_t)f * 2 * B2F_DRIFT_ROW_STRIDE(m0);
            res = rows_scan(c, rows2, rows2 + B2F_DRIFT_ROW_STRIDE(m0), tid, nt);
        }
        if (tid == 0) {
            res = fmin(fmax(res, 0.0), 1.0);
            s_keep = rows_scan_trusted(res, m, n, (2 * h) / ng + 1);
            if (s_keep) p.p_val[out] = res;
        }
        __syncthreads(); /* also: the ring's last read is done before a sweep reuses the shared memory */
        if (s_keep) return;
    }
    if (too_wide) {
        double *bufs = p.wide_scratch + (int64_t)f * 2 * p.wide_ring;
        if (!p.wide_scratch || ring_need > p.wide_ring) { /* the host sizes the scratch for every band this batch size allows */
            if (tid == 0) p.p_val[out] = nan("");
            return;
        }
        res = sweep_wide(c, tid, nt, bufs, bufs + ring_need);
    } else if (ring == 32) {
        if (tid >= 32) return;
        res = sweep_warp(c, tid);
    } else {
        if (tid >= ring) return; /* whole warps leave (ring is a multiple of 32); the rest meet on named barrier 1 */
        const int active = min(nt, ring);
        double *bufs = reinterpret_cast<double *>(drift_smem);
        const int ns = ring / active;
        if (ns == 1) res = sweep_block<1>(c, tid, active, bufs, bufs + ring);
        else if (ns == 2) res = sweep_block<2>(c, tid, active, bufs, bufs + ring);
        else res = sweep_block<4>(c, tid, active, bufs, bufs + ring);
    }
    if (tid == 0) p.p_val[out] = fmin(fmax(res, 0.0), 1.0);
}
