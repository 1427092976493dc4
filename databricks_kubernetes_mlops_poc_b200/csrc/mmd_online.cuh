/*
 * mmd_online.cuh -- K13: the online MMD drift detector (alibi-detect's MMDDriftOnline) in K9's space (sm_90a, FP64).
 *
 * A reference of n_ref rows with row sums r_i = sum_{j != i} k(i, j) (K9's r_ref) and T = sum r.  A window size W and
 * E = 2W - 1.  A row sequence x_0 .. x_{n-1} (a bootstrap's E reference rows, or the stream's last W - 1 rows followed by
 * a pushed piece) is described per row s by
 *     c_s     = sum_{i in R} k(i, x_s)                     (R: the sub-reference of rw = n_ref - E rows)
 *     P[s][L] = sum_{d = 1 .. L} k(x_s, x_{s-d}),  L < W     (band prefixes, d ascending; P[s][0] = 0)
 * and the window starting at w (rows w .. w + W - 1) by
 *     S_RW(w) = sum_s c_s,  S_WW(w) = 2 sum_s P[s][s - w]   (s ascending: oldest first)
 *     stat(w) = K_RR / (rw (rw - 1)) + S_WW / (W (W - 1)) - 2 S_RW / (rw W)
 * mmd_online_window is that one helper; the bootstrap and the stream both go through it.  For a bootstrap y (E reference
 * positions, R the other rows): q_s = sum_{i in y, i != s} k(y_s, y_i), c_s = r_{y_s} - q_s and K_RR = T - 2 sum r_y + sum q.
 * For the stream, c_s comes from K9's k_mmd_row_sums against the compacted R and K_RR from the configuration.
 *
 * P is stored transposed, band[L * n + s], so that the window threads w, w + 1, ... read consecutive doubles.  Each P[s][L]
 * depends on x_s and its L predecessors only, so a row's values, and every window statistic, are the same bits however the
 * stream is cut into pushes and pieces.  No float atomics.
 *
 *   k_mmd_online_gather  rows by index: the compacted sub-reference and the initial window
 *   k_mmd_online_total   T = sum of r over the reference (one block, fixed order)
 *   k_mmd_online_band    grid (A tiles, sequences): P of every row; in the bootstrap form also q and c
 *   k_mmd_online_boot    block = bootstrap: K_RR and the statistic of every window position
 *   k_mmd_online_steps   thread = pushed row: the statistic of the window that ends at it
 */
#pragma once
#include "mmd_drift.cuh"

#define B2F_MMD_ONLINE_THREADS 256

/* one thread per row: dst row i = src row idx[i] (z and codes) */
__global__ void __launch_bounds__(256) k_mmd_online_gather(const double *__restrict__ zs, const int32_t *__restrict__ cs, const int32_t *__restrict__ idx,
                                                           long long n, int n_cat, int n_num, double *__restrict__ zd, int32_t *__restrict__ cd) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long src = __ldg(idx + i);
    for (int k = 0; k < n_num; ++k) zd[i * n_num + k] = zs[src * n_num + k];
    for (int k = 0; k < n_cat; ++k) cd[i * n_cat + k] = cs[src * n_cat + k];
}

/* one block of B2F_MMD_ONLINE_THREADS: *out = sum of r[0 .. n), strided per thread, then mmd_block_sum */
__global__ void __launch_bounds__(B2F_MMD_ONLINE_THREADS) k_mmd_online_total(const double *__restrict__ r, long long n, double *__restrict__ out) {
    __shared__ double sh[B2F_MMD_ONLINE_THREADS];
    double v = 0.0;
    for (long long i = threadIdx.x; i < n; i += B2F_MMD_ONLINE_THREADS) v += r[i];
    v = mmd_block_sum(v, sh);
    if (threadIdx.x == 0) *out = v;
}

/* grid (A tiles, sequences): sequence q has n rows, row s at pool index pos[q * n + s] (BOOT) or s (the stream's sequence is
 * the pool's reference part).  band[(q * W + L) * n + s] = P[s][L] for L <= min(s, W - 1), summed d ascending: the B tiles
 * are walked from the row's own tile down, each from its last row down.  BOOT: the walk covers all n rows, and
 * qsum[q * n + s] = q_s (i descending), c[q * n + s] = r[pos] - q_s. */
template <bool BOOT>
__global__ void __launch_bounds__(B2F_MMD_TILE)
    k_mmd_online_band(const __grid_constant__ MmdPool P, const int32_t *__restrict__ pos, long long n, int W, double coef,
                      const double *__restrict__ r, double *__restrict__ band, double *__restrict__ qsum, double *__restrict__ c) {
    extern __shared__ __align__(16) unsigned char mmd_smem[];
    const MmdTiles s_ = mmd_tiles(mmd_smem, P.n_cat, P.n_num);
    const int t = threadIdx.x;
    const long long q = blockIdx.y, s0 = (long long)blockIdx.x * B2F_MMD_TILE, s = s0 + t;
    const int32_t *pq = BOOT ? pos + q * n : nullptr;
    double *bq = band + q * W * n;
    const bool live = s < n;
    mmd_load(P, live ? (BOOT ? (long long)__ldg(pq + s) : s) : -1, s_, t, true);
    if (live) bq[s] = 0.0;
    const long long lo = BOOT ? 0 : max(0LL, s0 - (W - 1)) / B2F_MMD_TILE;
    const long long hi = BOOT ? (n - 1) / B2F_MMD_TILE : s0 / B2F_MMD_TILE;
    double acc = 0.0, qs = 0.0;
    for (long long J = hi; J >= lo; --J) {
        const long long b0 = J * B2F_MMD_TILE;
        __syncthreads(); /* the previous B tile is consumed */
        mmd_load(P, b0 + t < n ? (BOOT ? (long long)__ldg(pq + b0 + t) : b0 + t) : -1, s_, t, false);
        __syncthreads();
        const int nb = (int)min((long long)B2F_MMD_TILE, n - b0);
        for (int j0 = ((nb - 1) / B2F_MMD_SUB) * B2F_MMD_SUB; j0 >= 0; j0 -= B2F_MMD_SUB) {
            double d[B2F_MMD_SUB];
            mmd_dists(s_, P.n_cat, P.n_num, t, j0, d);
#pragma unroll
            for (int jj = B2F_MMD_SUB - 1; jj >= 0; --jj) {
                const long long i = b0 + j0 + jj, L = s - i;
                if (!live || j0 + jj >= nb || L == 0 || (!BOOT && (L < 0 || L >= W))) continue;
                const double kv = exp(-d[jj] * coef);
                if (BOOT) qs += kv;
                if (L > 0 && L < W) {
                    acc += kv;
                    bq[L * n + s] = acc;
                }
            }
        }
    }
    if (BOOT && live) {
        qsum[q * n + s] = qs;
        c[q * n + s] = r[__ldg(pq + s)] - qs;
    }
}

/* the window of W rows starting at row w of a sequence of n rows: S_RW and S_WW from c and the transposed band prefixes,
 * oldest row first */
__device__ __forceinline__ void mmd_online_window(const double *__restrict__ c, const double *__restrict__ band, long long n, int W, long long w,
                                                  double &s_rw, double &s_ww) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < W; ++k) {
        a += c[w + k];
        b += band[(long long)k * n + w + k];
    }
    s_rw = a;
    s_ww = 2.0 * b;
}

__device__ __forceinline__ double mmd_online_stat(double k_rr, double s_ww, double s_rw, long long rw, int W) {
    const double r = (double)rw, w = (double)W;
    return k_rr / (r * (r - 1.0)) + s_ww / (w * (w - 1.0)) - 2.0 * s_rw / (r * w);
}

/* block = bootstrap q (E = 2W - 1 rows): K_RR = *total - 2 sum r_y + sum q, then stats[q * W + w] for every window
 * position w; k_rr[q] = K_RR */
__global__ void __launch_bounds__(B2F_MMD_ONLINE_THREADS)
    k_mmd_online_boot(const double *__restrict__ r, const int32_t *__restrict__ pos, const double *__restrict__ total, const double *__restrict__ qsum,
                      const double *__restrict__ c, const double *__restrict__ band, int W, long long rw, double *__restrict__ stats,
                      double *__restrict__ k_rr) {
    __shared__ double sh[B2F_MMD_ONLINE_THREADS];
    const int t = threadIdx.x;
    const long long q = blockIdx.x, E = 2LL * W - 1;
    double v = 0.0;
    for (long long s = t; s < E; s += B2F_MMD_ONLINE_THREADS) v += r[__ldg(pos + q * E + s)];
    const double ry = mmd_block_sum(v, sh);
    v = 0.0;
    for (long long s = t; s < E; s += B2F_MMD_ONLINE_THREADS) v += qsum[q * E + s];
    const double see = mmd_block_sum(v, sh);
    const double krr = *total - 2.0 * ry + see;
    if (t < W) {
        double s_rw, s_ww;
        mmd_online_window(c + q * E, band + q * W * E, E, W, t, s_rw, s_ww);
        stats[q * W + t] = mmd_online_stat(krr, s_ww, s_rw, rw, W);
    }
    if (t == 0) k_rr[q] = krr;
}

/* thread = pushed row i < m of a sequence of n = W - 1 + m rows: out[i] = the statistic of the window ending at row
 * W - 1 + i (starting at row i) */
__global__ void __launch_bounds__(B2F_MMD_ONLINE_THREADS)
    k_mmd_online_steps(const double *__restrict__ c, const double *__restrict__ band, long long n, int W, long long m, long long rw, double k_rr,
                       double *__restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    double s_rw, s_ww;
    mmd_online_window(c, band, n, W, i, s_rw, s_ww);
    out[i] = mmd_online_stat(k_rr, s_ww, s_rw, rw, W);
}
