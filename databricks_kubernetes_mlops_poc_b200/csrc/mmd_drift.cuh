/*
 * mmd_drift.cuh -- K9: the kernel two-sample (MMD) drift test of a batch against a reference table (sm_90a, FP64).
 *
 * alibi-detect's MMDDrift on the classifier's input vectors: a row is its one-hot categoricals (an unknown or missing code
 * is the all-zero block) and its numerics as scored (float32, NaN imputed with the training median), z-scored in float64
 * with the reference's mean and population std.  Squared distance of two rows:
 *     d(a, b) = sum_num (z_a - z_b)^2 + sum_cat cost,  cost = 2 (both codes known and different), 1 (exactly one is -1), 0
 * which is the squared Euclidean distance of the dense vectors, computed by direct differences, the numerics in field order
 * with separate multiplies and adds (no FMA) and the integer cost added last: numpy's d + x * x in that order gives the
 * same bits, so the select's sigma is exact against a host count.  k(a, b) = exp(-d * coef) with coef = 1 / (2 sigma^2).
 *
 * Pool: [reference (n_ref rows); batch (m rows)], pool index p < n_ref in the reference arrays, else the batch's.  Per row:
 * n_num doubles (z) and n_cat int32 codes, row-major.
 *
 * Every pair kernel works on 128 x 128 tiles: thread t holds row a_t of the A tile (transposed in shared memory, za[f][t]),
 * the B tile sits row-major (zb[j][f], read as broadcasts), and each thread sums its pairs over j in order.  Block sums use
 * one fixed tree; integers are the only atomics (the select's histogram), so results are bit-identical from run to run.
 *
 *   k_mmd_embed        rows (B2F_ROWS_WORDS24 / B2F_ROWS_PACKED64) -> z, codes
 *   k_mmd_select_hist  one digit pass of the exact radix select of a pair distance over the reference triangle
 *   k_mmd_row_sums     grid (A tiles, column chunks): partial[chunk][a] = sum over the chunk's b != a of k(a, b)
 *   k_mmd_row_finish   r[a] = base[a] + sum over chunks of partial[chunk][a], in chunk order
 *   k_mmd_subset_pairs grid (J tile, I tile <= J, subset): the sum of k over the subset's pairs in tile pair (I, J)
 *   k_mmd_finish       block = subset: T = sum r, R_U = sum of r over the subset, S_UU from the tile sums -> mmd^2
 */
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#define B2F_MMD_TILE 128
#define B2F_MMD_SUB 8            /* B rows per inner step: their distances live in registers */
#define B2F_MMD_CHUNK_TILES 16   /* column tiles per k_mmd_row_sums block */
#define B2F_MMD_DIGIT_BITS 11    /* radix select digit: 6 passes over the 64-bit key */
#define B2F_MMD_FINISH_THREADS 256

struct MmdParams {
    int n_cat, n_num;
    float impute[24];  /* per row word: the blob's float32 training median (numeric words) */
    double mean[24];   /* per numeric (index k, not row word): the reference's mean */
    double scale[24];  /* per numeric: the reference's population std, 1 where it is 0 */
};

struct MmdPool {
    const double *zr;  /* reference: n_ref x n_num */
    const int32_t *cr; /* reference: n_ref x n_cat */
    const double *zb;  /* batch: m x n_num */
    const int32_t *cb; /* batch: m x n_cat */
    long long n_ref;
    int n_cat, n_num;
};

/* one thread per row: the embedding of row i into z[i * n_num + k] and c[i * n_cat + j] */
template <bool PACKED>
__global__ void __launch_bounds__(256) k_mmd_embed(const __grid_constant__ MmdParams p, const uint32_t *__restrict__ rows, long long n,
                                                   double *__restrict__ z, int32_t *__restrict__ c) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned long long codes = 0;
    const uint32_t *row = rows + i * (PACKED ? 16 : 24);
    if (PACKED) codes = ((unsigned long long)row[1] << 32) | row[0];
    for (int j = 0; j < p.n_cat; ++j) c[i * p.n_cat + j] = PACKED ? (int32_t)((codes >> (7 * j)) & 0x7fu) - 1 : (int32_t)row[j];
    for (int k = 0; k < p.n_num; ++k) {
        float v = __uint_as_float(row[(PACKED ? 2 : p.n_cat) + k]);
        if (isnan(v)) v = p.impute[p.n_cat + k];
        z[i * p.n_num + k] = ((double)v - p.mean[k]) / p.scale[k];
    }
}

/* dynamic shared memory of the pair kernels: an A and a B tile of z and codes */
static inline size_t mmd_smem_bytes(int n_cat, int n_num) { return (size_t)2 * B2F_MMD_TILE * (8 * n_num + 4 * n_cat); }

struct MmdTiles {
    double *za, *zb;  /* za[f * TILE + t], zb[j * n_num + f] */
    int32_t *ca, *cb; /* ca[f * TILE + t], cb[j * n_cat + f] */
};

__device__ __forceinline__ MmdTiles mmd_tiles(unsigned char *smem, int n_cat, int n_num) {
    MmdTiles s;
    s.za = reinterpret_cast<double *>(smem);
    s.zb = s.za + (size_t)B2F_MMD_TILE * n_num;
    s.ca = reinterpret_cast<int32_t *>(s.zb + (size_t)B2F_MMD_TILE * n_num);
    s.cb = s.ca + (size_t)B2F_MMD_TILE * n_cat;
    return s;
}

/* pool row pi (pi < 0: an empty slot, zeros) into slot t of the A tile (a) or the B tile (!a) */
__device__ __forceinline__ void mmd_load(const MmdPool &P, long long pi, const MmdTiles &s, int t, bool a) {
    const double *z = nullptr;
    const int32_t *c = nullptr;
    if (pi >= 0) {
        if (pi < P.n_ref) z = P.zr + pi * P.n_num, c = P.cr + pi * P.n_cat;
        else z = P.zb + (pi - P.n_ref) * P.n_num, c = P.cb + (pi - P.n_ref) * P.n_cat;
    }
    for (int f = 0; f < P.n_num; ++f) (a ? s.za[f * B2F_MMD_TILE + t] : s.zb[t * P.n_num + f]) = z ? __ldg(z + f) : 0.0;
    for (int f = 0; f < P.n_cat; ++f) (a ? s.ca[f * B2F_MMD_TILE + t] : s.cb[t * P.n_cat + f]) = c ? __ldg(c + f) : -1;
}

/* d[jj] = d(row t of the A tile, row j0 + jj of the B tile) for jj < B2F_MMD_SUB: numerics first, then the categorical cost */
__device__ __forceinline__ void mmd_dists(const MmdTiles &s, int n_cat, int n_num, int t, int j0, double (&d)[B2F_MMD_SUB]) {
#pragma unroll
    for (int jj = 0; jj < B2F_MMD_SUB; ++jj) d[jj] = 0.0;
    for (int f = 0; f < n_num; ++f) {
        const double a = s.za[f * B2F_MMD_TILE + t];
#pragma unroll
        for (int jj = 0; jj < B2F_MMD_SUB; ++jj) {
            const double x = a - s.zb[(j0 + jj) * n_num + f];
            d[jj] = __dadd_rn(d[jj], __dmul_rn(x, x)); /* not fused: numpy's d + x * x gives the same bits */
        }
    }
    int cost[B2F_MMD_SUB];
#pragma unroll
    for (int jj = 0; jj < B2F_MMD_SUB; ++jj) cost[jj] = 0;
    for (int f = 0; f < n_cat; ++f) {
        const int32_t a = s.ca[f * B2F_MMD_TILE + t];
#pragma unroll
        for (int jj = 0; jj < B2F_MMD_SUB; ++jj) {
            const int32_t b = s.cb[(j0 + jj) * n_cat + f];
            cost[jj] += a == b ? 0 : ((a < 0 || b < 0) ? 1 : 2);
        }
    }
#pragma unroll
    for (int jj = 0; jj < B2F_MMD_SUB; ++jj) d[jj] += (double)cost[jj];
}

/* fixed-order block sum over blockDim.x (a power of two) threads; sh holds blockDim.x values */
template <typename V>
__device__ __forceinline__ V mmd_block_sum(V v, V *sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    const V r = sh[0];
    __syncthreads();
    return r;
}

/* One digit pass of the select over the reference's pairs a < b: hist[digit] += the pairs whose key (the bits of the
 * non-negative double d) equals prefix on mask, by digit (key >> shift) & (2^width - 1).  Integer counts: the order of the
 * atomics does not matter.  grid (J tile, I tile); I > J exits. */
__global__ void __launch_bounds__(B2F_MMD_TILE)
    k_mmd_select_hist(const __grid_constant__ MmdPool P, unsigned long long prefix, unsigned long long mask, int shift, int width,
                      unsigned long long *__restrict__ hist) {
    const int I = blockIdx.y, J = blockIdx.x;
    if (I > J) return;
    extern __shared__ __align__(16) unsigned char mmd_smem[];
    __shared__ unsigned int sh[1 << B2F_MMD_DIGIT_BITS];
    const MmdTiles s = mmd_tiles(mmd_smem, P.n_cat, P.n_num);
    const int t = threadIdx.x;
    for (int b = t; b < (1 << B2F_MMD_DIGIT_BITS); b += B2F_MMD_TILE) sh[b] = 0;
    const long long a = (long long)I * B2F_MMD_TILE + t, b0 = (long long)J * B2F_MMD_TILE;
    mmd_load(P, a < P.n_ref ? a : -1, s, t, true);
    mmd_load(P, b0 + t < P.n_ref ? b0 + t : -1, s, t, false);
    __syncthreads();
    const int nb = (int)min((long long)B2F_MMD_TILE, P.n_ref - b0);
    const unsigned long long dmask = (1ull << width) - 1ull;
    if (a < P.n_ref) {
        for (int j0 = 0; j0 < nb; j0 += B2F_MMD_SUB) {
            double d[B2F_MMD_SUB];
            mmd_dists(s, P.n_cat, P.n_num, t, j0, d);
#pragma unroll
            for (int jj = 0; jj < B2F_MMD_SUB; ++jj) {
                const unsigned long long key = (unsigned long long)__double_as_longlong(d[jj]);
                if (j0 + jj < nb && a < b0 + j0 + jj && (key & mask) == prefix) atomicAdd(&sh[(key >> shift) & dmask], 1u);
            }
        }
    }
    __syncthreads();
    for (int b = t; b < (1 << B2F_MMD_DIGIT_BITS); b += B2F_MMD_TILE)
        if (sh[b]) atomicAdd(hist + b, (unsigned long long)sh[b]);
}

/* grid (A tiles, column chunks of B2F_MMD_CHUNK_TILES tiles): partial[chunk * na + i] = the sum, over pool columns
 * b in [b_lo + chunk * CH, ...) below b_hi with b != a, of k(a, b), a = a_lo + i, summed in column order */
__global__ void __launch_bounds__(B2F_MMD_TILE)
    k_mmd_row_sums(const __grid_constant__ MmdPool P, long long a_lo, long long na, long long b_lo, long long b_hi, double coef,
                   double *__restrict__ partial) {
    extern __shared__ __align__(16) unsigned char mmd_smem[];
    const MmdTiles s = mmd_tiles(mmd_smem, P.n_cat, P.n_num);
    const int t = threadIdx.x;
    const long long i = (long long)blockIdx.x * B2F_MMD_TILE + t, a = a_lo + i;
    mmd_load(P, i < na ? a : -1, s, t, true);
    const long long c0 = b_lo + (long long)blockIdx.y * B2F_MMD_CHUNK_TILES * B2F_MMD_TILE;
    const long long c1 = min(b_hi, c0 + (long long)B2F_MMD_CHUNK_TILES * B2F_MMD_TILE);
    double acc = 0.0;
    for (long long b0 = c0; b0 < c1; b0 += B2F_MMD_TILE) {
        __syncthreads(); /* the previous B tile is consumed */
        mmd_load(P, b0 + t < c1 ? b0 + t : -1, s, t, false);
        __syncthreads();
        const int nb = (int)min((long long)B2F_MMD_TILE, c1 - b0);
        for (int j0 = 0; j0 < nb; j0 += B2F_MMD_SUB) {
            double d[B2F_MMD_SUB];
            mmd_dists(s, P.n_cat, P.n_num, t, j0, d);
#pragma unroll
            for (int jj = 0; jj < B2F_MMD_SUB; ++jj)
                if (j0 + jj < nb && b0 + j0 + jj != a) acc += exp(-d[jj] * coef);
        }
    }
    if (i < na) partial[(long long)blockIdx.y * na + i] = acc;
}

/* r[i] = (base ? base[i] : 0) + partial[0][i] + partial[1][i] + ... */
__global__ void __launch_bounds__(256)
    k_mmd_row_finish(const double *__restrict__ partial, int chunks, long long na, const double *__restrict__ base, double *__restrict__ r) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= na) return;
    double v = base ? base[i] : 0.0;
    for (int c = 0; c < chunks; ++c) v += partial[(long long)c * na + i];
    r[i] = v;
}

/* grid (J tile, I tile, subset u): partial[(u * nt + I) * nt + J] = the sum of k over the pairs of positions p < q of subset
 * u (pool indices sub[u * s + p]) with p in tile I and q in tile J; I > J exits */
__global__ void __launch_bounds__(B2F_MMD_TILE)
    k_mmd_subset_pairs(const __grid_constant__ MmdPool P, const int32_t *__restrict__ sub, long long s, int nt, double coef,
                       double *__restrict__ partial) {
    const int I = blockIdx.y, J = blockIdx.x;
    if (I > J) return;
    extern __shared__ __align__(16) unsigned char mmd_smem[];
    __shared__ double sh[B2F_MMD_TILE];
    const MmdTiles s_ = mmd_tiles(mmd_smem, P.n_cat, P.n_num);
    const int t = threadIdx.x;
    const int32_t *su = sub + (long long)blockIdx.z * s;
    const long long p = (long long)I * B2F_MMD_TILE + t, q0 = (long long)J * B2F_MMD_TILE;
    mmd_load(P, p < s ? (long long)__ldg(su + p) : -1, s_, t, true);
    mmd_load(P, q0 + t < s ? (long long)__ldg(su + q0 + t) : -1, s_, t, false);
    __syncthreads();
    const int nb = (int)min((long long)B2F_MMD_TILE, s - q0);
    double acc = 0.0;
    if (p < s) {
        for (int j0 = 0; j0 < nb; j0 += B2F_MMD_SUB) {
            double d[B2F_MMD_SUB];
            mmd_dists(s_, P.n_cat, P.n_num, t, j0, d);
#pragma unroll
            for (int jj = 0; jj < B2F_MMD_SUB; ++jj)
                if (j0 + jj < nb && p < q0 + j0 + jj) acc += exp(-d[jj] * coef);
        }
    }
    acc = mmd_block_sum(acc, sh);
    if (t == 0) partial[((long long)blockIdx.z * nt + I) * nt + J] = acc;
}

/* block = subset u: the statistic of the split whose side U is subset u (the batch-sized side when u_is_batch, else the
 * reference-sized side) and whose other side V is the rest of the pool.  With r_i = sum_{j != i} k(i, j) over the pool,
 * T = sum r, R_U = sum_{i in U} r_i and S_UU = 2 * (the pair sum inside U):  S_UV = R_U - S_UU,  S_VV = T - S_UU - 2 S_UV,
 * mmd^2 = S_XX / (n (n - 1)) + S_YY / (m (m - 1)) - 2 S_XY / (n m). */
__global__ void __launch_bounds__(B2F_MMD_FINISH_THREADS)
    k_mmd_finish(const double *__restrict__ r, long long N, const int32_t *__restrict__ sub, long long s, const double *__restrict__ partial,
                 int nt, long long n_ref, long long m, int u_is_batch, double *__restrict__ out) {
    __shared__ double sh[B2F_MMD_FINISH_THREADS];
    const int t = threadIdx.x;
    const int32_t *su = sub + (long long)blockIdx.x * s;
    double v = 0.0;
    for (long long i = t; i < N; i += B2F_MMD_FINISH_THREADS) v += r[i];
    const double T = mmd_block_sum(v, sh);
    v = 0.0;
    for (long long i = t; i < s; i += B2F_MMD_FINISH_THREADS) v += r[su[i]];
    const double RU = mmd_block_sum(v, sh);
    v = 0.0;
    const double *pu = partial + (long long)blockIdx.x * nt * nt;
    for (long long k = t; k < (long long)nt * nt; k += B2F_MMD_FINISH_THREADS)
        if (k / nt <= k % nt) v += pu[k];
    const double S = mmd_block_sum(v, sh);
    if (t == 0) {
        const double Suu = 2.0 * S, Suv = RU - Suu, Svv = T - Suu - 2.0 * Suv;
        const double Sxx = u_is_batch ? Svv : Suu, Syy = u_is_batch ? Suu : Svv;
        const double n = (double)n_ref, mm = (double)m;
        out[blockIdx.x] = Sxx / (n * (n - 1.0)) + Syy / (mm * (mm - 1.0)) - 2.0 * Suv / (n * mm);
    }
}
