/*
 * knn.cuh -- K11: exact k-nearest reference rows of each query row, per class (sm_90a, FP64); the device half of trust scores.
 *
 * The space is K9's (mmd_drift.cuh): rows embedded by k_mmd_embed with the trust reference's mean and scale, and the squared
 * distance d(a, b) of mmd_dists (numerics in field order as d + x * x without FMA, then the integer categorical cost), so every
 * distance equals numpy's bit for bit.  A NaN distance (only infinite inputs make one) ranks as +inf.
 *
 * The reference sits class-sorted in the pool's reference arrays: class c holds positions [lo_c, lo_c + n_c), each class in
 * the original row order.  The queries are the pool's batch side (pool index n_ref + q).  Candidates are ordered by the pair
 * (d, position): ties go to the lower position, which is the lower original index.  No float atomics, no order that depends on
 * scheduling: two calls give the same bytes.
 *
 *   k_knn_chunk  grid (query tiles, chunks, class): thread t = query row, the A tile transposed in shared memory, B tiles of the
 *                class's chunk read as broadcasts.  Each thread keeps its sorted top-k list in shared memory (list[j][t]) and
 *                its k-th distance in a register: a candidate is looked at only when it beats that.  With one chunk the
 *                list is the answer (sqrt and the original index are written); else it goes to the candidate scratch.
 *   k_knn_merge  block = (query, class): each candidate's rank in the union of the chunk lists is its position in its own
 *                list plus, per other list, how many entries precede it (a binary search); rank < k is written.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "mmd_drift.cuh" /* and include/b2f.h before it: B2F_KNN_MAX_K */

#define B2F_KNN_MERGE_THREADS 128
#define B2F_KNN_NONE 0x7fffffff /* the index of an empty candidate slot (distance +inf) */

struct KnnArgs {
    long long nq;             /* query rows of this launch (pool indices n_ref .. n_ref + nq) */
    long long lo[2], n[2];    /* class c: reference positions [lo[c], lo[c] + n[c]) */
    long long chunk_rows;     /* rows per chunk, a multiple of B2F_MMD_TILE */
    int k, chunks;            /* chunks == 1: the lists are written as the answer */
    const int32_t *orig;      /* reference position -> original row index */
    double *dist;             /* chunks == 1: [q][class][k] sqrt(d) */
    int32_t *index;           /* chunks == 1: [q][class][k] original index */
    double *cand_d;           /* chunks > 1: [q][class][chunk][k] d */
    int32_t *cand_i;          /* chunks > 1: [q][class][chunk][k] reference position, B2F_KNN_NONE when empty */
};

/* dynamic shared memory of k_knn_chunk: K9's A and B tiles, then the per-thread lists (doubles first, then positions) */
static inline size_t knn_smem_bytes(int n_cat, int n_num, int k) {
    return mmd_smem_bytes(n_cat, n_num) + (size_t)B2F_MMD_TILE * k * (8 + 4);
}

/* (d, i) before (e, j) in the lexicographic order */
__device__ __forceinline__ bool knn_before(double d, int32_t i, double e, int32_t j) { return d < e || (d == e && i < j); }

__global__ void __launch_bounds__(B2F_MMD_TILE) k_knn_chunk(const __grid_constant__ MmdPool P, const __grid_constant__ KnnArgs A) {
    extern __shared__ __align__(16) unsigned char knn_smem[];
    const MmdTiles s = mmd_tiles(knn_smem, P.n_cat, P.n_num);
    double *ld = reinterpret_cast<double *>(s.cb + (size_t)B2F_MMD_TILE * P.n_cat); /* past the B tile: 8-byte aligned */
    int32_t *li = reinterpret_cast<int32_t *>(ld + (size_t)B2F_MMD_TILE * A.k);
    const int t = threadIdx.x, cls = blockIdx.z, chunk = blockIdx.y;
    const long long b_lo = A.lo[cls] + (long long)chunk * A.chunk_rows;
    const long long b_end = A.lo[cls] + A.n[cls];
    if (b_lo >= b_end) return; /* this class has fewer chunks than the grid */
    const long long b_hi = min(b_end, b_lo + A.chunk_rows);
    const long long q = (long long)blockIdx.x * B2F_MMD_TILE + t;
    mmd_load(P, q < A.nq ? P.n_ref + q : -1, s, t, true);
    int cnt = 0;         /* entries in the list */
    double kth = 0.0;    /* the list's last distance once it is full */
    for (long long b0 = b_lo; b0 < b_hi; b0 += B2F_MMD_TILE) {
        __syncthreads(); /* the previous B tile is consumed */
        mmd_load(P, b0 + t < b_hi ? b0 + t : -1, s, t, false);
        __syncthreads();
        if (q >= A.nq) continue;
        const int nb = (int)min((long long)B2F_MMD_TILE, b_hi - b0);
        for (int j0 = 0; j0 < nb; j0 += B2F_MMD_SUB) {
            double d[B2F_MMD_SUB];
            mmd_dists(s, P.n_cat, P.n_num, t, j0, d);
#pragma unroll
            for (int jj = 0; jj < B2F_MMD_SUB; ++jj) {
                const double v = isnan(d[jj]) ? (double)INFINITY : d[jj];
                /* positions rise along the scan: an equal distance comes after every entry already listed */
                if (j0 + jj < nb && (cnt < A.k || v < kth)) {
                    int j = cnt < A.k ? cnt : A.k - 1;
                    while (j > 0 && ld[(j - 1) * B2F_MMD_TILE + t] > v) {
                        ld[j * B2F_MMD_TILE + t] = ld[(j - 1) * B2F_MMD_TILE + t];
                        li[j * B2F_MMD_TILE + t] = li[(j - 1) * B2F_MMD_TILE + t];
                        --j;
                    }
                    ld[j * B2F_MMD_TILE + t] = v;
                    li[j * B2F_MMD_TILE + t] = (int32_t)(b0 + j0 + jj);
                    if (cnt < A.k) ++cnt;
                    if (cnt == A.k) kth = ld[(A.k - 1) * B2F_MMD_TILE + t];
                }
            }
        }
    }
    if (q >= A.nq) return;
    if (A.chunks == 1) {
        const long long o = (q * 2 + cls) * A.k;
        for (int j = 0; j < A.k; ++j) {
            A.dist[o + j] = __dsqrt_rn(ld[j * B2F_MMD_TILE + t]);
            A.index[o + j] = __ldg(A.orig + li[j * B2F_MMD_TILE + t]);
        }
        return;
    }
    const long long o = ((q * 2 + cls) * A.chunks + chunk) * A.k;
    for (int j = 0; j < A.k; ++j) {
        const bool has = j < cnt;
        A.cand_d[o + j] = has ? ld[j * B2F_MMD_TILE + t] : (double)INFINITY;
        A.cand_i[o + j] = has ? li[j * B2F_MMD_TILE + t] : B2F_KNN_NONE;
    }
}

/* block = (query q, class c) as blockIdx.x = q * 2 + c; the class's chunk lists -> its top k, in order */
__global__ void __launch_bounds__(B2F_KNN_MERGE_THREADS) k_knn_merge(const __grid_constant__ KnnArgs A) {
    const long long qc = blockIdx.x;
    const int cls = (int)(qc & 1);
    const int lists = (int)((A.n[cls] + A.chunk_rows - 1) / A.chunk_rows);
    const double *cd = A.cand_d + qc * A.chunks * A.k;
    const int32_t *ci = A.cand_i + qc * A.chunks * A.k;
    for (int e = threadIdx.x; e < lists * A.k; e += B2F_KNN_MERGE_THREADS) {
        const int32_t i = ci[e];
        if (i == B2F_KNN_NONE) continue;
        const double d = cd[e];
        const int own = e / A.k;
        int rank = e - own * A.k;
        for (int l = 0; l < lists && rank < A.k; ++l) {
            if (l == own) continue;
            /* entries of list l before (d, i): the lists are sorted, empty slots last */
            int a = 0, b = A.k;
            while (a < b) {
                const int mid = (a + b) >> 1;
                const int32_t mi = ci[l * A.k + mid];
                if (mi != B2F_KNN_NONE && knn_before(cd[l * A.k + mid], mi, d, i)) a = mid + 1;
                else b = mid;
            }
            rank += a;
        }
        if (rank < A.k) {
            A.dist[qc * A.k + rank] = __dsqrt_rn(d);
            A.index[qc * A.k + rank] = __ldg(A.orig + i);
        }
    }
}
