/*
 * feature_moments.cuh -- K2: per-feature (count, mean, M2) over N encoded rows, sm_90a.
 *
 * BASELINE config 5 ("drift-monitor path: per-feature mean/var reduction").  The reference has no
 * mean/var computation; the nearest call on its path is `self.drift.predict(df[all].values)`
 * (reference databricks/src/02-register-model.ipynb:338).  This is a pure HBM-bound streaming
 * reduction: 96 B read per row, 24*3 float64 written per launch.
 *
 * Structure: a TMA-fed shared-memory ring per CTA.  A producer warp streams 256-row slabs (24 KB,
 * contiguous) with cp.async.bulk + mbarrier complete_tx into a 3-stage ring; 12 consumer warps read
 * 16-byte vectors of the rows from shared memory.  WARP w owns vector q = w mod 6 of every row (its
 * lanes take consecutive rows), so which of its four words are categorical (integer) and which numeric
 * (float32, NaN = missing) is WARP-UNIFORM and compiled in (consume_slabs<NC>): no per-word type select,
 * no NaN test on integer words, and the missing-value case is a predicate on the three accumulations
 * instead of selects.  (Round 1 gave thread t vector t mod 6: every word went through both conversions
 * and a select chain, 83 instructions per vector: issue-bound, not memory-bound.)
 * Memory-level parallelism comes from the ring (3 CTAs x 3 stages x 24 KB = 216 KB in flight per SM),
 * not from registers: a first version that relied on unrolled LDG.128 got one or two loads in flight
 * per warp from ptxas and stalled on the long scoreboard.
 * Arithmetic: shifted float64 sums sum(x-K), sum((x-K)^2) and an integer count per word (K = the word's
 * value in row 0; the shift removes the cancellation of the raw sum-of-squares form).  Block partials are
 * reduced through shared memory in a fixed order, written to global memory, and the last block to finish
 * (atomic ticket) reduces the partials in a fixed order, so the result is deterministic.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b2f.h"

#include "forest_predict.cuh" /* mbarrier / TMA helpers */

#define B2F_MOM_ROWS_PER_BLOCK 64
#define B2F_MOM_CONSUMERS (B2F_MOM_ROWS_PER_BLOCK * 6) /* 384 consumer threads = 12 warps */
#define B2F_MOM_THREADS (B2F_MOM_CONSUMERS + 32)       /* + 1 producer warp */
#define B2F_MOM_VALUES (B2F_ROW_WORDS * 3)
#define B2F_MOM_SLAB_ROWS 256
#define B2F_MOM_SLAB_BYTES (B2F_MOM_SLAB_ROWS * B2F_ROW_BYTES) /* 24 576 */
#define B2F_MOM_STAGES 3
#define B2F_MOM_SMEM (B2F_MOM_STAGES * B2F_MOM_SLAB_BYTES)     /* 73 728 B dynamic */

__device__ __forceinline__ double mom_word_value(uint32_t w, int word, int n_cat) {
    return word < n_cat ? (double)(int32_t)w : (double)__uint_as_float(w);
}

__device__ __forceinline__ void mbar_arrive_cta(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}

/* One consumer warp, its vector q of every row of its slabs; NC = how many of the vector's four words are categorical
 * (integers, never missing): the words' types are compile-time, the accumulations of a missing numeric are predicated off. */
template <int NC>
__device__ __forceinline__ void consume_slabs(const uint8_t *ring, uint64_t *full_bar, uint64_t *empty_bar, long long my_slabs, long long n, int q,
                                              int half, int lane, const double (&K)[4], unsigned int (&cnt)[4], double (&s)[4], double (&ss)[4]) {
    for (long long k = 0; k < my_slabs; ++k) {
        const int st = (int)(k % B2F_MOM_STAGES);
        mbar_wait(&full_bar[st], (uint32_t)((k / B2F_MOM_STAGES) & 1));
        const long long r0 = ((long long)blockIdx.x + k * gridDim.x) * B2F_MOM_SLAB_ROWS;
        const int rows_here = (int)min((long long)B2F_MOM_SLAB_ROWS, n - r0);
        const uint4 *slab = reinterpret_cast<const uint4 *>(ring + st * B2F_MOM_SLAB_BYTES);
#pragma unroll
        for (int i = 0; i < B2F_MOM_SLAB_ROWS / 64; ++i) {
            const int row = i * 64 + half * 32 + lane;
            if (row < rows_here) {
                const uint4 v = slab[row * 6 + q];
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    if (c < NC) {
                        const double d = (double)(int32_t)w[c] - K[c];
                        cnt[c] += 1u;
                        s[c] += d;
                        ss[c] = fma(d, d, ss[c]);
                    } else {
                        const float xf = __uint_as_float(w[c]);
                        const double d = (double)xf - K[c];
                        if (xf == xf) { /* a missing value contributes nothing */
                            cnt[c] += 1u;
                            s[c] += d;
                            ss[c] = fma(d, d, ss[c]);
                        }
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive_cta(&empty_bar[st]);
    }
}

__global__ void __launch_bounds__(B2F_MOM_THREADS, 3)
    k_feature_moments(const uint4 *__restrict__ rows, long long n, int n_cat, double *__restrict__ partials,
                      unsigned int *__restrict__ ticket, double *__restrict__ out) {
    extern __shared__ __align__(128) uint8_t ring[]; /* B2F_MOM_STAGES slabs; reused as `red` at the end */
    __shared__ __align__(8) uint64_t full_bar[B2F_MOM_STAGES];
    __shared__ __align__(8) uint64_t empty_bar[B2F_MOM_STAGES];
    __shared__ double tot[B2F_MOM_VALUES];
    __shared__ double tot_seg[4][B2F_MOM_VALUES];
    __shared__ bool is_last;
    double(*red)[12 + 1] = reinterpret_cast<double(*)[12 + 1]>(ring); /* [384][13] doubles = 39 936 B */

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < B2F_MOM_STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], B2F_MOM_CONSUMERS / 32);
        }
        fence_mbar_init();
        fence_proxy_async();
    }
    __syncthreads();

    const long long n_slabs = (n + B2F_MOM_SLAB_ROWS - 1) / B2F_MOM_SLAB_ROWS;
    const long long my_slabs = blockIdx.x < n_slabs ? (n_slabs - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (warp == B2F_MOM_CONSUMERS / 32) {
        /* ===== producer warp: one lane feeds the ring with TMA bulk copies ===== */
        if (lane == 0) {
            for (long long k = 0; k < my_slabs; ++k) {
                const int st = (int)(k % B2F_MOM_STAGES);
                const long long j = k / B2F_MOM_STAGES;
                if (j > 0) mbar_wait(&empty_bar[st], (uint32_t)((j - 1) & 1));
                const long long slab = blockIdx.x + k * gridDim.x;
                const long long r0 = slab * B2F_MOM_SLAB_ROWS;
                const uint32_t bytes = (uint32_t)(min((long long)B2F_MOM_SLAB_ROWS, n - r0) * B2F_ROW_BYTES);
                mbar_arrive_expect_tx(&full_bar[st], bytes);
                tma_bulk_g2s(ring + st * B2F_MOM_SLAB_BYTES, reinterpret_cast<const uint8_t *>(rows) + r0 * B2F_ROW_BYTES, bytes, &full_bar[st]);
            }
        }
    } else {
        /* ===== consumer warps: warp w reads vector q = w mod 6 of rows half*32 + lane (+ 64 i) of every slab ===== */
        const int q = warp % 6, half = warp / 6;
        double K[4];
        {
            const uint4 v0 = n > 0 ? __ldg(rows + q) : make_uint4(0, 0, 0, 0);
            const uint32_t w0[4] = {v0.x, v0.y, v0.z, v0.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const double x = mom_word_value(w0[k], q * 4 + k, n_cat);
                K[k] = (x == x) ? x : 0.0;
            }
        }
        unsigned int cnt[4] = {0, 0, 0, 0};
        double s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
        const int nc = min(4, max(0, n_cat - q * 4)); /* categorical words of this warp's vector: warp-uniform */
        switch (nc) {
            case 0: consume_slabs<0>(ring, full_bar, empty_bar, my_slabs, n, q, half, lane, K, cnt, s, ss); break;
            case 1: consume_slabs<1>(ring, full_bar, empty_bar, my_slabs, n, q, half, lane, K, cnt, s, ss); break;
            case 2: consume_slabs<2>(ring, full_bar, empty_bar, my_slabs, n, q, half, lane, K, cnt, s, ss); break;
            case 3: consume_slabs<3>(ring, full_bar, empty_bar, my_slabs, n, q, half, lane, K, cnt, s, ss); break;
            default: consume_slabs<4>(ring, full_bar, empty_bar, my_slabs, n, q, half, lane, K, cnt, s, ss); break;
        }
        /* `red` aliases the ring: every consumer must be done reading slabs before anyone overwrites it */
        asm volatile("bar.sync 1, %0;" ::"n"(B2F_MOM_CONSUMERS) : "memory");
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            red[threadIdx.x][k * 3 + 0] = (double)cnt[k];
            red[threadIdx.x][k * 3 + 1] = s[k];
            red[threadIdx.x][k * 3 + 2] = ss[k];
        }
    }
    __syncthreads();

    /* (word, component) -> fixed-order sum over the 64 threads of that vector, in 4 segments of 16 so 288 threads
     * share the latency-bound chain; the 4 segment sums are then added in order */
    if (threadIdx.x < 4 * B2F_MOM_VALUES) {
        const int v = threadIdx.x % B2F_MOM_VALUES, sg = threadIdx.x / B2F_MOM_VALUES;
        const int word = v / 3, comp = v % 3;
        const int wq = word / 4, wk = word % 4;
        /* the 64 threads that hold vector wq: warps wq and wq + 6, lanes in order */
        const int first = ((sg >> 1) * 6 + wq) * 32 + (sg & 1) * 16;
        double a = 0.0;
#pragma unroll 4
        for (int r = first; r < first + 16; ++r) a += red[r][wk * 3 + comp];
        tot_seg[sg][v] = a;
    }
    __syncthreads();
    if (threadIdx.x < B2F_MOM_VALUES)
        partials[(size_t)blockIdx.x * B2F_MOM_VALUES + threadIdx.x] =
            ((tot_seg[0][threadIdx.x] + tot_seg[1][threadIdx.x]) + tot_seg[2][threadIdx.x]) + tot_seg[3][threadIdx.x];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!is_last) return;
    __threadfence();

    /* last block: reduce the block partials in a fixed order -- 5 interleaved segments per value so
     * 360 threads work and every thread's loads are independent (the adds form 5 short chains) */
    {
        double *seg = &red[0][0]; /* reuse: [5][72] */
        __syncthreads();
        if (threadIdx.x < 5 * B2F_MOM_VALUES) {
            const int v = threadIdx.x % B2F_MOM_VALUES, sgm = threadIdx.x / B2F_MOM_VALUES;
            double a = 0.0;
#pragma unroll 8
            for (unsigned int b = sgm; b < gridDim.x; b += 5) a += __ldcg(partials + (size_t)b * B2F_MOM_VALUES + v);
            seg[sgm * B2F_MOM_VALUES + v] = a;
        }
        __syncthreads();
        if (threadIdx.x < B2F_MOM_VALUES) {
            double a = 0.0;
            for (int sgm = 0; sgm < 5; ++sgm) a += seg[sgm * B2F_MOM_VALUES + threadIdx.x];
            tot[threadIdx.x] = a;
        }
    }
    __syncthreads();
    if (threadIdx.x < B2F_ROW_WORDS) {
        const int word = threadIdx.x;
        const double c = tot[word * 3 + 0], S = tot[word * 3 + 1], SS = tot[word * 3 + 2];
        double Kw = 0.0; /* this word's pivot: its value in row 0 (NaN -> 0), as above */
        if (n > 0) {
            const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t *>(rows) + word);
            Kw = mom_word_value(w0, word, n_cat);
            if (!(Kw == Kw)) Kw = 0.0;
        }
        double mean = 0.0, m2 = 0.0;
        if (c > 0.0) {
            mean = Kw + S / c;
            m2 = SS - S * S / c;
            if (m2 < 0.0) m2 = 0.0;
        }
        out[word * 3 + 0] = c;
        out[word * 3 + 1] = mean;
        out[word * 3 + 2] = m2;
    }
    if (threadIdx.x == 0) *ticket = 0; /* re-arm for the next launch on this stream */
}
