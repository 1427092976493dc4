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
 * Arithmetic: shifted float64 sums sum(x-K), sum((x-K)^2) and an integer count per word; the shift removes the
 * cancellation of the raw sum-of-squares form when it is a value of the column.  Each warp takes as K the first present
 * value of the word it meets (no search: until then it has accumulated nothing, so adopting K is exact), so a column that
 * is missing in row 0, over a long leading run or everywhere costs nothing extra.  Partials shifted by different pivots
 * are combined by re-shifting (mom_absorb): the two warps of a vector in shared memory, the blocks' (count, S, SS, K) in
 * a fixed order by the last block to finish (atomic ticket), so the result is deterministic.
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
#define B2F_MOM_PARTIAL_VALUES (B2F_MOM_VALUES + B2F_ROW_WORDS) /* per block: (count, S, SS) per word, then its pivots */
#define B2F_MOM_FINAL_SEGS 16

__device__ __forceinline__ double mom_word_value(uint32_t w, int word, int n_cat) {
    return word < n_cat ? (double)(int32_t)w : (double)__uint_as_float(w);
}

/* Sums (c, S, SS) shifted by pivot K absorb a partial (cb, Sb, SSb) shifted by its own pivot Kb: the partial is re-shifted
 * to K (S' = Sb + cb d, SS' = SSb + d (2 Sb + cb d), d = Kb - K).  Until something has been accumulated the partial's pivot
 * is adopted as is, so the first present value met stays the pivot.  Both pivots are values of the column, so d is of the
 * order of its spread and the re-shift keeps SS - S^2/c free of cancellation. */
__device__ __forceinline__ void mom_absorb(double &c, double &S, double &SS, double &K, double cb, double Sb, double SSb, double Kb) {
    if (!(cb > 0.0)) return;
    if (c == 0.0) K = Kb;
    const double d = Kb - K;
    c += cb;
    S += Sb + cb * d;
    SS += SSb + d * (2.0 * Sb + cb * d);
}

__device__ __forceinline__ void mbar_arrive_cta(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}

/* One consumer warp, rows half*32 + lane + 64 i of one landed slab, its vector q; NC = how many of the vector's four words
 * are categorical (integers, never missing): the words' types are compile-time, the accumulations of a missing numeric
 * are predicated off.  SETTLE: some word (bit c of `todo`) has no pivot yet, because this warp has met no present value
 * of it: before each row group the warp ballots, and the first present value becomes the word's pivot K[c].  Nothing has
 * been accumulated for that word until then, so the change of pivot is exact.  An all-missing word keeps K = 0 and costs
 * one ballot per row group; once every word has a pivot the warp takes the SETTLE = false form. */
template <int NC, bool SETTLE>
__device__ __forceinline__ void consume_slab(const uint4 *slab, int rows_here, int q, int half, int lane, unsigned int &todo, double (&K)[4],
                                             unsigned int (&cnt)[4], double (&s)[4], double (&ss)[4]) {
#pragma unroll
    for (int i = 0; i < B2F_MOM_SLAB_ROWS / 64; ++i) {
        const int row = i * 64 + half * 32 + lane;
        const bool live = row < rows_here;
        const uint4 v = (SETTLE || live) ? slab[row * 6 + q] : make_uint4(0, 0, 0, 0); /* in the ring either way */
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        if (SETTLE) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                if ((todo >> c) & 1u) {
                    const double x = c < NC ? (double)(int32_t)w[c] : (double)__uint_as_float(w[c]);
                    const unsigned int present = __ballot_sync(0xFFFFFFFFu, live && (c < NC || x == x));
                    if (present != 0u) {
                        K[c] = __shfl_sync(0xFFFFFFFFu, x, __ffs(present) - 1);
                        todo &= ~(1u << c);
                    }
                }
            }
        }
        if (live) {
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
}

template <int NC>
__device__ __forceinline__ void consume_slabs(const uint8_t *ring, uint64_t *full_bar, uint64_t *empty_bar, long long my_slabs, long long n, int q,
                                              int half, int lane, double (&K)[4], unsigned int (&cnt)[4], double (&s)[4], double (&ss)[4]) {
    unsigned int todo = 0xFu; /* words of this warp without a pivot yet: warp-uniform */
    for (long long k = 0; k < my_slabs; ++k) {
        const int st = (int)(k % B2F_MOM_STAGES);
        mbar_wait(&full_bar[st], (uint32_t)((k / B2F_MOM_STAGES) & 1));
        const long long r0 = ((long long)blockIdx.x + k * gridDim.x) * B2F_MOM_SLAB_ROWS;
        const int rows_here = (int)min((long long)B2F_MOM_SLAB_ROWS, n - r0);
        const uint4 *slab = reinterpret_cast<const uint4 *>(ring + st * B2F_MOM_SLAB_BYTES);
        if (todo != 0u)
            consume_slab<NC, true>(slab, rows_here, q, half, lane, todo, K, cnt, s, ss);
        else
            consume_slab<NC, false>(slab, rows_here, q, half, lane, todo, K, cnt, s, ss);
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
    __shared__ double tot_seg[4][B2F_MOM_VALUES];
    __shared__ double piv[B2F_MOM_CONSUMERS / 32][4]; /* each consumer warp's pivots of its vector's four words */
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
        double K[4] = {0.0, 0.0, 0.0, 0.0}; /* set per word by consume_slabs from the first present value this warp meets */
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
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < 4; ++k) piv[warp][k] = K[k];
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
    /* the block's partial per word: warp wq's sums (segments 0, 1) absorb warp wq + 6's (segments 2, 3), re-shifted to the
     * first warp's pivot unless that warp met no value; stored with the pivot they are shifted by */
    if (threadIdx.x < B2F_ROW_WORDS) {
        const int word = threadIdx.x, v = word * 3, wq = word / 4, wk = word % 4;
        double c = 0.0, S = 0.0, SS = 0.0, K = 0.0;
        mom_absorb(c, S, SS, K, tot_seg[0][v] + tot_seg[1][v], tot_seg[0][v + 1] + tot_seg[1][v + 1], tot_seg[0][v + 2] + tot_seg[1][v + 2], piv[wq][wk]);
        mom_absorb(c, S, SS, K, tot_seg[2][v] + tot_seg[3][v], tot_seg[2][v + 1] + tot_seg[3][v + 1], tot_seg[2][v + 2] + tot_seg[3][v + 2], piv[wq + 6][wk]);
        double *p = partials + (size_t)blockIdx.x * B2F_MOM_PARTIAL_VALUES;
        p[v + 0] = c;
        p[v + 1] = S;
        p[v + 2] = SS;
        p[B2F_MOM_VALUES + word] = K;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!is_last) return;
    __threadfence();

    /* last block: absorb the block partials in a fixed order -- 16 interleaved segments per word so 384 threads work
     * and every thread's loads are independent (the absorptions form 16 short chains), then the 16 segments in order */
    double(*seg)[B2F_ROW_WORDS][4] = reinterpret_cast<double(*)[B2F_ROW_WORDS][4]>(ring); /* reuse: [16][24][4] */
    __syncthreads();
    if (threadIdx.x < B2F_MOM_FINAL_SEGS * B2F_ROW_WORDS) {
        const int word = threadIdx.x % B2F_ROW_WORDS, sgm = threadIdx.x / B2F_ROW_WORDS;
        double c = 0.0, S = 0.0, SS = 0.0, K = 0.0;
#pragma unroll 4
        for (unsigned int b = sgm; b < gridDim.x; b += B2F_MOM_FINAL_SEGS) {
            const double *p = partials + (size_t)b * B2F_MOM_PARTIAL_VALUES;
            mom_absorb(c, S, SS, K, __ldcg(p + word * 3), __ldcg(p + word * 3 + 1), __ldcg(p + word * 3 + 2), __ldcg(p + B2F_MOM_VALUES + word));
        }
        seg[sgm][word][0] = c;
        seg[sgm][word][1] = S;
        seg[sgm][word][2] = SS;
        seg[sgm][word][3] = K;
    }
    __syncthreads();
    if (threadIdx.x < B2F_ROW_WORDS) {
        const int word = threadIdx.x;
        double c = 0.0, S = 0.0, SS = 0.0, K = 0.0;
        for (int sgm = 0; sgm < B2F_MOM_FINAL_SEGS; ++sgm) mom_absorb(c, S, SS, K, seg[sgm][word][0], seg[sgm][word][1], seg[sgm][word][2], seg[sgm][word][3]);
        double mean = 0.0, m2 = 0.0;
        if (c > 0.0) {
            mean = K + S / c;
            m2 = SS - S * S / c;
            if (m2 < 0.0) m2 = 0.0;
        }
        out[word * 3 + 0] = c;
        out[word * 3 + 1] = mean;
        out[word * 3 + 2] = m2;
    }
    if (threadIdx.x == 0) *ticket = 0; /* re-arm for the next launch on this stream */
}
