/*
 * forest_predict.cuh -- K1: fused impute -> one-hot-as-equality -> tree walk -> aggregate kernel
 * for sm_90a.  No tensor cores: the path is a branchy pointer walk, not a contraction.
 *
 * Replaces, on the GPU, what `classifier.predict_proba(df[all_features])[:, 1]` computes on the CPU
 * (reference databricks/src/02-register-model.ipynb:335-337; pipeline definition
 * 01-train-model.ipynb:195-231): SimpleImputer(median) + OneHotEncoder(ignore unknown) +
 * RandomForestClassifier.predict_proba (float32 inputs, float64 mean of leaf class fractions), and
 * for BASELINE configs 2-4 the binary GBDT form expit(init + sum lr*leaf).
 *
 * Geometry: ONE WARP PER ROW (R rows interleaved per warp for ILP); lane l walks tree 32*g + l of
 * group g.  The encoded row lives in registers, one 32-bit word per lane (lanes 0..23), fetched with
 * one coalesced 96-byte load per row; a split's feature value is a warp shuffle from the lane that
 * holds it, so rows never touch shared memory.  The forest lives in shared memory as the
 * tree-interleaved SoA described in forest_blob.h, brought in once per CTA by TMA bulk copies
 * (cp.async.bulk, one mbarrier per tree group so walking group 0 overlaps the copy of groups 1..);
 * CTAs are persistent (grid = #SMs) and stride over the batch.  Per-lane float64 partial sums are
 * combined with a shuffle butterfly.  Forests that do not fit 227 KB of shared memory are walked
 * from global memory / L2 with the same code (WALK_GLOBAL).
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b2f.h"
#include "forest_blob.h"

#define B2F_PREDICT_THREADS 1024
#define B2F_PREDICT_WARPS (B2F_PREDICT_THREADS / 32)
#define B2F_BULK_PIECE (32u * 1024u) /* bytes per cp.async.bulk */
#define B2F_PACKED_ROW_WORDS 16

struct KGroup {
    uint32_t chunk_off;
    uint32_t chunk_bytes;
    uint32_t n_slots;
    uint32_t n_leaf_slots;
    uint32_t depth;
};

struct KParams {
    const uint8_t *chunks; /* device pointer to the first chunk (256-byte aligned) */
    int32_t n_groups;
    int32_t agg_mode;
    int32_t n_cat;
    int32_t n_num;
    double init_raw;
    double denom;
    double threshold; /* isolation forest: is_outlier = score > threshold */
    float impute[24];
    KGroup g[B2F_MAX_GROUPS];
};

/* ---------------------------------------------------------------- PTX helpers */
__device__ __forceinline__ uint32_t smem_addr(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_addr(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(smem_addr(bar)),
        "r"(parity)
        : "memory");
}

/* Node addresses are 32-bit shared-window addresses (SMEM) or 64-bit global addresses (GLOBAL). */
template <bool SMEM>
struct AddrOf {
    using type = uint64_t;
};
template <>
struct AddrOf<true> {
    using type = uint32_t;
};
template <bool SMEM>
__device__ __forceinline__ typename AddrOf<SMEM>::type node_addr(const uint8_t *p) {
    if constexpr (SMEM) {
        return smem_addr(p);
    } else {
        return reinterpret_cast<uint64_t>(p);
    }
}
template <bool SMEM>
__device__ __forceinline__ uint2 ld_node(typename AddrOf<SMEM>::type a) {
    uint2 v;
    if constexpr (SMEM) {
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
    } else {
        asm volatile("ld.global.nc.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(a));
    }
    return v;
}
template <bool SMEM>
__device__ __forceinline__ uint32_t ld_word(typename AddrOf<SMEM>::type a) {
    uint32_t v;
    if constexpr (SMEM) {
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    } else {
        asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(a));
    }
    return v;
}
template <bool SMEM>
__device__ __forceinline__ double ld_leaf(typename AddrOf<SMEM>::type a) {
    double v;
    if constexpr (SMEM) {
        asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
    } else {
        asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(v) : "l"(a));
    }
    return v;
}

/* Branch-free split decision (forest_blob.h): second = (x ==bits t) or (geu(x, t) and not cat);
 * returns `if_second` or `if_first` -- three predicate instructions and one select. */
__device__ __forceinline__ bool take_second(uint32_t x, uint32_t t, uint32_t m) {
    uint32_t c;
    asm("{\n\t"
        ".reg .pred pc, p1, p2;\n\t"
        ".reg .b32 cbit;\n\t"
        "and.b32 cbit, %3, 0x04000000;\n\t"
        "setp.ne.u32 pc, cbit, 0;\n\t"
        "setp.geu.and.f32 p1, %1, %2, !pc;\n\t"
        "setp.eq.or.u32 p2, %4, %5, p1;\n\t"
        "selp.u32 %0, 1, 0, p2;\n\t"
        "}"
        : "=r"(c)
        : "f"(__uint_as_float(x)), "f"(__uint_as_float(t)), "r"(m), "r"(x), "r"(t));
    return c != 0;
}
template <typename A>
__device__ __forceinline__ A pick_child(uint32_t x, uint32_t t, uint32_t m, A if_first, A if_second) {
    return take_second(x, t, m) ? if_second : if_first;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

/* sum of leaf payloads -> (score, label); shared by all predict kernels.
 *   RF       : p1 = s / n_trees, label = argmax (class 1 iff p1 > p0)        (sklearn: proba /= n_estimators)
 *   GBDT     : p1 = expit(init + s), label = raw >= 0   (sklearn >= 1.4 `_gb.py` predict: `raw_predictions >= 0`, the
 *              library the oracle runs; the reference's pin 1.1.1 takes argmax([1-p, p]) and differs only on the exact
 *              tie raw == 0, where it picks class 0.  The reference itself serves a RandomForest, never a GBDT.)
 *   IFOREST  : score = 2^(-s / (n_trees * c(max_samples))) + offset_, flag = score > user threshold, decided as
 *              s <= `threshold`, the largest path-length sum whose score numpy puts above the user threshold (flatten.py)
 *              (sklearn IsolationForest: -decision_function; alibi-detect IForest.predict,
 *              reference databricks/src/02-register-model.ipynb:232-233,339,344)
 * Labels and flags of rows inside the rounding band of the decision are re-decided by forest_decide.cuh. */
__device__ __forceinline__ void aggregate(int agg_mode, double init_raw, double denom, double threshold, double s, double &p1, int &lab) {
    if (agg_mode == B2F_AGG_RF_MEAN) {
        p1 = s / denom;
        lab = s > (denom - s);
    } else if (agg_mode == B2F_AGG_GBDT_LOGISTIC) {
        const double raw = init_raw + s;
        p1 = 1.0 / (1.0 + exp(-raw)); /* expit */
        lab = raw >= 0.0;
    } else {
        p1 = exp2(-(s / denom)) + init_raw;
        lab = s <= threshold; /* threshold: the host's path-length bound, score > user threshold <=> s <= bound */
    }
}

/* Output strides travel in one int: low 16 bits = stride of `proba` in OutT elements, high 16 bits = stride of
 * `label` in int32 elements (0: same as proba's).  1 = two plain arrays; 2 = interleaved {float, int32} pairs
 * (b2f_scored); B2F_OSTRIDE(3, 6) / B2F_OSTRIDE(6, 6) = the double / float fields of a 24-byte b2f_scored_full. */
#define B2F_OSTRIDE(ps, ls) ((ps) | ((ls) << 16))
__device__ __forceinline__ int ostride_p(int o) { return o & 0xffff; }
__device__ __forceinline__ int ostride_l(int o) { return (o >> 16) ? (o >> 16) : (o & 0xffff); }

#include "forest_decide.cuh"

/* aggregate -> (probability, label) for one row per lane; rows < 0 are empty slots */
template <bool PACKED, typename OutT>
__device__ __forceinline__ void finalize_store(const KParams &p, double s, long long row, const uint32_t *__restrict__ rows,
                                               OutT *__restrict__ proba, int32_t *__restrict__ label, int ostride) {
    if (row < 0) return;
    double p1;
    int lab;
    aggregate(p.agg_mode, p.init_raw, p.denom, p.threshold, s, p1, lab);
    if (label && decide_exactly(p.agg_mode, s, p.denom, p.threshold)) lab = decide_row_blob<PACKED>(p, rows, row);
    if (proba) proba[row * ostride_p(ostride)] = (OutT)p1;
    if (label) label[row * ostride_l(ostride)] = lab;
}

/* ---------------------------------------------------------------- the kernel */
/* One group for R rows: D dependent levels, R independent chains interleaved for ILP.
 * D > 0: fully unrolled (the common shallow forests); D == 0: run-time depth. */
template <int R, bool SMEM, int D>
__device__ __forceinline__ void walk_group(typename AddrOf<SMEM>::type a_first, typename AddrOf<SMEM>::type a_leaf, int depth,
                                           const uint32_t (&w)[R], double (&acc)[R]) {
    using addr_t = typename AddrOf<SMEM>::type;
    const addr_t a_second = a_first + B2F_NODE_STRIDE;
    addr_t at[R]; /* address of this lane's current node */
#pragma unroll
    for (int r = 0; r < R; ++r) at[r] = a_first;

    auto level = [&]() {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const uint2 tm = ld_node<SMEM>(at[r]);
            const uint32_t x = __shfl_sync(0xffffffffu, w[r], (int)(tm.y >> B2F_META_FEAT_SHIFT));
            /* (M << 8): top byte (word index, flags) falls out, slot index becomes a byte offset */
            at[r] = pick_child(x, tm.x, tm.y, a_first, a_second) + (addr_t)(tm.y << 8);
        }
    };
    if constexpr (D > 0) {
#pragma unroll
        for (int d = 0; d < D; ++d) level();
    } else {
#pragma unroll 4
        for (int d = 0; d < depth; ++d) level();
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const uint32_t leaf_id = ld_word<SMEM>(at[r]);
        acc[r] += ld_leaf<SMEM>(a_leaf + (addr_t)(leaf_id << 8));
    }
}

template <int R, bool SMEM, bool PACKED, typename OutT>
__global__ void __launch_bounds__(B2F_PREDICT_THREADS, 1)
    k_forest_predict(const __grid_constant__ KParams p, const uint32_t *__restrict__ rows, long long n,
                     OutT *__restrict__ proba, int32_t *__restrict__ label, int ostride) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t bars[B2F_MAX_GROUPS];
    /* per group: {node area, leaf area, depth}: shared-window addresses (SMEM) or byte offsets from
     * p.chunks (GLOBAL); one broadcast 16-byte load per group instead of indexed constant loads */
    __shared__ uint4 gtab[B2F_MAX_GROUPS];

    using addr_t = typename AddrOf<SMEM>::type;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int n_groups = p.n_groups;

    if (threadIdx.x < n_groups) {
        const KGroup gd = p.g[threadIdx.x];
        const uint32_t origin = SMEM ? smem_addr(smem) : 0u;
        gtab[threadIdx.x] = make_uint4(origin + gd.chunk_off, origin + gd.chunk_off + gd.n_slots * B2F_NODE_STRIDE, gd.depth, 0u);
    }
    if constexpr (SMEM) {
        /* one thread arms one mbarrier per tree group and issues the TMA bulk copies */
        if (threadIdx.x == 0) {
            for (int g = 0; g < n_groups; ++g) mbar_init(&bars[g], 1);
            fence_mbar_init();
            fence_proxy_async();
            for (int g = 0; g < n_groups; ++g) {
                const uint32_t bytes = p.g[g].chunk_bytes;
                mbar_arrive_expect_tx(&bars[g], bytes);
                for (uint32_t o = 0; o < bytes; o += B2F_BULK_PIECE) {
                    const uint32_t piece = min(B2F_BULK_PIECE, bytes - o);
                    tma_bulk_g2s(smem + p.g[g].chunk_off + o, p.chunks + p.g[g].chunk_off + o, piece, &bars[g]);
                }
            }
        }
    }
    __syncthreads();

    const uint32_t all_ready = n_groups >= 32 ? 0xffffffffu : ((1u << n_groups) - 1u);
    uint32_t ready = SMEM ? 0u : all_ready; /* bit g: this warp has seen group g's chunk land in shared memory */

    const long long n_batches = (n + R - 1) / R;
    /* CTA-minor numbering: consecutive row batches go to different SMs, so small batches spread
     * over the whole chip instead of filling the first CTAs */
    const long long warp_global = (long long)warp * gridDim.x + blockIdx.x;
    const long long warp_stride = (long long)gridDim.x * B2F_PREDICT_WARPS;

    /* numeric lanes impute NaN with the training median; lanes >= 23 hold the sentinel 0xFFFFFFFF */
    const bool lane_numeric = lane >= p.n_cat && lane < p.n_cat + p.n_num;
    const uint32_t impute_bits = lane < 24 ? __float_as_uint(p.impute[lane]) : 0u;
    const uint32_t lane8 = (uint32_t)lane * 8u; /* this lane's node inside a 256-byte slot */
    const addr_t origin_lane = (SMEM ? (addr_t)0 : (addr_t)reinterpret_cast<uint64_t>(p.chunks)) + lane8;

    /* raw load of this lane's word of a row (decoded by unpack_row when the row is consumed):
     * 96-byte rows: lane l < 23 holds word l;  packed 64-byte rows: lane l < 16 holds word l */
    auto load_row = [&](long long row) -> uint32_t {
        uint32_t v = B2F_SENTINEL_BITS;
        if constexpr (PACKED) {
            if (row < n && lane < B2F_PACKED_ROW_WORDS) v = __ldg(rows + row * B2F_PACKED_ROW_WORDS + lane);
        } else {
            if (row < n && lane < (int)B2F_SENTINEL_WORD) v = __ldg(rows + row * B2F_ROW_WORDS + lane);
        }
        return v;
    };
    /* -> one row word per lane: lanes 0..n_cat-1 category codes, then float32 numerics, sentinel above */
    auto unpack_row = [&](uint32_t v) -> uint32_t {
        if constexpr (PACKED) {
            /* words 0..1: nine 7-bit fields (code + 1, 0 = unknown); words 2..15: the 14 numerics */
            const uint32_t lo = __shfl_sync(0xffffffffu, v, 0), hi = __shfl_sync(0xffffffffu, v, 1);
            const uint32_t num = __shfl_sync(0xffffffffu, v, (lane - 7) & 31);
            const uint32_t field = (uint32_t)(((((unsigned long long)hi) << 32) | lo) >> (7 * (lane < 9 ? lane : 0))) & 0x7fu;
            v = lane < 9 ? field - 1u : (lane < (int)B2F_SENTINEL_WORD ? num : B2F_SENTINEL_BITS);
        }
        if (lane_numeric && isnan(__uint_as_float(v))) v = impute_bits;
        return v;
    };

    double pend_sum = 0.0; /* lane j: tree sum of the j-th row this warp finished since the last flush */
    long long pend_row = -1;
    int pend_n = 0;

    uint32_t wnext[R];
#pragma unroll
    for (int r = 0; r < R; ++r) wnext[r] = warp_global < n_batches ? load_row(warp_global * R + r) : B2F_SENTINEL_BITS;

    for (long long b = warp_global; b < n_batches; b += warp_stride) {
        uint32_t w[R];
        double acc[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            w[r] = unpack_row(wnext[r]);
            acc[r] = 0.0;
        }
        /* prefetch the next batch's rows; the loads complete behind this batch's walk */
        if (b + warp_stride < n_batches) {
#pragma unroll
            for (int r = 0; r < R; ++r) wnext[r] = load_row((b + warp_stride) * R + r);
        }

        for (int g = 0; g < n_groups; ++g) {
            if constexpr (SMEM) {
                if (ready != all_ready) { /* only while the forest is still streaming in */
                    if (!((ready >> g) & 1u)) {
                        mbar_wait(&bars[g], 0);
                        ready |= 1u << g;
                    }
                }
            }
            const uint4 gd = gtab[g];
            const addr_t a_first = origin_lane + gd.x;
            const addr_t a_leaf = origin_lane + gd.y;
            switch (gd.z) {
                case 1: walk_group<R, SMEM, 1>(a_first, a_leaf, 1, w, acc); break;
                case 2: walk_group<R, SMEM, 2>(a_first, a_leaf, 2, w, acc); break;
                case 3: walk_group<R, SMEM, 3>(a_first, a_leaf, 3, w, acc); break;
                case 4: walk_group<R, SMEM, 4>(a_first, a_leaf, 4, w, acc); break;
                case 5: walk_group<R, SMEM, 5>(a_first, a_leaf, 5, w, acc); break;
                case 6: walk_group<R, SMEM, 6>(a_first, a_leaf, 6, w, acc); break;
                case 7: walk_group<R, SMEM, 7>(a_first, a_leaf, 7, w, acc); break;
                case 8: walk_group<R, SMEM, 8>(a_first, a_leaf, 8, w, acc); break;
                default: walk_group<R, SMEM, 0>(a_first, a_leaf, (int)gd.z, w, acc); break;
            }
        }

        /* every lane now holds the row's tree sum; lane `pend_n` keeps it.  The float64 divide / exp
         * of the aggregate and the stores then run once per 32 rows with all lanes busy, instead of
         * once per row on a single lane. */
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const double s = warp_sum(acc[r]);
            const long long row = b * R + r;
            if (lane == pend_n) {
                pend_sum = s;
                pend_row = row < n ? row : -1;
            }
            if (++pend_n == 32) {
                finalize_store<PACKED>(p, pend_sum, pend_row, rows, proba, label, ostride);
                pend_n = 0;
                pend_row = -1;
            }
        }
    }
    if (pend_n > 0) finalize_store<PACKED>(p, pend_sum, pend_row, rows, proba, label, ostride);

    if constexpr (SMEM) {
        /* never retire a CTA while a bulk copy into its shared memory is still in flight */
        for (int g = 0; g < n_groups; ++g)
            if (!((ready >> g) & 1u)) mbar_wait(&bars[g], 0);
    }
}


/* ---------------------------------------------------------------- small batches: groups across warps
 * k_forest_predict_split: the latency form of the warp-per-row kernel.  For a handful of rows the
 * dependent chain -- groups x depth node visits per row -- is what the caller waits for, so the tree
 * GROUPS of one row go to different warps of one CTA (blockDim = 32 * n_groups, one CTA per R rows):
 * every warp walks one group straight from global memory / L2 (no shared-memory fill of a forest that a
 * few rows would not amortise), lane sums are reduced with shuffles, the per-group sums meet in shared
 * memory and are added in group order (deterministic), then finalised.  500 trees x depth 8: the chain
 * drops from 16 x 9 dependent loads to 9. */
template <int R, bool PACKED, typename OutT>
__global__ void __launch_bounds__(1024, 1)
    k_forest_predict_split(const __grid_constant__ KParams p, const uint32_t *__restrict__ rows, long long n,
                           OutT *__restrict__ proba, int32_t *__restrict__ label, int ostride) {
    __shared__ double part[B2F_MAX_GROUPS][R];
    const int lane = threadIdx.x & 31;
    const int g = threadIdx.x >> 5; /* this warp's tree group */
    const long long b = blockIdx.x;
    const bool lane_numeric = lane >= p.n_cat && lane < p.n_cat + p.n_num;
    const uint32_t impute_bits = lane < 24 ? __float_as_uint(p.impute[lane]) : 0u;
    const uint32_t lane8 = (uint32_t)lane * 8u;

    uint32_t w[R];
    double acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const long long row = b * R + r;
        uint32_t v = B2F_SENTINEL_BITS;
        if constexpr (PACKED) {
            if (row < n && lane < B2F_PACKED_ROW_WORDS) v = __ldg(rows + row * B2F_PACKED_ROW_WORDS + lane);
            const uint32_t lo = __shfl_sync(0xffffffffu, v, 0), hi = __shfl_sync(0xffffffffu, v, 1);
            const uint32_t num = __shfl_sync(0xffffffffu, v, (lane - 7) & 31);
            const uint32_t field = (uint32_t)(((((unsigned long long)hi) << 32) | lo) >> (7 * (lane < 9 ? lane : 0))) & 0x7fu;
            v = row < n ? (lane < 9 ? field - 1u : (lane < (int)B2F_SENTINEL_WORD ? num : B2F_SENTINEL_BITS)) : B2F_SENTINEL_BITS;
        } else {
            if (row < n && lane < (int)B2F_SENTINEL_WORD) v = __ldg(rows + row * B2F_ROW_WORDS + lane);
        }
        if (lane_numeric && isnan(__uint_as_float(v))) v = impute_bits;
        w[r] = v;
        acc[r] = 0.0;
    }
    {
        const KGroup gd = p.g[g];
        const uint64_t nodes = reinterpret_cast<uint64_t>(p.chunks) + gd.chunk_off + lane8;
        const uint64_t leaves = nodes + (uint64_t)gd.n_slots * B2F_NODE_STRIDE;
        walk_group<R, false, 0>(nodes, leaves, (int)gd.depth, w, acc);
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const double s = warp_sum(acc[r]);
        if (lane == 0) part[g][r] = s;
    }
    __syncthreads();
    if (threadIdx.x < R) {
        const int r = threadIdx.x;
        double s = 0.0;
        for (int k = 0; k < p.n_groups; ++k) s += part[k][r]; /* group order: deterministic */
        const long long row = b * R + r;
        finalize_store<PACKED>(p, s, row < n ? row : -1, rows, proba, label, ostride);
    }
}
