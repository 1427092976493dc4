/*
 * forest_predict_tile.cuh -- K1b: the large-batch form of the fused scoring kernel (sm_90a).
 *
 * Same arithmetic as k_forest_predict (forest_predict.cuh) -- it replaces
 * `classifier.predict_proba(df[all_features])[:, 1]` (reference databricks/src/02-register-model.ipynb:335-337)
 * -- with the opposite geometry:
 *
 *   k_forest_predict       one WARP per row, lane = tree.  Lowest latency (one row spreads over 32 lanes),
 *                          used for small batches and for forests whose trees do not fit a shared-memory piece.
 *   k_forest_predict_tile  one THREAD per row, a warp owns a TILE of 32 consecutive rows and walks the trees one
 *                          U-group (8 trees) at a time, all lanes in the same trees.  Node loads are
 *                          near-broadcast (the 32 lanes sit in the same breadth-first level of the same tree, a
 *                          contiguous <= 256-byte run), there is no cross-lane reduction, no 32-tree quantisation,
 *                          the float64 sum runs in tree order (exactly sklearn's order), row tiles are read with
 *                          16-byte vector loads and results are written as coalesced 128-byte stores.
 *
 * Memory plan per CTA (persistent, 1 CTA/SM, W = 16..24 consumer warps + 1 producer warp):
 *   xs[W][24][32]   the warp's 32 encoded rows, TRANSPOSED (word-major) so a per-lane dynamic feature index is
 *                   one conflict-free LDS:  bank = lane.
 *   ring[n_slots]   forest PIECES (whole U-groups of trees, tree-major nodes + leaf payloads) streamed by the
 *                   producer warp with TMA bulk copies (cp.async.bulk + mbarrier complete_tx).  If the forest has
 *                   no more pieces than slots it is loaded once and stays resident; otherwise the ring is
 *                   recycled (full/empty mbarriers) and the forest streams through shared memory once per pass
 *                   of W tiles while accumulators stay in registers.
 *
 * Node format here ("tile layout", built by the library from the forest blob at model creation):
 *   T  as in forest_blob.h (t' | category code | leaf id)
 *   M  bits 16..31 first-child index inside the tree, bits 13..15 zero, bit 12 categorical flag,
 *      bits 7..11 row word index (i.e. bits 0..11 hold word*128, the byte offset of xs[word][0]).
 *      child byte offset = M >> 13 (one LEA.HI; bits 13..15 are zero so this is index*8 exactly);
 *      feature address   = xs_lane | (M & 0xF80) (one LOP3; each warp's xs block is 4 KB aligned).
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "forest_predict.cuh"

#define B2F_TILE_ROWS 32
#ifndef B2F_TILE_U
#define B2F_TILE_U 8                 /* trees walked concurrently by one thread (independent chains) */
#endif
#define B2F_TILE_WARPS_MIN 16        /* consumer warps per CTA: 16 when the forest streams, up to 24 when it is */
#define B2F_TILE_WARPS_MAX 24        /* resident and shared memory allows (more warps hide more smem latency) */
#define B2F_TILE_THREADS_MAX ((B2F_TILE_WARPS_MAX + 1) * 32)
#define B2F_TILE_XS_BYTES 4096 /* per warp: 24 words x 32 lanes x 4 B = 3072 B, padded so the block is 4 KB aligned */
#define B2F_TILE_MAX_SLOTS 8
#define B2F_TILE_META_CAT 0x1000u
#define B2F_TILE_CHILD_SHIFT 16u
#define B2F_TILE_FEAT_SHIFT 7u
#define B2F_TILE_MAX_TREE_NODES 65536u

/* one U-group descriptor inside a piece (offsets in bytes from the piece start) */
struct TUGroup {
    uint32_t node_off[B2F_TILE_U];
    uint32_t leaf_off[B2F_TILE_U];
    uint32_t depth; /* max depth of the U trees: walk iterations */
    uint32_t pad[3];
};
static_assert(sizeof(TUGroup) == 8 * B2F_TILE_U + 16 && sizeof(TUGroup) % 16 == 0, "TUGroup size");

struct TPiece {
    uint32_t off;   /* bytes from the tile-layout base (128-byte aligned) */
    uint32_t bytes; /* multiple of 128 */
    uint32_t n_ug;
    uint32_t pad;
};

struct TParams {
    const uint8_t *layout;  /* device: pieces back to back */
    const TPiece *pieces;   /* device: piece table */
    int32_t n_pieces;
    int32_t n_slots;
    uint32_t slot_bytes;
    int32_t agg_mode;
    int32_t n_cat;
    int32_t n_num;
    double init_raw;
    double denom;
    double threshold;
    float impute[24];
    const KParams *blob;    /* device copy of the blob parameters: rows inside the rounding band are re-decided on it */
};

__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}

__device__ __forceinline__ uint2 lds64(uint32_t a) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ double lds_f64(uint32_t a) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
    return v;
}

/* split decision, tile-layout flag position */
__device__ __forceinline__ bool take_second_tile(uint32_t x, uint32_t t, uint32_t m) {
    uint32_t c;
    asm("{\n\t"
        ".reg .pred pc, p1, p2;\n\t"
        ".reg .b32 cbit;\n\t"
        "and.b32 cbit, %3, 0x1000;\n\t"
        "setp.ne.u32 pc, cbit, 0;\n\t"
        "setp.geu.and.f32 p1, %1, %2, !pc;\n\t"
        "setp.eq.or.u32 p2, %4, %5, p1;\n\t"
        "selp.u32 %0, 1, 0, p2;\n\t"
        "}"
        : "=r"(c)
        : "f"(__uint_as_float(x)), "f"(__uint_as_float(t)), "r"(m), "r"(x), "r"(t));
    return c != 0;
}

/* walk one U-group for this lane's row; values are added to acc in tree order */
template <int D>
__device__ __forceinline__ void tile_walk_ugroup(uint32_t piece_addr, uint32_t ug_addr, uint32_t xs_lane, int depth, double &acc) {
    uint32_t base[B2F_TILE_U], lbase[B2F_TILE_U];
#pragma unroll
    for (int u = 0; u < B2F_TILE_U; u += 4) {
        const uint4 no = *reinterpret_cast<const uint4 *>(__cvta_shared_to_generic(ug_addr + 4 * u));
        const uint4 lo = *reinterpret_cast<const uint4 *>(__cvta_shared_to_generic(ug_addr + 4 * B2F_TILE_U + 4 * u));
        base[u] = piece_addr + no.x, base[u + 1] = piece_addr + no.y, base[u + 2] = piece_addr + no.z, base[u + 3] = piece_addr + no.w;
        lbase[u] = piece_addr + lo.x, lbase[u + 1] = piece_addr + lo.y, lbase[u + 2] = piece_addr + lo.z, lbase[u + 3] = piece_addr + lo.w;
    }
    uint32_t at[B2F_TILE_U];
#pragma unroll
    for (int u = 0; u < B2F_TILE_U; ++u) at[u] = base[u];

    auto level = [&]() {
#pragma unroll
        for (int u = 0; u < B2F_TILE_U; ++u) {
            const uint2 tm = lds64(at[u]);
            const uint32_t x = lds32(xs_lane | (tm.y & 0xF80u)); /* xs[word][lane] */
            const uint32_t c = take_second_tile(x, tm.x, tm.y) ? base[u] + 8u : base[u];
            at[u] = (tm.y >> 13) + c; /* child index * 8 */
        }
    };
    if constexpr (D > 0) {
#pragma unroll
        for (int d = 0; d < D; ++d) level();
    } else {
#pragma unroll 2
        for (int d = 0; d < depth; ++d) level();
    }
#pragma unroll
    for (int u = 0; u < B2F_TILE_U; ++u) {
        const uint32_t leaf_id = lds32(at[u]);
        acc += lds_f64(lbase[u] + leaf_id * 8u);
    }
}

template <bool PACKED, typename OutT>
__global__ void __launch_bounds__(B2F_TILE_THREADS_MAX, 1)
    k_forest_predict_tile(const __grid_constant__ TParams p, const uint32_t *__restrict__ rows, long long n,
                          OutT *__restrict__ proba, int32_t *__restrict__ label, int ostride) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t full_bar[B2F_TILE_MAX_SLOTS];
    __shared__ __align__(8) uint64_t empty_bar[B2F_TILE_MAX_SLOTS];

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int n_pieces = p.n_pieces, n_slots = p.n_slots;
    const int n_cwarps = (int)(blockDim.x >> 5) - 1; /* consumer warps; the last warp is the producer */
    const bool resident = n_pieces <= n_slots;

    /* xs blocks must be 4 KB aligned in the shared window (the feature address is formed with OR) */
    const uint32_t pad = (4096u - (smem_addr(smem) & 4095u)) & 4095u;
    uint8_t *xs_all = smem + pad;                                  /* [W] x 4 KB: [24][32] words each */
    uint8_t *ring = xs_all + n_cwarps * B2F_TILE_XS_BYTES;         /* [n_slots][slot_bytes] */

    if (threadIdx.x == 0) {
        for (int s = 0; s < n_slots; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], n_cwarps);
        }
        fence_mbar_init();
        fence_proxy_async();
    }
    __syncthreads();

    const long long n_tiles = (n + B2F_TILE_ROWS - 1) / B2F_TILE_ROWS;
    const long long tiles_per_pass = (long long)gridDim.x * n_cwarps;
    /* every warp of every CTA runs the same number of passes so the ring hand-shake stays in step;
     * tiles are numbered CTA-minor so a small batch spreads over all SMs */
    const long long n_pass = (n_tiles + tiles_per_pass - 1) / tiles_per_pass;

    if (warp == n_cwarps) {
        /* ===== producer warp: one lane streams forest pieces into the ring with TMA bulk copies ===== */
        if (lane == 0) {
            const long long fills = resident ? (n_pass > 0 ? n_pieces : 0) : n_pass * n_pieces;
            for (long long f = 0; f < fills; ++f) {
                const int piece = (int)(f % n_pieces);
                const int slot = (int)(f % n_slots);
                const long long j = f / n_slots; /* fill number of this slot */
                if (j > 0) mbar_wait(&empty_bar[slot], (uint32_t)((j - 1) & 1));
                const TPiece pc = p.pieces[piece];
                mbar_arrive_expect_tx(&full_bar[slot], pc.bytes);
                uint8_t *dst = ring + (size_t)slot * p.slot_bytes;
                for (uint32_t o = 0; o < pc.bytes; o += B2F_BULK_PIECE) {
                    const uint32_t part = min(B2F_BULK_PIECE, pc.bytes - o);
                    tma_bulk_g2s(dst + o, p.layout + pc.off + o, part, &full_bar[slot]);
                }
            }
        }
        return;
    }

    /* ===== consumer warps ===== */
    const uint32_t xs_warp = smem_addr(xs_all + warp * B2F_TILE_XS_BYTES);
    const uint32_t xs_lane = xs_warp + lane * 4u;
    const uint32_t ring_addr = smem_addr(ring);

    for (long long pass = 0; pass < n_pass; ++pass) {
        const long long tile = (pass * n_cwarps + warp) * gridDim.x + blockIdx.x;
        const long long row = tile * B2F_TILE_ROWS + lane;
        const bool live = tile < n_tiles && row < n;

        /* ---- stage this lane's row: six 16-byte vector loads, impute, transpose into xs[word][lane] ---- */
        __syncwarp();
        {
            uint32_t w[B2F_ROW_WORDS];
#pragma unroll
            for (int k = 0; k < B2F_ROW_WORDS; ++k) w[k] = B2F_SENTINEL_BITS;
            if (live) {
                if constexpr (PACKED) {
                    /* 64-byte row: words 0..1 = nine 7-bit (code + 1) fields, words 2..15 = 14 numerics */
                    const uint4 *src = reinterpret_cast<const uint4 *>(rows + row * B2F_PACKED_ROW_WORDS);
                    uint32_t q[B2F_PACKED_ROW_WORDS];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const uint4 v = __ldg(src + k);
                        q[4 * k + 0] = v.x, q[4 * k + 1] = v.y, q[4 * k + 2] = v.z, q[4 * k + 3] = v.w;
                    }
                    const unsigned long long codes = (((unsigned long long)q[1]) << 32) | q[0];
#pragma unroll
                    for (int k = 0; k < 9; ++k) w[k] = ((uint32_t)(codes >> (7 * k)) & 0x7fu) - 1u;
#pragma unroll
                    for (int k = 0; k < 14; ++k) w[9 + k] = q[2 + k];
                } else {
                    const uint4 *src = reinterpret_cast<const uint4 *>(rows + row * B2F_ROW_WORDS);
#pragma unroll
                    for (int k = 0; k < 6; ++k) {
                        const uint4 v = __ldg(src + k);
                        w[4 * k + 0] = v.x, w[4 * k + 1] = v.y, w[4 * k + 2] = v.z, w[4 * k + 3] = v.w;
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < B2F_ROW_WORDS; ++k) {
                uint32_t v = w[k];
                if (k >= p.n_cat && k < p.n_cat + p.n_num && isnan(__uint_as_float(v))) v = __float_as_uint(p.impute[k]);
                if (k >= (int)B2F_SENTINEL_WORD) v = B2F_SENTINEL_BITS;
                asm volatile("st.shared.u32 [%0], %1;" ::"r"(xs_lane + k * 128u), "r"(v) : "memory");
            }
        }
        __syncwarp();

        /* GBDT: start from the init estimator's raw value and add trees in order -- sklearn's own order */
        double acc = p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? p.init_raw : 0.0;
        const bool warp_live = tile < n_tiles; /* warp-uniform: a warp without a tile only keeps the ring protocol */
        for (int piece = 0; piece < n_pieces; ++piece) {
            const long long f = resident ? piece : pass * n_pieces + piece;
            const int slot = (int)(f % n_slots);
            if (!resident || pass == 0) mbar_wait(&full_bar[slot], (uint32_t)((f / n_slots) & 1));
            if (warp_live) {
                const uint32_t piece_addr = ring_addr + slot * p.slot_bytes;
                const int n_ug = (int)p.pieces[piece].n_ug;
                for (int g = 0; g < n_ug; ++g) {
                    const uint32_t ug_addr = piece_addr + g * (uint32_t)sizeof(TUGroup);
                    const int depth = (int)lds32(ug_addr + 8 * B2F_TILE_U);
                    switch (depth) {
                        case 1: tile_walk_ugroup<1>(piece_addr, ug_addr, xs_lane, 1, acc); break;
                        case 2: tile_walk_ugroup<2>(piece_addr, ug_addr, xs_lane, 2, acc); break;
                        case 3: tile_walk_ugroup<3>(piece_addr, ug_addr, xs_lane, 3, acc); break;
                        case 4: tile_walk_ugroup<4>(piece_addr, ug_addr, xs_lane, 4, acc); break;
                        case 5: tile_walk_ugroup<5>(piece_addr, ug_addr, xs_lane, 5, acc); break;
                        case 6: tile_walk_ugroup<6>(piece_addr, ug_addr, xs_lane, 6, acc); break;
                        case 7: tile_walk_ugroup<7>(piece_addr, ug_addr, xs_lane, 7, acc); break;
                        case 8: tile_walk_ugroup<8>(piece_addr, ug_addr, xs_lane, 8, acc); break;
                        default: tile_walk_ugroup<0>(piece_addr, ug_addr, xs_lane, depth, acc); break;
                    }
                }
            }
            if (!resident) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[slot]);
            }
        }

        /* ---- aggregate -> probability + label, one row per lane, coalesced stores ---- */
        if (live) {
            double p1;
            int lab;
            /* the GBDT init value is already in acc (added first, as sklearn does) */
            aggregate(p.agg_mode, p.agg_mode == B2F_AGG_GBDT_LOGISTIC ? 0.0 : p.init_raw, p.denom, p.threshold, acc, p1, lab);
            if (label && decide_exactly(p.agg_mode, acc, p.denom, p.threshold)) lab = decide_row_blob<PACKED>(*p.blob, rows, row);
            if (proba) proba[row * ostride_p(ostride)] = (OutT)p1;
            if (label) label[row * ostride_l(ostride)] = lab;
        }
    }
}
