/*
 * forest_rank.h -- host side of the "ranked" row format and of the rank-quantised forest layout (no GPU involved).
 *
 * What the reference's classifier compares is `x <= threshold` with x a float32 feature value
 * (sklearn `_tree.pyx` `_apply_dense`, reached from `classifier.predict_proba`, reference
 * databricks/src/02-register-model.ipynb:335-337).  A forest only ever compares a feature with the finitely many
 * thresholds its nodes hold, so the value can be replaced, EXACTLY, by its rank among them:
 *
 *     t'_0 < t'_1 < ... < t'_{m-1}   the distinct float32 split values t' of numeric feature k over the whole forest
 *                                    (t' = nextup(floor32(threshold)), forest_blob.h:  x <= thr  <=>  x < t')
 *     rank_k(x) = #{ j : t'_j <= x }                                    (0 .. m)
 *     x >= t'_j  <=>  rank_k(x) >= j + 1
 *
 * so a numeric node becomes the INTEGER test  rank >= j + 1, a node shrinks from 8 to 4 bytes, and a row from 14 float32
 * to 14 uint16.  Missing values: the row carries the rank of the imputation value (the training median; or m, "beyond
 * every threshold", where the blob's imputation value is NaN as in an isolation forest).  Categorical features keep their
 * dictionary code (+1, 0 = unknown / missing), bit-packed.
 *
 * B2F_ROWS_RANKED row (include/b2f.h), little-endian:
 *     bytes 0 .. cat_bytes-1        the categorical fields, LSB first, field j at bit cat_shift[j], cat_bits[j] wide
 *                                   (cat_bytes = 4 when they fit 32 bits, else 8)
 *     then n_num x uint16           rank of numeric feature k
 *     zero padding to a multiple of 8 bytes            (credit-default schema: 4 + 28 = 32 bytes per row)
 *
 * Rank layout of the forest (what k_forest_predict_rank walks, forest_predict_rank.cuh): every tree is padded to a COMPLETE
 * binary tree of the forest's depth D in breadth-first order, so the child of node i is 2i+1 (+1) and no child pointer
 * is stored; a tree is 2^D 4-byte node words (the last one unused) followed by 2^D float64 leaf payloads.
 * EVERY test is a rank test "value[f] >= t" over 16-bit values: pseudo-feature f is either numeric feature k (f = k, value
 * = its rank) or one (categorical feature j, category c) pair that some node of the forest tests (f = even(n_num) + pair
 * index; value = 1 if the row's code is c, else 0; t = 1) -- the one-hot column sklearn's tree splits on (x_j <= 0.5), restated.
 *     node word   bits 16..31  t     (second child iff value[f] >= t)
 *                 bits 0..15   byte offset of value[f] inside the kernel's per-tile value block: (f >> 1) * 128 + (f & 1) * 2
 *                              (two 16-bit values per 32-bit word of a lane's column, so a lane's fetch always hits its own bank)
 *     0x00000000 = "always second child", 0xFFFF0000 = "never" (values stay below 65535).
 *     a leaf above depth D is replicated downwards (its subtree's nodes are 0, all its leaf slots hold its payload).
 */
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <thread>
#include <vector>

#include "../../include/b2f.h"
#include "forest_blob.h"

/* host SIMD (csrc/host_simd.cpp, compiled by g++): 16-ary rank tables, one 64-byte compare per level */
extern "C" {
struct b2f_ranktab {
    int32_t levels;
    int32_t count;
    int32_t fan[4]; /* fan-out per level (multiples of 16); capacity prod(fan) > count */
    const float *lvl[4];
};
int b2f_simd_level(void);
void b2f_simd_rank_column(const b2f_ranktab *t, const float *x, int64_t n, int64_t x_stride, uint16_t *out, int64_t out_stride, uint16_t nan_rank);
int b2f_simd_cvt_column(const double *src, int64_t stride, int64_t n, float *dst); /* float64 -> float32; 1 = an inf / overflow was seen */
int64_t b2f_simd_hash_codes(const void *offsets, int offsets_are_64, const uint8_t *data, int64_t data_bytes, int64_t nb, uint64_t m1, uint64_t m2,
                            uint64_t m3, int shift, const void *slots, int32_t *codes); /* rows done from the start; -2 = hit that needs the full compare */
void b2f_simd_pack_rows64(const int32_t *codes, const float *cols, int64_t ld, int n_cat, int n_num, int64_t nb, uint32_t *out);
}

#define B2F_RANK_BLOCK 256 /* rows ranked per call of the column kernel (the transposed block stays in L1) */
#define B2F_RANK_MAX_DEPTH 8
#define B2F_RANK_MAX_FEATS 128 /* pseudo-features per row: numerics + tested (categorical feature, category) pairs */
#define B2F_RANK_MAX_THRESHOLDS 65534

struct b2f_ranker {
    int n_cat = 0, n_num = 0, n_trees = 0, depth = 0, agg_mode = 0;
    bool ok = false;          /* the forest has a rank layout (depth <= 8, thresholds and categories fit 16 bits) */
    char why[160] = "";       /* when !ok */
    int cat_bytes = 0, row_bytes = 0;
    int cat_shift[16] = {0}, cat_bits[16] = {0}, vocab[16] = {0};
    float impute[24] = {0};
    std::vector<std::vector<float>> thr; /* per numeric feature: sorted distinct t' */
    std::vector<uint16_t> nan_rank;      /* per numeric feature: rank a missing value gets */
    std::vector<std::vector<float>> tab_store; /* per numeric feature: the 16-ary rank table, levels back to back */
    std::vector<b2f_ranktab> tabs;             /* views into tab_store (re-pointed by ranker_fix_tabs after a copy) */
    std::vector<uint32_t> pairs;         /* tested (categorical feature j, category code c) pairs: j << 16 | c, ascending;
                                            pair i is pseudo-feature n_num + i */
    uint32_t tree_stride = 0;            /* bytes per tree in the layout: 2^D * 12 */
    std::vector<uint8_t> layout;         /* n_trees_padded * tree_stride */
    int n_trees_padded = 0;              /* multiple of 8 (stub trees: all-zero nodes and payloads) */
};

/* pseudo-feature index of the first one-hot value: numerics occupy 0 .. n_num-1, one-hot values start at the next EVEN index so
 * that no 32-bit word of the kernel's value block mixes a rank with a one-hot value */
static inline int rank_onehot_base(int n_num) { return (n_num + 1) & ~1; }

namespace rankdetail {

struct Tree {
    std::vector<uint32_t> T, M; /* blob words per slot (this tree's lane) */
    std::vector<double> leaves;
};

static inline int bits_for(uint32_t max_value) { /* bits needed for 0..max_value */
    int b = 1;
    while ((max_value >> b) != 0) ++b;
    return b;
}

/* slot-indexed copy of one tree out of the 32-interleaved blob group */
static void read_tree(const uint8_t *blob, const b2f_blob_header &h, const b2f_blob_group &gr, uint32_t lane, Tree &t) {
    const uint32_t *N = reinterpret_cast<const uint32_t *>(blob + h.chunks_off + gr.chunk_off);
    const double *LV = reinterpret_cast<const double *>(blob + h.chunks_off + gr.chunk_off + (size_t)gr.n_slots * 256);
    t.T.resize(gr.n_slots);
    t.M.resize(gr.n_slots);
    for (uint32_t s = 0; s < gr.n_slots; ++s) {
        t.T[s] = N[(s * 32 + lane) * 2];
        t.M[s] = N[(s * 32 + lane) * 2 + 1];
    }
    t.leaves.resize(gr.n_leaf_slots);
    for (uint32_t i = 0; i < gr.n_leaf_slots; ++i) t.leaves[i] = LV[i * 32 + lane];
}

static inline bool is_leaf(const Tree &t, uint32_t s) { return (t.M[s] & B2F_META_SLOT_MASK) == s; }

static int tree_depth(const Tree &t, uint32_t s, int d, int limit) {
    if (is_leaf(t, s) || d > limit) return d;
    const uint32_t c = t.M[s] & B2F_META_SLOT_MASK;
    return std::max(tree_depth(t, c, d + 1, limit), tree_depth(t, c + 1, d + 1, limit));
}

}  // namespace rankdetail

/* The sorted distinct split values t' of each numeric feature over the whole forest, at any depth: thr[k] for row word
 * n_cat + k.  -0.0 and +0.0 collapse (float ==), as the comparison sees them.  Every lane of a group below its tree count is
 * read, node slot by node slot.  Returns NULL, or why the forest has no such table (thr is then unspecified). */
static const char *forest_split_values(const uint8_t *blob, const b2f_blob_header &h, std::vector<std::vector<float>> &thr) {
    const int n_cat = (int)h.n_cat, n_num = (int)h.n_num;
    thr.assign(n_num, {});
    const b2f_blob_group *gt = reinterpret_cast<const b2f_blob_group *>(blob + h.groups_off);
    for (uint32_t t = 0; t < h.n_trees; ++t) {
        const b2f_blob_group &gr = gt[t / 32];
        const uint32_t *N = reinterpret_cast<const uint32_t *>(blob + h.chunks_off + gr.chunk_off);
        for (uint32_t s = 0; s < gr.n_slots; ++s) {
            const uint32_t T = N[(s * 32 + t % 32) * 2], M = N[(s * 32 + t % 32) * 2 + 1];
            if ((M & B2F_META_SLOT_MASK) == s || (M & B2F_META_CAT)) continue; /* leaf, categorical test */
            const uint32_t w = M >> B2F_META_FEAT_SHIFT;
            if (w == B2F_SENTINEL_WORD) continue; /* "always second child" node */
            if ((int)w < n_cat || (int)w >= n_cat + n_num) return "numeric test on a non-numeric row word";
            float f;
            memcpy(&f, &T, 4);
            if (f != f) return "NaN split value";
            thr[w - n_cat].push_back(f);
        }
    }
    for (auto &v : thr) {
        std::sort(v.begin(), v.end());
        v.erase(std::unique(v.begin(), v.end()), v.end());
    }
    return nullptr;
}

/* rank tables (host_simd.cpp): lvl[j][i] = largest value of the i-th chunk at level j; +inf padding.  Upper levels fan out
 * 16 ways, the last one 16..64 ways, chosen as the shallowest / narrowest shape whose capacity exceeds the value count. */
static void rank_tab_shape(size_t m, int *levels, int32_t fan[4]) {
    int L = 1;
    size_t upper = 1; /* 16^(L-1) */
    while (upper * 64 <= m) upper *= 16, ++L;
    int F = 16;
    while (upper * (size_t)F <= m) F += 16;
    for (int j = 0; j < 4; ++j) fan[j] = j < L - 1 ? 16 : (j == L - 1 ? F : 0);
    *levels = L;
}
static void ranker_fix_tabs(b2f_ranker *r) {
    r->tabs.assign(r->thr.size(), b2f_ranktab{});
    for (size_t k = 0; k < r->thr.size(); ++k) {
        b2f_ranktab &t = r->tabs[k];
        rank_tab_shape(r->thr[k].size(), &t.levels, t.fan);
        t.count = (int32_t)r->thr[k].size();
        size_t off = 0, sz = 1;
        for (int j = 0; j < t.levels; ++j) {
            sz *= (size_t)t.fan[j];
            t.lvl[j] = r->tab_store[k].data() + off;
            off += sz;
        }
    }
}
static void ranker_build_tabs(b2f_ranker *r) {
    r->tab_store.assign(r->thr.size(), {});
    for (size_t k = 0; k < r->thr.size(); ++k) {
        const std::vector<float> &v = r->thr[k];
        int L;
        int32_t fan[4];
        rank_tab_shape(v.size(), &L, fan);
        size_t cap = 1;
        for (int j = 0; j < L; ++j) cap *= (size_t)fan[j]; /* > m: the last chunk always ends in +inf */
        std::vector<float> full(cap, INFINITY);
        std::copy(v.begin(), v.end(), full.begin());
        std::vector<float> &st = r->tab_store[k];
        size_t sz = 1;
        for (int j = 0; j < L; ++j) {
            sz *= (size_t)fan[j];
            const size_t step = cap / sz;
            for (size_t i = 0; i < sz; ++i) st.push_back(full[(i + 1) * step - 1]);
        }
    }
    ranker_fix_tabs(r);
}

/* Fill r from a validated blob.  Returns false (r->ok = false, r->why set) when the forest has no rank layout; the
 * row-format fields are still valid whenever the schema itself fits. */
static bool ranker_build(b2f_ranker *r, const uint8_t *blob, const b2f_blob_header &h) {
    using namespace rankdetail;
    r->n_cat = (int)h.n_cat;
    r->n_num = (int)h.n_num;
    r->n_trees = (int)h.n_trees;
    r->agg_mode = (int)h.agg_mode;
    memcpy(r->impute, h.impute, sizeof(r->impute));
    r->ok = false;
    auto fail = [&](const char *msg) {
        snprintf(r->why, sizeof(r->why), "%s", msg);
        return false;
    };
    /* categorical block */
    int bit = 0;
    if (r->n_cat > 16) return fail("more than 16 categorical features");
    for (int j = 0; j < r->n_cat; ++j) {
        const int v = h.vocab[j];
        if (v < 0 || v > 65533) return fail("a categorical vocabulary does not fit 16 bits");
        r->cat_bits[j] = bits_for((uint32_t)v); /* values 0 .. v (code + 1) */
        r->vocab[j] = v;
        r->cat_shift[j] = bit;
        bit += r->cat_bits[j];
    }
    if (bit > 64) return fail("categorical fields need more than 64 bits");
    r->cat_bytes = bit <= 32 ? 4 : 8;
    r->row_bytes = (r->cat_bytes + 2 * r->n_num + 7) / 8 * 8;

    /* trees */
    const b2f_blob_group *gt = reinterpret_cast<const b2f_blob_group *>(blob + h.groups_off);
    std::vector<Tree> trees(h.n_trees);
    int depth = 0;
    for (uint32_t t = 0; t < h.n_trees; ++t) {
        read_tree(blob, h, gt[t / 32], t % 32, trees[t]);
        depth = std::max(depth, tree_depth(trees[t], 0, 0, B2F_RANK_MAX_DEPTH + 1));
    }
    if (depth > B2F_RANK_MAX_DEPTH) return fail("trees deeper than 8 levels");
    if (depth < 1) depth = 1;
    r->depth = depth;

    /* tested (categorical feature, category) pairs; distinct split values per numeric feature */
    r->pairs.clear();
    for (const Tree &t : trees)
        for (uint32_t s = 0; s < t.T.size(); ++s) {
            if (is_leaf(t, s) || !(t.M[s] & B2F_META_CAT)) continue;
            const uint32_t w = t.M[s] >> B2F_META_FEAT_SHIFT;
            if (t.T[s] == 0x7FFFFFFFu) continue; /* "never equal" */
            if ((int)w >= r->n_cat || t.T[s] > 65533u) return fail("categorical test outside the schema");
            r->pairs.push_back((w << 16) | t.T[s]);
        }
    if (const char *why = forest_split_values(blob, h, r->thr)) return fail(why);
    std::sort(r->pairs.begin(), r->pairs.end());
    r->pairs.erase(std::unique(r->pairs.begin(), r->pairs.end()), r->pairs.end());
    if (rank_onehot_base(r->n_num) + (int)r->pairs.size() > B2F_RANK_MAX_FEATS) return fail("more than 128 numeric features + tested categories");
    for (uint32_t pr : r->pairs)
        if ((pr & 0xFFFFu) >= 64u) return fail("a tested category code does not fit the kernel's 64-bit per-feature mask");
    r->nan_rank.assign(r->n_num, 0);
    for (int k = 0; k < r->n_num; ++k) {
        const auto &v = r->thr[k];
        if (v.size() > B2F_RANK_MAX_THRESHOLDS) return fail("more than 65534 distinct split values on one feature");
        const float imp = r->impute[r->n_cat + k];
        r->nan_rank[k] = (imp != imp) ? (uint16_t)v.size() : (uint16_t)(std::upper_bound(v.begin(), v.end(), imp) - v.begin());
    }

    ranker_build_tabs(r);

    /* complete-tree layout */
    const uint32_t n_slots = 1u << depth;
    r->tree_stride = n_slots * 12u;
    r->n_trees_padded = (r->n_trees + 7) / 8 * 8;
    r->layout.assign((size_t)r->n_trees_padded * r->tree_stride, 0);
    bool bad = false;
    for (uint32_t ti = 0; ti < h.n_trees; ++ti) {
        const Tree &t = trees[ti];
        uint32_t *nodes = reinterpret_cast<uint32_t *>(r->layout.data() + (size_t)ti * r->tree_stride);
        double *leaves = reinterpret_cast<double *>(r->layout.data() + (size_t)ti * r->tree_stride + n_slots * 4u);
        /* (slot, level, position inside the level) */
        struct Item {
            uint32_t s;
            int d;
            uint32_t pos;
        };
        std::vector<Item> stack{{0u, 0, 0u}};
        while (!stack.empty()) {
            const Item it = stack.back();
            stack.pop_back();
            if (is_leaf(t, it.s)) {
                const uint32_t id = t.T[it.s];
                const double v = id < t.leaves.size() ? t.leaves[id] : 0.0;
                const uint32_t span = 1u << (depth - it.d);
                for (uint32_t q = 0; q < span; ++q) leaves[it.pos * span + q] = v; /* the subtree's nodes stay 0 */
                continue;
            }
            if (it.d >= depth) {
                bad = true;
                continue;
            }
            const uint32_t m = t.M[it.s], w = m >> B2F_META_FEAT_SHIFT, first = m & B2F_META_SLOT_MASK;
            uint32_t word;
            auto feat_off = [](uint32_t f) { return (f >> 1) * 128u + (f & 1u) * 2u; };
            if (m & B2F_META_CAT) {
                if (t.T[it.s] == 0x7FFFFFFFu) { /* "never equal": always first child */
                    word = 0xFFFF0000u;
                } else {
                    const uint32_t key = (w << 16) | t.T[it.s];
                    const uint32_t pi = (uint32_t)(std::lower_bound(r->pairs.begin(), r->pairs.end(), key) - r->pairs.begin());
                    if (pi >= r->pairs.size() || r->pairs[pi] != key) bad = true;
                    word = (1u << 16) | feat_off((uint32_t)rank_onehot_base(r->n_num) + pi); /* one-hot value >= 1 */
                }
            } else if (w == B2F_SENTINEL_WORD) {
                word = 0u; /* always second child */
            } else {
                float f;
                memcpy(&f, &t.T[it.s], 4);
                const auto &v = r->thr[w - r->n_cat];
                const uint32_t j = (uint32_t)(std::lower_bound(v.begin(), v.end(), f) - v.begin());
                word = ((j + 1u) << 16) | feat_off(w - (uint32_t)r->n_cat);
            }
            nodes[(1u << it.d) - 1u + it.pos] = word;
            stack.push_back({first, it.d + 1, it.pos * 2u});
            stack.push_back({first + 1u, it.d + 1, it.pos * 2u + 1u});
        }
    }
    if (bad) return fail("forest blob does not map onto the rank layout");
    r->ok = true;
    r->why[0] = 0;
    return true;
}

static inline uint16_t rank_value(const b2f_ranker *r, int k, float f) {
    uint16_t out;
    b2f_simd_rank_column(&r->tabs[k], &f, 1, 1, &out, 1, r->nan_rank[k]);
    return out;
}

/* the categorical block + zero padding of one ranked row (the uint16 ranks are written by rank_block) */
static inline void rank_write_cats(const b2f_ranker *r, const int32_t *codes, uint8_t *out) {
    uint64_t cw = 0;
    for (int j = 0; j < r->n_cat; ++j) cw |= (uint64_t)(uint32_t)(codes[j] + 1) << r->cat_shift[j];
    memcpy(out, &cw, (size_t)r->cat_bytes);
    for (int b = r->cat_bytes + 2 * r->n_num; b < r->row_bytes; ++b) out[b] = 0;
}

/* ranks of a block of rows: cols = float32 numerics column-major, cols[k * B2F_RANK_BLOCK + i]; out = first row of the block */
static inline void rank_block(const b2f_ranker *r, const float *cols, int64_t nb, uint8_t *out) {
    uint16_t *q = reinterpret_cast<uint16_t *>(out + r->cat_bytes);
    for (int k = 0; k < r->n_num; ++k)
        b2f_simd_rank_column(&r->tabs[k], cols + (size_t)k * B2F_RANK_BLOCK, nb, 1, q + k, r->row_bytes / 2, r->nan_rank[k]);
}

static void rank_rows_range(const b2f_ranker *r, const uint8_t *rows, int64_t lo, int64_t hi, int row_format, uint8_t *out) {
    int32_t codes[16];
    float cols[24 * B2F_RANK_BLOCK];
    for (int64_t b0 = lo; b0 < hi; b0 += B2F_RANK_BLOCK) {
        const int64_t nb = std::min<int64_t>(B2F_RANK_BLOCK, hi - b0);
        for (int64_t i = 0; i < nb; ++i) {
            const uint32_t *nums;
            if (row_format == B2F_ROWS_PACKED64) {
                const uint32_t *w = reinterpret_cast<const uint32_t *>(rows + (size_t)(b0 + i) * B2F_PACKED_ROW_BYTES);
                const uint64_t c = ((uint64_t)w[1] << 32) | w[0];
                for (int j = 0; j < r->n_cat; ++j) {
                    const int32_t cj = (int32_t)((c >> (7 * j)) & 0x7f) - 1;
                    codes[j] = cj >= r->vocab[j] ? -1 : cj;
                }
                nums = w + 2;
            } else {
                const uint32_t *w = reinterpret_cast<const uint32_t *>(rows + (size_t)(b0 + i) * B2F_ROW_BYTES);
                for (int j = 0; j < r->n_cat; ++j) {
                    const int32_t c = (int32_t)w[j];
                    codes[j] = (c < 0 || c >= r->vocab[j]) ? -1 : c; /* codes outside the vocabulary match nothing */
                }
                nums = w + r->n_cat;
            }
            for (int k = 0; k < r->n_num; ++k) memcpy(&cols[(size_t)k * B2F_RANK_BLOCK + i], &nums[k], 4);
            rank_write_cats(r, codes, out + (size_t)(b0 + i) * r->row_bytes);
        }
        rank_block(r, cols, nb, out + (size_t)b0 * r->row_bytes);
    }
}
