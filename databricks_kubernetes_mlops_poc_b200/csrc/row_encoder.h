/*
 * row_encoder.h -- native host-side row encoder (no GPU involved; compiled into libb200forest.so).
 *
 * The host half of the "fused preprocess": what the reference does with pandas + sklearn's
 * SimpleImputer(constant) / OneHotEncoder lookup before any arithmetic
 * (reference app/main.py:54 `pd.DataFrame(data)`, databricks/src/01-train-model.ipynb:197-221).
 * Input is columnar, exactly as pandas / Arrow hold it:
 *   - categorical columns as Arrow string arrays (validity bitmap, int32 or int64 offsets, UTF-8 bytes),
 *   - numeric columns as float64 arrays (pointer + element stride).
 * Output is encoded rows in either layout of include/b2f.h, written straight into the caller's (pinned)
 * staging buffer by a few host threads.  Semantics are those of databricks_kubernetes_mlops_poc_b200/encode.py
 * (which remains the portable implementation and the one used for tiny requests):
 *   string in the feature's vocabulary -> its index; unknown string -> -1; null -> the feature's "missing" code
 *   (the imputer's constant, if it was a training category) else -1;  float64 -> float32 round-to-nearest, NaN kept
 *   (the kernel imputes), +-inf or float32 overflow -> error (sklearn raises ValueError there).
 */
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <string>
#include <thread>
#include <vector>

#include "../../include/b2f.h"
#include "forest_rank.h"

struct EncEntry {
    uint64_t prefix; /* first min(len, 8) bytes, zero padded */
    uint64_t suffix; /* last 8 bytes (len >= 8), else the prefix again */
    uint32_t len;    /* 0xFFFFFFFF = empty slot */
    int32_t code;
};

/* Per categorical feature a PERFECT hash of its vocabulary: slot = ((prefix * m1) ^ (suffix * m2) ^ (len * m3)) >> shift,
 * multipliers searched at construction until no two vocabulary strings share a slot.  A lookup is two unaligned 8-byte loads,
 * three multiplies, ONE table probe and three integer compares -- no scan over the vocabulary, no data-dependent branch
 * except hit / miss (a linear (length, prefix) scan mispredicts on nearly every row). */
struct EncHash {
    uint64_t m1 = 0, m2 = 0, m3 = 0;
    int shift = 58;
    std::vector<EncEntry> slots;
};

struct b2f_encoder {
    int n_cat = 0, n_num = 0;
    std::vector<std::vector<std::string>> vocab; /* per categorical feature, in code order */
    std::vector<EncHash> hash;                   /* per categorical feature */
    std::vector<int32_t> null_code;              /* per categorical feature: code of a null entry, or -1 */
    bool packed_ok = false;
    b2f_ranker *ranker = nullptr; /* copy of the forest's split-value tables (b2f_encoder_attach_ranker): B2F_ROWS_RANKED output */
};

static inline uint64_t enc_prefix(const uint8_t *s, int64_t len) {
    uint64_t p = 0;
    memcpy(&p, s, (size_t)(len < 8 ? len : 8));
    return p;
}
static inline uint64_t enc_suffix(const uint8_t *s, int64_t len, uint64_t prefix) {
    if (len < 8) return prefix;
    uint64_t q;
    memcpy(&q, s + len - 8, 8);
    return q;
}
static inline size_t enc_slot(const EncHash &h, uint64_t p, uint64_t q, uint64_t len) { return (size_t)(((p * h.m1) ^ (q * h.m2) ^ (len * h.m3)) >> h.shift); }

static bool enc_build_hash(const std::vector<std::string> &vocab, EncHash &h) {
    int bits = 4;
    while ((size_t)1 << bits < 2 * vocab.size() + 2) ++bits;
    uint64_t seed = 0x9E3779B97F4A7C15ull;
    auto next = [&seed] { /* splitmix64 */
        uint64_t z = (seed += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    };
    for (; bits <= 16; ++bits) {
        for (int attempt = 0; attempt < 2000; ++attempt) {
            h.m1 = next() | 1ull, h.m2 = next() | 1ull, h.m3 = next() | 1ull;
            h.shift = 64 - bits;
            h.slots.assign((size_t)1 << bits, EncEntry{0, 0, 0xFFFFFFFFu, -1});
            bool ok = true;
            for (size_t k = 0; k < vocab.size() && ok; ++k) {
                const uint8_t *w = reinterpret_cast<const uint8_t *>(vocab[k].data());
                const int64_t len = (int64_t)vocab[k].size();
                const uint64_t p = enc_prefix(w, len), q = enc_suffix(w, len, p);
                EncEntry &e = h.slots[enc_slot(h, p, q, (uint64_t)len)];
                if (e.len != 0xFFFFFFFFu) ok = false; /* duplicate vocabulary strings cannot happen (OneHotEncoder categories are unique) */
                e = EncEntry{p, q, (uint32_t)len, (int32_t)k};
            }
            if (ok) return true;
        }
    }
    return false;
}

static inline int32_t enc_lookup(const b2f_encoder *e, int j, const uint8_t *s, int64_t len, bool can_read8) {
    /* prefix: one unaligned 8-byte load masked to the string's length whenever 8 bytes are readable (always, except at the
     * very end of the buffer) */
    uint64_t p;
    if (can_read8) {
        memcpy(&p, s, 8);
        if (len < 8) p &= (len == 0 ? 0ull : (~0ull >> (64 - 8 * len)));
    } else {
        p = enc_prefix(s, len);
    }
    const uint64_t q = enc_suffix(s, len, p);
    const EncHash &h = e->hash[j];
    const EncEntry &en = h.slots[enc_slot(h, p, q, (uint64_t)len)];
    if (en.len != (uint32_t)len || en.prefix != p || en.suffix != q) return -1;
    /* up to 16 bytes the two words cover the whole string; longer ones are compared in full */
    if (len > 16 && memcmp(e->vocab[j][en.code].data() + 8, s + 8, (size_t)len - 16) != 0) return -1;
    return en.code;
}

static inline int32_t enc_code(const b2f_encoder *e, int j, const b2f_str_column &c, int64_t i) {
    const int64_t k = i + c.offset;
    if (c.validity && !((c.validity[k >> 3] >> (k & 7)) & 1)) return e->null_code[j];
    int64_t a, b;
    if (c.offsets_are_64) {
        a = static_cast<const int64_t *>(c.offsets)[k], b = static_cast<const int64_t *>(c.offsets)[k + 1];
    } else {
        a = static_cast<const int32_t *>(c.offsets)[k], b = static_cast<const int32_t *>(c.offsets)[k + 1];
    }
    return enc_lookup(e, j, c.data + a, b - a, a + 8 <= c.data_bytes);
}

/* codes of rows [i0, i0 + nb) of categorical column j into out[0 .. nb): eight strings per step where the column allows it
 * (no nulls -- host_simd.cpp), the scalar lookup for the rest and for hits that need their middle compared */
static inline void enc_codes_block(const b2f_encoder *e, int j, const b2f_str_column &c, int64_t i0, int64_t nb, int32_t *out) {
    int64_t done = 0;
    if (!c.validity) {
        static_assert(sizeof(EncEntry) == 24, "the vector lookup gathers 24-byte entries");
        const EncHash &h = e->hash[j];
        const int64_t k0 = i0 + c.offset;
        const void *off = c.offsets_are_64 ? static_cast<const void *>(static_cast<const int64_t *>(c.offsets) + k0)
                                           : static_cast<const void *>(static_cast<const int32_t *>(c.offsets) + k0);
        done = b2f_simd_hash_codes(off, c.offsets_are_64, c.data, c.data_bytes, nb, h.m1, h.m2, h.m3, h.shift, h.slots.data(), out);
        for (int64_t i = 0; i < done; ++i)
            if (out[i] == -2) out[i] = enc_code(e, j, c, i0 + i);
    }
    for (int64_t i = done; i < nb; ++i) out[i] = enc_code(e, j, c, i0 + i);
}

/* ranked rows: blocks of B2F_RANK_BLOCK rows -- categorical block per row, float32 numerics transposed into a
 * column-major scratch, then one SIMD rank pass per feature over the block (forest_rank.h / host_simd.cpp) */
static int enc_range_ranked(const b2f_encoder *e, int64_t lo, int64_t hi, const b2f_str_column *cats, const double *const *nums,
                            const int64_t *num_strides, uint8_t *out) {
    const b2f_ranker *r = e->ranker;
    const int nc = e->n_cat, nn = e->n_num;
    int bad = 0;
    float cols[24 * B2F_RANK_BLOCK];
    int32_t codes[16];
    for (int64_t b0 = lo; b0 < hi; b0 += B2F_RANK_BLOCK) {
        const int64_t nb = std::min<int64_t>(B2F_RANK_BLOCK, hi - b0);
        for (int64_t i = 0; i < nb; ++i) {
            for (int j = 0; j < nc; ++j) {
                const int32_t c = enc_code(e, j, cats[j], b0 + i);
                codes[j] = c >= r->vocab[j] ? -1 : c;
            }
            rank_write_cats(r, codes, out + (size_t)(b0 + i) * r->row_bytes);
        }
        for (int k = 0; k < nn; ++k) bad |= b2f_simd_cvt_column(nums[k] + b0 * num_strides[k], num_strides[k], nb, cols + (size_t)k * B2F_RANK_BLOCK);
        rank_block(r, cols, nb, out + (size_t)b0 * r->row_bytes);
    }
    return bad;
}

/* packed 64-byte rows, block by block: the category codes of one column at a time (the feature's hash parameters stay in
 * registers, the column's offsets and bytes stream), the float64 -> float32 conversion of one column at a time (vector converts),
 * then one transposing pass that writes whole 64-byte rows (host_simd.cpp) */
static int enc_range_packed(const b2f_encoder *e, int64_t lo, int64_t hi, const b2f_str_column *cats, const double *const *nums,
                            const int64_t *num_strides, uint32_t *out) {
    const int nc = e->n_cat, nn = e->n_num;
    int bad = 0;
    float cols[14 * B2F_RANK_BLOCK];
    int32_t codes[9 * B2F_RANK_BLOCK];
    for (int64_t b0 = lo; b0 < hi; b0 += B2F_RANK_BLOCK) {
        const int64_t nb = std::min<int64_t>(B2F_RANK_BLOCK, hi - b0);
        for (int j = 0; j < nc; ++j) enc_codes_block(e, j, cats[j], b0, nb, codes + (size_t)j * B2F_RANK_BLOCK);
        for (int k = 0; k < nn; ++k) bad |= b2f_simd_cvt_column(nums[k] + b0 * num_strides[k], num_strides[k], nb, cols + (size_t)k * B2F_RANK_BLOCK);
        b2f_simd_pack_rows64(codes, cols, B2F_RANK_BLOCK, nc, nn, nb, out + (size_t)b0 * 16);
    }
    return bad;
}

static int enc_range(const b2f_encoder *e, int64_t lo, int64_t hi, const b2f_str_column *cats, const double *const *nums,
                     const int64_t *num_strides, int row_format, uint32_t *out) {
    if (row_format == B2F_ROWS_RANKED) return enc_range_ranked(e, lo, hi, cats, nums, num_strides, reinterpret_cast<uint8_t *>(out));
    if (row_format == B2F_ROWS_PACKED64 && e->n_cat == 9 && e->n_num <= 14) return enc_range_packed(e, lo, hi, cats, nums, num_strides, out);
    const int nc = e->n_cat, nn = e->n_num;
    const bool packed = row_format == B2F_ROWS_PACKED64;
    const int words = packed ? 16 : B2F_ROW_WORDS;
    int bad = 0;
    for (int64_t i = lo; i < hi; ++i) {
        int32_t codes[16];
        for (int j = 0; j < nc; ++j) codes[j] = enc_code(e, j, cats[j], i);
        uint32_t *row = out + (size_t)i * words;
        uint32_t *numw;
        if (packed) {
            uint64_t w = 0;
            for (int j = 0; j < nc; ++j) w |= (uint64_t)(uint32_t)(codes[j] + 1) << (7 * j);
            row[0] = (uint32_t)w;
            row[1] = (uint32_t)(w >> 32);
            numw = row + 2;
            for (int k = nn; k < 14; ++k) numw[k] = 0;
        } else {
            for (int j = 0; j < nc; ++j) row[j] = (uint32_t)codes[j];
            numw = row + nc;
            for (int k = nc + nn; k < B2F_ROW_WORDS; ++k) row[k] = 0;
        }
        for (int k = 0; k < nn; ++k) {
            const double v = nums[k][i * num_strides[k]];
            const float f = (float)v; /* round-to-nearest-even, as numpy astype(float32) */
            if (!(v != v) && !isfinite(f)) bad = 1; /* inf, or a finite float64 that overflows float32 */
            memcpy(&numw[k], &f, 4);
        }
    }
    return bad;
}

extern "C" b2f_encoder *b2f_encoder_create(int n_cat, int n_num, const int32_t *vocab_counts, const char *vocab_bytes,
                                           const int64_t *vocab_offsets, const int32_t *null_codes) {
    if (n_cat < 0 || n_cat > 16 || n_num < 0 || n_cat + n_num > 23 || (n_cat > 0 && (!vocab_counts || !vocab_bytes || !vocab_offsets)))
        return nullptr;
    b2f_encoder *e = new b2f_encoder();
    e->n_cat = n_cat;
    e->n_num = n_num;
    e->vocab.resize(n_cat);
    e->null_code.assign(n_cat, -1);
    int64_t s = 0;
    e->packed_ok = n_cat == 9 && n_num <= 14; /* the kernels' decode is fixed to nine 7-bit fields + numerics from word 2 */
    for (int j = 0; j < n_cat; ++j) {
        for (int k = 0; k < vocab_counts[j]; ++k, ++s)
            e->vocab[j].emplace_back(vocab_bytes + vocab_offsets[s], (size_t)(vocab_offsets[s + 1] - vocab_offsets[s]));
        if (null_codes) e->null_code[j] = null_codes[j];
        if (vocab_counts[j] > 126) e->packed_ok = false;
        e->hash.emplace_back();
        if (!enc_build_hash(e->vocab[j], e->hash[j])) {
            delete e;
            return nullptr;
        }
    }
    return e;
}

extern "C" void b2f_encoder_destroy(b2f_encoder *e) {
    if (e) delete e->ranker;
    delete e;
}

extern "C" int b2f_encoder_attach_ranker(b2f_encoder *e, const b2f_ranker *r) {
    if (!e || !r || !r->ok || r->n_cat != e->n_cat || r->n_num != e->n_num) return B2F_EINVAL;
    b2f_ranker *copy = new b2f_ranker(*r);
    std::vector<uint8_t>().swap(copy->layout); /* the encoder only needs the tables */
    ranker_fix_tabs(copy);                     /* the table views must point into the copy's own storage */
    delete e->ranker;
    e->ranker = copy;
    return B2F_OK;
}

/* category codes only, column-major (codes_out[j * n + i]): the drift detector's view of a request (its reference categories are
 * this encoder's vocabulary); -1 = not a reference category, nulls take the feature's null code */
extern "C" int b2f_encoder_codes(const b2f_encoder *e, int64_t n, const b2f_str_column *cat_cols, int32_t *codes_out, int threads) {
    if (!e || n < 0 || !codes_out || (e->n_cat > 0 && !cat_cols)) return B2F_EINVAL;
    threads = (int)std::min<int64_t>(std::max(threads, 1), std::max<int64_t>(1, n / 8192));
    auto work = [&](int64_t lo, int64_t hi) {
        for (int j = 0; j < e->n_cat; ++j) {
            int32_t *out = codes_out + (size_t)j * n;
            enc_codes_block(e, j, cat_cols[j], lo, hi - lo, out + lo);
        }
    };
    if (threads == 1) {
        work(0, n);
        return B2F_OK;
    }
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back(work, n * t / threads, n * (t + 1) / threads);
    work(0, n / threads);
    for (auto &th : pool) th.join();
    return B2F_OK;
}

extern "C" int b2f_encoder_encode(const b2f_encoder *e, int64_t n, const b2f_str_column *cat_cols, const double *const *num_cols,
                                  const int64_t *num_strides, int row_format, void *rows_out, int threads) {
    if (!e || n < 0 || !rows_out || (e->n_cat > 0 && !cat_cols) || (e->n_num > 0 && (!num_cols || !num_strides))) return B2F_EINVAL;
    if (row_format != B2F_ROWS_WORDS24 && row_format != B2F_ROWS_PACKED64 && row_format != B2F_ROWS_RANKED) return B2F_EINVAL;
    if (row_format == B2F_ROWS_PACKED64 && !e->packed_ok) return B2F_EINVAL;
    if (row_format == B2F_ROWS_RANKED && !e->ranker) return B2F_EINVAL;
    if (threads < 1) threads = 1;
    threads = (int)std::min<int64_t>(threads, std::max<int64_t>(1, n / 4096));
    uint32_t *out = static_cast<uint32_t *>(rows_out);
    if (threads == 1) return enc_range(e, 0, n, cat_cols, num_cols, num_strides, row_format, out) ? B2F_ERANGE : B2F_OK;
    std::vector<int> bad(threads, 0);
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t)
        pool.emplace_back([&, t] { bad[t] = enc_range(e, n * t / threads, n * (t + 1) / threads, cat_cols, num_cols, num_strides, row_format, out); });
    bad[0] = enc_range(e, 0, n / threads, cat_cols, num_cols, num_strides, row_format, out);
    for (auto &th : pool) th.join();
    for (int b : bad)
        if (b) return B2F_ERANGE;
    return B2F_OK;
}
