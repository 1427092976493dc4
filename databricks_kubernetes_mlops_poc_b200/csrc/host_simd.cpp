/*
 * host_simd.cpp -- host-side SIMD for the ranked-row encoder (compiled by g++, not nvcc; linked into libb200forest.so).
 *
 * rank_k(x) = #{ j : t'_j <= x } over the sorted distinct split values of numeric feature k (csrc/forest_rank.h) is the
 * one piece of arithmetic the ranked row format moves from the GPU kernel to the request encoder (reference
 * counterpart: the float32-vs-threshold compares inside sklearn's tree walk, databricks/src/02-register-model.ipynb:335-337).
 * A request batch needs n_rows x 14 of them, so it is done without branches and without per-element gathers:
 *
 *   the split values of a feature are stored as a wide search tree laid out level by level ("rank table"):
 *     fan[j]   = fan-out of level j: 16 for the upper levels, 16 / 32 / 48 / 64 for the last one
 *     full     = the sorted values padded with +inf to prod(fan) entries (> m, so every level's count stays below its fan-out)
 *     lvl[j][i] = full[(i + 1) * S_j - 1], S_j = prod(fan[j+1..])      the LARGEST value of the i-th chunk at level j
 *   one level = fan/16 64-byte loads of consecutive chunk maxima, vector compares against the broadcast x, popcounts:
 *   c_j = #{chunk maxima <= x} is the digit of the rank in the mixed radix, and selects the chunk to descend into.
 *   m <= 63: one level; m <= 1023: two (16 x up to 64: 4 KB per feature, so 14 features stay in L1); m <= 16383: three.
 *
 * AVX-512F path when the CPU has it, else an AVX2 form of the same walk (2 x 8 lanes), else scalar.
 */
#include <immintrin.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

extern "C" {

struct b2f_ranktab {
    int32_t levels;      /* 1..4 */
    int32_t count;       /* m: real split values */
    int32_t fan[4];      /* fan-out per level: multiples of 16 */
    const float *lvl[4]; /* lvl[j]: prod(fan[0..j]) floats */
};

int b2f_simd_level(void) {
    static int level = -1;
    if (level < 0) {
        __builtin_cpu_init();
        level = __builtin_cpu_supports("avx512f") ? 2 : (__builtin_cpu_supports("avx2") ? 1 : 0);
        const char *cap = getenv("B2F_SIMD"); /* test hook: "0" scalar, "1" at most AVX2 */
        if (cap && cap[0] >= '0' && cap[0] <= '2' && (cap[0] - '0') < level) level = cap[0] - '0';
    }
    return level;
}

static inline uint32_t rank_scalar(const b2f_ranktab *t, float x) {
    uint32_t idx = 0;
    for (int j = 0; j < t->levels; ++j) {
        const int fan = t->fan[j];
        const float *p = t->lvl[j] + (size_t)idx * fan;
        uint32_t c = 0;
        for (int i = 0; i < fan; ++i) c += p[i] <= x ? 1u : 0u;
        idx = idx * fan + c;
    }
    return idx;
}

__attribute__((target("avx2,popcnt"))) static inline uint32_t rank_avx2(const b2f_ranktab *t, float x) {
    const __m256 vx = _mm256_set1_ps(x);
    uint32_t idx = 0;
    for (int j = 0; j < t->levels; ++j) {
        const int fan = t->fan[j];
        const float *p = t->lvl[j] + (size_t)idx * fan;
        uint32_t c = 0;
        for (int i = 0; i < fan; i += 8) c += (uint32_t)__builtin_popcount((unsigned)_mm256_movemask_ps(_mm256_cmp_ps(_mm256_loadu_ps(p + i), vx, _CMP_LE_OQ)));
        idx = idx * fan + c;
    }
    return idx;
}

__attribute__((target("avx512f,popcnt"))) static inline uint32_t rank_avx512(const b2f_ranktab *t, float x) {
    const __m512 vx = _mm512_set1_ps(x);
    uint32_t idx = 0;
    for (int j = 0; j < t->levels; ++j) {
        const int fan = t->fan[j];
        const float *p = t->lvl[j] + (size_t)idx * fan;
        uint32_t c = (uint32_t)__builtin_popcount((unsigned)_mm512_cmp_ps_mask(_mm512_loadu_ps(p), vx, _CMP_LE_OQ));
        for (int i = 16; i < fan; i += 16) c += (uint32_t)__builtin_popcount((unsigned)_mm512_cmp_ps_mask(_mm512_loadu_ps(p + i), vx, _CMP_LE_OQ));
        idx = idx * fan + c;
    }
    return idx;
}

#define RANK_COLUMN_BODY(RANKFN)                                                              \
    for (int64_t i = 0; i < n; ++i) {                                                         \
        const float v = x[i * x_stride];                                                      \
        out[i * out_stride] = (v != v) ? nan_rank : (uint16_t)RANKFN(t, v);                   \
    }

__attribute__((target("avx512f,popcnt"))) static void rank_column_avx512(const b2f_ranktab *t, const float *x, int64_t n, int64_t x_stride, uint16_t *out,
                                                                           int64_t out_stride, uint16_t nan_rank) {
    RANK_COLUMN_BODY(rank_avx512)
}
__attribute__((target("avx2,popcnt"))) static void rank_column_avx2(const b2f_ranktab *t, const float *x, int64_t n, int64_t x_stride, uint16_t *out,
                                                                      int64_t out_stride, uint16_t nan_rank) {
    RANK_COLUMN_BODY(rank_avx2)
}
static void rank_column_scalar(const b2f_ranktab *t, const float *x, int64_t n, int64_t x_stride, uint16_t *out, int64_t out_stride, uint16_t nan_rank) {
    RANK_COLUMN_BODY(rank_scalar)
}

/* ranks of n values of ONE feature: x[i * x_stride] -> out[i * out_stride] (strides in elements); NaN -> nan_rank */
void b2f_simd_rank_column(const b2f_ranktab *t, const float *x, int64_t n, int64_t x_stride, uint16_t *out, int64_t out_stride, uint16_t nan_rank) {
    switch (b2f_simd_level()) {
        case 2: rank_column_avx512(t, x, n, x_stride, out, out_stride, nan_rank); break;
        case 1: rank_column_avx2(t, x, n, x_stride, out, out_stride, nan_rank); break;
        default: rank_column_scalar(t, x, n, x_stride, out, out_stride, nan_rank); break;
    }
}

/* ---- float64 column -> float32 block (round to nearest even, as numpy astype(float32)); returns 1 when some value is +-inf
 *      or a finite float64 beyond float32 (sklearn raises ValueError there), NaN passes through (the kernel imputes) ---- */
static int cvt_column_scalar(const double *src, int64_t stride, int64_t n, float *dst) {
    int bad = 0;
    for (int64_t i = 0; i < n; ++i) {
        const double v = src[i * stride];
        const float f = (float)v;
        if (!(v != v) && !isfinite(f)) bad = 1;
        dst[i] = f;
    }
    return bad;
}

__attribute__((target("avx512f"))) static int cvt_column_avx512(const double *src, int64_t n, float *dst) {
    const __m512i absmask = _mm512_set1_epi32(0x7fffffff), inf = _mm512_set1_epi32(0x7f800000);
    __mmask16 bad = 0;
    int64_t i = 0;
    for (; i + 16 <= n; i += 16) {
        const __m256 a = _mm512_cvtpd_ps(_mm512_loadu_pd(src + i)), b = _mm512_cvtpd_ps(_mm512_loadu_pd(src + i + 8));
        const __m512 f = _mm512_castpd_ps(_mm512_insertf64x4(_mm512_castpd256_pd512(_mm256_castps_pd(a)), _mm256_castps_pd(b), 1));
        /* |f| == inf: the source was +-inf or overflowed; a NaN source stays NaN (exponent all ones, mantissa non-zero) */
        bad |= _mm512_cmpeq_epi32_mask(_mm512_and_si512(_mm512_castps_si512(f), absmask), inf);
        _mm512_storeu_ps(dst + i, f);
    }
    return (bad ? 1 : 0) | (i < n ? cvt_column_scalar(src + i, 1, n - i, dst + i) : 0);
}

int b2f_simd_cvt_column(const double *src, int64_t stride, int64_t n, float *dst) {
    if (stride == 1 && b2f_simd_level() == 2) return cvt_column_avx512(src, n, dst);
    return cvt_column_scalar(src, stride, n, dst);
}

/* ---- B2F_ROWS_PACKED64 rows from a column-major block: codes[j * ld + i] (int32, -1 = unknown) and cols[k * ld + i]
 *      (float32) -> row i = { uint64 of nine 7-bit (code + 1) fields, 14 float32 }, 64 bytes.  AVX-512: sixteen rows at a time,
 *      the two halves of the categorical word and the 14 numerics as sixteen 16-lane vectors, one 16 x 16 transpose of 32-bit
 *      elements (64 shuffles), sixteen 64-byte stores -- non-temporal when the destination is 64-byte aligned (pinned staging
 *      that only the DMA engine reads: no read-for-ownership of the row's cache line). ---- */
static void pack_rows64_scalar(const int32_t *codes, const float *cols, int64_t ld, int n_cat, int n_num, int64_t i0, int64_t i1, uint32_t *out) {
    for (int64_t i = i0; i < i1; ++i) {
        uint64_t w = 0;
        for (int j = 0; j < n_cat; ++j) w |= (uint64_t)(uint32_t)(codes[j * ld + i] + 1) << (7 * j);
        uint32_t *row = out + (size_t)i * 16;
        row[0] = (uint32_t)w;
        row[1] = (uint32_t)(w >> 32);
        for (int k = 0; k < n_num; ++k) memcpy(&row[2 + k], &cols[k * ld + i], 4);
        for (int k = n_num; k < 14; ++k) row[2 + k] = 0;
    }
}

__attribute__((target("avx512f"))) static void pack_rows64_avx512(const int32_t *codes, const float *cols, int64_t ld, int n_cat, int n_num, int64_t nb,
                                                                  uint32_t *out) {
    const bool nt = ((uintptr_t)out & 63u) == 0;
    const __m512i one = _mm512_set1_epi32(1);
    int64_t g = 0;
    for (; g + 16 <= nb; g += 16) {
        __m512i c[16];
        __m512i lo = _mm512_setzero_si512(), hi = _mm512_setzero_si512();
        for (int j = 0; j < n_cat; ++j) {
            const __m512i v = _mm512_add_epi32(_mm512_loadu_si512(codes + j * ld + g), one); /* 1..127, 0 = unknown */
            const int sh = 7 * j;
            if (sh < 32) lo = _mm512_or_si512(lo, _mm512_sllv_epi32(v, _mm512_set1_epi32(sh)));
            if (sh + 7 > 32) hi = _mm512_or_si512(hi, sh >= 32 ? _mm512_sllv_epi32(v, _mm512_set1_epi32(sh - 32)) : _mm512_srlv_epi32(v, _mm512_set1_epi32(32 - sh)));
        }
        c[0] = lo;
        c[1] = hi;
        for (int k = 0; k < 14; ++k) c[2 + k] = k < n_num ? _mm512_castps_si512(_mm512_loadu_ps(cols + k * ld + g)) : _mm512_setzero_si512();
        __m512i t[16], u[16];
        for (int a = 0; a < 8; ++a) {
            t[2 * a] = _mm512_unpacklo_epi32(c[2 * a], c[2 * a + 1]);
            t[2 * a + 1] = _mm512_unpackhi_epi32(c[2 * a], c[2 * a + 1]);
        }
        for (int a = 0; a < 4; ++a) { /* u[4a + r]: 128-bit lane L = row 4L + r, columns 4a .. 4a + 3 */
            u[4 * a + 0] = _mm512_unpacklo_epi64(t[4 * a], t[4 * a + 2]);
            u[4 * a + 1] = _mm512_unpackhi_epi64(t[4 * a], t[4 * a + 2]);
            u[4 * a + 2] = _mm512_unpacklo_epi64(t[4 * a + 1], t[4 * a + 3]);
            u[4 * a + 3] = _mm512_unpackhi_epi64(t[4 * a + 1], t[4 * a + 3]);
        }
        for (int r = 0; r < 4; ++r) {
            const __m512i v0 = _mm512_shuffle_i32x4(u[r], u[4 + r], 0x88), v1 = _mm512_shuffle_i32x4(u[r], u[4 + r], 0xdd);
            const __m512i v2 = _mm512_shuffle_i32x4(u[8 + r], u[12 + r], 0x88), v3 = _mm512_shuffle_i32x4(u[8 + r], u[12 + r], 0xdd);
            const __m512i row[4] = {_mm512_shuffle_i32x4(v0, v2, 0x88), _mm512_shuffle_i32x4(v1, v3, 0x88), _mm512_shuffle_i32x4(v0, v2, 0xdd),
                                    _mm512_shuffle_i32x4(v1, v3, 0xdd)}; /* rows 4L + r, L = 0..3 */
            for (int L = 0; L < 4; ++L) {
                uint32_t *dst = out + (size_t)(g + 4 * L + r) * 16;
                if (nt)
                    _mm512_stream_si512(reinterpret_cast<__m512i *>(dst), row[L]);
                else
                    _mm512_storeu_si512(dst, row[L]);
            }
        }
    }
    if (nt) _mm_sfence(); /* the rows are handed to a DMA copy next: order the non-temporal stores before it */
    if (g < nb) pack_rows64_scalar(codes, cols, ld, n_cat, n_num, g, nb, out);
}

void b2f_simd_pack_rows64(const int32_t *codes, const float *cols, int64_t ld, int n_cat, int n_num, int64_t nb, uint32_t *out) {
    if (b2f_simd_level() == 2 && n_cat <= 9 && n_num <= 14)
        pack_rows64_avx512(codes, cols, ld, n_cat, n_num, nb, out);
    else
        pack_rows64_scalar(codes, cols, ld, n_cat, n_num, 0, nb, out);
}

/* ---- vocabulary codes of a block of one string column, eight strings at a time (AVX-512F + DQ) ----------------------------
 * The scalar lookup (row_encoder.h: enc_lookup) is ~30 instructions per string; here the same perfect hash runs on eight rows
 * per step: two loads of the Arrow offsets (int32 or int64), a gather of the first 8 bytes and one of the last 8 bytes of each
 * string, the length mask, three 64-bit multiplies, and three gathers of the 24-byte table entry {prefix, suffix, len | code}.
 * Returns how many rows from the start were done (a multiple of 8; the caller finishes the rest with the scalar lookup).
 * A hit on a string longer than 16 bytes still needs its middle compared: those rows get B2F_CODE_RECHECK. */
#define B2F_CODE_RECHECK (-2)

__attribute__((target("avx512f,avx512dq,avx512vl"))) static inline __m256i hash_codes_step(__m512i a, __m512i len64, const uint8_t *data, __m512i vm1,
                                                                                            __m512i vm2, __m512i vm3, __m128i vshift, const void *slots) {
    const __m512i one = _mm512_set1_epi64(1), three = _mm512_set1_epi64(3), lo32 = _mm512_set1_epi64(0xFFFFFFFFll);
    const __m512i off2 = _mm512_max_epi64(_mm512_sub_epi64(len64, _mm512_set1_epi64(8)), _mm512_setzero_si512());
    const __m512i p_raw = _mm512_i64gather_epi64(a, data, 1);
    const __m512i q_raw = _mm512_i64gather_epi64(_mm512_add_epi64(a, off2), data, 1);
    /* (1 << 8 len) - 1: a shift count >= 64 gives 0, minus one = all ones -- exactly the mask of a string of >= 8 bytes */
    const __m512i mask = _mm512_sub_epi64(_mm512_sllv_epi64(one, _mm512_slli_epi64(len64, 3)), one);
    const __m512i pp = _mm512_and_si512(p_raw, mask), qq = _mm512_and_si512(q_raw, mask);
    const __m512i h = _mm512_xor_si512(_mm512_xor_si512(_mm512_mullo_epi64(pp, vm1), _mm512_mullo_epi64(qq, vm2)), _mm512_mullo_epi64(len64, vm3));
    const __m512i idx = _mm512_mullo_epi64(_mm512_srl_epi64(h, vshift), three); /* entry = 3 x 8 bytes */
    const __m512i ep = _mm512_i64gather_epi64(idx, slots, 8);
    const __m512i es = _mm512_i64gather_epi64(_mm512_add_epi64(idx, one), slots, 8);
    const __m512i el = _mm512_i64gather_epi64(_mm512_add_epi64(idx, _mm512_set1_epi64(2)), slots, 8);
    const __mmask8 hit = _mm512_cmpeq_epi64_mask(ep, pp) & _mm512_cmpeq_epi64_mask(es, qq) & _mm512_cmpeq_epi64_mask(_mm512_and_si512(el, lo32), len64);
    const __mmask8 longs = hit & _mm512_cmpgt_epi64_mask(len64, _mm512_set1_epi64(16));
    __m256i code = _mm512_cvtepi64_epi32(_mm512_srli_epi64(el, 32));
    code = _mm256_mask_blend_epi32(hit, _mm256_set1_epi32(-1), code);
    return _mm256_mask_blend_epi32(longs, code, _mm256_set1_epi32(B2F_CODE_RECHECK));
}

__attribute__((target("avx512f,avx512dq,avx512vl"))) static int64_t hash_codes_avx512(const void *offsets, int offsets_are_64, const uint8_t *data,
                                                                                      int64_t data_bytes, int64_t nb, uint64_t m1, uint64_t m2, uint64_t m3,
                                                                                      int shift, const void *slots, int32_t *codes) {
    const __m512i vm1 = _mm512_set1_epi64((long long)m1), vm2 = _mm512_set1_epi64((long long)m2), vm3 = _mm512_set1_epi64((long long)m3);
    const __m128i vshift = _mm_cvtsi32_si128(shift);
    int64_t i = 0;
    if (offsets_are_64) {
        const int64_t *o = static_cast<const int64_t *>(offsets);
        for (; i + 8 <= nb; i += 8) {
            if (o[i + 8] + 8 > data_bytes) break; /* the 8-byte loads of the last strings would leave the buffer */
            const __m512i a = _mm512_loadu_si512(o + i), b = _mm512_loadu_si512(o + i + 1);
            _mm256_storeu_si256(reinterpret_cast<__m256i *>(codes + i), hash_codes_step(a, _mm512_sub_epi64(b, a), data, vm1, vm2, vm3, vshift, slots));
        }
    } else {
        const int32_t *o = static_cast<const int32_t *>(offsets);
        for (; i + 8 <= nb; i += 8) {
            if ((int64_t)o[i + 8] + 8 > data_bytes) break;
            const __m512i a = _mm512_cvtepi32_epi64(_mm256_loadu_si256(reinterpret_cast<const __m256i *>(o + i)));
            const __m512i b = _mm512_cvtepi32_epi64(_mm256_loadu_si256(reinterpret_cast<const __m256i *>(o + i + 1)));
            _mm256_storeu_si256(reinterpret_cast<__m256i *>(codes + i), hash_codes_step(a, _mm512_sub_epi64(b, a), data, vm1, vm2, vm3, vshift, slots));
        }
    }
    return i;
}

int64_t b2f_simd_hash_codes(const void *offsets, int offsets_are_64, const uint8_t *data, int64_t data_bytes, int64_t nb, uint64_t m1, uint64_t m2,
                            uint64_t m3, int shift, const void *slots, int32_t *codes) {
    static int ok = -1;
    if (ok < 0) {
        __builtin_cpu_init();
        ok = (b2f_simd_level() == 2 && __builtin_cpu_supports("avx512dq") && __builtin_cpu_supports("avx512vl")) ? 1 : 0;
    }
    if (!ok || nb < 8) return 0;
    return hash_codes_avx512(offsets, offsets_are_64, data, data_bytes, nb, m1, m2, m3, shift, slots, codes);
}

} /* extern "C" */
