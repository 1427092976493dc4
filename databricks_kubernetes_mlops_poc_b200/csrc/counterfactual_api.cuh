/*
 * counterfactual_api.cuh -- C ABI of nearest single-field counterfactuals (include/b2f.h: b2f_counterfactual*,
 * b2f_blob_split_values); included by b2f_api.cu.
 *
 * Host side of K7 (counterfactual.cuh).  A host call is a job of the host pipeline (HostJob in b2f_api.cu): its chunks
 * ride the same slots and streams as scores, with the per-(row, segment) candidates in the slot's scratch.
 */
#pragma once

static_assert(sizeof(struct b2f_counterfactual) == 32 && offsetof(struct b2f_counterfactual, lower) == 16 &&
                  offsetof(struct b2f_counterfactual, value) == 24,
              "b2f_counterfactual layout");
static_assert(sizeof(CfCand) == 32, "CfCand layout");

extern "C" int64_t b2f_blob_split_values(const void *forest_blob, size_t nbytes, int word, float *out, int64_t cap) {
    b2f_blob_header h;
    const uint8_t *blob = static_cast<const uint8_t *>(forest_blob);
    int rc = validate_blob(blob, nbytes, &h);
    if (rc) return rc;
    if (word < (int)h.n_cat || word >= (int)(h.n_cat + h.n_num))
        return set_err(B2F_EINVAL, "row word %d is not one of the numeric words %u..%u", word, h.n_cat, h.n_cat + h.n_num - 1);
    if (cap < 0 || (cap > 0 && !out)) return set_err(B2F_EINVAL, "bad output buffer");
    std::vector<std::vector<float>> thr;
    if (const char *why = forest_split_values(blob, h, thr)) return set_err(B2F_EINVAL, "forest blob: %s", why);
    const std::vector<float> &v = thr[word - h.n_cat];
    if (cap > 0) memcpy(out, v.data(), (size_t)std::min<int64_t>(cap, (int64_t)v.size()) * sizeof(float));
    return (int64_t)v.size();
}

/* device bytes of one chunk's candidates: the chunk's rows are this over the row's bytes, 1 024 to 16 384 */
#define B2F_CF_CHUNK_BYTES (64ll << 20)
static int64_t cf_chunk_rows(const b2f_model *m) {
    const int64_t rows = B2F_CF_CHUNK_BYTES / ((int64_t)m->cf.cp.seg0[m->cf.cp.n_words] * (int64_t)sizeof(CfCand));
    return std::max<int64_t>(1024, std::min<int64_t>(B2F_CHUNK_ROWS, rows / 32 * 32));
}

/* the split-value table, built from the device copy of the blob on the first call and kept for the model's life */
static int cf_build_table(b2f_model *m) {
    Counterfactual &cf = m->cf;
    if (cf.built) return B2F_OK;
    CUDA_TRY(cudaSetDevice(m->device));
    std::vector<uint8_t> blob(m->hdr.total_bytes);
    CUDA_TRY(cudaMemcpy(blob.data(), m->d_blob, blob.size(), cudaMemcpyDeviceToHost));
    std::vector<std::vector<float>> thr;
    if (const char *why = forest_split_values(blob.data(), m->hdr, thr)) return set_err(B2F_EINVAL, "counterfactuals: %s", why);
    std::vector<uint32_t> &t = cf.table;
    t.assign(B2F_CF_TAB_HEAD, 0u);
    for (size_t k = 0; k < thr.size(); ++k) {
        const uint32_t w = m->hdr.n_cat + (uint32_t)k;
        t[w] = (uint32_t)(t.size() - B2F_CF_TAB_HEAD);
        t[B2F_ROW_WORDS + w] = (uint32_t)thr[k].size();
        const size_t at = t.size();
        t.resize(at + thr[k].size());
        memcpy(t.data() + at, thr[k].data(), thr[k].size() * sizeof(float));
    }
    const size_t bytes = t.size() * sizeof(uint32_t);
    int rc = cf.dev.reserve(m->compute, bytes, bytes);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpy(cf.dev.p, t.data(), bytes, cudaMemcpyHostToDevice));
    cf.cp.tab = static_cast<const uint32_t *>(cf.dev.p);
    cf.built = true;
    return B2F_OK;
}

/* check a call's arguments, then set the probe fields of m->cf.cp (builds the table on the first call) */
static int cf_prepare(b2f_model *m, int64_t n, int fmt, const int32_t *words, int n_words, double cutoff, bool have_out) {
    const b2f_blob_header &h = m->hdr;
    if (fmt == B2F_ROWS_RANKED)
        return set_err(B2F_EINVAL, "counterfactuals take float32 rows (B2F_ROWS_WORDS24 / B2F_ROWS_PACKED64): ranked rows carry no values");
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    if (!have_out) return set_err(B2F_EINVAL, "out is NULL");
    if (!words) return set_err(B2F_EINVAL, "words is NULL");
    if (n_words < 1 || n_words > B2F_CF_MAX_WORDS) return set_err(B2F_EINVAL, "n_words = %d: expected 1..%d", n_words, B2F_CF_MAX_WORDS);
    for (int i = 0; i < n_words; ++i)
        if (words[i] < (int)h.n_cat || words[i] >= (int)(h.n_cat + h.n_num))
            return set_err(B2F_EINVAL,
                           "words[%d] = %d: counterfactuals probe the numeric row words %u..%u; a categorical field has no order "
                           "(score its categories with b2f_partial_dependence)",
                           i, words[i], h.n_cat, h.n_cat + h.n_num - 1);
    if (!std::isfinite(cutoff) || cutoff < 0.0 || cutoff > 1.0) return set_err(B2F_EINVAL, "cutoff %g: expected a number in [0, 1]", cutoff);
    if (h.max_depth > B2F_PD_STACK) return set_err(B2F_EINVAL, "counterfactuals walk trees of depth <= %d; this forest has depth %u", B2F_PD_STACK, h.max_depth);
    int rc = cf_build_table(m);
    if (rc) return rc;
    CfParams &cp = m->cf.cp;
    cp.cutoff = cutoff;
    cp.n_words = n_words;
    uint32_t segs = 0;
    for (int i = 0; i < n_words; ++i) {
        cp.word[i] = (uint32_t)words[i];
        cp.seg0[i] = segs;
        segs += (m->cf.table[B2F_ROW_WORDS + words[i]] + 1u + B2F_PD_SEG - 1u) / B2F_PD_SEG; /* m + 1 pieces */
    }
    cp.seg0[n_words] = segs;
    return B2F_OK;
}

/* n device rows of format fmt on stream st: candidates in scratch, then out (records, row stride out_stride bytes) and
 * proba (may be NULL, row stride proba_stride bytes) */
static int launch_counterfactual(b2f_model *m, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, uint8_t *out, long long out_stride,
                                 uint8_t *proba, long long proba_stride, DevBuf &scratch) {
    if (n <= 0) return B2F_OK;
    CfParams cp = m->cf.cp;
    const int64_t segs = cp.seg0[cp.n_words];
    const size_t need = (size_t)n * (size_t)segs * sizeof(CfCand);
    int rc = scratch.reserve(st, need, need);
    if (rc) return rc;
    CfCand *cand = static_cast<CfCand *>(scratch.p);
    const uint32_t *rows = static_cast<const uint32_t *>(rows_dev);
    const bool pk = fmt == B2F_ROWS_PACKED64;
    const unsigned bx = (unsigned)((n + B2F_PD_WARPS * 32 - 1) / (B2F_PD_WARPS * 32));
    for (int64_t s = 0; s < segs; s += 65535) { /* gridDim.y <= 65535 */
        cp.seg_base = (int32_t)s;
        const dim3 grid(bx, (unsigned)std::min<int64_t>(65535, segs - s));
        if (pk)
            k_counterfactual<true><<<grid, B2F_PD_WARPS * 32, 0, st>>>(cp, rows, (long long)n, cand);
        else
            k_counterfactual<false><<<grid, B2F_PD_WARPS * 32, 0, st>>>(cp, rows, (long long)n, cand);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return set_err(B2F_ECUDA, "k_counterfactual launch failed: %s", cudaGetErrorString(e));
        m->launches++;
    }
    const dim3 fgrid((unsigned)((n + 127) / 128), (unsigned)cp.n_words);
    if (pk)
        k_counterfactual_finish<true><<<fgrid, 128, 0, st>>>(cp, rows, (long long)n, cand, out, out_stride, proba, proba_stride);
    else
        k_counterfactual_finish<false><<<fgrid, 128, 0, st>>>(cp, rows, (long long)n, cand, out, out_stride, proba, proba_stride);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_err(B2F_ECUDA, "k_counterfactual_finish launch failed: %s", cudaGetErrorString(e));
    m->launches++;
    return B2F_OK;
}

/* A host chunk's output row is the row's n_words records, then its p1: one D2H copy per chunk into a staging array, split
 * into the caller's out and proba afterwards. */
extern "C" int b2f_counterfactual(b2f_model *m, const void *rows, int64_t n, int row_format, const int32_t *words, int n_words, double cutoff,
                                  double *proba, struct b2f_counterfactual *out, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (device_ms) *device_ms = 0.0f;
    int rc = cf_prepare(m, n, row_format, words, n_words, cutoff, out || n == 0);
    if (rc) return rc;
    const size_t rec_bytes = (size_t)n_words * sizeof(struct b2f_counterfactual), row_bytes = rec_bytes + sizeof(double);
    std::vector<uint8_t> staged((size_t)std::max<int64_t>(n, 0) * row_bytes);
    const HostJob job{row_bytes, cf_chunk_rows(m), false, 0,
                      [](b2f_model *m, int, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, void *out_dev, int32_t *, DevBuf &scratch) {
                          const long long rec = (long long)m->cf.cp.n_words * (long long)sizeof(struct b2f_counterfactual), stride = rec + (long long)sizeof(double);
                          uint8_t *o = static_cast<uint8_t *>(out_dev);
                          return launch_counterfactual(m, st, rows_dev, n, fmt, o, stride, o + rec, stride, scratch);
                      }};
    rc = timed_host_batch(m, job, rows, n, row_format, reinterpret_cast<double *>(staged.data()), device_ms);
    if (rc) return rc;
    for (int64_t i = 0; i < n; ++i) {
        const uint8_t *r = staged.data() + (size_t)i * row_bytes;
        memcpy(out + (size_t)i * n_words, r, rec_bytes);
        if (proba) memcpy(proba + i, r + rec_bytes, sizeof(double));
    }
    return B2F_OK;
}

extern "C" int b2f_counterfactual_device(b2f_model *m, const void *rows_dev, int64_t n, int row_format, const int32_t *words, int n_words,
                                         double cutoff, double *proba_dev, struct b2f_counterfactual *out_dev) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    int rc = cf_prepare(m, n, row_format, words, n_words, cutoff, out_dev != nullptr || n == 0);
    if (rc == B2F_OK) rc = check_row_format(m, row_format);
    if (rc) return rc;
    if (n == 0) return B2F_OK;
    CUDA_TRY(cudaSetDevice(m->device));
    return launch_counterfactual(m, m->compute, rows_dev, n, row_format, reinterpret_cast<uint8_t *>(out_dev),
                                 (long long)n_words * (long long)sizeof(struct b2f_counterfactual), reinterpret_cast<uint8_t *>(proba_dev),
                                 (long long)sizeof(double), m->scratch);
}
