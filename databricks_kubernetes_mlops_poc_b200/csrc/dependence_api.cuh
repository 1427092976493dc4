/*
 * dependence_api.cuh -- C ABI of partial dependence (include/b2f.h: b2f_partial_dependence*); included by b2f_api.cu.
 *
 * Host side of K6 (partial_dependence.cuh).  A host call is a job of the host pipeline (HostJob in b2f_api.cu): its chunks
 * ride the same slots and streams as scores.
 */
#pragma once

/* device bytes of one chunk's partial-dependence curves: the chunk's rows are this over the row's bytes, 1 024 to 16 384 */
#define B2F_PD_CHUNK_BYTES (64ll << 20)
static int64_t pd_chunk_rows(const b2f_model *m) {
    const int64_t rows = B2F_PD_CHUNK_BYTES / ((int64_t)m->pd.points * (int64_t)sizeof(double));
    return std::max<int64_t>(1024, std::min<int64_t>(B2F_CHUNK_ROWS, rows / 32 * 32));
}

/* ------------------------------------------------------------------ partial dependence (K6: partial_dependence.cuh)
 * A call's probes and grid become one spec: a PdSeg per run of up to B2F_PD_SEG points of a probe, then every point's
 * word in output order (a row's output is its probes' points, concatenated), numerics imputed as the kernels impute rows.
 * The spec is checked and built on the host, uploaded once per call, and read by every chunk's launch. */
static int pd_check(int fmt, bool have_out) {
    const int rc = check_value_rows(fmt, "partial dependence takes");
    if (rc) return rc;
    if (!have_out) return set_err(B2F_EINVAL, "out is NULL");
    return B2F_OK;
}

static int pd_prepare(b2f_model *m, const b2f_pd_probe *probes, int n_probes, const uint32_t *grid_words) {
    const b2f_blob_header &h = m->hdr;
    if (!probes || !grid_words) return set_err(B2F_EINVAL, "probes or grid_words is NULL");
    if (n_probes < 1 || n_probes > B2F_PD_MAX_PROBES) return set_err(B2F_EINVAL, "n_probes = %d: expected 1..%d", n_probes, B2F_PD_MAX_PROBES);
    const int rc = check_walk_depth(m, "partial dependence walks");
    if (rc) return rc;
    const int fields = (int)(h.n_cat + h.n_num);
    std::vector<PdSeg> segs;
    std::vector<uint32_t> words;
    for (int i = 0; i < n_probes; ++i) {
        const b2f_pd_probe pr = probes[i];
        if (pr.word < 0 || pr.word >= fields) return set_err(B2F_EINVAL, "probe %d: row word %d outside the %d fields", i, pr.word, fields);
        if (pr.count < 1 || pr.count > B2F_PD_MAX_POINTS) return set_err(B2F_EINVAL, "probe %d: %d grid points, expected 1..%d", i, pr.count, B2F_PD_MAX_POINTS);
        if (pr.grid_offset < 0 || pr.grid_offset > B2F_PD_MAX_PROBES * B2F_PD_MAX_POINTS - pr.count)
            return set_err(B2F_EINVAL, "probe %d: grid offset %d out of range", i, pr.grid_offset);
        const bool cat = pr.word < (int)h.n_cat;
        for (int k = 0; k < pr.count; ++k) {
            uint32_t w = grid_words[pr.grid_offset + k];
            if (cat) {
                const int32_t code = (int32_t)w, vocab = h.vocab[pr.word];
                if (code < -1 || (vocab > 0 && code >= vocab))
                    return set_err(B2F_EINVAL, "probe %d point %d: category code %d outside [-1, %d)", i, k, code, vocab);
            } else {
                float f;
                memcpy(&f, &w, sizeof(f));
                if (std::isinf(f)) return set_err(B2F_ERANGE, "probe %d point %d: value is infinite or overflows float32", i, k);
                if (std::isnan(f)) memcpy(&w, &h.impute[pr.word], sizeof(w));
            }
            if (k % B2F_PD_SEG == 0) segs.push_back(PdSeg{(uint32_t)pr.word, 0u, (uint32_t)words.size(), 0u});
            segs.back().count++;
            words.push_back(w);
        }
    }
    Dependence &pd = m->pd;
    pd.n_segs = (int)segs.size();
    pd.points = (int32_t)words.size();
    pack_spec(pd.spec, segs, words);
    return B2F_OK;
}

/* out_dev[n][points] for n device rows of format fmt on stream st; spec_dev holds the call's spec */
static int launch_dependence(b2f_model *m, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, double *out_dev, const void *spec_dev) {
    if (n <= 0) return B2F_OK;
    PdParams pp = m->walk;
    pp.segs = static_cast<const PdSeg *>(spec_dev);
    pp.grid = reinterpret_cast<const uint32_t *>(pp.segs + m->pd.n_segs);
    pp.points = m->pd.points;
    const dim3 grid((unsigned)((n + B2F_PD_WARPS * 32 - 1) / (B2F_PD_WARPS * 32)), (unsigned)m->pd.n_segs);
    const uint32_t *rows = static_cast<const uint32_t *>(rows_dev);
    if (fmt == B2F_ROWS_PACKED64)
        k_partial_dependence<true><<<grid, B2F_PD_WARPS * 32, 0, st>>>(pp, rows, (long long)n, out_dev);
    else
        k_partial_dependence<false><<<grid, B2F_PD_WARPS * 32, 0, st>>>(pp, rows, (long long)n, out_dev);
    return launched(m, "k_partial_dependence");
}

/* the spec goes up once, before the chunks that read it; no earlier host call still reads it (each one synchronises) */
extern "C" int b2f_partial_dependence(b2f_model *m, const void *rows, int64_t n, int row_format, const b2f_pd_probe *probes, int n_probes,
                                      const uint32_t *grid_words, double *out, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (device_ms) *device_ms = 0.0f;
    int rc = pd_prepare(m, probes, n_probes, grid_words);
    if (rc) return rc;
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    if ((rc = pd_check(row_format, out || n == 0))) return rc;
    if (n > 0) {
        CUDA_TRY(cudaSetDevice(m->device));
        if ((rc = upload_spec(m, m->pd.host_spec, m->pd.spec, false, nullptr))) return rc;
    }
    const HostJob job{(size_t)m->pd.points * sizeof(double), pd_chunk_rows(m), false, 0,
                      [](b2f_model *m, int, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, void *out_dev, int32_t *, DevBuf &) {
                          return launch_dependence(m, st, rows_dev, n, fmt, static_cast<double *>(out_dev), m->pd.host_spec.p);
                      }};
    return timed_host_batch(m, job, rows, n, row_format, out, device_ms);
}
/* the spec is copied on the compute stream into the device form's own buffer, so it is ordered with the launch */
extern "C" int b2f_partial_dependence_device(b2f_model *m, const void *rows_dev, int64_t n, int row_format, const b2f_pd_probe *probes,
                                             int n_probes, const uint32_t *grid_words, double *out_dev) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    int rc = pd_prepare(m, probes, n_probes, grid_words);
    if (rc == B2F_OK) rc = pd_check(row_format, out_dev != nullptr || n == 0);
    if (rc == B2F_OK) rc = check_row_format(m, row_format);
    if (rc) return rc;
    if (n == 0) return B2F_OK;
    CUDA_TRY(cudaSetDevice(m->device));
    if ((rc = upload_spec(m, m->pd.device_spec, m->pd.spec, true, nullptr))) return rc;
    return launch_dependence(m, m->compute, rows_dev, n, row_format, out_dev, m->pd.device_spec.p);
}
