/*
 * pair_dependence_api.cuh -- C ABI of two-way partial dependence (include/b2f.h: b2f_pair_dependence*); included by b2f_api.cu.
 *
 * Host side of K10 (pair_dependence.cuh).  A call's probes and points become one spec: a PpSeg per run of up to
 * B2F_PD_SEG points of a probe, then every point's two words in output order, numerics imputed as the kernels impute rows.
 *   mean = 0: the curves, n x P doubles.  A host call is a job of the host pipeline (HostJob in b2f_api.cu), in chunks of
 *             at most B2F_PD_CHUNK_BYTES of curves.
 *   mean = 1: P doubles, each point's mean over the rows.  Not a host job: a point reads every row, so the rows go to the
 *             device once, on the compute stream, into buffers the model owns (grown on demand, never shrunk), and the
 *             points are scored in groups of whole segments whose per-CTA partial sums stay under B2F_PERM_SCRATCH_BYTES.
 */
#pragma once

static_assert(sizeof(b2f_pair_probe) == 16, "b2f_pair_probe layout");

static int pp_check(int fmt, bool have_out) {
    const int rc = check_value_rows(fmt, "pair dependence takes");
    if (rc) return rc;
    if (!have_out) return set_err(B2F_EINVAL, "out is NULL");
    return B2F_OK;
}

/* one point word of row word `word`: a category code in [-1, vocab), or float32 bits, NaN imputed; -> rc */
static int pp_point_word(const b2f_blob_header &h, int probe, int k, int word, uint32_t &w) {
    if (word < (int)h.n_cat) {
        const int32_t code = (int32_t)w, vocab = h.vocab[word];
        if (code < -1 || (vocab > 0 && code >= vocab))
            return set_err(B2F_EINVAL, "probe %d point %d: category code %d of word %d outside [-1, %d)", probe, k, code, word, vocab);
        return B2F_OK;
    }
    float f;
    memcpy(&f, &w, sizeof(f));
    if (std::isinf(f)) return set_err(B2F_ERANGE, "probe %d point %d: value of word %d is infinite or overflows float32", probe, k, word);
    if (std::isnan(f)) memcpy(&w, &h.impute[word], sizeof(w));
    return B2F_OK;
}

static int pp_prepare(b2f_model *m, const b2f_pair_probe *probes, int n_probes, const uint32_t *point_words, int mean) {
    const b2f_blob_header &h = m->hdr;
    if (!probes || !point_words) return set_err(B2F_EINVAL, "probes or point_words is NULL");
    if (mean != 0 && mean != 1) return set_err(B2F_EINVAL, "mean = %d: expected 0 or 1", mean);
    if (n_probes < 1 || n_probes > B2F_PAIR_MAX_PROBES) return set_err(B2F_EINVAL, "n_probes = %d: expected 1..%d", n_probes, B2F_PAIR_MAX_PROBES);
    int rc = check_walk_depth(m, "pair dependence walks");
    if (rc) return rc;
    const int fields = (int)(h.n_cat + h.n_num);
    int64_t total = 0;
    for (int i = 0; i < n_probes; ++i) {
        const b2f_pair_probe pr = probes[i];
        if (pr.word_a < 0 || pr.word_a >= fields) return set_err(B2F_EINVAL, "probe %d: word_a %d outside the %d fields", i, pr.word_a, fields);
        if (pr.word_b < -1 || pr.word_b >= fields) return set_err(B2F_EINVAL, "probe %d: word_b %d outside the %d fields (-1: one-way)", i, pr.word_b, fields);
        if (pr.word_b == pr.word_a) return set_err(B2F_EINVAL, "probe %d: word_a and word_b are both %d", i, pr.word_a);
        if (pr.count < 1 || pr.count > B2F_PAIR_MAX_POINTS) return set_err(B2F_EINVAL, "probe %d: %d points, expected 1..%d", i, pr.count, B2F_PAIR_MAX_POINTS);
        if (pr.point_offset < 0 || (int64_t)pr.point_offset > (int64_t)B2F_PAIR_MAX_PROBES * B2F_PAIR_MAX_POINTS - pr.count)
            return set_err(B2F_EINVAL, "probe %d: point offset %d out of range", i, pr.point_offset);
        total += pr.count;
    }
    if (!mean && total > B2F_PAIR_MAX_CURVE_POINTS)
        return set_err(B2F_EINVAL, "%lld points: the curves (mean = 0) take at most %d per row", (long long)total, B2F_PAIR_MAX_CURVE_POINTS);
    PairDependence &pp = m->pair;
    std::vector<PpSeg> segs;
    std::vector<uint32_t> words;
    words.reserve((size_t)total * 2);
    for (int i = 0; i < n_probes; ++i) {
        const b2f_pair_probe pr = probes[i];
        for (int k = 0; k < pr.count; ++k) {
            uint32_t a = point_words[2 * ((size_t)pr.point_offset + k)], b = point_words[2 * ((size_t)pr.point_offset + k) + 1];
            if ((rc = pp_point_word(h, i, k, pr.word_a, a))) return rc;
            if (pr.word_b >= 0 && (rc = pp_point_word(h, i, k, pr.word_b, b))) return rc;
            if (pr.word_b < 0) b = 0u;
            if (k % B2F_PD_SEG == 0)
                segs.push_back(PpSeg{(uint32_t)pr.word_a, pr.word_b < 0 ? B2F_PP_NO_WORD : (uint32_t)pr.word_b, 0u, (uint32_t)(words.size() / 2)});
            segs.back().count++;
            words.push_back(a);
            words.push_back(b);
        }
    }
    pp.n_segs = (int)segs.size();
    pp.points = total;
    pack_spec(pp.spec, segs, words);
    return B2F_OK;
}

/* the model's walk parameters with this call's point table at spec_dev */
static PdParams pp_params(const b2f_model *m, const void *spec_dev, const PpSeg **segs) {
    PdParams p = m->walk;
    *segs = static_cast<const PpSeg *>(spec_dev);
    p.grid = reinterpret_cast<const uint32_t *>(*segs + m->pair.n_segs);
    p.points = (int32_t)std::min<int64_t>(m->pair.points, INT_MAX);
    return p;
}

/* segments [s0, s1) of the spec at spec_dev over n device rows, launched in pieces of at most 65 535 segments (gridDim.y) */
static int pp_launch(b2f_model *m, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, bool mean, double *out_dev, const void *spec_dev,
                     int s0, int s1, int point0, int group_points) {
    const PpSeg *segs;
    const PdParams p = pp_params(m, spec_dev, &segs);
    const unsigned bx = (unsigned)((n + B2F_PD_WARPS * 32 - 1) / (B2F_PD_WARPS * 32));
    const uint32_t *rows = static_cast<const uint32_t *>(rows_dev);
    const bool packed = fmt == B2F_ROWS_PACKED64;
    for (int s = s0; s < s1; s += 65535) {
        const dim3 grid(bx, (unsigned)std::min(65535, s1 - s));
        if (mean) {
            if (packed) k_pair_dependence<true, true><<<grid, B2F_PD_WARPS * 32, 0, st>>>(p, segs + s, rows, (long long)n, out_dev, point0, group_points);
            else k_pair_dependence<false, true><<<grid, B2F_PD_WARPS * 32, 0, st>>>(p, segs + s, rows, (long long)n, out_dev, point0, group_points);
        } else {
            if (packed) k_pair_dependence<true, false><<<grid, B2F_PD_WARPS * 32, 0, st>>>(p, segs + s, rows, (long long)n, out_dev, 0, 0);
            else k_pair_dependence<false, false><<<grid, B2F_PD_WARPS * 32, 0, st>>>(p, segs + s, rows, (long long)n, out_dev, 0, 0);
        }
        const int rc = launched(m, "k_pair_dependence");
        if (rc) return rc;
    }
    return B2F_OK;
}

/* mean = 1 on the compute stream: n >= 1 device rows -> out_dev[P], the spec already at m->pair.spec_dev.  A group is a
 * run of whole segments of at most gp points, gp the most points whose partials (one double per CTA) fit the budget. */
static int pp_mean(b2f_model *m, const void *rows_dev, int64_t n, int fmt, double *out_dev) {
    PairDependence &pp = m->pair;
    const cudaStream_t st = m->compute;
    const int64_t n_cta = (n + B2F_PD_WARPS * 32 - 1) / (B2F_PD_WARPS * 32);
    const int64_t gp = std::min<int64_t>(pp.points, std::max<int64_t>(B2F_PD_SEG, B2F_PERM_SCRATCH_BYTES / (n_cta * (int64_t)sizeof(double))));
    int rc = compute_reserve(m, pp.partial, (size_t)(n_cta * gp) * sizeof(double), "pair dependence", "the per-CTA partial sums");
    if (rc) return rc;
    const PpSeg *segs = reinterpret_cast<const PpSeg *>(pp.spec.data());
    double *partial = static_cast<double *>(pp.partial.p);
    for (int s0 = 0; s0 < pp.n_segs;) {
        const int point0 = (int)segs[s0].off;
        int s1 = s0;
        while (s1 < pp.n_segs && (int64_t)segs[s1].off + segs[s1].count - point0 <= gp) ++s1;
        const int np = (int)(segs[s1 - 1].off + segs[s1 - 1].count - (uint32_t)point0);
        if ((rc = pp_launch(m, st, rows_dev, n, fmt, true, partial, pp.spec_dev.p, s0, s1, point0, np))) return rc;
        k_pair_dependence_finish<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(partial, (int)n_cta, np, (long long)n, out_dev + point0);
        if ((rc = launched(m, "k_pair_dependence_finish"))) return rc;
        s0 = s1;
    }
    return B2F_OK;
}

/* rows per chunk of the curves: a 64 MB output budget, a multiple of 32, at least 32 rows */
static int64_t pp_chunk_rows(const b2f_model *m) {
    const int64_t rows = B2F_PD_CHUNK_BYTES / (m->pair.points * (int64_t)sizeof(double));
    return std::max<int64_t>(32, std::min<int64_t>(B2F_CHUNK_ROWS, rows / 32 * 32));
}

extern "C" int b2f_pair_dependence(b2f_model *m, const void *rows, int64_t n, int row_format, const b2f_pair_probe *probes, int n_probes,
                                   const uint32_t *point_words, int mean, double *out, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (device_ms) *device_ms = 0.0f;
    int rc = pp_prepare(m, probes, n_probes, point_words, mean);
    if (rc) return rc;
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    if ((rc = pp_check(row_format, out || (n == 0 && !mean)))) return rc;
    if (!mean) {
        if (n > 0) {
            CUDA_TRY(cudaSetDevice(m->device));
            if ((rc = upload_spec(m, m->pair.host_spec, m->pair.spec, false, "pair dependence"))) return rc;
        }
        const HostJob job{(size_t)m->pair.points * sizeof(double), pp_chunk_rows(m), false, 0,
                          [](b2f_model *m, int, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, void *out_dev, int32_t *, DevBuf &) {
                              return pp_launch(m, st, rows_dev, n, fmt, false, static_cast<double *>(out_dev), m->pair.host_spec.p, 0,
                                               m->pair.n_segs, 0, 0);
                          }};
        return timed_host_batch(m, job, rows, n, row_format, out, device_ms);
    }
    if (n < 1 || n > (int64_t)INT_MAX) return set_err(B2F_EINVAL, "n = %lld: the mean needs 1 .. 2^31 - 1 rows", (long long)n);
    if (!rows) return set_err(B2F_EINVAL, "rows is NULL");
    if ((rc = check_row_format(m, row_format))) return rc;
    CUDA_TRY(cudaSetDevice(m->device));
    PairDependence &pp = m->pair;
    const cudaStream_t st = m->compute;
    const size_t row_bytes = row_bytes_of(m, row_format);
    if ((rc = compute_reserve(m, pp.rows, (size_t)n * row_bytes, "pair dependence", "the rows")) ||
        (rc = compute_reserve(m, pp.out, (size_t)pp.points * sizeof(double), "pair dependence", "the means")))
        return rc;
    TimedRegion timed{m, device_ms};
    if ((rc = timed.start())) return rc;
    if ((rc = upload_spec(m, pp.spec_dev, pp.spec, true, "pair dependence"))) return rc;
    CUDA_TRY(cudaMemcpyAsync(pp.rows.p, rows, (size_t)n * row_bytes, cudaMemcpyHostToDevice, st));
    if ((rc = pp_mean(m, pp.rows.p, n, row_format, static_cast<double *>(pp.out.p)))) return rc;
    CUDA_TRY(cudaMemcpyAsync(out, pp.out.p, (size_t)pp.points * sizeof(double), cudaMemcpyDeviceToHost, st));
    return timed.finish();
}

extern "C" int b2f_pair_dependence_device(b2f_model *m, const void *rows_dev, int64_t n, int row_format, const b2f_pair_probe *probes,
                                          int n_probes, const uint32_t *point_words, int mean, double *out_dev) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    int rc = pp_prepare(m, probes, n_probes, point_words, mean);
    if (rc == B2F_OK) rc = pp_check(row_format, out_dev != nullptr || (n == 0 && !mean));
    if (rc == B2F_OK) rc = check_row_format(m, row_format);
    if (rc) return rc;
    if (mean && (n < 1 || n > (int64_t)INT_MAX)) return set_err(B2F_EINVAL, "n = %lld: the mean needs 1 .. 2^31 - 1 rows", (long long)n);
    if (n == 0) return B2F_OK;
    CUDA_TRY(cudaSetDevice(m->device));
    if ((rc = upload_spec(m, m->pair.spec_dev, m->pair.spec, true, "pair dependence"))) return rc;
    if (mean) return pp_mean(m, rows_dev, n, row_format, out_dev);
    return pp_launch(m, m->compute, rows_dev, n, row_format, false, out_dev, m->pair.spec_dev.p, 0, m->pair.n_segs, 0, 0);
}
