/*
 * ale_api.cuh -- C ABI of accumulated local effects (include/b2f.h: b2f_ale*); included by b2f_api.cu.
 *
 * Host side of K12 (ale.cuh).  A call's probes become one spec: the AleSeg table (probes sorted by word, up to
 * B2F_ALE_SEG_PROBES per segment), then the call's float32 edges, each probe's K + 1 in probe order.  Everything runs on
 * the compute stream: the host form copies the rows once into a buffer the model keeps; the rows go through k_ale in
 * pieces of whole CTAs whose per-CTA partials stay under B2F_PERM_SCRATCH_BYTES, each piece followed by k_ale_finish,
 * which adds its partials to the running per-bin sums.
 */
#pragma once

static_assert(sizeof(b2f_ale_probe) == 12, "b2f_ale_probe layout");
static_assert(sizeof(AleSeg) % sizeof(uint32_t) == 0, "AleSeg packs into a spec");

static int ale_prepare(b2f_model *m, const b2f_ale_probe *probes, int n_probes, const float *edges) {
    const b2f_blob_header &h = m->hdr;
    if (!probes || !edges) return set_err(B2F_EINVAL, "probes or edges is NULL");
    if (n_probes < 1 || n_probes > (int)h.n_num) return set_err(B2F_EINVAL, "n_probes = %d: expected 1..%u (the numeric fields)", n_probes, h.n_num);
    int rc = check_walk_depth(m, "accumulated local effects walk");
    if (rc) return rc;
    const int lo_word = (int)h.n_cat, hi_word = (int)(h.n_cat + h.n_num);
    uint32_t seen = 0u;
    for (int i = 0; i < n_probes; ++i) {
        const b2f_ale_probe pr = probes[i];
        if (pr.word < lo_word || pr.word >= hi_word)
            return set_err(B2F_EINVAL, "probe %d: row word %d is not a numeric field (%d..%d): ALE needs an ordered field", i, pr.word, lo_word, hi_word - 1);
        if ((seen >> pr.word) & 1u) return set_err(B2F_EINVAL, "probe %d: row word %d is probed twice", i, pr.word);
        seen |= 1u << pr.word;
        if (pr.bins < 1 || pr.bins > B2F_ALE_MAX_BINS) return set_err(B2F_EINVAL, "probe %d: %d bins, expected 1..%d", i, pr.bins, B2F_ALE_MAX_BINS);
        if (pr.edge_offset < 0 || pr.edge_offset > B2F_ALE_MAX_EDGES - (pr.bins + 1))
            return set_err(B2F_EINVAL, "probe %d: edge offset %d out of range", i, pr.edge_offset);
        const float *z = edges + pr.edge_offset;
        for (int e = 0; e <= pr.bins; ++e) {
            if (!std::isfinite(z[e])) return set_err(B2F_ERANGE, "probe %d edge %d is not a finite number", i, e);
            if (e > 0 && !(z[e - 1] < z[e])) return set_err(B2F_EINVAL, "probe %d: edges %d and %d are not strictly increasing", i, e - 1, e);
        }
    }
    std::vector<int> order(n_probes);
    for (int i = 0; i < n_probes; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](int a, int b) { return probes[a].word < probes[b].word; });
    std::vector<uint32_t> boff(n_probes), eoff(n_probes);
    uint32_t bins = 0, n_edges = 0;
    for (int i = 0; i < n_probes; ++i) {
        boff[i] = bins, eoff[i] = n_edges;
        bins += (uint32_t)probes[i].bins;
        n_edges += (uint32_t)probes[i].bins + 1u;
    }
    std::vector<AleSeg> segs;
    for (int k = 0; k < n_probes; ++k) {
        const int i = order[k];
        if (k % B2F_ALE_SEG_PROBES == 0) segs.push_back(AleSeg{});
        AleSeg &s = segs.back();
        s.p[s.count++] = AleProbe{(uint32_t)probes[i].word, eoff[i], (uint32_t)probes[i].bins, boff[i]};
        s.words |= 1u << probes[i].word;
        s.bins += (uint32_t)probes[i].bins;
    }
    std::vector<uint32_t> words;
    words.reserve(n_edges);
    for (int i = 0; i < n_probes; ++i)
        for (int e = 0; e <= probes[i].bins; ++e) {
            uint32_t w;
            memcpy(&w, edges + probes[i].edge_offset + e, sizeof(w));
            words.push_back(w);
        }
    Ale &a = m->ale;
    a.n_segs = (int)segs.size();
    a.bins = (int)bins;
    pack_spec(a.spec, segs, words);
    return B2F_OK;
}

/* n >= 1 device rows on the compute stream -> sums_dev / counts_dev [a.bins]; the spec already at m->ale.spec_dev.  A piece
 * is the most whole CTAs whose partials (a double and a count per bin) fit the budget. */
static int ale_run(b2f_model *m, const void *rows_dev, int64_t n, int fmt, double *sums_dev, long long *counts_dev) {
    Ale &a = m->ale;
    const cudaStream_t st = m->compute;
    constexpr int64_t rows_per_cta = B2F_PD_WARPS * 32;
    const int64_t n_cta = (n + rows_per_cta - 1) / rows_per_cta;
    const int64_t per_cta = (int64_t)a.bins * (int64_t)(sizeof(double) + sizeof(uint32_t));
    const int64_t piece = std::min<int64_t>(n_cta, std::max<int64_t>(1, B2F_PERM_SCRATCH_BYTES / per_cta));
    int rc;
    if ((rc = compute_reserve(m, a.psum, (size_t)(piece * a.bins) * sizeof(double), "accumulated local effects", "the per-CTA sums")) ||
        (rc = compute_reserve(m, a.pcnt, (size_t)(piece * a.bins) * sizeof(uint32_t), "accumulated local effects", "the per-CTA counts")))
        return rc;
    PdParams p = m->walk;
    const AleSeg *segs = static_cast<const AleSeg *>(a.spec_dev.p);
    const float *edges = reinterpret_cast<const float *>(segs + a.n_segs);
    const bool packed = fmt == B2F_ROWS_PACKED64;
    const size_t row_words = packed ? B2F_PACKED_ROW_WORDS : B2F_ROW_WORDS;
    double *psum = static_cast<double *>(a.psum.p);
    uint32_t *pcnt = static_cast<uint32_t *>(a.pcnt.p);
    for (int64_t c0 = 0; c0 < n_cta; c0 += piece) {
        const int64_t c1 = std::min(n_cta, c0 + piece);
        const int64_t r0 = c0 * rows_per_cta, nr = std::min(n, c1 * rows_per_cta) - r0;
        const uint32_t *rows = static_cast<const uint32_t *>(rows_dev) + (size_t)r0 * row_words;
        const dim3 grid((unsigned)(c1 - c0), (unsigned)a.n_segs);
        if (packed) k_ale<true><<<grid, rows_per_cta, 0, st>>>(p, segs, edges, rows, (long long)nr, a.bins, psum, pcnt);
        else k_ale<false><<<grid, rows_per_cta, 0, st>>>(p, segs, edges, rows, (long long)nr, a.bins, psum, pcnt);
        if ((rc = launched(m, "k_ale"))) return rc;
        k_ale_finish<<<(unsigned)((a.bins + 255) / 256), 256, 0, st>>>(psum, pcnt, (int)(c1 - c0), a.bins, c0 == 0, sums_dev, counts_dev);
        if ((rc = launched(m, "k_ale_finish"))) return rc;
    }
    return B2F_OK;
}

static int ale_check(b2f_model *m, int64_t n, int fmt) {
    int rc = check_value_rows(fmt, "accumulated local effects take");
    if (rc) return rc;
    if (n < 1) return set_err(B2F_EINVAL, "n = %lld: expected at least 1 row", (long long)n);
    return check_row_format(m, fmt);
}

extern "C" int b2f_ale(b2f_model *m, const void *rows, int64_t n, int row_format, const b2f_ale_probe *probes, int n_probes, const float *edges,
                       double *bin_sums, int64_t *bin_rows, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (device_ms) *device_ms = 0.0f;
    int rc = ale_prepare(m, probes, n_probes, edges);
    if (rc) return rc;
    if ((rc = ale_check(m, n, row_format))) return rc;
    if (!rows || !bin_sums || !bin_rows) return set_err(B2F_EINVAL, "rows, bin_sums or bin_rows is NULL");
    CUDA_TRY(cudaSetDevice(m->device));
    Ale &a = m->ale;
    const cudaStream_t st = m->compute;
    const size_t row_bytes = row_bytes_of(m, row_format);
    if ((rc = compute_reserve(m, a.rows, (size_t)n * row_bytes, "accumulated local effects", "the rows")) ||
        (rc = compute_reserve(m, a.sums, (size_t)a.bins * sizeof(double), "accumulated local effects", "the bin sums")) ||
        (rc = compute_reserve(m, a.counts, (size_t)a.bins * sizeof(long long), "accumulated local effects", "the bin counts")))
        return rc;
    TimedRegion timed{m, device_ms};
    if ((rc = timed.start())) return rc;
    if ((rc = upload_spec(m, a.spec_dev, a.spec, true, "accumulated local effects"))) return rc;
    CUDA_TRY(cudaMemcpyAsync(a.rows.p, rows, (size_t)n * row_bytes, cudaMemcpyHostToDevice, st));
    if ((rc = ale_run(m, a.rows.p, n, row_format, static_cast<double *>(a.sums.p), static_cast<long long *>(a.counts.p)))) return rc;
    CUDA_TRY(cudaMemcpyAsync(bin_sums, a.sums.p, (size_t)a.bins * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(bin_rows, a.counts.p, (size_t)a.bins * sizeof(long long), cudaMemcpyDeviceToHost, st));
    return timed.finish();
}

extern "C" int b2f_ale_device(b2f_model *m, const void *rows_dev, int64_t n, int row_format, const b2f_ale_probe *probes, int n_probes,
                              const float *edges, double *bin_sums_dev, int64_t *bin_rows_dev) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    int rc = ale_prepare(m, probes, n_probes, edges);
    if (rc) return rc;
    if ((rc = ale_check(m, n, row_format))) return rc;
    if (!rows_dev || !bin_sums_dev || !bin_rows_dev) return set_err(B2F_EINVAL, "rows_dev, bin_sums_dev or bin_rows_dev is NULL");
    CUDA_TRY(cudaSetDevice(m->device));
    if ((rc = upload_spec(m, m->ale.spec_dev, m->ale.spec, true, "accumulated local effects"))) return rc;
    return ale_run(m, rows_dev, n, row_format, bin_sums_dev, reinterpret_cast<long long *>(bin_rows_dev));
}
