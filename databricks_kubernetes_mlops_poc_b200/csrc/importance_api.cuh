/*
 * importance_api.cuh -- C ABI of permutation importance (include/b2f.h: b2f_permutation_scores); included by b2f_api.cu.
 *
 * Host side of K8 (permutation_importance.cuh).  Not a job of the host pipeline: a row's points read other rows and the
 * ROC AUC needs a whole point at once, so one call uploads its rows, labels and permutations once, on the compute
 * stream, into buffers the model owns (grown on demand, never shrunk), and scores its points in groups whose keys, flags
 * and sort scratch stay under B2F_PERM_SCRATCH_BYTES.  Only the records come back.
 *
 * Points: 0 = the baseline (every row as it is), 1 + f * n_repeats + r = probed word f under permutation r.  A group is a
 * run of consecutive points; its segments (PiSeg) split each probe's repeats in the group into runs of up to 32.
 */
#pragma once

/* segmented_sort.cu */
cudaError_t pi_segmented_sort(void *temp, size_t *temp_bytes, unsigned long long *k0, unsigned long long *k1, uint8_t *f0, uint8_t *f1,
                              int items, int segs, const int *off, cudaStream_t st, int *current);

static_assert(sizeof(struct b2f_perm_score) == 64 && offsetof(struct b2f_perm_score, log_loss_sum) == 32 &&
                  offsetof(struct b2f_perm_score, auc_u2) == 48,
              "b2f_perm_score layout");
static_assert(sizeof(PiScore) == sizeof(struct b2f_perm_score) && offsetof(PiScore, auc_u2) == offsetof(struct b2f_perm_score, auc_u2),
              "PiScore layout");

/* reserve with the failure reported as B2F_ENOMEM and its byte count */
static int pi_reserve(b2f_model *m, DevBuf &b, size_t bytes, const char *what) {
    if (b.reserve(m->compute, bytes, bytes) == B2F_OK) return B2F_OK;
    (void)cudaGetLastError();
    return set_err(B2F_ENOMEM, "permutation scores: cannot allocate %zu device bytes for %s", bytes, what);
}

/* points of one group: the most whose keys, flags and their sort copies (18 bytes per row) fit the budget, at least one */
static int64_t pi_group_points(int64_t n, int64_t points) {
    const int64_t fit = std::max<int64_t>(1, B2F_PERM_SCRATCH_BYTES / (18 * n));
    return std::min<int64_t>({points, fit, (int64_t)INT_MAX / n});
}

extern "C" int b2f_permutation_scores(b2f_model *m, const void *rows, int64_t n, int row_format, const int32_t *labels, const int32_t *perm,
                                      int n_repeats, const int32_t *words, int n_words, struct b2f_perm_score *out,
                                      struct b2f_perm_score *baseline, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (device_ms) *device_ms = 0.0f;
    const b2f_blob_header &h = m->hdr;
    if (row_format == B2F_ROWS_RANKED)
        return set_err(B2F_EINVAL, "permutation scores take float32 rows (B2F_ROWS_WORDS24 / B2F_ROWS_PACKED64): ranked rows carry no values");
    int rc = check_row_format(m, row_format);
    if (rc) return rc;
    if (n < 1 || n > (int64_t)INT_MAX) return set_err(B2F_EINVAL, "n = %lld: expected 1 .. 2^31 - 1 rows", (long long)n);
    if (!rows || !labels || !perm || !words || !out || !baseline) return set_err(B2F_EINVAL, "rows, labels, perm, words, out or baseline is NULL");
    if (n_repeats < 1 || n_repeats > B2F_PERM_MAX_REPEATS) return set_err(B2F_EINVAL, "n_repeats = %d: expected 1..%d", n_repeats, B2F_PERM_MAX_REPEATS);
    const int fields = (int)(h.n_cat + h.n_num);
    if (n_words < 1 || n_words > fields) return set_err(B2F_EINVAL, "n_words = %d: expected 1..%d", n_words, fields);
    for (int i = 0; i < n_words; ++i)
        if (words[i] < 0 || words[i] >= fields) return set_err(B2F_EINVAL, "words[%d] = %d: outside the %d fields", i, words[i], fields);
    if (h.max_depth > B2F_PD_STACK)
        return set_err(B2F_EINVAL, "permutation scores walk trees of depth <= %d; this forest has depth %u", B2F_PD_STACK, h.max_depth);
    for (int64_t i = 0; i < n; ++i)
        if (labels[i] != 0 && labels[i] != 1) return set_err(B2F_EINVAL, "labels[%lld] = %d: expected 0 or 1", (long long)i, labels[i]);
    const int64_t perm_n = (int64_t)n_repeats * n;
    for (int64_t i = 0; i < perm_n; ++i)
        if (perm[i] < 0 || (int64_t)perm[i] >= n)
            return set_err(B2F_EINVAL, "perm[%lld] = %d (repeat %lld): not a row index in [0, %lld)", (long long)i, perm[i], (long long)(i / n), (long long)n);

    CUDA_TRY(cudaSetDevice(m->device));
    Importance &pi = m->pi;
    const cudaStream_t st = m->compute;
    const size_t row_bytes = row_format == B2F_ROWS_PACKED64 ? B2F_PACKED_ROW_WORDS * 4 : B2F_ROW_WORDS * 4;
    const int64_t points = 1 + (int64_t)n_words * n_repeats, gp = pi_group_points(n, points);
    if ((rc = pi_reserve(m, pi.rows, (size_t)n * row_bytes, "the rows")) || (rc = pi_reserve(m, pi.labels, (size_t)n, "the labels")) ||
        (rc = pi_reserve(m, pi.perm, (size_t)perm_n * 4, "the permutations")) ||
        (rc = pi_reserve(m, pi.keys, (size_t)gp * n * 16, "the ranking keys")) || (rc = pi_reserve(m, pi.flags, (size_t)gp * n * 2, "the flags")) ||
        (rc = pi_reserve(m, pi.scores, (size_t)gp * sizeof(PiScore), "the records")) ||
        (rc = pi_reserve(m, pi.offsets, (size_t)(gp + 1) * 4, "the segment offsets")) ||
        (rc = pi_reserve(m, pi.segs, (size_t)(gp + 2) * sizeof(PiSeg), "the segments")))
        return rc;
    uint8_t *d_labels = static_cast<uint8_t *>(pi.labels.p);
    unsigned long long *k0 = static_cast<unsigned long long *>(pi.keys.p), *k1 = k0 + gp * n;
    uint8_t *f0 = static_cast<uint8_t *>(pi.flags.p), *f1 = f0 + gp * n;
    PiScore *d_scores = static_cast<PiScore *>(pi.scores.p);
    int *d_off = static_cast<int *>(pi.offsets.p);
    /* the sort's temporary storage for the largest group */
    size_t temp_bytes = 0;
    CUDA_TRY(pi_segmented_sort(nullptr, &temp_bytes, k0, k1, f0, f1, (int)(gp * n), (int)gp, d_off, st, nullptr));
    if ((rc = pi_reserve(m, pi.temp, std::max<size_t>(temp_bytes, 1), "the sort's temporary storage"))) return rc;
    const size_t smem = pi_smem_bytes((int)h.max_depth);
    CUDA_TRY(cudaFuncSetAttribute(k_permutation_scores<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(cudaFuncSetAttribute(k_permutation_scores<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));

    Events evs;
    if (device_ms) {
        if ((rc = evs.create(2))) return rc;
        CUDA_TRY(cudaEventRecord(evs.e[0], st));
    }
    CUDA_TRY(cudaMemcpyAsync(pi.rows.p, rows, (size_t)n * row_bytes, cudaMemcpyHostToDevice, st));
    std::vector<uint8_t> lab8((size_t)n);
    for (int64_t i = 0; i < n; ++i) lab8[i] = (uint8_t)labels[i];
    CUDA_TRY(cudaMemcpyAsync(d_labels, lab8.data(), (size_t)n, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(pi.perm.p, perm, (size_t)perm_n * 4, cudaMemcpyHostToDevice, st));
    std::vector<int> off((size_t)gp + 1);
    for (int64_t p = 0; p <= gp; ++p) off[p] = (int)(p * n);
    CUDA_TRY(cudaMemcpyAsync(d_off, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice, st));

    std::vector<PiScore> res((size_t)points);
    const PdParams &pp = m->pd.pp; /* the forest fields (segs, grid and points unused) */
    const uint32_t *d_rows = static_cast<const uint32_t *>(pi.rows.p);
    const int32_t *d_perm = static_cast<const int32_t *>(pi.perm.p);
    const unsigned bx = (unsigned)((n + B2F_PD_WARPS * 32 - 1) / (B2F_PD_WARPS * 32));
    std::vector<PiSeg> segs;
    for (int64_t g0 = 0; g0 < points; g0 += gp) {
        const int64_t g1 = std::min(points, g0 + gp), np = g1 - g0;
        segs.clear();
        for (int64_t q = g0; q < g1;) { /* q: global point */
            PiSeg s;
            if (q == 0) {
                s = PiSeg{B2F_PI_NO_WORD, 0u, 1u, 0u};
            } else {
                const int64_t f = (q - 1) / n_repeats, r = (q - 1) % n_repeats;
                const int64_t c = std::min<int64_t>({(int64_t)B2F_PD_SEG, n_repeats - r, g1 - q});
                s = PiSeg{(uint32_t)words[f], (uint32_t)r, (uint32_t)c, (uint32_t)(q - g0)};
            }
            segs.push_back(s);
            q += s.count;
        }
        CUDA_TRY(cudaMemcpyAsync(pi.segs.p, segs.data(), segs.size() * sizeof(PiSeg), cudaMemcpyHostToDevice, st));
        const PiSeg *d_segs = static_cast<const PiSeg *>(pi.segs.p);
        for (size_t s = 0; s < segs.size(); s += 65535) { /* gridDim.y <= 65535 */
            const dim3 grid(bx, (unsigned)std::min<size_t>(65535, segs.size() - s));
            if (row_format == B2F_ROWS_PACKED64)
                k_permutation_scores<true><<<grid, B2F_PD_WARPS * 32, smem, st>>>(pp, d_segs + s, d_rows, d_labels, d_perm, (long long)n, k0, f0);
            else
                k_permutation_scores<false><<<grid, B2F_PD_WARPS * 32, smem, st>>>(pp, d_segs + s, d_rows, d_labels, d_perm, (long long)n, k0, f0);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) return set_err(B2F_ECUDA, "k_permutation_scores launch failed: %s", cudaGetErrorString(e));
            m->launches++;
        }
        k_permutation_metrics<<<(unsigned)np, B2F_PI_METRIC_THREADS, 0, st>>>(pp, k0, f0, (long long)n, d_scores);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return set_err(B2F_ECUDA, "k_permutation_metrics launch failed: %s", cudaGetErrorString(e));
        m->launches++;
        size_t tb = pi.temp.bytes;
        int cur = 0;
        CUDA_TRY(pi_segmented_sort(pi.temp.p, &tb, k0, k1, f0, f1, (int)(np * n), (int)np, d_off, st, &cur));
        k_permutation_auc<<<(unsigned)np, B2F_PI_METRIC_THREADS, 0, st>>>(cur ? k1 : k0, cur ? f1 : f0, (long long)n, d_scores);
        e = cudaGetLastError();
        if (e != cudaSuccess) return set_err(B2F_ECUDA, "k_permutation_auc launch failed: %s", cudaGetErrorString(e));
        m->launches++;
        CUDA_TRY(cudaMemcpyAsync(res.data() + g0, d_scores, (size_t)np * sizeof(PiScore), cudaMemcpyDeviceToHost, st));
    }
    if (device_ms) CUDA_TRY(cudaEventRecord(evs.e[1], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (device_ms) CUDA_TRY(cudaEventElapsedTime(device_ms, evs.e[0], evs.e[1]));
    memcpy(baseline, res.data(), sizeof(PiScore));
    memcpy(out, res.data() + 1, (size_t)(points - 1) * sizeof(PiScore));
    return B2F_OK;
}
