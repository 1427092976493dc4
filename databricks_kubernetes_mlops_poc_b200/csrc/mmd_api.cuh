/*
 * mmd_api.cuh -- C ABI of the MMD drift test (include/b2f.h: b2f_model_attach_mmd_reference, b2f_mmd_drift); included by
 * b2f_api.cu.
 *
 * Host side of K9 (mmd_drift.cuh).  The reference's embedding, its kernel row sums r_ref (reference x reference, diagonal
 * excluded) and sigma stay on the device with the model; a call embeds its batch, completes the pool's row sums with the
 * reference x batch and batch x pool blocks, and sums each subset's pairs.  Every buffer is on the compute stream, grown on
 * demand and never shrunk.
 */
#pragma once

/* reserve with the failure reported as B2F_ENOMEM and its byte count */
static int mmd_reserve(b2f_model *m, DevBuf &b, size_t bytes, const char *what) {
    if (b.reserve(m->compute, bytes, bytes) == B2F_OK) return B2F_OK;
    (void)cudaGetLastError();
    return set_err(B2F_ENOMEM, "MMD drift: cannot allocate %zu device bytes for %s", bytes, what);
}

static int mmd_launched(b2f_model *m, const char *what) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_err(B2F_ECUDA, "%s launch failed: %s", what, cudaGetErrorString(e));
    m->launches++;
    return B2F_OK;
}

static int mmd_check_rows(b2f_model *m, const void *rows, int64_t n, int row_format, int64_t lo, int64_t hi, const char *what) {
    if (row_format == B2F_ROWS_RANKED)
        return set_err(B2F_EINVAL, "MMD drift takes float32 rows (B2F_ROWS_WORDS24 / B2F_ROWS_PACKED64): ranked rows carry no values");
    const int rc = check_row_format(m, row_format);
    if (rc) return rc;
    if (!rows) return set_err(B2F_EINVAL, "%s: rows is NULL", what);
    if (n < lo || n > hi) return set_err(B2F_EINVAL, "%s: n = %lld rows, expected %lld .. %lld", what, (long long)n, (long long)lo, (long long)hi);
    return B2F_OK;
}

/* the pair kernels' dynamic shared memory (up to 47 KB, beside the select's static histogram) */
static int mmd_smem_attr(const Mmd &md) {
    const int smem = (int)mmd_smem_bytes(md.mp.n_cat, md.mp.n_num);
    CUDA_TRY(cudaFuncSetAttribute(k_mmd_select_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CUDA_TRY(cudaFuncSetAttribute(k_mmd_row_sums, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CUDA_TRY(cudaFuncSetAttribute(k_mmd_subset_pairs, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    return B2F_OK;
}

/* upload n rows and embed them into z / c on the compute stream */
static int mmd_embed(b2f_model *m, const void *rows, int64_t n, int row_format, DevBuf &z, DevBuf &c) {
    Mmd &md = m->mmd;
    const size_t row_bytes = row_format == B2F_ROWS_PACKED64 ? B2F_PACKED_ROW_WORDS * 4 : B2F_ROW_WORDS * 4;
    int rc;
    if ((rc = mmd_reserve(m, md.rows, (size_t)n * row_bytes, "the rows")) ||
        (rc = mmd_reserve(m, z, std::max<size_t>((size_t)n * md.mp.n_num * 8, 8), "the numerics")) ||
        (rc = mmd_reserve(m, c, std::max<size_t>((size_t)n * md.mp.n_cat * 4, 4), "the categories")))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(md.rows.p, rows, (size_t)n * row_bytes, cudaMemcpyHostToDevice, m->compute));
    const unsigned grid = (unsigned)((n + 255) / 256);
    const uint32_t *d_rows = static_cast<const uint32_t *>(md.rows.p);
    if (row_format == B2F_ROWS_PACKED64)
        k_mmd_embed<true><<<grid, 256, 0, m->compute>>>(md.mp, d_rows, (long long)n, static_cast<double *>(z.p), static_cast<int32_t *>(c.p));
    else
        k_mmd_embed<false><<<grid, 256, 0, m->compute>>>(md.mp, d_rows, (long long)n, static_cast<double *>(z.p), static_cast<int32_t *>(c.p));
    return mmd_launched(m, "k_mmd_embed");
}

static MmdPool mmd_pool(const Mmd &md, int64_t n_ref) {
    return MmdPool{static_cast<const double *>(md.ref_z.p), static_cast<const int32_t *>(md.ref_c.p), static_cast<const double *>(md.z.p),
                   static_cast<const int32_t *>(md.c.p), (long long)n_ref, md.mp.n_cat, md.mp.n_num};
}

/* r[i] = base[i] + sum over pool columns [b_lo, b_hi) other than a_lo + i of k(a_lo + i, b), i < na */
static int mmd_row_sums(b2f_model *m, const MmdPool &P, int64_t a_lo, int64_t na, int64_t b_lo, int64_t b_hi, const double *base, double *r) {
    Mmd &md = m->mmd;
    const int64_t ch = (int64_t)B2F_MMD_CHUNK_TILES * B2F_MMD_TILE, chunks = (b_hi - b_lo + ch - 1) / ch;
    int rc;
    if ((rc = mmd_reserve(m, md.partial, (size_t)(chunks * na) * 8, "the row-sum partials"))) return rc;
    const size_t smem = mmd_smem_bytes(P.n_cat, P.n_num);
    const dim3 grid((unsigned)((na + B2F_MMD_TILE - 1) / B2F_MMD_TILE), (unsigned)chunks);
    k_mmd_row_sums<<<grid, B2F_MMD_TILE, smem, m->compute>>>(P, (long long)a_lo, (long long)na, (long long)b_lo, (long long)b_hi, md.coef,
                                                              static_cast<double *>(md.partial.p));
    if ((rc = mmd_launched(m, "k_mmd_row_sums"))) return rc;
    k_mmd_row_finish<<<(unsigned)((na + 255) / 256), 256, 0, m->compute>>>(static_cast<const double *>(md.partial.p), (int)chunks, (long long)na, base, r);
    return mmd_launched(m, "k_mmd_row_finish");
}

/* the k-th smallest (0-based) distance over the reference's n (n - 1) / 2 pairs: an exact radix select on the bits of the
 * non-negative doubles, B2F_MMD_DIGIT_BITS per pass, recomputing the distances on each pass */
static int mmd_select(b2f_model *m, const MmdPool &P, unsigned long long k, double *v) {
    Mmd &md = m->mmd;
    constexpr int BINS = 1 << B2F_MMD_DIGIT_BITS;
    int rc;
    if ((rc = mmd_reserve(m, md.hist, BINS * 8, "the select histogram"))) return rc;
    unsigned long long *d_hist = static_cast<unsigned long long *>(md.hist.p);
    const unsigned nt = (unsigned)((P.n_ref + B2F_MMD_TILE - 1) / B2F_MMD_TILE);
    const size_t smem = mmd_smem_bytes(P.n_cat, P.n_num);
    std::vector<unsigned long long> h(BINS);
    unsigned long long prefix = 0, mask = 0;
    for (int hi = 64; hi > 0; hi -= B2F_MMD_DIGIT_BITS) {
        const int shift = std::max(hi - B2F_MMD_DIGIT_BITS, 0), width = hi - shift;
        CUDA_TRY(cudaMemsetAsync(d_hist, 0, BINS * 8, m->compute));
        k_mmd_select_hist<<<dim3(nt, nt), B2F_MMD_TILE, smem, m->compute>>>(P, prefix, mask, shift, width, d_hist);
        if ((rc = mmd_launched(m, "k_mmd_select_hist"))) return rc;
        CUDA_TRY(cudaMemcpyAsync(h.data(), d_hist, BINS * 8, cudaMemcpyDeviceToHost, m->compute));
        CUDA_TRY(cudaStreamSynchronize(m->compute));
        int digit = 0;
        while (digit < (1 << width) && h[digit] <= k) k -= h[digit++];
        if (digit == (1 << width)) return set_err(B2F_ECUDA, "MMD sigma: the pair select lost its rank (pass at bit %d)", shift);
        prefix |= (unsigned long long)digit << shift;
        mask |= ((1ull << width) - 1ull) << shift;
    }
    memcpy(v, &prefix, 8);
    return B2F_OK;
}

extern "C" int b2f_model_attach_mmd_reference(b2f_model *m, const void *rows, int64_t n, int row_format, const double *num_mean,
                                              const double *num_scale, double sigma, double *sigma_out, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (device_ms) *device_ms = 0.0f;
    Mmd &md = m->mmd;
    md.n_ref = 0; /* replaced: no reference until this one is complete */
    int rc = mmd_check_rows(m, rows, n, row_format, 2, B2F_MMD_MAX_REF, "MMD reference");
    if (rc) return rc;
    const b2f_blob_header &h = m->hdr;
    const int n_num = (int)h.n_num;
    if (n_num > 0 && (!num_mean || !num_scale)) return set_err(B2F_EINVAL, "MMD reference: num_mean or num_scale is NULL");
    for (int k = 0; k < n_num; ++k)
        if (!std::isfinite(num_mean[k]) || !std::isfinite(num_scale[k]) || !(num_scale[k] > 0.0))
            return set_err(B2F_EINVAL, "MMD reference: numeric %d has mean %g and scale %g: expected finite, scale > 0", k, num_mean[k], num_scale[k]);
    if (!std::isnan(sigma) && !(std::isfinite(sigma) && sigma > 0.0))
        return set_err(B2F_EINVAL, "MMD reference: sigma = %g: expected a finite positive number, or NaN for the median heuristic", sigma);

    CUDA_TRY(cudaSetDevice(m->device));
    md.mp.n_cat = (int)h.n_cat, md.mp.n_num = n_num;
    memcpy(md.mp.impute, h.impute, sizeof(md.mp.impute));
    for (int k = 0; k < 24; ++k) md.mp.mean[k] = k < n_num ? num_mean[k] : 0.0, md.mp.scale[k] = k < n_num ? num_scale[k] : 1.0;
    if ((rc = mmd_smem_attr(md))) return rc;
    const cudaStream_t st = m->compute;
    Events evs;
    if (device_ms) {
        if ((rc = evs.create(2))) return rc;
        CUDA_TRY(cudaEventRecord(evs.e[0], st));
    }
    if ((rc = mmd_embed(m, rows, n, row_format, md.ref_z, md.ref_c))) return rc;
    const MmdPool P = mmd_pool(md, n);
    if (std::isnan(sigma)) {
        const unsigned long long pairs = (unsigned long long)n * (unsigned long long)(n - 1) / 2ull;
        double v = 0.0;
        if ((rc = mmd_select(m, P, (pairs - 1ull) / 2ull, &v))) return rc;
        if (!(v > 0.0))
            return set_err(B2F_EINVAL, "MMD reference: the median pair distance is 0 (more than half the pairs are equal rows); pass sigma");
        sigma = std::sqrt(0.5 * v);
    }
    md.sigma = sigma;
    md.coef = 1.0 / (2.0 * sigma * sigma);
    if ((rc = mmd_reserve(m, md.r_ref, (size_t)n * 8, "the reference row sums"))) return rc;
    if ((rc = mmd_row_sums(m, P, 0, n, 0, n, nullptr, static_cast<double *>(md.r_ref.p)))) return rc;
    if (device_ms) CUDA_TRY(cudaEventRecord(evs.e[1], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (device_ms) CUDA_TRY(cudaEventElapsedTime(device_ms, evs.e[0], evs.e[1]));
    md.n_ref = n;
    if (sigma_out) *sigma_out = sigma;
    return B2F_OK;
}

extern "C" int b2f_mmd_drift(b2f_model *m, const void *rows, int64_t n, int row_format, const int32_t *subsets, int n_perm, double *mmd2_obs,
                             double *mmd2_perm, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (device_ms) *device_ms = 0.0f;
    Mmd &md = m->mmd;
    if (md.n_ref == 0) return set_err(B2F_ESTATE, "MMD drift: no reference attached (b2f_model_attach_mmd_reference)");
    int rc = mmd_check_rows(m, rows, n, row_format, 2, (int64_t)INT_MAX - md.n_ref, "MMD drift");
    if (rc) return rc;
    if (n_perm < 1 || n_perm > B2F_MMD_MAX_PERM) return set_err(B2F_EINVAL, "MMD drift: n_perm = %d, expected 1..%d", n_perm, B2F_MMD_MAX_PERM);
    if (!subsets || !mmd2_obs || !mmd2_perm) return set_err(B2F_EINVAL, "MMD drift: subsets, mmd2_obs or mmd2_perm is NULL");
    const int64_t n_ref = md.n_ref, N = n_ref + n, s = std::min(n, n_ref);
    const bool u_is_batch = n <= n_ref;
    for (int64_t b = 0; b < n_perm; ++b) {
        const int32_t *u = subsets + b * s;
        for (int64_t p = 0; p < s; ++p) {
            if (u[p] < 0 || u[p] >= N)
                return set_err(B2F_EINVAL, "MMD drift: subsets[%lld][%lld] = %d is outside the pool [0, %lld)", (long long)b, (long long)p, u[p], (long long)N);
            if (p > 0 && u[p] <= u[p - 1])
                return set_err(B2F_EINVAL, "MMD drift: subset %lld is not strictly increasing at %lld (sorted, no repeats)", (long long)b, (long long)p);
        }
    }

    CUDA_TRY(cudaSetDevice(m->device));
    if ((rc = mmd_smem_attr(md))) return rc;
    const cudaStream_t st = m->compute;
    const int64_t sets = (int64_t)n_perm + 1; /* subset 0: the observed split (the batch, or the reference when n > n_ref) */
    const int64_t nt = (s + B2F_MMD_TILE - 1) / B2F_MMD_TILE;
    if ((rc = mmd_reserve(m, md.r, (size_t)N * 8, "the pool row sums")) || (rc = mmd_reserve(m, md.sub, (size_t)(sets * s) * 4, "the subsets")) ||
        (rc = mmd_reserve(m, md.pairs, (size_t)(sets * nt * nt) * 8, "the subset tile sums")) ||
        (rc = mmd_reserve(m, md.out, (size_t)sets * 8, "the statistics")))
        return rc;
    Events evs;
    if (device_ms) {
        if ((rc = evs.create(2))) return rc;
        CUDA_TRY(cudaEventRecord(evs.e[0], st));
    }
    if ((rc = mmd_embed(m, rows, n, row_format, md.z, md.c))) return rc;
    std::vector<int32_t> obs((size_t)s);
    for (int64_t p = 0; p < s; ++p) obs[p] = (int32_t)(u_is_batch ? n_ref + p : p);
    int32_t *d_sub = static_cast<int32_t *>(md.sub.p);
    CUDA_TRY(cudaMemcpyAsync(d_sub, obs.data(), (size_t)s * 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(d_sub + s, subsets, (size_t)(n_perm * s) * 4, cudaMemcpyHostToDevice, st));
    const MmdPool P = mmd_pool(md, n_ref);
    double *d_r = static_cast<double *>(md.r.p);
    /* reference rows: r_ref plus the batch columns; batch rows: every pool column but their own */
    if ((rc = mmd_row_sums(m, P, 0, n_ref, n_ref, N, static_cast<const double *>(md.r_ref.p), d_r)) ||
        (rc = mmd_row_sums(m, P, n_ref, n, 0, N, nullptr, d_r + n_ref)))
        return rc;
    const size_t smem = mmd_smem_bytes(P.n_cat, P.n_num);
    double *d_pairs = static_cast<double *>(md.pairs.p);
    for (int64_t z0 = 0; z0 < sets; z0 += 65535) { /* gridDim.z <= 65535 */
        const unsigned nz = (unsigned)std::min<int64_t>(65535, sets - z0);
        k_mmd_subset_pairs<<<dim3((unsigned)nt, (unsigned)nt, nz), B2F_MMD_TILE, smem, st>>>(P, d_sub + z0 * s, (long long)s, (int)nt, md.coef,
                                                                                              d_pairs + z0 * nt * nt);
        if ((rc = mmd_launched(m, "k_mmd_subset_pairs"))) return rc;
    }
    k_mmd_finish<<<(unsigned)sets, B2F_MMD_FINISH_THREADS, 0, st>>>(d_r, (long long)N, d_sub, (long long)s, d_pairs, (int)nt, (long long)n_ref,
                                                                    (long long)n, u_is_batch ? 1 : 0, static_cast<double *>(md.out.p));
    if ((rc = mmd_launched(m, "k_mmd_finish"))) return rc;
    std::vector<double> res((size_t)sets);
    CUDA_TRY(cudaMemcpyAsync(res.data(), md.out.p, (size_t)sets * 8, cudaMemcpyDeviceToHost, st));
    if (device_ms) CUDA_TRY(cudaEventRecord(evs.e[1], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (device_ms) CUDA_TRY(cudaEventElapsedTime(device_ms, evs.e[0], evs.e[1]));
    *mmd2_obs = res[0];
    memcpy(mmd2_perm, res.data() + 1, (size_t)n_perm * 8);
    return B2F_OK;
}
