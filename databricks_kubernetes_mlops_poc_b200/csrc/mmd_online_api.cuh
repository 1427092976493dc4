/*
 * mmd_online_api.cuh -- C ABI of the online MMD drift detector (include/b2f.h: b2f_mmd_online_*); included by b2f_api.cu.
 *
 * Host side of K13 (mmd_online.cuh) on the attached MMD reference (K9: its embedding, sigma and r_ref).
 *   bootstrap: the statistic of every window position of n_boot bootstrap sequences, in slices whose band prefixes stay
 *              under B2F_PERM_SCRATCH_BYTES.
 *   configure: K_RR of the split (the bootstrap form on y = perm[rw:]), the compacted sub-reference perm[:rw], and the
 *              window state: the initial window's last W - 1 rows (perm[n_ref - W + 1:]), their embedding and their c from
 *              k_mmd_row_sums against the sub-reference.  A copy is kept for reset.
 *   push:      per piece, the piece's rows are embedded, their c computed the same way, and the sequence [carried W - 1
 *              rows; piece] gets its band prefixes and one statistic per row; its last W - 1 rows become the state.  The
 *              carried rows' prefixes are recomputed from the rows, which gives the same bits, so nothing else is carried.
 * Every buffer is on the compute stream, grown on demand and never shrunk.
 */
#pragma once

/* window in 2 .. B2F_MMD_ONLINE_MAX_WINDOW and n_ref >= 2W + 1 */
static int online_check_window(const Mmd &md, int window, const char *what) {
    if (window < 2 || window > B2F_MMD_ONLINE_MAX_WINDOW)
        return set_err(B2F_EINVAL, "%s: window = %d, expected 2..%d", what, window, B2F_MMD_ONLINE_MAX_WINDOW);
    if (md.ref.n_ref < 2LL * window + 1)
        return set_err(B2F_EINVAL, "%s: window %d needs a reference of at least 2W + 1 = %d rows; it has %lld", what, window, 2 * window + 1,
                       (long long)md.ref.n_ref);
    return B2F_OK;
}

/* every one of n_seq sequences of len positions lies in [0, n_ref) with no position twice */
static int online_check_positions(const int32_t *p, int64_t n_seq, int64_t len, int64_t n_ref, const char *what) {
    std::vector<int64_t> seen((size_t)n_ref, -1);
    for (int64_t b = 0; b < n_seq; ++b)
        for (int64_t s = 0; s < len; ++s) {
            const int32_t v = p[b * len + s];
            if (v < 0 || v >= n_ref)
                return set_err(B2F_EINVAL, "%s: position [%lld][%lld] = %d is outside the reference [0, %lld)", what, (long long)b, (long long)s, v,
                               (long long)n_ref);
            if (seen[v] == b) return set_err(B2F_EINVAL, "%s: position %d appears twice in sequence %lld", what, v, (long long)b);
            seen[v] = b;
        }
    return B2F_OK;
}

static int online_smem_attr(const Mmd &md) {
    const int smem = (int)mmd_smem_bytes(md.ref.mp.n_cat, md.ref.mp.n_num);
    CUDA_TRY(set_smem_limit(k_mmd_online_band<true>, smem));
    CUDA_TRY(set_smem_limit(k_mmd_online_band<false>, smem));
    return B2F_OK;
}

/* T = sum of r_ref into o.total */
static int online_total(b2f_model *m) {
    Mmd &md = m->mmd;
    int rc;
    if ((rc = compute_reserve(m, md.online.total, 8, "online MMD drift", "the reference total"))) return rc;
    k_mmd_online_total<<<1, B2F_MMD_ONLINE_THREADS, 0, m->compute>>>(static_cast<const double *>(md.r_ref.p), (long long)md.ref.n_ref,
                                                                     static_cast<double *>(md.online.total.p));
    return launched(m, "k_mmd_online_total");
}

/* stats (n_boot x W) and k_rr (n_boot) of n_boot bootstrap sequences of E = 2W - 1 reference positions (host memory), on
 * the compute stream; the caller has checked the positions and set the smem limits and o.total */
static int online_boot(b2f_model *m, const int32_t *etw, int64_t n_boot, int W, double *stats, double *k_rr) {
    Mmd &md = m->mmd;
    MmdOnline &o = md.online;
    const cudaStream_t st = m->compute;
    const int64_t E = 2LL * W - 1, rw = md.ref.n_ref - E;
    const int64_t per = E * 4 + (int64_t)W * E * 8 + 2 * E * 8 + (int64_t)W * 8 + 8;
    const int64_t slice = std::min<int64_t>({n_boot, 65535, std::max<int64_t>(1, (int64_t)B2F_PERM_SCRATCH_BYTES / per)});
    const char *who = "online MMD drift";
    int rc;
    if ((rc = compute_reserve(m, o.pos, (size_t)(slice * E) * 4, who, "the bootstrap positions")) ||
        (rc = compute_reserve(m, o.band, (size_t)(slice * W * E) * 8, who, "the band prefixes")) ||
        (rc = compute_reserve(m, o.qsum, (size_t)(slice * E) * 8, who, "the in-sequence row sums")) ||
        (rc = compute_reserve(m, o.cv, (size_t)(slice * E) * 8, who, "the sub-reference row sums")) ||
        (rc = compute_reserve(m, o.stats, (size_t)(slice * W) * 8, who, "the bootstrap statistics")) ||
        (rc = compute_reserve(m, o.krr, (size_t)slice * 8, who, "the bootstrap K_RR")))
        return rc;
    const MmdPool P = ref_pool(md.ref, md.ref.n_ref);
    const size_t smem = mmd_smem_bytes(P.n_cat, P.n_num);
    const double *d_r = static_cast<const double *>(md.r_ref.p);
    int32_t *d_pos = static_cast<int32_t *>(o.pos.p);
    double *d_band = static_cast<double *>(o.band.p), *d_q = static_cast<double *>(o.qsum.p), *d_c = static_cast<double *>(o.cv.p);
    for (int64_t b0 = 0; b0 < n_boot; b0 += slice) {
        const int64_t nb = std::min(slice, n_boot - b0);
        CUDA_TRY(cudaMemcpyAsync(d_pos, etw + b0 * E, (size_t)(nb * E) * 4, cudaMemcpyHostToDevice, st));
        const dim3 grid((unsigned)((E + B2F_MMD_TILE - 1) / B2F_MMD_TILE), (unsigned)nb);
        k_mmd_online_band<true><<<grid, B2F_MMD_TILE, smem, st>>>(P, d_pos, (long long)E, W, md.coef, d_r, d_band, d_q, d_c);
        if ((rc = launched(m, "k_mmd_online_band"))) return rc;
        k_mmd_online_boot<<<(unsigned)nb, B2F_MMD_ONLINE_THREADS, 0, st>>>(d_r, d_pos, static_cast<const double *>(o.total.p), d_q, d_c, d_band, W,
                                                                          (long long)rw, static_cast<double *>(o.stats.p),
                                                                          static_cast<double *>(o.krr.p));
        if ((rc = launched(m, "k_mmd_online_boot"))) return rc;
        CUDA_TRY(cudaMemcpyAsync(stats + b0 * W, o.stats.p, (size_t)(nb * W) * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(k_rr + b0, o.krr.p, (size_t)nb * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st)); /* the next slice overwrites the positions and the results */
    }
    return B2F_OK;
}

/* rows idx[0 .. n) of the reference's embedding into z / c */
static int online_gather(b2f_model *m, const int32_t *idx, int64_t n, DevBuf &z, DevBuf &c, const char *what) {
    Mmd &md = m->mmd;
    const int n_cat = md.ref.mp.n_cat, n_num = md.ref.mp.n_num;
    int rc;
    if ((rc = compute_reserve(m, md.online.pos, (size_t)n * 4, "online MMD drift", "the row positions")) ||
        (rc = compute_reserve(m, z, std::max<size_t>((size_t)n * n_num * 8, 8), "online MMD drift", what)) ||
        (rc = compute_reserve(m, c, std::max<size_t>((size_t)n * n_cat * 4, 4), "online MMD drift", what)))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(md.online.pos.p, idx, (size_t)n * 4, cudaMemcpyHostToDevice, m->compute));
    k_mmd_online_gather<<<(unsigned)((n + 255) / 256), 256, 0, m->compute>>>(static_cast<const double *>(md.ref.ref_z.p),
                                                                             static_cast<const int32_t *>(md.ref.ref_c.p),
                                                                             static_cast<const int32_t *>(md.online.pos.p), (long long)n, n_cat,
                                                                             n_num, static_cast<double *>(z.p), static_cast<int32_t *>(c.p));
    if ((rc = launched(m, "k_mmd_online_gather"))) return rc;
    CUDA_TRY(cudaStreamSynchronize(m->compute)); /* the positions' buffer is reused */
    return B2F_OK;
}

/* the pool of the c row sums: the compacted sub-reference, then rows z / c */
static MmdPool online_pool(const Mmd &md, const void *z, const void *c) {
    return MmdPool{static_cast<const double *>(md.online.rz.p), static_cast<const int32_t *>(md.online.rc.p), static_cast<const double *>(z),
                   static_cast<const int32_t *>(c), (long long)md.online.rw, md.ref.mp.n_cat, md.ref.mp.n_num};
}

/* n rows' z / c / cv from src to dst (device to device, on the compute stream) */
static int online_copy_rows(b2f_model *m, void *dz, void *dc, void *dcv, const void *sz, const void *sc, const void *scv, int64_t n) {
    const int n_cat = m->mmd.ref.mp.n_cat, n_num = m->mmd.ref.mp.n_num;
    if (n <= 0) return B2F_OK;
    if (n_num) CUDA_TRY(cudaMemcpyAsync(dz, sz, (size_t)n * n_num * 8, cudaMemcpyDeviceToDevice, m->compute));
    if (n_cat) CUDA_TRY(cudaMemcpyAsync(dc, sc, (size_t)n * n_cat * 4, cudaMemcpyDeviceToDevice, m->compute));
    CUDA_TRY(cudaMemcpyAsync(dcv, scv, (size_t)n * 8, cudaMemcpyDeviceToDevice, m->compute));
    return B2F_OK;
}

static int online_ready(b2f_model *m, const char *what) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (m->mmd.ref.n_ref == 0) return set_err(B2F_ESTATE, "%s: no MMD reference attached (b2f_model_attach_mmd_reference)", what);
    return B2F_OK;
}

extern "C" int b2f_mmd_online_bootstrap(b2f_model *m, const int32_t *etw, int n_boot, int window, double *stats, double *k_rr, float *device_ms) {
    const char *what = "online MMD bootstrap";
    int rc = online_ready(m, what);
    if (rc) return rc;
    if (device_ms) *device_ms = 0.0f;
    Mmd &md = m->mmd;
    if ((rc = online_check_window(md, window, what))) return rc;
    if (n_boot < 1 || n_boot > B2F_MMD_ONLINE_MAX_BOOT) return set_err(B2F_EINVAL, "%s: n_boot = %d, expected 1..%d", what, n_boot, B2F_MMD_ONLINE_MAX_BOOT);
    if (!etw || !stats || !k_rr) return set_err(B2F_EINVAL, "%s: etw, stats or k_rr is NULL", what);
    if ((rc = online_check_positions(etw, n_boot, 2LL * window - 1, md.ref.n_ref, what))) return rc;
    CUDA_TRY(cudaSetDevice(m->device));
    if ((rc = online_smem_attr(md))) return rc;
    TimedRegion timed{m, device_ms};
    if ((rc = timed.start()) || (rc = online_total(m)) || (rc = online_boot(m, etw, n_boot, window, stats, k_rr))) return rc;
    return timed.finish();
}

extern "C" int b2f_mmd_online_configure(b2f_model *m, const int32_t *perm, int window, float *device_ms) {
    const char *what = "online MMD configure";
    int rc = online_ready(m, what);
    if (rc) return rc;
    if (device_ms) *device_ms = 0.0f;
    Mmd &md = m->mmd;
    MmdOnline &o = md.online;
    o.window = 0; /* replaced: not configured until this one is complete */
    if ((rc = online_check_window(md, window, what))) return rc;
    if (!perm) return set_err(B2F_EINVAL, "%s: perm is NULL", what);
    const int64_t n_ref = md.ref.n_ref, E = 2LL * window - 1, rw = n_ref - E;
    if ((rc = online_check_positions(perm, 1, n_ref, n_ref, what))) return rc;
    CUDA_TRY(cudaSetDevice(m->device));
    if ((rc = online_smem_attr(md)) || (rc = mmd_smem_attr(md))) return rc;
    TimedRegion timed{m, device_ms};
    if ((rc = timed.start()) || (rc = online_total(m))) return rc;
    std::vector<double> st((size_t)window);
    double krr = 0.0;
    if ((rc = online_boot(m, perm + rw, 1, window, st.data(), &krr))) return rc;
    o.rw = rw;
    if ((rc = online_gather(m, perm, rw, o.rz, o.rc, "the sub-reference")) ||
        (rc = online_gather(m, perm + n_ref - (window - 1), window - 1, o.init_z, o.init_c, "the initial window")) ||
        (rc = compute_reserve(m, o.init_cv, (size_t)(window - 1) * 8, "online MMD drift", "the initial window")))
        return rc;
    if ((rc = mmd_row_sums(m, online_pool(md, o.init_z.p, o.init_c.p), rw, window - 1, 0, rw, nullptr, static_cast<double *>(o.init_cv.p))))
        return rc;
    const int n_cat = md.ref.mp.n_cat, n_num = md.ref.mp.n_num;
    if ((rc = compute_reserve(m, o.carry_z, std::max<size_t>((size_t)(window - 1) * n_num * 8, 8), "online MMD drift", "the window state")) ||
        (rc = compute_reserve(m, o.carry_c, std::max<size_t>((size_t)(window - 1) * n_cat * 4, 4), "online MMD drift", "the window state")) ||
        (rc = compute_reserve(m, o.carry_cv, (size_t)(window - 1) * 8, "online MMD drift", "the window state")))
        return rc;
    if ((rc = online_copy_rows(m, o.carry_z.p, o.carry_c.p, o.carry_cv.p, o.init_z.p, o.init_c.p, o.init_cv.p, window - 1))) return rc;
    if ((rc = timed.finish())) return rc;
    o.k_rr = krr;
    o.t = 0;
    o.window = window;
    return B2F_OK;
}

extern "C" int b2f_mmd_online_reset(b2f_model *m) {
    int rc = online_ready(m, "online MMD reset");
    if (rc) return rc;
    MmdOnline &o = m->mmd.online;
    if (!o.window) return set_err(B2F_ESTATE, "online MMD reset: not configured (b2f_mmd_online_configure)");
    CUDA_TRY(cudaSetDevice(m->device));
    if ((rc = online_copy_rows(m, o.carry_z.p, o.carry_c.p, o.carry_cv.p, o.init_z.p, o.init_c.p, o.init_cv.p, o.window - 1))) return rc;
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    o.t = 0;
    return B2F_OK;
}

extern "C" int b2f_mmd_online_push(b2f_model *m, const void *rows, int64_t n, int row_format, double *stat, int64_t *t_first, float *device_ms) {
    const char *what = "online MMD push";
    int rc = online_ready(m, what);
    if (rc) return rc;
    if (device_ms) *device_ms = 0.0f;
    Mmd &md = m->mmd;
    MmdOnline &o = md.online;
    if (!o.window) return set_err(B2F_ESTATE, "%s: not configured (b2f_mmd_online_configure)", what);
    if ((rc = ref_check_rows(m, rows, n, row_format, 1, (int64_t)INT_MAX, "online MMD drift takes", what))) return rc;
    if (!stat) return set_err(B2F_EINVAL, "%s: stat is NULL", what);
    CUDA_TRY(cudaSetDevice(m->device));
    if ((rc = online_smem_attr(md)) || (rc = mmd_smem_attr(md))) return rc;
    const cudaStream_t st = m->compute;
    const int W = o.window, n_cat = md.ref.mp.n_cat, n_num = md.ref.mp.n_num;
    const int64_t carry = W - 1, chunks = (o.rw + B2F_MMD_CHUNK_TILES * B2F_MMD_TILE - 1) / (B2F_MMD_CHUNK_TILES * B2F_MMD_TILE);
    const size_t row_bytes = row_bytes_of(m, row_format);
    /* per row: its upload, its embedding twice (the call's and the sequence's), c, its row-sum partials, its band prefixes
     * and its statistic */
    const int64_t per = (int64_t)row_bytes + 2 * (8LL * n_num + 4LL * n_cat) + 8 + chunks * 8 + 8LL * W + 8;
    const int64_t piece = std::min<int64_t>(n, std::max<int64_t>(1, (int64_t)B2F_PERM_SCRATCH_BYTES / per - carry));
    const int64_t ns = carry + piece;
    const char *who = "online MMD drift";
    if ((rc = compute_reserve(m, o.seq_z, std::max<size_t>((size_t)ns * n_num * 8, 8), who, "the sequence's numerics")) ||
        (rc = compute_reserve(m, o.seq_c, std::max<size_t>((size_t)ns * n_cat * 4, 4), who, "the sequence's categories")) ||
        (rc = compute_reserve(m, o.cv, (size_t)ns * 8, who, "the sub-reference row sums")) ||
        (rc = compute_reserve(m, o.band, (size_t)(ns * W) * 8, who, "the band prefixes")) ||
        (rc = compute_reserve(m, o.out, (size_t)piece * 8, who, "the statistics")))
        return rc;
    if (t_first) *t_first = o.t + 1;
    TimedRegion timed{m, device_ms};
    if ((rc = timed.start())) return rc;
    const size_t smem = mmd_smem_bytes(n_cat, n_num);
    double *seq_z = static_cast<double *>(o.seq_z.p), *cv = static_cast<double *>(o.cv.p), *band = static_cast<double *>(o.band.p);
    int32_t *seq_c = static_cast<int32_t *>(o.seq_c.p);
    for (int64_t r0 = 0; r0 < n; r0 += piece) {
        const int64_t np = std::min(piece, n - r0), nsq = carry + np;
        if ((rc = ref_embed(m, md.ref, static_cast<const unsigned char *>(rows) + (size_t)r0 * row_bytes, np, row_format, md.ref.z, md.ref.c, who)))
            return rc;
        if ((rc = online_copy_rows(m, seq_z, seq_c, cv, o.carry_z.p, o.carry_c.p, o.carry_cv.p, carry))) return rc;
        if (n_num) CUDA_TRY(cudaMemcpyAsync(seq_z + carry * n_num, md.ref.z.p, (size_t)np * n_num * 8, cudaMemcpyDeviceToDevice, st));
        if (n_cat) CUDA_TRY(cudaMemcpyAsync(seq_c + carry * n_cat, md.ref.c.p, (size_t)np * n_cat * 4, cudaMemcpyDeviceToDevice, st));
        if ((rc = mmd_row_sums(m, online_pool(md, md.ref.z.p, md.ref.c.p), o.rw, np, 0, o.rw, nullptr, cv + carry))) return rc;
        const MmdPool S{seq_z, seq_c, nullptr, nullptr, (long long)nsq, n_cat, n_num};
        k_mmd_online_band<false><<<dim3((unsigned)((nsq + B2F_MMD_TILE - 1) / B2F_MMD_TILE), 1), B2F_MMD_TILE, smem, st>>>(
            S, nullptr, (long long)nsq, W, md.coef, nullptr, band, nullptr, nullptr);
        if ((rc = launched(m, "k_mmd_online_band"))) return rc;
        k_mmd_online_steps<<<(unsigned)((np + B2F_MMD_ONLINE_THREADS - 1) / B2F_MMD_ONLINE_THREADS), B2F_MMD_ONLINE_THREADS, 0, st>>>(
            cv, band, (long long)nsq, W, (long long)np, (long long)o.rw, o.k_rr, static_cast<double *>(o.out.p));
        if ((rc = launched(m, "k_mmd_online_steps"))) return rc;
        CUDA_TRY(cudaMemcpyAsync(stat + r0, o.out.p, (size_t)np * 8, cudaMemcpyDeviceToHost, st));
        /* the sequence's last W - 1 rows are the next state */
        if ((rc = online_copy_rows(m, o.carry_z.p, o.carry_c.p, o.carry_cv.p, seq_z + np * n_num, seq_c + np * n_cat, cv + np, carry))) return rc;
        CUDA_TRY(cudaStreamSynchronize(st));
        o.t += np;
    }
    return timed.finish();
}
