/*
 * knn_api.cuh -- C ABI of the exact k-nearest reference search behind trust scores (include/b2f.h:
 * b2f_model_attach_knn_reference, b2f_knn); included by b2f_api.cu.
 *
 * Host side of K11 (knn.cuh).  The reference is kept class-sorted (each class in its original row order) as K9's embedding,
 * with the map back to original row indices.  A call embeds its queries piece by piece (at most B2F_KNN_PIECE_ROWS rows, and a
 * candidate scratch under B2F_KNN_SCRATCH_BYTES), splits each class into chunks so that small pieces still fill the GPU, and
 * merges the chunks' lists when there is more than one.  Every buffer is on the compute stream, grown on demand and never
 * shrunk.
 */
#pragma once

#define B2F_KNN_PIECE_ROWS 65536
#define B2F_KNN_SCRATCH_BYTES (256ull << 20)
#define B2F_KNN_MERGE_ENTRIES 1024 /* chunks * k at most this: the merge's binary searches stay short */

/* reserve with the failure reported as B2F_ENOMEM and its byte count */
static int knn_reserve(b2f_model *m, DevBuf &b, size_t bytes, const char *what) {
    if (b.reserve(m->compute, bytes, bytes) == B2F_OK) return B2F_OK;
    (void)cudaGetLastError();
    return set_err(B2F_ENOMEM, "trust neighbours: cannot allocate %zu device bytes for %s", bytes, what);
}

static int knn_check_rows(b2f_model *m, const void *rows, int64_t n, int row_format, int64_t lo, int64_t hi, const char *what) {
    if (row_format == B2F_ROWS_RANKED)
        return set_err(B2F_EINVAL, "%s takes float32 rows (B2F_ROWS_WORDS24 / B2F_ROWS_PACKED64): ranked rows carry no values", what);
    const int rc = check_row_format(m, row_format);
    if (rc) return rc;
    if (!rows) return set_err(B2F_EINVAL, "%s: rows is NULL", what);
    if (n < lo || n > hi) return set_err(B2F_EINVAL, "%s: n = %lld rows, expected %lld .. %lld", what, (long long)n, (long long)lo, (long long)hi);
    return B2F_OK;
}

static size_t knn_row_bytes(int row_format) { return row_format == B2F_ROWS_PACKED64 ? B2F_PACKED_ROW_WORDS * 4 : B2F_ROW_WORDS * 4; }

/* upload n rows and embed them (K9's k_mmd_embed with the trust reference's constants) into z / c on the compute stream */
static int knn_embed(b2f_model *m, const void *rows, int64_t n, int row_format, DevBuf &z, DevBuf &c) {
    Knn &kn = m->knn;
    const size_t row_bytes = knn_row_bytes(row_format);
    int rc;
    if ((rc = knn_reserve(m, kn.rows, (size_t)n * row_bytes, "the rows")) ||
        (rc = knn_reserve(m, z, std::max<size_t>((size_t)n * kn.mp.n_num * 8, 8), "the numerics")) ||
        (rc = knn_reserve(m, c, std::max<size_t>((size_t)n * kn.mp.n_cat * 4, 4), "the categories")))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(kn.rows.p, rows, (size_t)n * row_bytes, cudaMemcpyHostToDevice, m->compute));
    const unsigned grid = (unsigned)((n + 255) / 256);
    const uint32_t *d_rows = static_cast<const uint32_t *>(kn.rows.p);
    if (row_format == B2F_ROWS_PACKED64)
        k_mmd_embed<true><<<grid, 256, 0, m->compute>>>(kn.mp, d_rows, (long long)n, static_cast<double *>(z.p), static_cast<int32_t *>(c.p));
    else
        k_mmd_embed<false><<<grid, 256, 0, m->compute>>>(kn.mp, d_rows, (long long)n, static_cast<double *>(z.p), static_cast<int32_t *>(c.p));
    return mmd_launched(m, "k_mmd_embed");
}

extern "C" int b2f_model_attach_knn_reference(b2f_model *m, const void *rows, int64_t n, int row_format, const int32_t *cls,
                                              const double *num_mean, const double *num_scale) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    Knn &kn = m->knn;
    kn.n_ref = 0; /* replaced: no reference until this one is complete */
    int rc = knn_check_rows(m, rows, n, row_format, 2, B2F_MMD_MAX_REF, "trust reference");
    if (rc) return rc;
    if (!cls) return set_err(B2F_EINVAL, "trust reference: cls is NULL");
    int64_t count[2] = {0, 0};
    for (int64_t i = 0; i < n; ++i) {
        if (cls[i] != 0 && cls[i] != 1) return set_err(B2F_EINVAL, "trust reference: cls[%lld] = %d, expected 0 or 1", (long long)i, cls[i]);
        ++count[cls[i]];
    }
    if (count[0] == 0 || count[1] == 0)
        return set_err(B2F_EINVAL, "trust reference: class 0 has %lld rows and class 1 %lld; each needs at least one", (long long)count[0],
                       (long long)count[1]);
    const b2f_blob_header &h = m->hdr;
    const int n_num = (int)h.n_num;
    if (n_num > 0 && (!num_mean || !num_scale)) return set_err(B2F_EINVAL, "trust reference: num_mean or num_scale is NULL");
    for (int k = 0; k < n_num; ++k)
        if (!std::isfinite(num_mean[k]) || !std::isfinite(num_scale[k]) || !(num_scale[k] > 0.0))
            return set_err(B2F_EINVAL, "trust reference: numeric %d has mean %g and scale %g: expected finite, scale > 0", k, num_mean[k], num_scale[k]);

    CUDA_TRY(cudaSetDevice(m->device));
    kn.mp.n_cat = (int)h.n_cat, kn.mp.n_num = n_num;
    memcpy(kn.mp.impute, h.impute, sizeof(kn.mp.impute));
    for (int k = 0; k < 24; ++k) kn.mp.mean[k] = k < n_num ? num_mean[k] : 0.0, kn.mp.scale[k] = k < n_num ? num_scale[k] : 1.0;
    /* class-sorted, each class in row order: a tie on distance goes to the lower position, i.e. the lower original index */
    const size_t row_bytes = knn_row_bytes(row_format);
    std::vector<unsigned char> sorted((size_t)n * row_bytes);
    std::vector<int32_t> orig((size_t)n);
    int64_t at[2] = {0, count[0]};
    for (int64_t i = 0; i < n; ++i) {
        const int64_t p = at[cls[i]]++;
        memcpy(sorted.data() + p * row_bytes, static_cast<const unsigned char *>(rows) + i * row_bytes, row_bytes);
        orig[p] = (int32_t)i;
    }
    if ((rc = knn_reserve(m, kn.orig, (size_t)n * 4, "the reference's row map"))) return rc;
    if ((rc = knn_embed(m, sorted.data(), n, row_format, kn.ref_z, kn.ref_c))) return rc;
    CUDA_TRY(cudaMemcpyAsync(kn.orig.p, orig.data(), (size_t)n * 4, cudaMemcpyHostToDevice, m->compute));
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    kn.n_cls[0] = count[0], kn.n_cls[1] = count[1];
    kn.n_ref = n;
    return B2F_OK;
}

/* chunks per class for a piece of nq queries: enough blocks to fill the GPU a few times over, no chunk shorter than a tile,
 * chunks * k <= B2F_KNN_MERGE_ENTRIES; -> rows per chunk (a multiple of the tile) and the chunk count of the larger class */
static void knn_plan(const b2f_model *m, int64_t nq, int k, long long *chunk_rows, int *chunks) {
    const Knn &kn = m->knn;
    const int64_t tiles = (nq + B2F_MMD_TILE - 1) / B2F_MMD_TILE, n_max = std::max(kn.n_cls[0], kn.n_cls[1]);
    const int64_t target = 4 * (int64_t)std::max(m->sm_count, 1);
    int64_t c = (target + 2 * tiles - 1) / (2 * tiles);
    c = std::min<int64_t>({c, (n_max + B2F_MMD_TILE - 1) / B2F_MMD_TILE, std::max(1, B2F_KNN_MERGE_ENTRIES / k)});
    c = std::max<int64_t>(c, 1);
    const int64_t per = (n_max + c - 1) / c;
    *chunk_rows = (per + B2F_MMD_TILE - 1) / B2F_MMD_TILE * B2F_MMD_TILE;
    *chunks = (int)((n_max + *chunk_rows - 1) / *chunk_rows);
}

static size_t knn_scratch_bytes(int64_t nq, int k, int chunks) { return chunks > 1 ? (size_t)nq * 2 * chunks * k * 12 : 0; }

extern "C" int b2f_knn(b2f_model *m, const void *rows, int64_t n, int row_format, int k, double *dist, int32_t *index, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (device_ms) *device_ms = 0.0f;
    Knn &kn = m->knn;
    if (kn.n_ref == 0) return set_err(B2F_ESTATE, "trust neighbours: no reference attached (b2f_model_attach_knn_reference)");
    int rc = knn_check_rows(m, rows, n, row_format, 1, INT64_MAX / 2, "trust neighbours");
    if (rc) return rc;
    const int64_t k_max = std::min<int64_t>({(int64_t)B2F_KNN_MAX_K, kn.n_cls[0], kn.n_cls[1]});
    if (k < 1 || k > k_max)
        return set_err(B2F_EINVAL, "trust neighbours: k = %d, expected 1 .. %lld (at most %d, and the rows of the smaller class)", k,
                       (long long)k_max, B2F_KNN_MAX_K);
    if (!dist || !index) return set_err(B2F_EINVAL, "trust neighbours: dist or index is NULL");

    CUDA_TRY(cudaSetDevice(m->device));
    const int smem = (int)knn_smem_bytes(kn.mp.n_cat, kn.mp.n_num, k);
    CUDA_TRY(cudaFuncSetAttribute(k_knn_chunk, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const cudaStream_t st = m->compute;
    /* the piece size: at most B2F_KNN_PIECE_ROWS queries, halved until the candidate scratch fits the budget */
    int64_t piece = std::min<int64_t>(n, B2F_KNN_PIECE_ROWS);
    for (;;) {
        long long cr;
        int ch;
        knn_plan(m, piece, k, &cr, &ch);
        if (piece == 1 || knn_scratch_bytes(piece, k, ch) <= B2F_KNN_SCRATCH_BYTES) break;
        piece = (piece + 1) / 2;
    }
    const size_t out_bytes = (size_t)piece * 2 * k;
    if ((rc = knn_reserve(m, kn.dist, out_bytes * 8, "the distances")) || (rc = knn_reserve(m, kn.index, out_bytes * 4, "the indices")))
        return rc;
    Events evs;
    if (device_ms) {
        if ((rc = evs.create(2))) return rc;
        CUDA_TRY(cudaEventRecord(evs.e[0], st));
    }
    const size_t row_bytes = knn_row_bytes(row_format);
    for (int64_t off = 0; off < n; off += piece) {
        const int64_t nq = std::min(piece, n - off);
        KnnArgs a;
        knn_plan(m, nq, k, &a.chunk_rows, &a.chunks);
        const size_t scratch = knn_scratch_bytes(nq, k, a.chunks);
        if (scratch && ((rc = knn_reserve(m, kn.cand_d, scratch / 12 * 8, "the candidate distances")) ||
                        (rc = knn_reserve(m, kn.cand_i, scratch / 12 * 4, "the candidate indices"))))
            return rc;
        if ((rc = knn_embed(m, static_cast<const unsigned char *>(rows) + off * row_bytes, nq, row_format, kn.z, kn.c))) return rc;
        a.nq = nq, a.k = k;
        a.lo[0] = 0, a.n[0] = kn.n_cls[0], a.lo[1] = kn.n_cls[0], a.n[1] = kn.n_cls[1];
        a.orig = static_cast<const int32_t *>(kn.orig.p);
        a.dist = static_cast<double *>(kn.dist.p), a.index = static_cast<int32_t *>(kn.index.p);
        a.cand_d = static_cast<double *>(kn.cand_d.p), a.cand_i = static_cast<int32_t *>(kn.cand_i.p);
        const MmdPool P{static_cast<const double *>(kn.ref_z.p), static_cast<const int32_t *>(kn.ref_c.p), static_cast<const double *>(kn.z.p),
                        static_cast<const int32_t *>(kn.c.p), (long long)kn.n_ref, kn.mp.n_cat, kn.mp.n_num};
        const dim3 grid((unsigned)((nq + B2F_MMD_TILE - 1) / B2F_MMD_TILE), (unsigned)a.chunks, 2);
        k_knn_chunk<<<grid, B2F_MMD_TILE, smem, st>>>(P, a);
        if ((rc = mmd_launched(m, "k_knn_chunk"))) return rc;
        if (a.chunks > 1) {
            k_knn_merge<<<(unsigned)(nq * 2), B2F_KNN_MERGE_THREADS, 0, st>>>(a);
            if ((rc = mmd_launched(m, "k_knn_merge"))) return rc;
        }
        const size_t outs = (size_t)nq * 2 * k;
        CUDA_TRY(cudaMemcpyAsync(dist + off * 2 * k, kn.dist.p, outs * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(index + off * 2 * k, kn.index.p, outs * 4, cudaMemcpyDeviceToHost, st));
    }
    if (device_ms) CUDA_TRY(cudaEventRecord(evs.e[1], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (device_ms) CUDA_TRY(cudaEventElapsedTime(device_ms, evs.e[0], evs.e[1]));
    return B2F_OK;
}
