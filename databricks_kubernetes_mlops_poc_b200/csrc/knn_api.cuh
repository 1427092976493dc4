/*
 * knn_api.cuh -- C ABI of the exact k-nearest reference search behind trust scores (include/b2f.h:
 * b2f_model_attach_knn_reference, b2f_knn); included by b2f_api.cu.
 *
 * Host side of K11 (knn.cuh).  The reference is kept class-sorted (each class in its original row order) as K9's embedding
 * (EmbeddedRef; its row check, constants, upload and pool are mmd_api.cuh's ref_* functions), with the map back to original
 * row indices.  A call embeds its queries piece by piece (at most B2F_KNN_PIECE_ROWS rows, and a candidate scratch under
 * B2F_KNN_SCRATCH_BYTES), splits each class into chunks so that small pieces still fill the GPU, and merges the chunks'
 * lists when there is more than one.  Every buffer is on the compute stream, grown on demand and never
 * shrunk.
 */
#pragma once

#define B2F_KNN_PIECE_ROWS 65536
#define B2F_KNN_SCRATCH_BYTES (256ull << 20)
#define B2F_KNN_MERGE_ENTRIES 1024 /* chunks * k at most this: the merge's binary searches stay short */

extern "C" int b2f_model_attach_knn_reference(b2f_model *m, const void *rows, int64_t n, int row_format, const int32_t *cls,
                                              const double *num_mean, const double *num_scale) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    Knn &kn = m->knn;
    kn.ref.n_ref = 0; /* replaced: no reference until this one is complete */
    int rc = ref_check_rows(m, rows, n, row_format, 2, B2F_MMD_MAX_REF, "trust reference takes", "trust reference");
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
    if ((rc = ref_constants(m, kn.ref, num_mean, num_scale, "trust reference"))) return rc;

    CUDA_TRY(cudaSetDevice(m->device));
    /* class-sorted, each class in row order: a tie on distance goes to the lower position, i.e. the lower original index */
    const size_t row_bytes = row_bytes_of(m, row_format);
    std::vector<unsigned char> sorted((size_t)n * row_bytes);
    std::vector<int32_t> orig((size_t)n);
    int64_t at[2] = {0, count[0]};
    for (int64_t i = 0; i < n; ++i) {
        const int64_t p = at[cls[i]]++;
        memcpy(sorted.data() + p * row_bytes, static_cast<const unsigned char *>(rows) + i * row_bytes, row_bytes);
        orig[p] = (int32_t)i;
    }
    if ((rc = compute_reserve(m, kn.orig, (size_t)n * 4, "trust neighbours", "the reference's row map"))) return rc;
    if ((rc = ref_embed(m, kn.ref, sorted.data(), n, row_format, kn.ref.ref_z, kn.ref.ref_c, "trust neighbours"))) return rc;
    CUDA_TRY(cudaMemcpyAsync(kn.orig.p, orig.data(), (size_t)n * 4, cudaMemcpyHostToDevice, m->compute));
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    kn.n_cls[0] = count[0], kn.n_cls[1] = count[1];
    kn.ref.n_ref = n;
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
    if (kn.ref.n_ref == 0) return set_err(B2F_ESTATE, "trust neighbours: no reference attached (b2f_model_attach_knn_reference)");
    int rc = ref_check_rows(m, rows, n, row_format, 1, INT64_MAX / 2, "trust neighbours takes", "trust neighbours");
    if (rc) return rc;
    const int64_t k_max = std::min<int64_t>({(int64_t)B2F_KNN_MAX_K, kn.n_cls[0], kn.n_cls[1]});
    if (k < 1 || k > k_max)
        return set_err(B2F_EINVAL, "trust neighbours: k = %d, expected 1 .. %lld (at most %d, and the rows of the smaller class)", k,
                       (long long)k_max, B2F_KNN_MAX_K);
    if (!dist || !index) return set_err(B2F_EINVAL, "trust neighbours: dist or index is NULL");

    CUDA_TRY(cudaSetDevice(m->device));
    const int smem = (int)knn_smem_bytes(kn.ref.mp.n_cat, kn.ref.mp.n_num, k);
    CUDA_TRY(set_smem_limit(k_knn_chunk, smem));
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
    const char *who = "trust neighbours";
    if ((rc = compute_reserve(m, kn.dist, out_bytes * 8, who, "the distances")) || (rc = compute_reserve(m, kn.index, out_bytes * 4, who, "the indices")))
        return rc;
    TimedRegion timed{m, device_ms};
    if ((rc = timed.start())) return rc;
    const size_t row_bytes = row_bytes_of(m, row_format);
    for (int64_t off = 0; off < n; off += piece) {
        const int64_t nq = std::min(piece, n - off);
        KnnArgs a;
        knn_plan(m, nq, k, &a.chunk_rows, &a.chunks);
        const size_t scratch = knn_scratch_bytes(nq, k, a.chunks);
        if (scratch && ((rc = compute_reserve(m, kn.cand_d, scratch / 12 * 8, who, "the candidate distances")) ||
                        (rc = compute_reserve(m, kn.cand_i, scratch / 12 * 4, who, "the candidate indices"))))
            return rc;
        if ((rc = ref_embed(m, kn.ref, static_cast<const unsigned char *>(rows) + off * row_bytes, nq, row_format, kn.ref.z, kn.ref.c, who))) return rc;
        a.nq = nq, a.k = k;
        a.lo[0] = 0, a.n[0] = kn.n_cls[0], a.lo[1] = kn.n_cls[0], a.n[1] = kn.n_cls[1];
        a.orig = static_cast<const int32_t *>(kn.orig.p);
        a.dist = static_cast<double *>(kn.dist.p), a.index = static_cast<int32_t *>(kn.index.p);
        a.cand_d = static_cast<double *>(kn.cand_d.p), a.cand_i = static_cast<int32_t *>(kn.cand_i.p);
        const MmdPool P = ref_pool(kn.ref, kn.ref.n_ref);
        const dim3 grid((unsigned)((nq + B2F_MMD_TILE - 1) / B2F_MMD_TILE), (unsigned)a.chunks, 2);
        k_knn_chunk<<<grid, B2F_MMD_TILE, smem, st>>>(P, a);
        if ((rc = launched(m, "k_knn_chunk"))) return rc;
        if (a.chunks > 1) {
            k_knn_merge<<<(unsigned)(nq * 2), B2F_KNN_MERGE_THREADS, 0, st>>>(a);
            if ((rc = launched(m, "k_knn_merge"))) return rc;
        }
        const size_t outs = (size_t)nq * 2 * k;
        CUDA_TRY(cudaMemcpyAsync(dist + off * 2 * k, kn.dist.p, outs * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(index + off * 2 * k, kn.index.p, outs * 4, cudaMemcpyDeviceToHost, st));
    }
    return timed.finish();
}
