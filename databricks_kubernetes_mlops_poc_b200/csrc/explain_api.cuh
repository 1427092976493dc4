/*
 * explain_api.cuh -- C ABI of the explanations (include/b2f.h: b2f_paths_validate, b2f_model_attach_explainer,
 * b2f_model_attach_background, b2f_explain*); included by b2f_api.cu.
 *
 * Host side of K5 (tree_shap.cuh, tree_shap_interactions.cuh, tree_shap_interventional.cuh; path table: forest_paths.h).
 * A host call is a job of the host pipeline (HostJob in b2f_api.cu): its chunks ride the same slots and streams as scores.
 */
#pragma once

/* what a K5 launch computes: phi (k_tree_shap), the F x F interaction matrix (k_tree_shap_interactions), or phi against the
 * attached background (k_tree_shap_interventional) */
enum ShapVariant { SHAP_PHI, SHAP_INTERACTIONS, SHAP_INTERVENTIONAL, SHAP_VARIANTS };

/* the launch shape of one explanation kernel */
struct ExplainKernel {
    int smem_bytes = 0;
    int ctas_per_sm = 1; /* resident CTAs per SM */
};

/* an attached background set (b2f_model_attach_background; tree_shap_interventional.cuh) */
struct Background {
    void *d_table = nullptr; /* offsets[n_paths + 1] int64, then the {mask, count} entries */
    size_t bytes = 0;
    int64_t rows = 0;        /* 0: none attached */
    double base_value = 0.0; /* mean over the background rows of the prediction, in the output space */
    VParams vp{};            /* vp.s: the explainer's SParams with denom * rows */
};

/* an attached path table (b2f_model_attach_explainer) */
struct Explainer {
    b2f_paths_header hdr;
    void *d_table = nullptr;
    IParams ip;   /* k_tree_shap takes ip.s; k_tree_shap_interactions also each warp's fields (inter_assign) */
    int maxl = 9; /* length bucket of the kernels: 9, 16 or 24 */
    ExplainKernel kernels[SHAP_VARIANTS];
    Background bg; /* k_tree_shap_interventional's table (b2f_model_attach_background) */
};

/* frees an explainer's tables; nothing on the device may still use them */
static void explainer_free(Explainer *ex) {
    if (ex->d_table) cudaFree(ex->d_table);
    if (ex->bg.d_table) cudaFree(ex->bg.d_table);
    delete ex;
}

/* rows per chunk of an interactions batch (4 232 B of output per row for 23 fields), with no chunk plan: every chunk of
 * 16 384 rows is 512 row tiles, more than the SMs hold at once, so it runs as one range and needs no scratch */
#define B2F_INTER_CHUNK_ROWS 16384

static int explain_fields(const b2f_model *m) { return (int)(m->hdr.n_cat + m->hdr.n_num); }
static size_t explain_row_bytes(const b2f_model *m, int v) {
    const size_t F = (size_t)explain_fields(m);
    return (v == SHAP_INTERACTIONS ? F * F : F) * sizeof(double);
}

/* the checks of an explain call that follow the explainer's own (m->ex is set) */
static int explain_check(const b2f_model *m, int fmt, int v, bool have_out) {
    if (v == SHAP_INTERVENTIONAL && !m->ex->bg.rows) return set_err(B2F_ESTATE, "no background attached (b2f_model_attach_background)");
    const int rc = check_value_rows(fmt, "explanations take");
    if (rc) return rc;
    if (!have_out) return set_err(B2F_EINVAL, v == SHAP_INTERACTIONS ? "phi2 is NULL" : "phi is NULL");
    return B2F_OK;
}

/* row tiles x path ranges of one launch: one range from a full grid of row tiles up; below, enough ranges to fill every SM
 * (at least sixteen paths per range: two per warp for k_tree_shap).  The partials of several ranges take ranges * n * values
 * doubles (values: fields, or F(F+1)/2 triangle slots for interactions); since ranges > 1 only when tiles < target, that is
 * below 2 * target * 32 rows' worth: bounded by the GPU, not by n or the number of paths. */
static int64_t explain_ranges(const b2f_model *m, int64_t n, int v) {
    const int64_t tiles = (n + 31) / 32, target = (int64_t)m->sm_count * m->ex->kernels[v].ctas_per_sm;
    int64_t r = tiles >= target ? 1 : (target + tiles - 1) / tiles;
    r = std::min<int64_t>(r, std::max<int64_t>(1, (int64_t)m->ex->hdr.n_paths / (2 * B2F_SHAP_WARPS)));
    return std::max<int64_t>(1, std::min<int64_t>(r, 65535));
}

template <int MAXL>
static const void *explain_kernel_l(int v, bool pk) {
    if (v == SHAP_INTERACTIONS)
        return pk ? (const void *)k_tree_shap_interactions<MAXL, true> : (const void *)k_tree_shap_interactions<MAXL, false>;
    if (v == SHAP_INTERVENTIONAL)
        return pk ? (const void *)k_tree_shap_interventional<MAXL, true> : (const void *)k_tree_shap_interventional<MAXL, false>;
    return pk ? (const void *)k_tree_shap<MAXL, true> : (const void *)k_tree_shap<MAXL, false>;
}
/* the variant's kernel for the path-length bucket maxl and the row format.  All take (params, rows, n, out, partials): IParams
 * for interactions, the background's VParams for interventional values, the SParams otherwise. */
static const void *explain_kernel(int v, int maxl, bool pk) {
    return maxl <= 9 ? explain_kernel_l<9>(v, pk) : (maxl <= 16 ? explain_kernel_l<16>(v, pk) : explain_kernel_l<24>(v, pk));
}

/* out_dev[n] rows of explain_row_bytes (phi, or the F x F interaction matrix) for n device rows of format fmt, on stream st,
 * partial sums (phi, or the triangle) in scratch */
static int launch_explain(b2f_model *m, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, int v, double *out_dev, DevBuf &scratch) {
    if (n <= 0) return B2F_OK;
    Explainer &ex = *m->ex;
    const bool inter = v == SHAP_INTERACTIONS, interv = v == SHAP_INTERVENTIONAL;
    const char *name = inter ? "k_tree_shap_interactions" : (interv ? "k_tree_shap_interventional" : "k_tree_shap");
    void *params = inter ? static_cast<void *>(&ex.ip) : (interv ? static_cast<void *>(&ex.bg.vp) : static_cast<void *>(&ex.ip.s));
    const double denom = interv ? ex.bg.vp.s.denom : ex.hdr.denom; /* phi = sum / denom (interventional: / (denom * rows)) */
    const int F = explain_fields(m), values = inter ? inter_slots(F) : F; /* partial sums per row */
    if (ex.hdr.n_paths == 0) { /* every tree a single leaf: nothing moves away from base_value */
        CUDA_TRY(cudaMemsetAsync(out_dev, 0, (size_t)n * explain_row_bytes(m, v), st));
        return B2F_OK;
    }
    const int64_t ranges = explain_ranges(m, n, v);
    int rc;
    if (ranges > 1) {
        const size_t bytes = (size_t)ranges * (size_t)n * values * sizeof(double);
        if ((rc = scratch.reserve(st, bytes, bytes))) return rc;
    }
    double *partials = static_cast<double *>(scratch.p);
    const uint32_t *rows = static_cast<const uint32_t *>(rows_dev);
    long long n_rows = n;
    void *args[] = {params, &rows, &n_rows, &out_dev, &partials};
    /* a failed launch is also the thread's last error, taken (and cleared) below as after <<< >>> */
    cudaLaunchKernel(explain_kernel(v, ex.maxl, fmt == B2F_ROWS_PACKED64), dim3((unsigned)((n + 31) / 32), (unsigned)ranges),
                     dim3(B2F_SHAP_THREADS), args, (size_t)ex.kernels[v].smem_bytes, st);
    if ((rc = launched(m, name))) return rc;
    if (ranges > 1) {
        if (inter) { /* one CTA per row, its triangle in shared memory */
            const unsigned blocks = (unsigned)std::min<int64_t>(n, (int64_t)m->sm_count * 8);
            k_tree_shap_interactions_finish<<<blocks, 256, (size_t)values * sizeof(double), st>>>(partials, (int)ranges, n_rows, F, denom,
                                                                                                  out_dev);
        } else {
            const int64_t n_values = n * F;
            const unsigned blocks = (unsigned)std::min<int64_t>((n_values + 255) / 256, (int64_t)m->sm_count * 8);
            k_tree_shap_finish<<<blocks, 256, 0, st>>>(partials, (int)ranges, (long long)n_values, denom, out_dev);
        }
        return launched(m, (std::string(name) + "_finish").c_str());
    }
    return B2F_OK;
}

/* ------------------------------------------------------------------ explainer: path table check, attach, explain */
static int validate_paths(const uint8_t *t, size_t nbytes, b2f_paths_header *hdr_out) {
    if (!t || nbytes < sizeof(b2f_paths_header)) return set_err(B2F_EINVAL, "path table too small (%zu bytes)", nbytes);
    b2f_paths_header h;
    memcpy(&h, t, sizeof(h));
    if (memcmp(h.magic, B2F_PATHS_MAGIC, 8) != 0) return set_err(B2F_EINVAL, "path table: bad magic");
    if (h.version != B2F_PATHS_VERSION) return set_err(B2F_EINVAL, "path table: version %u, expected %u", h.version, B2F_PATHS_VERSION);
    if (h.header_bytes != B2F_PATHS_HEADER_BYTES) return set_err(B2F_EINVAL, "path table: header_bytes=%u unsupported", h.header_bytes);
    if (h.agg_mode != B2F_AGG_RF_MEAN && h.agg_mode != B2F_AGG_GBDT_LOGISTIC)
        return set_err(B2F_EINVAL, "path table: agg_mode %u (only RandomForest and GBDT classifiers are explained)", h.agg_mode);
    if (h.n_cat + h.n_num > B2F_SENTINEL_WORD || h.n_cat + h.n_num == 0)
        return set_err(B2F_EINVAL, "path table: n_cat+n_num=%u out of range [1,%u]", h.n_cat + h.n_num, B2F_SENTINEL_WORD);
    if (h.n_trees == 0 || h.n_trees > B2F_MAX_TREES) return set_err(B2F_EINVAL, "path table: n_trees=%u out of range", h.n_trees);
    if (h.max_len > B2F_PATHS_MAX_LEN) return set_err(B2F_EINVAL, "path table: max_len=%u exceeds %u", h.max_len, B2F_PATHS_MAX_LEN);
    if (!(h.denom > 0.0) || !std::isfinite(h.base_value)) return set_err(B2F_EINVAL, "path table: bad denom or base_value");
    const uint64_t elems_off = (h.paths_off + (uint64_t)h.n_paths * sizeof(b2f_path) + 15) / 16 * 16;
    if (h.paths_off != B2F_PATHS_HEADER_BYTES || h.elems_off != elems_off || h.total_bytes != nbytes ||
        h.elems_off + (uint64_t)h.n_elems * sizeof(b2f_path_elem) != nbytes)
        return set_err(B2F_EINVAL, "path table: sections do not match its size (%zu bytes; truncated?)", nbytes);
    const b2f_path *P = reinterpret_cast<const b2f_path *>(t + h.paths_off);
    const b2f_path_elem *E = reinterpret_cast<const b2f_path_elem *>(t + h.elems_off);
    const uint32_t F = h.n_cat + h.n_num;
    uint64_t next = 0;
    uint32_t longest = 0;
    for (uint32_t p = 0; p < h.n_paths; ++p) {
        b2f_path pr;
        memcpy(&pr, &P[p], sizeof(pr));
        if (pr.first != next || pr.len < 2 || pr.len > h.max_len || (uint64_t)pr.first + pr.len > h.n_elems || pr.tree >= h.n_trees ||
            !std::isfinite(pr.leaf))
            return set_err(B2F_EINVAL, "path table: path %u malformed (first %u, len %u)", p, pr.first, pr.len);
        next += pr.len;
        longest = std::max(longest, pr.len);
        uint32_t seen = 0;
        for (uint32_t k = 0; k < pr.len; ++k) {
            b2f_path_elem e;
            memcpy(&e, &E[pr.first + k], sizeof(e));
            if (k == 0) {
                if (e.field != B2F_PATH_BIAS_FIELD || e.kind != B2F_PE_BIAS) return set_err(B2F_EINVAL, "path table: path %u has no bias element", p);
                continue;
            }
            const bool cat = e.kind == B2F_PE_CAT, num = (e.kind & ~B2F_PE_HAS_HI) == B2F_PE_NUM;
            if (e.field >= F || (cat && e.field >= h.n_cat) || (num && e.field < h.n_cat) || !(cat || num))
                return set_err(B2F_EINVAL, "path table: path %u element %u: field %u / kind %u invalid", p, k, e.field, e.kind);
            if (seen & (1u << e.field)) return set_err(B2F_EINVAL, "path table: path %u tests field %u twice (elements must be merged)", p, e.field);
            seen |= 1u << e.field;
            if (!(e.zero_fraction > 0.0 && e.zero_fraction <= 1.0) || !(e.inv_zero_fraction >= 1.0) || !std::isfinite(e.inv_zero_fraction))
                return set_err(B2F_EINVAL, "path table: path %u element %u: bad zero fraction", p, k);
        }
    }
    if (next != h.n_elems || longest != h.max_len) return set_err(B2F_EINVAL, "path table: element count or max_len inconsistent");
    *hdr_out = h;
    return B2F_OK;
}

extern "C" int b2f_paths_validate(const void *paths, size_t nbytes) {
    b2f_paths_header h;
    return validate_paths(static_cast<const uint8_t *>(paths), nbytes, &h);
}

/* flatten.py blob_fingerprint: sum of splitmix64(w_i ^ i * golden) over the blob's 64-bit words */
static uint64_t blob_fingerprint(const uint8_t *blob, size_t nbytes) {
    uint64_t sum = 0;
    for (size_t i = 0; i < nbytes / 8; ++i) {
        uint64_t z;
        memcpy(&z, blob + 8 * i, 8);
        z ^= (uint64_t)i * 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        sum += z ^ (z >> 31);
    }
    return sum;
}

/* the fields each warp of k_tree_shap_interactions owns, balancing the counted pair work: per path of d elements that holds
 * field f, its owner unwinds f (d steps) and takes the unwound sum of every element of a higher field (d - 1 steps each).
 * Longest work first, each field to the warp with the least work so far (ties: the lower field, the lower warp). */
static void inter_assign(const uint8_t *t, const b2f_paths_header &h, uint32_t own[B2F_SHAP_WARPS]) {
    const int F = (int)(h.n_cat + h.n_num);
    const b2f_path *P = reinterpret_cast<const b2f_path *>(t + h.paths_off);
    const b2f_path_elem *E = reinterpret_cast<const b2f_path_elem *>(t + h.elems_off);
    std::vector<double> work(F, 0.0);
    for (uint32_t p = 0; p < h.n_paths; ++p) {
        b2f_path pr;
        memcpy(&pr, &P[p], sizeof(pr));
        uint32_t fields[B2F_PATHS_MAX_LEN];
        for (uint32_t k = 1; k < pr.len; ++k) memcpy(&fields[k], &E[pr.first + k].field, sizeof(uint32_t));
        const double d = pr.len - 1.0;
        for (uint32_t k = 1; k < pr.len; ++k) {
            int higher = 0;
            for (uint32_t j = 1; j < pr.len; ++j) higher += fields[j] > fields[k];
            work[fields[k]] += d + higher * (d - 1.0);
        }
    }
    std::vector<int> order(F);
    for (int f = 0; f < F; ++f) order[f] = f;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return work[a] > work[b]; });
    double load[B2F_SHAP_WARPS] = {};
    for (int w = 0; w < B2F_SHAP_WARPS; ++w) own[w] = 0;
    for (int f : order) {
        const int w = (int)(std::min_element(load, load + B2F_SHAP_WARPS) - load);
        own[w] |= 1u << f;
        load[w] += work[f];
    }
}

extern "C" int b2f_model_attach_explainer(b2f_model *m, const void *paths, size_t nbytes) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    b2f_paths_header h;
    int rc = validate_paths(static_cast<const uint8_t *>(paths), nbytes, &h);
    if (rc) return rc;
    if (h.n_cat != m->hdr.n_cat || h.n_num != m->hdr.n_num || h.agg_mode != m->hdr.agg_mode || h.n_trees != m->hdr.n_trees)
        return set_err(B2F_EINVAL, "path table: shape (%u cat, %u num, agg %u, %u trees) differs from the model's (%u, %u, %u, %u)", h.n_cat, h.n_num,
                       h.agg_mode, h.n_trees, m->hdr.n_cat, m->hdr.n_num, m->hdr.agg_mode, m->hdr.n_trees);
    CUDA_TRY(cudaSetDevice(m->device));
    std::vector<uint8_t> blob(m->hdr.total_bytes);
    CUDA_TRY(cudaMemcpy(blob.data(), m->d_blob, blob.size(), cudaMemcpyDeviceToHost));
    if (blob_fingerprint(blob.data(), blob.size()) != h.fingerprint)
        return set_err(B2F_EINVAL, "path table: built from another forest (fingerprint mismatch)");
    /* replacing an explainer: nothing may still read the old table.  Waited for before anything new is allocated, so a
     * failure here leaves the model as it was and leaks nothing. */
    if (m->ex) CUDA_TRY(cudaDeviceSynchronize());
    Explainer *ex = new (std::nothrow) Explainer();
    if (!ex) return set_err(B2F_ENOMEM, "out of host memory");
    auto fail = [&](int code) {
        explainer_free(ex);
        return code;
    };
    ex->hdr = h;
    if (cudaMalloc(&ex->d_table, nbytes) != cudaSuccess || cudaMemcpy(ex->d_table, paths, nbytes, cudaMemcpyHostToDevice) != cudaSuccess)
        return fail(set_err(B2F_ENOMEM, "path table upload (%zu bytes) failed: %s", nbytes, cudaGetErrorString(cudaGetLastError())));
    SParams &sp = ex->ip.s;
    memset(&sp, 0, sizeof(sp));
    sp.paths = reinterpret_cast<const b2f_path *>(static_cast<uint8_t *>(ex->d_table) + h.paths_off);
    sp.elems = reinterpret_cast<const b2f_path_elem *>(static_cast<uint8_t *>(ex->d_table) + h.elems_off);
    sp.n_paths = (int)h.n_paths;
    sp.n_cat = (int)h.n_cat;
    sp.n_num = (int)h.n_num;
    sp.denom = h.denom;
    memcpy(sp.impute, m->hdr.impute, sizeof(sp.impute));
    ex->maxl = h.max_len <= 9 ? 9 : (h.max_len <= 16 ? 16 : 24);
    inter_assign(static_cast<const uint8_t *>(paths), h, ex->ip.own);
    /* the EXTEND / UNWIND factors (no division in the kernel) */
    double tab[4][B2F_SHAP_TAB_L][B2F_SHAP_TAB_L]; /* per call: concurrent attaches (other handles) share nothing on the host */
    for (int l = 0; l < B2F_SHAP_TAB_L; ++l)
        for (int i = 0; i < B2F_SHAP_TAB_L; ++i) {
            tab[0][l][i] = (i + 1.0) / (l + 1.0);
            tab[1][l][i] = (l - i) / (l + 1.0);
            tab[2][l][i] = (l + 1.0) / (i + 1.0);
            tab[3][l][i] = l > i ? (l + 1.0) / (l - i) : 0.0;
        }
    cudaError_t e = cudaMemcpyToSymbol(c_shap_tab, tab, sizeof(tab));
    for (int v = 0; v < SHAP_VARIANTS; ++v) {
        ExplainKernel &k = ex->kernels[v];
        const int F = sp.n_cat + sp.n_num;
        k.smem_bytes = v == SHAP_INTERACTIONS ? inter_smem_bytes(F) : (v == SHAP_INTERVENTIONAL ? interv_smem_bytes(F) : shap_smem_bytes(F));
        for (bool pk : {false, true})
            if (e == cudaSuccess) e = set_smem_limit(explain_kernel(v, ex->maxl, pk), k.smem_bytes);
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&k.ctas_per_sm, explain_kernel(v, ex->maxl, false), B2F_SHAP_THREADS, k.smem_bytes);
        k.ctas_per_sm = std::max(1, k.ctas_per_sm);
    }
    if (e != cudaSuccess) return fail(set_err(B2F_ECUDA, "explainer set-up failed: %s", cudaGetErrorString(e)));
    if (m->ex) explainer_free(m->ex); /* the device was synchronised above */
    m->ex = ex;
    return B2F_OK;
}

/* b2f_explain / b2f_explain_interactions / b2f_explain_interventional: a host job of variant v */
static int explain_host(b2f_model *m, const void *rows, int64_t n, int row_format, double *out, int v, double *base_value, float *device_ms) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (!m->ex) return set_err(B2F_ESTATE, "no explainer attached (b2f_model_attach_explainer)");
    if (base_value) *base_value = v == SHAP_INTERVENTIONAL ? m->ex->bg.base_value : m->ex->hdr.base_value;
    if (device_ms) *device_ms = 0.0f;
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    int rc = explain_check(m, row_format, v, out || n == 0);
    if (rc) return rc;
    const HostJob job{explain_row_bytes(m, v), v == SHAP_INTERACTIONS ? B2F_INTER_CHUNK_ROWS : 0, false, v,
                      [](b2f_model *m, int v, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, void *out_dev, int32_t *, DevBuf &scratch) {
                          return launch_explain(m, st, rows_dev, n, fmt, v, static_cast<double *>(out_dev), scratch);
                      }};
    return timed_host_batch(m, job, rows, n, row_format, out, device_ms);
}

extern "C" int b2f_explain(b2f_model *m, const void *rows, int64_t n, int row_format, double *phi, double *base_value, float *device_ms) {
    return explain_host(m, rows, n, row_format, phi, SHAP_PHI, base_value, device_ms);
}
extern "C" int b2f_explain_interactions(b2f_model *m, const void *rows, int64_t n, int row_format, double *phi2, double *base_value,
                                        float *device_ms) {
    return explain_host(m, rows, n, row_format, phi2, SHAP_INTERACTIONS, base_value, device_ms);
}

/* b2f_explain_device / b2f_explain_interactions_device / b2f_explain_interventional_device */
static int explain_device(b2f_model *m, const void *rows_dev, int64_t n, int row_format, double *out_dev, int v) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    if (!m->ex) return set_err(B2F_ESTATE, "no explainer attached (b2f_model_attach_explainer)");
    int rc = explain_check(m, row_format, v, out_dev != nullptr || n == 0);
    if (rc == B2F_OK) rc = check_row_format(m, row_format);
    if (rc) return rc;
    CUDA_TRY(cudaSetDevice(m->device));
    return launch_explain(m, m->compute, rows_dev, n, row_format, v, out_dev, m->scratch);
}
extern "C" int b2f_explain_device(b2f_model *m, const void *rows_dev, int64_t n, int row_format, double *phi_dev) {
    return explain_device(m, rows_dev, n, row_format, phi_dev, SHAP_PHI);
}
extern "C" int b2f_explain_interactions_device(b2f_model *m, const void *rows_dev, int64_t n, int row_format, double *phi2_dev) {
    return explain_device(m, rows_dev, n, row_format, phi2_dev, SHAP_INTERACTIONS);
}

/* The background table of n host rows (tree_shap_interventional.cuh): the rows' imputed words in tiles, a counting pass,
 * the offsets (scanned on the host), one allocation sized from them, a fill pass.  base_value = the path table's
 * path-dependent base value plus each path's move to the background mean (k_background_table), added in path order. */
extern "C" int b2f_model_attach_background(b2f_model *m, const void *rows, int64_t n, int row_format, size_t *table_bytes) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    if (!m->ex) return set_err(B2F_ESTATE, "no explainer attached (b2f_model_attach_explainer)");
    if (n <= 0) return set_err(B2F_EINVAL, "background needs at least one row (n = %lld)", (long long)n);
    if (!rows) return set_err(B2F_EINVAL, "rows is NULL");
    int rc = check_value_rows(row_format, "a background takes");
    if (rc == B2F_OK) rc = check_row_format(m, row_format);
    if (rc) return rc;
    CUDA_TRY(cudaSetDevice(m->device));
    Explainer &ex = *m->ex;
    const int64_t P = ex.hdr.n_paths, tiles = (n + 31) / 32;
    const int F = explain_fields(m);
    const bool pk = row_format == B2F_ROWS_PACKED64;
    Background bg;
    bg.rows = n;
    bg.vp.s = ex.ip.s;
    bg.vp.s.denom = ex.hdr.denom * (double)n;
    void *d_rows = nullptr, *d_words = nullptr, *d_counts = nullptr, *d_moved = nullptr;
    auto done = [&](int code) { /* frees the scratch, and the new table unless it was attached */
        for (void *b : {d_rows, d_words, d_counts, d_moved})
            if (b) cudaFree(b);
        if (code != B2F_OK && bg.d_table) cudaFree(bg.d_table);
        return code;
    };
    auto cuda_fail = [&](const char *what) {
        return done(set_err(B2F_ECUDA, "background %s failed: %s", what, cudaGetErrorString(cudaGetLastError())));
    };
    const size_t rows_bytes = (size_t)n * row_bytes_of(m, row_format), words_bytes = (size_t)tiles * F * 32 * sizeof(uint32_t);
    if (cudaMalloc(&d_rows, rows_bytes) != cudaSuccess || cudaMalloc(&d_words, words_bytes) != cudaSuccess ||
        cudaMalloc(&d_counts, (size_t)std::max<int64_t>(P, 1) * sizeof(long long)) != cudaSuccess ||
        cudaMalloc(&d_moved, (size_t)std::max<int64_t>(P, 1) * sizeof(double)) != cudaSuccess)
        return done(set_err(B2F_ENOMEM, "background scratch (%zu bytes of rows, %zu of words) allocation failed: %s", rows_bytes, words_bytes,
                            cudaGetErrorString(cudaGetLastError())));
    if (cudaMemcpy(d_rows, rows, rows_bytes, cudaMemcpyHostToDevice) != cudaSuccess) return cuda_fail("upload");
    const uint32_t *rw = static_cast<const uint32_t *>(d_rows);
    uint32_t *words = static_cast<uint32_t *>(d_words);
    long long *counts = static_cast<long long *>(d_counts);
    double *moved = static_cast<double *>(d_moved);
    if (pk)
        k_background_words<true><<<(unsigned)tiles, B2F_SHAP_THREADS>>>(bg.vp.s, rw, (long long)n, words);
    else
        k_background_words<false><<<(unsigned)tiles, B2F_SHAP_THREADS>>>(bg.vp.s, rw, (long long)n, words);
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(P, (int64_t)m->sm_count * 32));
    if (P) k_background_table<false><<<grid, B2F_SHAP_THREADS>>>(bg.vp, words, (long long)n, counts, nullptr, nullptr);
    if (cudaGetLastError() != cudaSuccess) return cuda_fail("counting pass");
    std::vector<long long> off((size_t)P + 1, 0);
    if (P && cudaMemcpy(off.data() + 1, counts, (size_t)P * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess)
        return cuda_fail("counting pass");
    for (int64_t p = 0; p < P; ++p) off[p + 1] += off[p];
    const size_t off_bytes = off.size() * sizeof(long long);
    bg.bytes = off_bytes + (size_t)off[P] * sizeof(uint2);
    if (cudaMalloc(&bg.d_table, bg.bytes) != cudaSuccess) {
        bg.d_table = nullptr;
        return done(set_err(B2F_ENOMEM, "background table (%zu bytes) allocation failed: %s", bg.bytes, cudaGetErrorString(cudaGetLastError())));
    }
    bg.vp.offsets = static_cast<const long long *>(bg.d_table);
    bg.vp.entries = reinterpret_cast<const uint2 *>(static_cast<uint8_t *>(bg.d_table) + off_bytes);
    if (cudaMemcpy(bg.d_table, off.data(), off_bytes, cudaMemcpyHostToDevice) != cudaSuccess) return cuda_fail("offsets upload");
    if (P)
        k_background_table<true><<<grid, B2F_SHAP_THREADS>>>(bg.vp, words, (long long)n, nullptr, const_cast<uint2 *>(bg.vp.entries), moved);
    if (cudaGetLastError() != cudaSuccess) return cuda_fail("fill pass");
    std::vector<double> mv((size_t)P);
    if (P && cudaMemcpy(mv.data(), moved, (size_t)P * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) return cuda_fail("fill pass");
    double sum = 0.0;
    for (double v : mv) sum += v;
    bg.base_value = ex.hdr.base_value + sum / ex.hdr.denom;
    /* replacing a background: nothing may still read the old table */
    if (cudaDeviceSynchronize() != cudaSuccess) return cuda_fail("synchronise");
    if (ex.bg.d_table) cudaFree(ex.bg.d_table);
    ex.bg = bg;
    if (table_bytes) *table_bytes = bg.bytes;
    return done(B2F_OK);
}

extern "C" int b2f_explain_interventional(b2f_model *m, const void *rows, int64_t n, int row_format, double *phi, double *base_value,
                                          float *device_ms) {
    return explain_host(m, rows, n, row_format, phi, SHAP_INTERVENTIONAL, base_value, device_ms);
}
extern "C" int b2f_explain_interventional_device(b2f_model *m, const void *rows_dev, int64_t n, int row_format, double *phi_dev) {
    return explain_device(m, rows_dev, n, row_format, phi_dev, SHAP_INTERVENTIONAL);
}
