/*
 * drift_api.cuh -- C ABI of the batch drift detector (include/b2f.h, b2f_drift_*); included by b2f_api.cu.
 *
 * Host side of K3 (drift_stats.cuh): the reference table lives in HBM from b2f_drift_create on (numeric columns
 * pre-sorted, category counts pre-computed -- the reference re-derives both on every request,
 * databricks/src/02-register-model.ipynb:338); a request costs two small H2D copies, one memset of the
 * histograms, two kernels and one D2H copy of 23 (p, statistic, flag) triples.
 */
#pragma once
#include "drift_stats.cuh"

struct b2f_drift {
    int device = 0;
    int sm_count = 0;
    int64_t n_ref = 0;
    int n_num = 0, n_cat = 0;
    int cat_total = 0;
    std::vector<int32_t> cat_off; /* host copy */
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    double *d_ref = nullptr;
    int32_t *d_cat_off = nullptr;
    int64_t *d_ref_counts = nullptr;
    void *d_hist = nullptr; /* hist_a | hist_b | nan_count | cat_hist, one memset */
    size_t hist_bytes = 0;
    DevBuf x, codes; /* the batch's numeric columns and category codes, n + n/2 rows' worth */
    int32_t *d_new_off = nullptr;
    DevBuf new_counts;
    double *d_rows = nullptr; /* row-scan scratch: [n_num][2][B2F_DRIFT_ROW_STRIDE(n_ref)] */
    int rowscan_max_n = 0, rowscan_smem_max_n = 0;
    DevBuf wide; /* wide-band sweep scratch: [n_num][2][ring slots] for the widest ring a batch needed so far */
    size_t finish_smem = 0;
    void *d_out = nullptr; /* p_val[F] | stat[F] | flags[F] */
    void *h_out = nullptr; /* pinned mirror */
    int64_t launches = 0;
};

extern "C" void b2f_drift_destroy(b2f_drift *d) {
    if (!d) return;
    cudaSetDevice(d->device);
    if (d->stream) cudaStreamSynchronize(d->stream);
    if (d->d_ref) cudaFree(d->d_ref);
    if (d->d_cat_off) cudaFree(d->d_cat_off);
    if (d->d_ref_counts) cudaFree(d->d_ref_counts);
    if (d->d_hist) cudaFree(d->d_hist);
    for (DevBuf *b : {&d->x, &d->codes, &d->new_counts, &d->wide}) b->release();
    if (d->d_new_off) cudaFree(d->d_new_off);
    if (d->d_rows) cudaFree(d->d_rows);
    if (d->d_out) cudaFree(d->d_out);
    if (d->h_out) cudaFreeHost(d->h_out);
    if (d->ev0) cudaEventDestroy(d->ev0);
    if (d->ev1) cudaEventDestroy(d->ev1);
    if (d->stream) cudaStreamDestroy(d->stream);
    delete d;
}

static int drift_init(b2f_drift *d, const double *ref_sorted, const int32_t *cat_sizes, const int64_t *ref_counts) {
    CUDA_TRY(cudaSetDevice(d->device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, d->device));
    if (prop.major != 9 || prop.minor != 0) return set_err(B2F_ENODEV, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", d->device, prop.major, prop.minor);
    d->sm_count = prop.multiProcessorCount;
    d->cat_off.assign(d->n_cat + 1, 0);
    for (int c = 0; c < d->n_cat; ++c) {
        if (cat_sizes[c] < 0 || cat_sizes[c] > B2F_DRIFT_MAX_CATS) return set_err(B2F_EINVAL, "drift: categorical feature %d has %d reference categories (max %d)", c, cat_sizes[c], B2F_DRIFT_MAX_CATS);
        d->cat_off[c + 1] = d->cat_off[c] + cat_sizes[c];
    }
    d->cat_total = d->cat_off[d->n_cat];
    for (int f = 0; f < d->n_num; ++f) {
        if (ref_sorted[(int64_t)f * d->n_ref] != ref_sorted[(int64_t)f * d->n_ref]) /* the loop below sees a NaN only after row 0 */
            return set_err(B2F_EINVAL, "drift: reference column %d holds NaN at row 0", f);
        for (int64_t j = 1; j < d->n_ref; ++j)
            if (!(ref_sorted[(int64_t)f * d->n_ref + j - 1] <= ref_sorted[(int64_t)f * d->n_ref + j]))
                return set_err(B2F_EINVAL, "drift: reference column %d is not sorted ascending (or holds NaN) at row %lld", f, (long long)j);
    }
    CUDA_TRY(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreate(&d->ev0));
    CUDA_TRY(cudaEventCreate(&d->ev1));
    const size_t ref_bytes = (size_t)d->n_num * d->n_ref * sizeof(double);
    CUDA_TRY(cudaMalloc((void **)&d->d_ref, std::max<size_t>(ref_bytes, 8)));
    CUDA_TRY(cudaMemcpy(d->d_ref, ref_sorted, ref_bytes, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc((void **)&d->d_cat_off, (d->n_cat + 1) * sizeof(int32_t)));
    CUDA_TRY(cudaMemcpy(d->d_cat_off, d->cat_off.data(), (d->n_cat + 1) * sizeof(int32_t), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc((void **)&d->d_ref_counts, std::max<size_t>((size_t)d->cat_total * sizeof(int64_t), 8)));
    if (d->cat_total) CUDA_TRY(cudaMemcpy(d->d_ref_counts, ref_counts, (size_t)d->cat_total * sizeof(int64_t), cudaMemcpyHostToDevice));
    d->hist_bytes = ((size_t)2 * d->n_num * (d->n_ref + 1) + d->n_num + d->cat_total) * sizeof(uint32_t);
    CUDA_TRY(cudaMalloc(&d->d_hist, std::max<size_t>(d->hist_bytes, 8)));
    const int F = d->n_num + d->n_cat;
    const size_t out_bytes = (size_t)F * (2 * sizeof(double) + sizeof(int32_t));
    CUDA_TRY(cudaMalloc(&d->d_out, out_bytes));
    CUDA_TRY(cudaHostAlloc(&d->h_out, out_bytes, cudaHostAllocPortable));
    CUDA_TRY(cudaMalloc((void **)&d->d_new_off, (d->n_cat + 1) * sizeof(int32_t)));
    /* row-scan form of the exact p-value for request-sized batches (B2F_DRIFT_ROWSCAN=0 keeps the anti-diagonal sweep) */
    d->rowscan_max_n = B2F_DRIFT_ROWSCAN_MAX;
    if (const char *rs = getenv("B2F_DRIFT_ROWSCAN")) d->rowscan_max_n = std::max(0, std::min(B2F_DRIFT_ROWSCAN_MAX, atoi(rs)));
    if (d->rowscan_max_n > 0 && d->n_num > 0 && d->n_ref >= 1024)
        CUDA_TRY(cudaMalloc((void **)&d->d_rows, (size_t)d->n_num * 2 * (size_t)B2F_DRIFT_ROW_STRIDE(d->n_ref) * sizeof(double)));
    /* B2F_DRIFT_ROWSCAN=0 switches both row-scan forms off; B2F_DRIFT_ROWSCAN_SMEM=<n> caps the shared-memory form alone */
    d->rowscan_smem_max_n = getenv("B2F_DRIFT_ROWSCAN") && d->rowscan_max_n == 0 ? 0 : B2F_DRIFT_ROWSCAN_SMEM_MAX;
    if (const char *rs = getenv("B2F_DRIFT_ROWSCAN_SMEM")) d->rowscan_smem_max_n = std::max(0, std::min(B2F_DRIFT_ROWSCAN_SMEM_LIMIT, atoi(rs)));
    d->finish_smem = 2 * B2F_DRIFT_RING_MAX * sizeof(double);
    if (d->rowscan_smem_max_n > 0) d->finish_smem = std::max(d->finish_smem, (size_t)B2F_DRIFT_ROWSCAN_CAP * sizeof(double));
    CUDA_TRY(set_smem_limit(k_drift_finish, (int)std::max<size_t>(d->finish_smem, (size_t)B2F_DRIFT_ROWSCAN_CAP * sizeof(double))));
    return B2F_OK;
}

extern "C" b2f_drift *b2f_drift_create(int device, int64_t n_ref, int n_num, const double *ref_sorted, int n_cat, const int32_t *cat_sizes,
                                       const int64_t *ref_counts) {
    int ndev = b2f_device_count();
    if (ndev < 0) return nullptr;
    if (device < 0 || device >= ndev) {
        set_err(B2F_EINVAL, "device %d out of range (have %d)", device, ndev);
        return nullptr;
    }
    if (n_ref < 1 || n_ref > (1 << 26) || n_num < 0 || n_cat < 0 || n_num + n_cat < 1 || n_num + n_cat > 1024 || (n_num > 0 && !ref_sorted) ||
        (n_cat > 0 && (!cat_sizes || !ref_counts))) {
        set_err(B2F_EINVAL, "drift: bad reference table description");
        return nullptr;
    }
    b2f_drift *d = new (std::nothrow) b2f_drift();
    if (!d) {
        set_err(B2F_ENOMEM, "out of host memory");
        return nullptr;
    }
    d->device = device;
    d->n_ref = n_ref;
    d->n_num = n_num;
    d->n_cat = n_cat;
    if (drift_init(d, ref_sorted, cat_sizes, ref_counts) != B2F_OK) {
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        b2f_drift_destroy(d);
        memcpy(g_err, keep, sizeof(keep));
        return nullptr;
    }
    return d;
}

/* ---- the asymptotic branch of scipy's ks_2samp, natively (host; a handful of scalar formulas) ---------------------------------
 * Where lcm(m, n) >= 2^31 scipy itself leaves the exact lattice-path method and returns kstwo.sf(D, round(m n / (m + n)))
 * (scipy/stats/_stats_py.py `_attempt_exact_2kssamp` / `ks_2samp`), i.e. the ONE-sample two-sided K-S survival function
 * `scipy.stats._ksstats._kolmogn(n, x, cdf=False)` (Simard & L'Ecuyer 2011).  Its decision tree is restated here for the
 * sample sizes that can reach this branch (n_eff in the thousands):
 *   n x <= 1 and n x >= n - 1        Ruben-Gambino closed forms
 *   x >= 0.5, or n x^2 >= 2.2        2 * Smirnov's one-sided exact formula  P(D+ >= x) = x sum_j C(n,j) (x + j/n)^(j-1) (1 - x - j/n)^(n-j)
 *                                    (all terms positive: summed in log space, lgamma-limited to ~1e-10 relative)
 *   n x^2 >= 370                     0
 *   otherwise                        1 - Pelz-Good (1976) four-term expansion of the CDF  (scipy runs Durbin's matrix algorithm
 *                                    for n x^1.5 <= 1.4; there the CDF is below 1e-8 and both agree to ~1e-13 in the survival value)
 * Checked against scipy itself in tests/test_drift_cpu.py.  The response carries float32 p-values. */
static double smirnov_sf(double n, double x) {
    if (x <= 0.0) return 1.0;
    if (x >= 1.0) return 0.0;
    const double lgn = lgamma(n + 1.0);
    double sum = 0.0;
    const double jmax = floor(n * (1.0 - x));
    for (double j = 0.0; j <= jmax; j += 1.0) {
        const double a = x + j / n, b = 1.0 - x - j / n;
        if (b < 0.0) break;
        double lt = lgn - lgamma(j + 1.0) - lgamma(n - j + 1.0) + (j - 1.0) * log(a);
        if (n - j > 0.0) {
            if (b <= 0.0) continue;
            lt += (n - j) * log(b);
        }
        sum += exp(lt);
    }
    return std::min(1.0, std::max(0.0, x * sum));
}

static double pelz_good_cdf(double n, double x) {
    const double PI = 3.14159265358979323846, PI2 = PI * PI, PI4 = PI2 * PI2, PI6 = PI4 * PI2;
    const double z = sqrt(n) * x, z2 = z * z, z3 = z2 * z, z4 = z2 * z2, z6 = z4 * z2, z8 = z4 * z4;
    const double qlog = -PI2 / 8.0 / z2;
    if (qlog < -745.0) return 0.0;
    double q = exp(qlog);
    const double k1a = -z2, k1b = PI2 / 4.0;
    const double k2a = 6.0 * z6 + 2.0 * z4, k2b = (2.0 * z4 - 5.0 * z2) * PI2 / 4.0, k2c = PI4 * (1.0 - 2.0 * z2) / 16.0;
    const double k3d = PI6 * (5.0 - 30.0 * z2) / 64.0, k3c = PI4 * (-60.0 * z2 + 212.0 * z4) / 16.0, k3b = PI2 * (135.0 * z4 - 96.0 * z6) / 4.0,
                 k3a = -30.0 * z6 - 90.0 * z8;
    double K[4] = {0.0, 0.0, 0.0, 0.0};
    const int maxk = (int)ceil(16.0 * z / PI);
    for (int k = maxk; k > 0; --k) {
        const double m = 2.0 * k - 1.0, m2 = m * m, m4 = m2 * m2, m6 = m4 * m2;
        const double qp = pow(q, 8.0 * k);
        const double c[4] = {1.0, k1a + k1b * m2, k2a + k2b * m2 + k2c * m4, k3a + k3b * m2 + k3c * m4 + k3d * m6};
        for (int i = 0; i < 4; ++i) K[i] = K[i] * qp + c[i];
    }
    const double SQRT2PI = sqrt(2.0 * PI);
    const double div[4] = {z, 6.0 * z4, 72.0 * z4 * z3, 6480.0 * z8 * z2};
    for (int i = 0; i < 4; ++i) K[i] = K[i] * q * SQRT2PI / div[i];
    q = exp(-PI2 / 2.0 / z2);
    double k2e = 0.0, k3e = 0.0;
    const double s3z = sqrt(3.0) * z;
    for (int k = maxk; k > 0; --k) {
        const double k2 = (double)k * k, qp = pow(q, k2), kp = PI * k;
        k2e += k2 * qp;
        k3e += (s3z + kp) * (s3z - kp) * k2 * qp;
    }
    K[2] += k2e * PI2 * SQRT2PI / (-36.0 * z3);
    K[3] += k3e * PI2 * SQRT2PI / (216.0 * z6);
    return K[0] + K[1] / sqrt(n) + K[2] / n + K[3] / (n * sqrt(n));
}

/* scipy.stats.kstwo.sf(x, n): survival function of the one-sample two-sided K-S statistic (large n) */
extern "C" double b2f_kstwo_sf(double x, double n) {
    if (!(n >= 1.0) || x != x) return nan("");
    auto clip = [](double p) { return std::min(1.0, std::max(0.0, p)); };
    if (x >= 1.0) return 0.0;
    if (x <= 0.0) return 1.0;
    const double t = n * x;
    if (t <= 1.0) {
        if (t <= 0.5) return 1.0;
        const double cdf = exp(lgamma(n + 1.0) - n * log(n) + n * log(2.0 * t - 1.0));
        return clip(1.0 - cdf);
    }
    if (t >= n - 1.0) return clip(2.0 * pow(1.0 - x, n));
    if (x >= 0.5) return clip(2.0 * smirnov_sf(n, x));
    const double nx2 = t * x;
    if (nx2 >= 370.0) return 0.0;
    if (nx2 >= 2.2) return clip(2.0 * smirnov_sf(n, x));
    return clip(1.0 - pelz_good_cdf(n, x));
}

extern "C" int b2f_drift_score(b2f_drift *d, int64_t n, const double *num_cols, const int32_t *cat_codes, const int32_t *new_offsets,
                               const int64_t *new_counts, double *p_val, double *stat, int32_t *flags, float *device_ms) {
    if (!d) return set_err(B2F_EINVAL, "drift handle is NULL");
    if (n < 1) return set_err(B2F_EINVAL, "drift: the batch must hold at least one row"); /* scipy: "Data passed to ks_2samp must not be empty" */
    if ((d->n_num > 0 && !num_cols) || (d->n_cat > 0 && !cat_codes) || !p_val) return set_err(B2F_EINVAL, "drift: NULL argument");
    if (n > (1 << 26)) return set_err(B2F_EINVAL, "drift: batch too large");
    CUDA_TRY(cudaSetDevice(d->device));
    const size_t cap = (size_t)std::max<int64_t>(n + n / 2, 1024), x_row = d->n_num * sizeof(double), codes_row = d->n_cat * sizeof(int32_t);
    int rc = d->x.reserve(d->stream, std::max<size_t>(n * x_row, 8), std::max<size_t>(cap * x_row, 8));
    if (rc == B2F_OK) rc = d->codes.reserve(d->stream, std::max<size_t>(n * codes_row, 8), std::max<size_t>(cap * codes_row, 8));
    if (rc) return rc;
    /* the widest sweep ring this batch size can need (h <= lcm: D <= 1); beyond B2F_DRIFT_RING_MAX slots the sweep keeps its two
     * rings in a global scratch.  Where lcm >= 2^31 (flag 1) no sweep runs. */
    int64_t wide_need = 0;
    if (d->n_num > 0) {
        int64_t g = d->n_ref;
        for (int64_t b = n; b;) {
            const int64_t t = g % b;
            g = b;
            b = t;
        }
        const int64_t mg = std::max(d->n_ref, n) / g, ng = std::min(d->n_ref, n) / g;
        if ((double)(d->n_ref / g) < 2147483647.0 / (double)(n / g)) {
            const int64_t width = (2 * mg * ng * g) / (ng + mg) + 2;
            int64_t ring = 32;
            while (ring < width + 3) ring <<= 1;
            if (ring > B2F_DRIFT_RING_MAX) wide_need = ring;
        }
    }
    const size_t wide_slot = (size_t)d->n_num * 2 * sizeof(double); /* bytes per ring slot over the features */
    if ((rc = d->wide.reserve(d->stream, wide_slot * wide_need, wide_slot * wide_need))) return rc;
    int64_t n_new = 0;
    if (new_offsets) {
        if (!new_counts && new_offsets[d->n_cat] > 0) return set_err(B2F_EINVAL, "drift: new_counts is NULL");
        for (int c = 0; c < d->n_cat; ++c) {
            const int k = new_offsets[c + 1] - new_offsets[c];
            if (k < 0 || k + (d->cat_off[c + 1] - d->cat_off[c]) > B2F_DRIFT_MAX_CATS) return set_err(B2F_EINVAL, "drift: too many categories for feature %d", c);
        }
        n_new = new_offsets[d->n_cat];
        if ((rc = d->new_counts.reserve(d->stream, (size_t)n_new * sizeof(int64_t), (size_t)(n_new + 64) * sizeof(int64_t)))) return rc;
        CUDA_TRY(cudaMemcpyAsync(d->d_new_off, new_offsets, (d->n_cat + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, d->stream));
        if (n_new) CUDA_TRY(cudaMemcpyAsync(d->new_counts.p, new_counts, (size_t)n_new * sizeof(int64_t), cudaMemcpyHostToDevice, d->stream));
    }
    const int F = d->n_num + d->n_cat;
    CUDA_TRY(cudaEventRecord(d->ev0, d->stream));
    /* the batch arrives feature-major with stride n: one copy per kind */
    if (d->n_num) CUDA_TRY(cudaMemcpyAsync(d->x.p, num_cols, (size_t)n * d->n_num * sizeof(double), cudaMemcpyHostToDevice, d->stream));
    if (d->n_cat) CUDA_TRY(cudaMemcpyAsync(d->codes.p, cat_codes, (size_t)n * d->n_cat * sizeof(int32_t), cudaMemcpyHostToDevice, d->stream));
    CUDA_TRY(cudaMemsetAsync(d->d_hist, 0, d->hist_bytes, d->stream));
    DriftParams p;
    memset(&p, 0, sizeof(p));
    p.n_ref = d->n_ref;
    p.n = n;
    p.n_num = d->n_num;
    p.n_cat = d->n_cat;
    p.ref_sorted = d->d_ref;
    p.x = static_cast<double *>(d->x.p);
    p.codes = static_cast<int32_t *>(d->codes.p);
    uint32_t *hp = static_cast<uint32_t *>(d->d_hist);
    p.hist_a = hp;
    p.hist_b = hp + (size_t)d->n_num * (d->n_ref + 1);
    p.nan_count = hp + (size_t)2 * d->n_num * (d->n_ref + 1);
    p.cat_hist = p.nan_count + d->n_num;
    p.cat_off = d->d_cat_off;
    p.ref_counts = d->d_ref_counts;
    p.new_off = new_offsets ? d->d_new_off : nullptr;
    p.new_counts = static_cast<int64_t *>(d->new_counts.p);
    p.p_val = static_cast<double *>(d->d_out);
    p.stat = p.p_val + F;
    p.flags = reinterpret_cast<int32_t *>(p.stat + F);
    p.row_scratch = d->d_rows;
    p.rowscan_max_n = d->rowscan_max_n;
    p.rowscan_smem_max_n = (n >= 2 && n <= d->rowscan_smem_max_n) ? d->rowscan_smem_max_n : 0;
    p.rowscan_cap = B2F_DRIFT_ROWSCAN_CAP;
    p.wide_scratch = static_cast<double *>(d->wide.p);
    p.wide_ring = d->n_num ? (int64_t)(d->wide.bytes / wide_slot) : 0;
    const int64_t total = n * F;
    const unsigned blocks = (unsigned)std::max<int64_t>(1, std::min<int64_t>((total + 255) / 256, (int64_t)d->sm_count * 8));
    k_drift_count<<<blocks, 256, 0, d->stream>>>(p);
    /* the big shared-memory ring only when this batch can take the shared-memory row scan: with 208 KB of shared memory the SM
     * keeps almost no L1, which the first part of the kernel (histogram scan) and k_drift_count's searches like to have */
    const size_t ring_smem = 2 * B2F_DRIFT_RING_MAX * sizeof(double);
    static const bool force_big = getenv("B2F_DRIFT_FORCE_BIG_SMEM") != nullptr; /* experiment: the cost of the big launch alone */
    const size_t smem = ((n >= 2 && n <= d->rowscan_smem_max_n) || force_big) ? std::max(d->finish_smem, (size_t)B2F_DRIFT_ROWSCAN_CAP * sizeof(double)) : ring_smem;
    k_drift_finish<<<(unsigned)F, B2F_DRIFT_THREADS, smem, d->stream>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_err(B2F_ECUDA, "drift kernel launch failed: %s", cudaGetErrorString(e));
    d->launches += 2;
    const size_t out_bytes = (size_t)F * (2 * sizeof(double) + sizeof(int32_t));
    CUDA_TRY(cudaMemcpyAsync(d->h_out, d->d_out, out_bytes, cudaMemcpyDeviceToHost, d->stream));
    CUDA_TRY(cudaEventRecord(d->ev1, d->stream));
    CUDA_TRY(cudaStreamSynchronize(d->stream));
    double *hp_p = static_cast<double *>(d->h_out);
    {
        /* flag 1 (lcm of the sample sizes >= 2^31): scipy's own asymptotic branch, kstwo.sf(D, round(m n / (m + n))) */
        const int32_t *hf = reinterpret_cast<const int32_t *>(hp_p + 2 * F);
        const double en = nearbyint((double)d->n_ref * (double)n / ((double)d->n_ref + (double)n));
        for (int f = 0; f < F; ++f)
            if (hf[f] == 1) hp_p[f] = b2f_kstwo_sf(hp_p[F + f], en);
    }
    memcpy(p_val, hp_p, (size_t)F * sizeof(double));
    if (stat) memcpy(stat, hp_p + F, (size_t)F * sizeof(double));
    if (flags) memcpy(flags, hp_p + 2 * F, (size_t)F * sizeof(int32_t));
    if (device_ms) CUDA_TRY(cudaEventElapsedTime(device_ms, d->ev0, d->ev1));
    return B2F_OK;
}

extern "C" int64_t b2f_drift_launches(const b2f_drift *d) { return d ? d->launches : 0; }
