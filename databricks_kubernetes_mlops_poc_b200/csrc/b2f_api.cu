/*
 * b2f_api.cu -- C ABI (include/b2f.h) of libb200forest.so: model lifetime, the pinned-ring /
 * multi-stream staging around the kernels, timing helpers and the NCCL plumbing.
 *
 * The reference's counterpart of this file is Python glue: `lifespan` loading the model
 * (reference app/main.py:20-31), `CustomModel.load_context` / `.predict`
 * (databricks/src/02-register-model.ipynb:317-353).  Here the model is a flattened forest in HBM
 * and "predict" is H2D copy -> one fused kernel -> D2H copy, pipelined over CUDA streams.
 * There is no CPU fallback anywhere in this file: no device, no result.
 */
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <limits.h>
#include <nccl.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <mutex>
#include <string>
#include <thread>
#include <new>
#include <vector>

#include "../../include/b2f.h"
#include "feature_moments.cuh"
#include "forest_blob.h"
#include "forest_predict.cuh"
#include "forest_predict_tile.cuh"
#include "forest_predict_rank.cuh"
#include "forest_rank.h"
#include "partial_dependence.cuh"
#include "counterfactual.cuh"
#include "permutation_importance.cuh"
#include "pair_dependence.cuh"
#include "ale.cuh"
#include "mmd_drift.cuh"
#include "mmd_online.cuh"
#include "knn.cuh"
#include "tree_shap.cuh"
#include "tree_shap_interactions.cuh"
#include "tree_shap_interventional.cuh"
#include "json_rows.h"
#include "row_encoder.h"

#define B2F_VERSION_STR "b200forest 0.1.0 (sm_90a)"
#define B2F_STREAMS 4
#define B2F_TICKETS 256
#define B2F_CHUNK_ROWS 16384
#define B2F_FLUSH_BYTES (256ull << 20) /* > 50 MB L2 */

/* ------------------------------------------------------------------ errors */
static thread_local char g_err[512] = "";

static int set_err(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CUDA_TRY(expr)                                                                         \
    do {                                                                                       \
        cudaError_t e_ = (expr);                                                               \
        if (e_ != cudaSuccess)                                                                 \
            return set_err(B2F_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

extern "C" const char *b2f_last_error(void) { return g_err; }
extern "C" const char *b2f_version(void) { return B2F_VERSION_STR; }

extern "C" int b2f_device_count(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) return set_err(B2F_ENODEV, "no CUDA device: %s", cudaGetErrorString(e));
    return n;
}

/* ------------------------------------------------------------------ NCCL (lazy dlopen) */
struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t *, int, const int *) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)(void) = nullptr;
    ncclResult_t (*GroupEnd)(void) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;

static int nccl_load(void) {
    if (g_nccl.handle) return B2F_OK;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    void *h = nullptr;
    for (const char *nm : names) {
        h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
        if (h) break;
    }
    if (!h) return set_err(B2F_ENCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
#define LOADSYM(field, sym)                                                        \
    do {                                                                           \
        *(void **)(&g_nccl.field) = dlsym(h, sym);                                 \
        if (!g_nccl.field) return set_err(B2F_ENCCL, "NCCL symbol %s missing", sym); \
    } while (0)
    LOADSYM(GetUniqueId, "ncclGetUniqueId");
    LOADSYM(CommInitRank, "ncclCommInitRank");
    LOADSYM(CommInitAll, "ncclCommInitAll");
    LOADSYM(CommDestroy, "ncclCommDestroy");
    LOADSYM(AllGather, "ncclAllGather");
    LOADSYM(GroupStart, "ncclGroupStart");
    LOADSYM(GroupEnd, "ncclGroupEnd");
    LOADSYM(GetErrorString, "ncclGetErrorString");
#undef LOADSYM
    g_nccl.handle = h;
    return B2F_OK;
}
#define NCCL_TRY(expr)                                                                                      \
    do {                                                                                                    \
        ncclResult_t r_ = (expr);                                                                           \
        if (r_ != ncclSuccess) return set_err(B2F_ENCCL, "%s failed: %s", #expr, g_nccl.GetErrorString(r_)); \
    } while (0)

/* ------------------------------------------------------------------ model */
/* A device buffer grown on demand and used by one stream at a time.  reserve: when need exceeds the capacity, wait for the
 * stream st, which orders every use of the buffer, then free it and allocate alloc bytes; a failed allocation leaves it empty. */
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    int reserve(cudaStream_t st, size_t need, size_t alloc) {
        if (need <= bytes) return B2F_OK;
        CUDA_TRY(cudaStreamSynchronize(st));
        release();
        const cudaError_t e = cudaMalloc(&p, alloc);
        if (e != cudaSuccess) {
            p = nullptr;
            return set_err(B2F_ECUDA, "cudaMalloc(%zu bytes) failed: %s", alloc, cudaGetErrorString(e));
        }
        bytes = alloc;
        return B2F_OK;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
};

/* one stream of the host pipeline and a chunk's device buffers, whatever the job: chunks on a slot are ordered by its stream */
struct Slot {
    cudaStream_t stream = nullptr;
    DevBuf rows;    /* the chunk's rows, 96 B per row */
    DevBuf out;     /* its output rows: scores, records, explanations or curves */
    DevBuf label;   /* its labels */
    DevBuf scratch; /* per-range partial sums of an explain chunk (launch_explain) */
};

struct Explainer; /* an attached path table (explain_api.cuh) */
static void explainer_free(Explainer *ex);

/* partial dependence (b2f_partial_dependence; partial_dependence.cuh): the current call's spec and point count */
struct Dependence {
    int32_t points = 0; /* doubles per output row */
    int n_segs = 0;
    std::vector<uint32_t> spec; /* the call's PdSeg table, then its grid words */
    DevBuf host_spec;           /* a host call's spec on the device */
    DevBuf device_spec;         /* the device form's: a host call never overwrites a spec an enqueued device-form launch reads */
};

/* two-way partial dependence (b2f_pair_dependence; pair_dependence.cuh): the current call's spec (PpSeg table, then two
 * words per point); the mean form's rows, partial sums and means, on the compute stream, grown on demand and kept */
struct PairDependence {
    int n_segs = 0;
    int64_t points = 0;
    std::vector<uint32_t> spec;
    DevBuf host_spec; /* a curve call's spec, read by its host job's chunks */
    DevBuf spec_dev;  /* the spec of the mean form and of the device form, written on the compute stream */
    DevBuf rows, partial, out;
};

/* accumulated local effects (b2f_ale; ale.cuh): the current call's spec (AleSeg table, then the edges) and bins; the
 * rows of the host form, the per-CTA partials of a piece and the per-bin results, on the compute stream, grown on demand */
struct Ale {
    int n_segs = 0;
    int bins = 0;
    std::vector<uint32_t> spec;
    DevBuf spec_dev, rows, psum, pcnt, sums, counts;
};

/* nearest single-field counterfactuals (b2f_counterfactual; counterfactual.cuh).  The split-value table is built on the
 * first call; cp.pd is the model's walk parameters, set at model creation, the probe fields are the current call's. */
struct Counterfactual {
    CfParams cp;
    bool built = false;
    std::vector<uint32_t> table; /* offset[24], count[24] per row word, then the float32 split values */
    DevBuf dev;                  /* the table on the device */
};

/* permutation importance (b2f_permutation_scores; permutation_importance.cuh): a call's rows, labels and permutations and
 * its groups' scratch, on the compute stream; grown on demand and kept for the model's life */
struct Importance {
    DevBuf rows, labels, perm;
    DevBuf keys;    /* two [point][row] key arrays of a group: the kernel's and the sort's other buffer */
    DevBuf flags;   /* the same for the flags bytes */
    DevBuf temp;    /* the segmented sort's temporary storage */
    DevBuf offsets; /* point p of a group starts at p * n */
    DevBuf segs;    /* the group's PiSeg table */
    DevBuf scores;  /* the group's records */
};

/* a reference table in K9's embedding (k_mmd_embed; mmd_drift.cuh), which MMD drift and trust scores share: its constants and
 * embedding, kept between calls, and a call's rows and their embedding; all on the compute stream, grown on demand */
struct EmbeddedRef {
    MmdParams mp;
    int64_t n_ref = 0;   /* 0: no reference */
    DevBuf ref_z, ref_c; /* the reference's embedding */
    DevBuf rows, z, c;   /* a call's rows and their embedding */
};

/* the online MMD detector (b2f_mmd_online_*; mmd_online.cuh): its configuration, the window state carried between pushes
 * (the stream's last W - 1 rows: embedding and c) and its copy at configure for reset, and a call's buffers; all on the
 * compute stream, grown on demand */
struct MmdOnline {
    int window = 0; /* 0: not configured */
    int64_t rw = 0, t = 0;
    double k_rr = 0.0;
    DevBuf total;                          /* T = sum of r_ref */
    DevBuf rz, rc;                         /* the sub-reference's embedding, compacted */
    DevBuf carry_z, carry_c, carry_cv;     /* the window state */
    DevBuf init_z, init_c, init_cv;        /* the window state at configure */
    DevBuf pos, band, qsum, cv, stats, krr; /* a bootstrap slice's or a push piece's scratch */
    DevBuf seq_z, seq_c, out;              /* a piece's sequence: the carried rows, then its own */
};

/* the MMD drift test (b2f_model_attach_mmd_reference / b2f_mmd_drift; mmd_drift.cuh): the reference and its kernel row
 * sums, kept between calls, and a call's buffers; all on the compute stream, grown on demand */
struct Mmd {
    EmbeddedRef ref;
    double sigma = 0.0, coef = 0.0;
    DevBuf r_ref; /* sum_{j != i} k(i, j) over the reference */
    DevBuf r, partial, sub, pairs, out, hist;
    MmdOnline online; /* configured against this reference: attaching another drops it */
};

/* the k-nearest reference search of trust scores (b2f_model_attach_knn_reference / b2f_knn; knn.cuh): the class-sorted
 * reference and its row map, kept between calls, and a call's buffers; all on the compute stream, grown on demand */
struct Knn {
    EmbeddedRef ref; /* class 0 rows, then class 1; a call embeds a piece of its queries */
    int64_t n_cls[2] = {0, 0};
    DevBuf orig; /* reference position -> original row */
    DevBuf cand_d, cand_i, dist, index;
};

struct TicketRec {
    uint64_t id = 0;
    cudaEvent_t ev[B2F_STREAMS] = {nullptr, nullptr, nullptr, nullptr};
    uint32_t used_mask = 0;
};

struct b2f_model {
    int device = 0;
    int sm_count = 0;
    int max_smem_optin = 0;
    KParams kp;
    b2f_blob_header hdr;
    int walk_mode = B2F_WALK_GLOBAL;
    int smem_bytes = 0;
    int rows_per_warp_max = 2;
    int64_t chunk_rows = B2F_CHUNK_ROWS;
    std::vector<int64_t> chunk_plan; /* per-chunk share of a batch in 1/1024ths */
    /* tile kernel (large batches) */
    bool tile_ok = false;
    TParams tp;
    void *d_tile_layout = nullptr;
    KParams *d_kp = nullptr; /* device copy of kp: the tile kernel re-decides rows inside the rounding band on it */
    TPiece *d_tile_pieces = nullptr;
    int tile_smem_bytes = 0;
    int tile_cwarps = B2F_TILE_WARPS_MIN;
    int64_t tile_min_rows = 32768;
    int64_t tile_layout_bytes = 0;
    int64_t launches_tile = 0;
    int64_t launches_split = 0;
    int64_t split_max_rows = 0;
    bool packed_ok = false;
    /* rank kernel (B2F_ROWS_RANKED rows; forest resident in its 4-byte-node complete-tree layout) */
    b2f_ranker rk;
    bool rank_ok = false;
    RParams rp;
    void *d_rank_layout = nullptr;
    int rank_smem_bytes = 0;
    int rank_u = 4;
    bool rank_stream = false; /* the rank layout streams through shared memory in pieces (too large to stay resident) */
    bool rank_pdl = true;     /* launch the rank kernel with programmatic stream serialization (B2F_NO_PDL at model creation: off) */
    int64_t launches_rank = 0;
    void *d_blob = nullptr;
    int64_t forest_bytes = 0;
    Explainer *ex = nullptr; /* attached TreeSHAP path table (b2f_model_attach_explainer) */
    PdParams walk; /* the forest fields every mask-walk kernel reads (K6, K7, K8, K10, K12); segs, grid and points are a call's */
    Dependence pd;
    PairDependence pair;
    Ale ale;
    Counterfactual cf;
    Importance pi;
    Mmd mmd;
    Knn knn;
    b2f_model *outlier = nullptr; /* attached isolation forest (b2f_model_attach_outlier_forest): a child handle on the
                                     same device whose kernels are launched on this handle's streams and rows */
    Slot slots[B2F_STREAMS];
    cudaStream_t compute = nullptr; /* device-resident interface + moments */
    DevBuf scratch;                 /* per-range partial sums of the explain launches on compute */
    TicketRec tickets[B2F_TICKETS];
    uint64_t next_ticket = 1;
    uint64_t next_slot = 0;
    /* moments */
    DevBuf mom_rows;
    double *d_mom_partials = nullptr;
    int mom_blocks = 0;
    unsigned int *d_mom_ticket = nullptr;
    double *d_mom_out = nullptr;
    DevBuf gather; /* (nranks + 1) * 72 doubles */
    /* L2 flush scratch */
    DevBuf flush;
    /* nccl */
    ncclComm_t comm = nullptr;
    int nranks = 0;
    int rank = 0;
    int64_t launches = 0;
};

static int validate_blob(const uint8_t *blob, size_t nbytes, b2f_blob_header *hdr_out) {
    if (!blob || nbytes < sizeof(b2f_blob_header)) return set_err(B2F_EINVAL, "forest blob too small (%zu bytes)", nbytes);
    b2f_blob_header h;
    memcpy(&h, blob, sizeof(h));
    if (memcmp(h.magic, B2F_BLOB_MAGIC, 8) != 0) return set_err(B2F_EINVAL, "forest blob: bad magic");
    if (h.version != B2F_BLOB_VERSION) return set_err(B2F_EINVAL, "forest blob: version %u, expected %u", h.version, B2F_BLOB_VERSION);
    if (h.header_bytes != B2F_BLOB_HEADER_BYTES || h.row_words != B2F_ROW_WORDS)
        return set_err(B2F_EINVAL, "forest blob: header_bytes=%u row_words=%u unsupported", h.header_bytes, h.row_words);
    if (h.agg_mode != B2F_AGG_RF_MEAN && h.agg_mode != B2F_AGG_GBDT_LOGISTIC && h.agg_mode != B2F_AGG_IFOREST)
        return set_err(B2F_EINVAL, "forest blob: unknown agg_mode %u", h.agg_mode);
    if (h.n_trees == 0 || h.n_trees > B2F_MAX_TREES) return set_err(B2F_EINVAL, "forest blob: n_trees=%u out of range [1,%d]", h.n_trees, B2F_MAX_TREES);
    if (h.n_groups != (h.n_trees + 31) / 32) return set_err(B2F_EINVAL, "forest blob: n_groups=%u inconsistent with n_trees=%u", h.n_groups, h.n_trees);
    if (h.n_cat + h.n_num > B2F_SENTINEL_WORD) return set_err(B2F_EINVAL, "forest blob: n_cat+n_num=%u exceeds %u", h.n_cat + h.n_num, B2F_SENTINEL_WORD);
    if (h.total_bytes != nbytes) return set_err(B2F_EINVAL, "forest blob: total_bytes=%llu but %zu given", (unsigned long long)h.total_bytes, nbytes);
    if (h.groups_off < sizeof(h) || h.groups_off + (uint64_t)h.n_groups * sizeof(b2f_blob_group) > nbytes)
        return set_err(B2F_EINVAL, "forest blob: group table out of bounds");
    if (h.chunks_off % 256 || h.chunks_off + h.chunks_bytes > nbytes) return set_err(B2F_EINVAL, "forest blob: chunk area out of bounds");
    if (!(h.denom > 0.0)) return set_err(B2F_EINVAL, "forest blob: denom must be positive");
    const b2f_blob_group *gt = reinterpret_cast<const b2f_blob_group *>(blob + h.groups_off);
    uint64_t expect_off = 0;
    for (uint32_t g = 0; g < h.n_groups; ++g) {
        b2f_blob_group gr;
        memcpy(&gr, &gt[g], sizeof(gr));
        if (gr.chunk_off != expect_off || gr.n_slots == 0 || gr.n_leaf_slots == 0 ||
            gr.chunk_bytes != (gr.n_slots + gr.n_leaf_slots) * 256u || (uint64_t)gr.chunk_off + gr.chunk_bytes > h.chunks_bytes ||
            gr.n_slots >= (1u << 24) || gr.n_leaf_slots >= (1u << 24) || gr.n_trees == 0 || gr.n_trees > 32)
            return set_err(B2F_EINVAL, "forest blob: group %u descriptor invalid", g);
        expect_off += gr.chunk_bytes;
        /* every node word must keep the walk in bounds: check all slots */
        const uint32_t *N = reinterpret_cast<const uint32_t *>(blob + h.chunks_off + gr.chunk_off);
        for (uint32_t s = 0; s < gr.n_slots; ++s)
            for (uint32_t l = 0; l < 32; ++l) {
                const uint32_t t = N[(s * 32 + l) * 2], m = N[(s * 32 + l) * 2 + 1];
                const uint32_t feat = m >> B2F_META_FEAT_SHIFT, first = m & B2F_META_SLOT_MASK;
                const bool leaf = (first == s);
                if ((m & 0x03000000u) || feat > B2F_SENTINEL_WORD)
                    return set_err(B2F_EINVAL, "forest blob: group %u slot %u lane %u: bad meta word 0x%08x", g, s, l, m);
                if (leaf) {
                    if (!(m & B2F_META_CAT) || feat != B2F_SENTINEL_WORD || t >= gr.n_leaf_slots)
                        return set_err(B2F_EINVAL, "forest blob: group %u slot %u lane %u: malformed leaf", g, s, l);
                } else {
                    if (first <= s || first + 1 >= gr.n_slots) return set_err(B2F_EINVAL, "forest blob: group %u slot %u lane %u: child %u out of range", g, s, l, first);
                    if ((m & B2F_META_CAT) && feat >= h.n_cat && feat != B2F_SENTINEL_WORD)
                        return set_err(B2F_EINVAL, "forest blob: group %u slot %u lane %u: categorical test on numeric word", g, s, l);
                }
            }
    }
    if (expect_off != h.chunks_bytes) return set_err(B2F_EINVAL, "forest blob: chunks_bytes mismatch");
    *hdr_out = h;
    return B2F_OK;
}

extern "C" int b2f_blob_validate(const void *forest_blob, size_t nbytes) {
    b2f_blob_header h;
    return validate_blob(static_cast<const uint8_t *>(forest_blob), nbytes, &h);
}

/* ------------------------------------------------------------------ ranked rows: host-side tables (forest_rank.h) */
extern "C" b2f_ranker *b2f_ranker_create(const void *forest_blob, size_t nbytes) {
    b2f_blob_header h;
    if (validate_blob(static_cast<const uint8_t *>(forest_blob), nbytes, &h) != B2F_OK) return nullptr;
    b2f_ranker *r = new (std::nothrow) b2f_ranker();
    if (!r) {
        set_err(B2F_ENOMEM, "out of host memory");
        return nullptr;
    }
    ranker_build(r, static_cast<const uint8_t *>(forest_blob), h);
    return r;
}
extern "C" void b2f_ranker_destroy(b2f_ranker *r) { delete r; }

static void fill_rank_info(const b2f_ranker *r, bool ok, b2f_rank_info *out) {
    memset(out, 0, sizeof(*out));
    out->ok = ok ? 1 : 0;
    out->row_bytes = r->row_bytes;
    out->cat_bytes = r->cat_bytes;
    out->n_cat = r->n_cat;
    out->n_num = r->n_num;
    out->depth = r->depth;
    out->n_trees = r->n_trees;
    out->layout_bytes = (int32_t)r->layout.size();
    for (int j = 0; j < 16; ++j) {
        out->cat_shift[j] = r->cat_shift[j];
        out->cat_bits[j] = r->cat_bits[j];
    }
    for (size_t k = 0; k < r->thr.size() && k < 24; ++k) out->n_thresholds[k] = (int32_t)r->thr[k].size();
    out->n_pairs = (int32_t)r->pairs.size();
    for (size_t i = 0; i < r->pairs.size() && i < 128; ++i) out->pairs[i] = r->pairs[i];
    snprintf(out->why, sizeof(out->why), "%s", r->why);
}
extern "C" int b2f_ranker_info(const b2f_ranker *r, b2f_rank_info *out) {
    if (!r || !out) return set_err(B2F_EINVAL, "null argument");
    fill_rank_info(r, r->ok, out);
    return B2F_OK;
}
extern "C" const float *b2f_ranker_thresholds(const b2f_ranker *r, int k, int32_t *count) {
    if (!r || k < 0 || k >= (int)r->thr.size()) {
        if (count) *count = 0;
        return nullptr;
    }
    if (count) *count = (int32_t)r->thr[k].size();
    return r->thr[k].data();
}
extern "C" const void *b2f_ranker_layout(const b2f_ranker *r, int64_t *nbytes) {
    if (!r || !r->ok) {
        if (nbytes) *nbytes = 0;
        return nullptr;
    }
    if (nbytes) *nbytes = (int64_t)r->layout.size();
    return r->layout.data();
}
extern "C" int b2f_ranker_rank_rows(const b2f_ranker *r, const void *rows, int64_t n, int row_format, void *ranked_out, int threads) {
    if (!r || n < 0 || (n > 0 && (!rows || !ranked_out))) return set_err(B2F_EINVAL, "bad argument");
    if (!r->ok) return set_err(B2F_EINVAL, "no rank layout for this forest (%s)", r->why);
    if (row_format != B2F_ROWS_WORDS24 && row_format != B2F_ROWS_PACKED64) return set_err(B2F_EINVAL, "rows must be B2F_ROWS_WORDS24 or B2F_ROWS_PACKED64");
    if (row_format == B2F_ROWS_PACKED64 && !(r->n_cat == 9 && r->n_num <= 14)) return set_err(B2F_EINVAL, "schema does not fit the packed 64-byte row");
    threads = (int)std::min<int64_t>(std::max(threads, 1), std::max<int64_t>(1, n / 4096));
    const uint8_t *in = static_cast<const uint8_t *>(rows);
    uint8_t *out = static_cast<uint8_t *>(ranked_out);
    if (threads == 1) {
        rank_rows_range(r, in, 0, n, row_format, out);
        return B2F_OK;
    }
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back([=] { rank_rows_range(r, in, n * t / threads, n * (t + 1) / threads, row_format, out); });
    rank_rows_range(r, in, 0, n / threads, row_format, out);
    for (auto &th : pool) th.join();
    return B2F_OK;
}

/* ------------------------------------------------------------------ kernel instantiations
 * Launches and cudaFuncSetAttribute calls both take the instantiation from here, so each template axis is switched once. */
template <typename OutT>
using RankKernel = void (*)(RParams, const uint8_t *, long long, OutT *, int32_t *, int);

template <int R, typename OutT>
static auto warp_kernel_r(bool smem, bool pk) {
    if (smem) return pk ? k_forest_predict<R, true, true, OutT> : k_forest_predict<R, true, false, OutT>;
    return pk ? k_forest_predict<R, false, true, OutT> : k_forest_predict<R, false, false, OutT>;
}
template <typename OutT>
static auto warp_kernel(int rows_per_warp, bool smem, bool pk) {
    if (rows_per_warp == 4) return warp_kernel_r<4, OutT>(smem, pk);
    return rows_per_warp == 2 ? warp_kernel_r<2, OutT>(smem, pk) : warp_kernel_r<1, OutT>(smem, pk);
}
template <typename OutT>
static auto tile_kernel(bool pk) {
    return pk ? k_forest_predict_tile<true, OutT> : k_forest_predict_tile<false, OutT>;
}
template <typename OutT>
static auto split_kernel(bool pk) {
    return pk ? k_forest_predict_split<2, true, OutT> : k_forest_predict_split<2, false, OutT>;
}
/* depths 1..8; NULL for any other depth */
template <typename OutT, int D = 1>
static RankKernel<OutT> rank_kernel(const b2f_model *m) {
    if constexpr (D > 8) {
        return nullptr;
    } else {
        if (m->rp.depth != D) return rank_kernel<OutT, D + 1>(m);
        /* a GBDT has no exact re-decision (forest_decide.cuh): its instances carry none of that code */
        if (m->hdr.agg_mode == B2F_AGG_GBDT_LOGISTIC) {
            if (m->rank_stream) return k_forest_predict_rank<D, 4, true, false, OutT>;
            return m->rank_u == 8 ? k_forest_predict_rank<D, 8, false, false, OutT> : k_forest_predict_rank<D, 4, false, false, OutT>;
        }
        if (m->rank_stream) return k_forest_predict_rank<D, 4, true, true, OutT>;
        return m->rank_u == 8 ? k_forest_predict_rank<D, 8, false, true, OutT> : k_forest_predict_rank<D, 4, false, true, OutT>;
    }
}
/* The dynamic shared-memory limit belongs to the kernel function on the current device, not to a model: every model of the
 * process that launches `kernel` shares it.  So it only ever rises -- a later model with a smaller need (an attached
 * outlier forest, a second engine, an explainer of fewer fields, a shallower forest's permutation scores, a smaller k)
 * must not lower it under an earlier model's launches, which would then fail.  Every kernel with dynamic shared memory
 * sets its limit here, at attach or per call, and never through cudaFuncSetAttribute directly
 * (tests/test_models_together_cpu.py). */
template <typename K>
static cudaError_t set_smem_limit(K kernel, int bytes) {
    if (!kernel) return cudaErrorInvalidValue;
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    cudaFuncAttributes a;
    const cudaError_t e = cudaFuncGetAttributes(&a, kernel);
    if (e != cudaSuccess || a.maxDynamicSharedSizeBytes >= bytes) return e;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

/* ------------------------------------------------------------------ environment hooks read at model creation (INTEGRATION.md) */
enum { KN_AUTO, KN_WARP, KN_TILE, KN_SPLIT };
struct EnvHooks {
    int kernel = KN_AUTO;      /* B2F_KERNEL: "warp" | "tile" | "split" pins one predict kernel (tests) */
    bool walk_global = false;  /* B2F_FORCE_WALK=global: walk the forest from global memory (test hook) */
    bool walk_smem = false;    /* B2F_FORCE_WALK=smem: shared-memory walk, an error if the forest does not fit */
    int64_t chunk_rows = B2F_CHUNK_ROWS; /* B2F_CHUNK_ROWS (>= 1024): rows per pipelined H2D/kernel/D2H chunk */
    /* B2F_CHUNK_PLAN="a,b,c": per-chunk share of a batch in 1/1024ths.  65 536-row batches: 3/4 of the batch, then the rest.
     * tools/chunk_plan_sweep.py on an H100 80GB HBM3 (700 W): the best of nine plans for both row formats -- 88 us p50 per
     * ranked-row call against 108 us in one chunk, 145 us against 158 us with 64-byte rows */
    std::vector<int64_t> chunk_plan{768};
    /* B2F_SPLIT_MAX_ROWS: the latency form (one CTA per 2 rows, warp = tree group) hands over to the warp-per-row kernel at
     * 2 048 rows: below that the warp-per-row kernel leaves most SMs idle while the latency form spreads one row's trees over a
     * CTA's warps.  tools/split_threshold.py on an H100 80GB HBM3 (700 W), synchronous 64-byte-row calls, GBDT 500 x d8: 38 vs
     * 64 us at 512 rows, 72 vs 80 at 2 048, 89 vs 79 at 3 072; GBDT 100 x d6: within ~5 us of each other at every size up to
     * 4 096. */
    int64_t split_max_rows = 2048;
    int rows_per_warp = 2;      /* B2F_ROWS_PER_WARP: 1 | 2 | 4 */
    int64_t tile_min_rows = -1; /* B2F_TILE_MIN_ROWS (>= 0); -1 = by the tile layout */
    int tile_warps = 0;         /* B2F_TILE_WARPS (clamped to 1..B2F_TILE_WARPS_MAX); 0 = choose */
    bool rank_off = false;      /* B2F_RANK=0: no rank kernel */
    int rank_max_tiles = INT_MAX; /* B2F_RANK_MAX_TILES (>= 1): cap on the resident rank kernel's row tiles */
    int rank_stream = -1;       /* B2F_RANK_STREAM: 1 / 0 force / forbid the streamed rank kernel; -1 = by size */
    int rank_u = 4;             /* B2F_RANK_U: 4 | 8 trees in flight per thread */
    bool rank_wait_first = false; /* B2F_RANK_WAIT_FIRST=1: the rank kernel's dependency wait back at kernel entry (A/B) */
    bool no_pdl = false;        /* B2F_NO_PDL: launch the rank kernel without programmatic stream serialization */
};

static EnvHooks read_env_hooks(void) {
    EnvHooks h;
    if (const char *v = getenv("B2F_KERNEL"))
        h.kernel = !strcmp(v, "warp") ? KN_WARP : !strcmp(v, "tile") ? KN_TILE : !strcmp(v, "split") ? KN_SPLIT : KN_AUTO;
    if (const char *v = getenv("B2F_FORCE_WALK")) {
        h.walk_global = !strcmp(v, "global");
        h.walk_smem = !strcmp(v, "smem");
    }
    if (const char *v = getenv("B2F_CHUNK_ROWS"))
        if (atoll(v) >= 1024) h.chunk_rows = atoll(v);
    if (const char *v = getenv("B2F_CHUNK_PLAN")) {
        h.chunk_plan.clear();
        for (const char *q = v; *q;) {
            h.chunk_plan.push_back(atoll(q));
            while (*q && *q != ',') ++q;
            if (*q == ',') ++q;
        }
    }
    if (const char *v = getenv("B2F_SPLIT_MAX_ROWS")) h.split_max_rows = atoll(v);
    if (const char *v = getenv("B2F_ROWS_PER_WARP")) {
        const int r = atoi(v);
        if (r == 1 || r == 2 || r == 4) h.rows_per_warp = r;
    }
    if (const char *v = getenv("B2F_TILE_MIN_ROWS"))
        if (atoll(v) >= 0) h.tile_min_rows = atoll(v);
    if (const char *v = getenv("B2F_TILE_WARPS")) h.tile_warps = std::min(B2F_TILE_WARPS_MAX, std::max(1, atoi(v)));
    if (const char *v = getenv("B2F_RANK")) h.rank_off = !strcmp(v, "0");
    if (const char *v = getenv("B2F_RANK_MAX_TILES")) h.rank_max_tiles = std::max(1, atoi(v));
    if (const char *v = getenv("B2F_RANK_STREAM")) h.rank_stream = atoi(v) != 0;
    if (const char *v = getenv("B2F_RANK_U")) h.rank_u = atoi(v) == 8 ? 8 : 4;
    if (const char *v = getenv("B2F_RANK_WAIT_FIRST")) h.rank_wait_first = atoi(v) != 0;
    h.no_pdl = getenv("B2F_NO_PDL") != nullptr;
    return h;
}


/* ------------------------------------------------------------------ tile layout (forest_predict_tile.cuh)
 * Re-pack the interleaved blob tree-major: per tree its breadth-first nodes then its leaf payloads, trees in
 * U-groups of B2F_TILE_U (8) with an 80-byte descriptor, U-groups packed into pieces that fit a shared-memory ring slot. */
struct TileTree {
    std::vector<uint32_t> nodes; /* T, M pairs */
    std::vector<double> leaves;
    uint32_t depth = 0;
};

static bool extract_tree(const uint8_t *blob, const b2f_blob_header &h, const b2f_blob_group &gr, uint32_t lane, TileTree &out) {
    const uint32_t *N = reinterpret_cast<const uint32_t *>(blob + h.chunks_off + gr.chunk_off);
    const double *LV = reinterpret_cast<const double *>(blob + h.chunks_off + gr.chunk_off + (size_t)gr.n_slots * 256);
    std::vector<uint32_t> depth_of(gr.n_slots, 0);
    uint32_t reach = 0, max_leaf = 0, max_depth = 0;
    for (uint32_t s = 0; s <= reach; ++s) {
        const uint32_t t = N[(s * 32 + lane) * 2], m = N[(s * 32 + lane) * 2 + 1];
        const uint32_t feat = m >> B2F_META_FEAT_SHIFT, first = m & B2F_META_SLOT_MASK;
        const bool cat = (m & B2F_META_CAT) != 0;
        if (first >= B2F_TILE_MAX_TREE_NODES) return false;
        out.nodes.push_back(t);
        out.nodes.push_back((first << B2F_TILE_CHILD_SHIFT) | (cat ? B2F_TILE_META_CAT : 0u) | (feat << B2F_TILE_FEAT_SHIFT));
        if (first == s) { /* leaf */
            max_leaf = std::max(max_leaf, t);
            max_depth = std::max(max_depth, depth_of[s]);
        } else {
            reach = std::max(reach, first + 1);
            depth_of[first] = depth_of[first + 1] = depth_of[s] + 1;
        }
    }
    out.leaves.resize(max_leaf + 1);
    for (uint32_t i = 0; i <= max_leaf; ++i) out.leaves[i] = LV[i * 32 + lane];
    out.depth = max_depth;
    return true;
}

static bool build_tile_layout(const uint8_t *blob, const b2f_blob_header &h, uint32_t avail_smem, std::vector<uint8_t> &layout,
                              std::vector<TPiece> &pieces, uint32_t *slot_bytes, int *n_slots) {
    const b2f_blob_group *gt = reinterpret_cast<const b2f_blob_group *>(blob + h.groups_off);
    std::vector<TileTree> trees(h.n_trees);
    for (uint32_t t = 0; t < h.n_trees; ++t)
        if (!extract_tree(blob, h, gt[t / 32], t % 32, trees[t])) return false;
    /* U-groups */
    struct UG {
        uint32_t first, count, bytes;
    };
    std::vector<UG> ugs;
    uint64_t total = 0;
    for (uint32_t t = 0; t < h.n_trees; t += B2F_TILE_U) {
        UG u{t, std::min<uint32_t>(B2F_TILE_U, h.n_trees - t), (uint32_t)sizeof(TUGroup)};
        for (uint32_t k = 0; k < B2F_TILE_U; ++k)
            u.bytes += k < u.count ? (uint32_t)(trees[t + k].nodes.size() * 4 + trees[t + k].leaves.size() * 8) : 16u; /* stub: 1 node + 1 leaf */
        ugs.push_back(u);
        total += u.bytes;
    }
    /* piece size: if everything fits the ring, cut it into at most B2F_TILE_MAX_SLOTS pieces (resident: loaded
     * once per CTA, and walking starts when the first piece lands); otherwise ~32 KB pieces streamed through */
    uint32_t max_ug = 0;
    for (const UG &u : ugs) max_ug = std::max(max_ug, u.bytes);
    const bool fits = total + (uint64_t)(max_ug + 128) * B2F_TILE_MAX_SLOTS <= avail_smem;
    uint32_t target = fits ? (uint32_t)((total + B2F_TILE_MAX_SLOTS - 1) / B2F_TILE_MAX_SLOTS) + max_ug : 32u * 1024u;
    layout.clear();
    pieces.clear();
    size_t i = 0;
    uint32_t max_piece = 0;
    while (i < ugs.size()) {
        size_t j = i;
        uint32_t bytes = 0;
        while (j < ugs.size() && (j == i || bytes + ugs[j].bytes <= target)) bytes += ugs[j++].bytes;
        /* emit piece [i, j) */
        const uint32_t n_ug = (uint32_t)(j - i);
        const size_t start = layout.size();
        std::vector<uint8_t> buf((size_t)n_ug * sizeof(TUGroup));
        for (uint32_t g = 0; g < n_ug; ++g) {
            TUGroup d;
            memset(&d, 0, sizeof(d));
            for (uint32_t k = 0; k < B2F_TILE_U; ++k) {
                while (buf.size() % 8) buf.push_back(0);
                d.node_off[k] = (uint32_t)buf.size();
                if (k < ugs[i + g].count) {
                    const TileTree &tr = trees[ugs[i + g].first + k];
                    const uint8_t *np = reinterpret_cast<const uint8_t *>(tr.nodes.data());
                    buf.insert(buf.end(), np, np + tr.nodes.size() * 4);
                    d.leaf_off[k] = (uint32_t)buf.size();
                    const uint8_t *lp = reinterpret_cast<const uint8_t *>(tr.leaves.data());
                    buf.insert(buf.end(), lp, lp + tr.leaves.size() * 8);
                    d.depth = std::max(d.depth, tr.depth);
                } else { /* stub tree: one self-looping leaf worth 0.0 */
                    const uint32_t stub[2] = {0u, (0u << B2F_TILE_CHILD_SHIFT) | B2F_TILE_META_CAT | (B2F_SENTINEL_WORD << B2F_TILE_FEAT_SHIFT)};
                    const uint8_t *sp = reinterpret_cast<const uint8_t *>(stub);
                    buf.insert(buf.end(), sp, sp + 8);
                    d.leaf_off[k] = (uint32_t)buf.size();
                    const double z = 0.0;
                    const uint8_t *zp = reinterpret_cast<const uint8_t *>(&z);
                    buf.insert(buf.end(), zp, zp + 8);
                }
            }
            memcpy(buf.data() + (size_t)g * sizeof(TUGroup), &d, sizeof(d));
        }
        while (buf.size() % 128) buf.push_back(0);
        layout.insert(layout.end(), buf.begin(), buf.end());
        pieces.push_back(TPiece{(uint32_t)start, (uint32_t)buf.size(), n_ug, 0u});
        max_piece = std::max<uint32_t>(max_piece, (uint32_t)buf.size());
        i = j;
    }
    *slot_bytes = max_piece;
    if ((size_t)max_piece * pieces.size() <= avail_smem && pieces.size() <= B2F_TILE_MAX_SLOTS) {
        *n_slots = (int)pieces.size(); /* resident */
    } else {
        int s = (int)std::min<uint64_t>(B2F_TILE_MAX_SLOTS, avail_smem / max_piece);
        if (s < 2) return false; /* a single U-group does not fit a ring slot: tile kernel not applicable */
        *n_slots = s;
    }
    return true;
}

/* What the kernels' aggregate() compares with: an isolation forest flags `s <= bound` on its path-length sum s (forest_predict.cuh).
 * The blob carries the bound flatten.py derived with numpy, the library's own arithmetic; for a blob written without one the same
 * search runs here with libm's pow.  Other modes: the header's threshold, unused. */
static double decision_threshold(const b2f_blob_header &h) {
    if (h.agg_mode != B2F_AGG_IFOREST) return h.threshold;
    if (h.flags & B2F_BLOB_HAS_PATH_BOUND) return h.path_bound;
    auto flagged = [&](int64_t bits) {
        double s;
        memcpy(&s, &bits, sizeof(s));
        return std::pow(2.0, -(s / h.denom)) + h.init_raw > h.threshold;
    };
    const double inf = std::numeric_limits<double>::infinity();
    int64_t lo = 0, hi;
    memcpy(&hi, &inf, sizeof(hi));
    if (!flagged(lo)) return -inf;
    if (flagged(hi)) return inf;
    while (hi - lo > 1) {
        const int64_t mid = lo + (hi - lo) / 2;
        (flagged(mid) ? lo : hi) = mid;
    }
    double s;
    memcpy(&s, &lo, sizeof(s));
    return s;
}

/* rank kernel: 4-byte integer nodes, complete trees, rows as ranks (forest_rank.h) */
static int rank_init(b2f_model *m, const uint8_t *blob, const EnvHooks &env) {
    m->rank_ok = false;
    ranker_build(&m->rk, blob, m->hdr);
    if (!m->rk.ok) return B2F_OK; /* no rank layout for this forest: the other kernels serve it */
    if (env.rank_off) return B2F_OK;
    const int64_t layout_bytes = (int64_t)m->rk.layout.size();
    const int64_t base = B2F_RANK_XS_BYTES /* alignment slack */ + (int64_t)B2F_RANK_PARTIALS * 32 * 8 + 256;
    m->rank_u = env.rank_u;
    /* resident: the CTA copies and walks the first ceil(n_trees / U) groups only (stub trees complete the last one) */
    const int n_groups = (m->rk.n_trees + m->rank_u - 1) / m->rank_u;
    const int64_t walked_bytes = (int64_t)n_groups * m->rank_u * m->rk.tree_stride;
    int max_tiles = (int)std::min<int64_t>(B2F_RANK_MAX_TILES, ((int64_t)m->max_smem_optin - base - walked_bytes) / B2F_RANK_XS_BYTES);
    max_tiles = std::min(max_tiles, env.rank_max_tiles);
    /* resident while the walked trees fit next to a useful number of row tiles and their top levels fit the parameter block's
     * table; otherwise the layout streams through a two-slot ring in pieces of 8 trees (2 groups of 4: warp w owns
     * (tile w / 2, group w mod 2), so <= 16 tiles per round) */
    const bool top_fits = m->rk.n_trees <= B2F_RANK_TOP_TREES;
    if (env.rank_stream == 0 && !top_fits) return B2F_OK; /* resident forced but impossible: no rank kernel */
    m->rank_stream = env.rank_stream < 0 ? (max_tiles < 8 || !top_fits) : env.rank_stream != 0;
    int64_t forest_smem = walked_bytes;
    if (m->rank_stream) {
        m->rank_u = 4;
        const int64_t piece = 8 * (int64_t)m->rk.tree_stride; /* n_trees_padded is a multiple of 8 */
        forest_smem = 2 * piece;
        max_tiles = (int)std::min<int64_t>(B2F_RANK_MAX_TILES, ((int64_t)m->max_smem_optin - base - forest_smem) / B2F_RANK_XS_BYTES);
        if (max_tiles < 4 || piece % 16) return B2F_OK;
    }
    CUDA_TRY(cudaMalloc(&m->d_rank_layout, (size_t)layout_bytes));
    CUDA_TRY(cudaMemcpy(m->d_rank_layout, m->rk.layout.data(), (size_t)layout_bytes, cudaMemcpyHostToDevice));
    RParams &rp = m->rp;
    memset(&rp, 0, sizeof(rp));
    rp.layout = static_cast<const uint8_t *>(m->d_rank_layout);
    rp.layout_bytes = (uint32_t)(m->rank_stream ? layout_bytes : walked_bytes);
    rp.tree_stride = m->rk.tree_stride;
    rp.n_trees_padded = m->rk.n_trees_padded;
    rp.n_groups = n_groups;
    if (!m->rank_stream) {
        for (int t = 0; t < m->rk.n_trees; ++t) {
            const uint32_t *nodes = reinterpret_cast<const uint32_t *>(m->rk.layout.data() + (size_t)t * m->rk.tree_stride);
            rp.top_root[t] = nodes[0];
            if (m->rk.depth >= 2) rp.top_kids[t] = make_uint2(nodes[1], nodes[2]); /* stumps have no level 1 */
        }
    }
    rp.depth = m->rk.depth;
    rp.agg_mode = (int)m->hdr.agg_mode;
    rp.n_cat = m->rk.n_cat;
    rp.n_num = m->rk.n_num;
    rp.row_bytes = m->rk.row_bytes;
    rp.cat_bytes = m->rk.cat_bytes;
    rp.max_tiles = max_tiles;
    rp.groups_per_piece = 2;
    rp.piece_bytes = 8u * m->rk.tree_stride;
    rp.n_pieces = m->rk.n_trees_padded / 8;
    rp.init_raw = m->hdr.init_raw;
    rp.denom = m->hdr.denom;
    rp.threshold = decision_threshold(m->hdr);
    rp.mul_two = 2u;
    rp.mul_64k = 65536u;
    rp.add_64k = 65535u;
    rp.n_pairs = (int)m->rk.pairs.size();
    rp.wait_first = env.rank_wait_first;
    m->rank_pdl = !env.no_pdl;
    for (int j = 0; j < 16; ++j) {
        rp.cat_shift[j] = (uint8_t)m->rk.cat_shift[j];
        rp.cat_bits[j] = (uint8_t)m->rk.cat_bits[j];
        rp.cat_start[j] = 0;
        rp.cat_mask[j] = 0ull;
    }
    for (int i = rp.n_pairs - 1; i >= 0; --i) { /* pairs are sorted by (feature, category): the last write per feature is its first pair */
        const uint32_t j = m->rk.pairs[i] >> 16, c = m->rk.pairs[i] & 0xFFFFu;
        rp.cat_start[j] = (uint8_t)i;
        rp.cat_mask[j] |= 1ull << c;
    }
    m->rank_smem_bytes = (int)(B2F_RANK_XS_BYTES + (int64_t)max_tiles * B2F_RANK_XS_BYTES + (int64_t)B2F_RANK_PARTIALS * 32 * 8 + forest_smem);
    CUDA_TRY(set_smem_limit(rank_kernel<float>(m), m->rank_smem_bytes));
    CUDA_TRY(set_smem_limit(rank_kernel<double>(m), m->rank_smem_bytes));
    m->rank_ok = true;
    return B2F_OK;
}

/* warp-per-row and latency kernels: the walk mode, the split hand-over and the chunking of host batches */
static int warp_init(b2f_model *m, const uint8_t *blob, const EnvHooks &env) {
    KParams &kp = m->kp;
    memset(&kp, 0, sizeof(kp));
    kp.chunks = static_cast<const uint8_t *>(m->d_blob) + m->hdr.chunks_off;
    kp.n_groups = (int)m->hdr.n_groups;
    kp.agg_mode = (int)m->hdr.agg_mode;
    kp.n_cat = (int)m->hdr.n_cat;
    kp.n_num = (int)m->hdr.n_num;
    kp.init_raw = m->hdr.init_raw;
    kp.denom = m->hdr.denom;
    kp.threshold = decision_threshold(m->hdr);
    memcpy(kp.impute, m->hdr.impute, sizeof(kp.impute));
    const b2f_blob_group *gt = reinterpret_cast<const b2f_blob_group *>(blob + m->hdr.groups_off);
    for (uint32_t g = 0; g < m->hdr.n_groups; ++g) {
        kp.g[g].chunk_off = gt[g].chunk_off;
        kp.g[g].chunk_bytes = gt[g].chunk_bytes;
        kp.g[g].n_slots = gt[g].n_slots;
        kp.g[g].n_leaf_slots = gt[g].n_leaf_slots;
        kp.g[g].depth = gt[g].depth;
    }
    PdParams &pp = m->walk;
    memset(&pp, 0, sizeof(pp));
    pp.chunks = kp.chunks;
    pp.n_groups = kp.n_groups;
    pp.agg_mode = kp.agg_mode;
    pp.n_cat = kp.n_cat;
    pp.n_num = kp.n_num;
    pp.init_raw = kp.init_raw;
    pp.denom = kp.denom;
    pp.threshold = kp.threshold;
    memcpy(pp.impute, kp.impute, sizeof(pp.impute));
    for (uint32_t g = 0; g < m->hdr.n_groups; ++g) {
        pp.g_off[g] = gt[g].chunk_off;
        pp.g_slots[g] = gt[g].n_slots;
        pp.g_trees[g] = gt[g].n_trees;
    }
    memset(&m->cf.cp, 0, sizeof(m->cf.cp));
    m->cf.cp.pd = pp;

    /* the packed 64-byte row needs the credit-default shape: exactly 9 categoricals of <= 126 categories, <= 14 numerics */
    m->packed_ok = m->hdr.n_cat == 9 && m->hdr.n_num <= 14; /* the kernels decode word L-7 / q[2+k] for exactly nine 7-bit fields */
    for (uint32_t f = 0; f < m->hdr.n_cat; ++f)
        if (m->hdr.vocab[f] > 126) m->packed_ok = false;

    /* shared-memory residency: whole forest + static barriers must fit the opt-in limit */
    const int64_t need = (int64_t)m->hdr.chunks_bytes;
    const bool fits = need + 1024 <= (int64_t)m->max_smem_optin && !env.walk_global;
    if (env.walk_smem && !fits) return set_err(B2F_EINVAL, "B2F_FORCE_WALK=smem but forest needs %lld bytes", (long long)need);
    m->walk_mode = fits ? B2F_WALK_SMEM : B2F_WALK_GLOBAL;
    m->smem_bytes = fits ? (int)need : 0;
    if (fits)
        for (bool pk : {false, true})
            for (int r : {1, 2, 4}) {
                CUDA_TRY(set_smem_limit(warp_kernel<float>(r, true, pk), m->smem_bytes));
                CUDA_TRY(set_smem_limit(warp_kernel<double>(r, true, pk), m->smem_bytes));
            }
    m->chunk_rows = env.chunk_rows;
    m->chunk_plan = env.chunk_plan;
    m->split_max_rows = env.split_max_rows;
    if (env.kernel == KN_WARP || env.kernel == KN_TILE) m->split_max_rows = 0;
    if (env.kernel == KN_SPLIT) m->split_max_rows = INT64_MAX;
    m->rows_per_warp_max = env.rows_per_warp;
    return B2F_OK;
}

/* tile kernel (large batches): tree-major layout + shared-memory ring plan */
static int tile_init(b2f_model *m, const uint8_t *blob, const EnvHooks &env) {
    std::vector<uint8_t> layout;
    std::vector<TPiece> pieces;
    uint32_t slot_bytes = 0;
    int n_slots = 0;
    bool ok = false;
    /* most consumer warps for which the forest still stays resident, else 16 warps and a streamed forest (B2F_TILE_WARPS: that many) */
    int cwarps = B2F_TILE_WARPS_MIN;
    const int w_hi = env.tile_warps ? env.tile_warps : B2F_TILE_WARPS_MAX, w_lo = env.tile_warps ? env.tile_warps : B2F_TILE_WARPS_MIN;
    for (int w = w_hi; env.kernel != KN_WARP && w >= w_lo && !ok; w -= 4) {
        const uint32_t avail = (uint32_t)m->max_smem_optin - 1024u - 4096u - (uint32_t)w * B2F_TILE_XS_BYTES;
        const bool built = build_tile_layout(blob, m->hdr, avail, layout, pieces, &slot_bytes, &n_slots);
        const bool res = built && (int)pieces.size() <= n_slots;
        if (built && (res || w == w_lo)) {
            ok = true;
            cwarps = w;
        }
    }
    if (!ok) {
        if (env.kernel == KN_TILE) return set_err(B2F_EINVAL, "B2F_KERNEL=tile but the forest's trees do not fit the tile kernel's shared-memory ring");
        return B2F_OK;
    }
    CUDA_TRY(cudaMalloc(&m->d_tile_layout, layout.size()));
    CUDA_TRY(cudaMemcpy(m->d_tile_layout, layout.data(), layout.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc((void **)&m->d_tile_pieces, pieces.size() * sizeof(TPiece)));
    CUDA_TRY(cudaMemcpy(m->d_tile_pieces, pieces.data(), pieces.size() * sizeof(TPiece), cudaMemcpyHostToDevice));
    const KParams &kp = m->kp;
    TParams &tp = m->tp;
    memset(&tp, 0, sizeof(tp));
    CUDA_TRY(cudaMalloc((void **)&m->d_kp, sizeof(KParams)));
    CUDA_TRY(cudaMemcpy(m->d_kp, &m->kp, sizeof(KParams), cudaMemcpyHostToDevice));
    tp.layout = static_cast<const uint8_t *>(m->d_tile_layout);
    tp.pieces = m->d_tile_pieces;
    tp.n_pieces = (int)pieces.size();
    tp.n_slots = n_slots;
    tp.slot_bytes = slot_bytes;
    tp.agg_mode = kp.agg_mode;
    tp.n_cat = kp.n_cat;
    tp.n_num = kp.n_num;
    tp.init_raw = kp.init_raw;
    tp.denom = kp.denom;
    tp.threshold = kp.threshold;
    tp.blob = m->d_kp;
    memcpy(tp.impute, kp.impute, sizeof(tp.impute));
    m->tile_cwarps = cwarps;
    m->tile_smem_bytes = 4096 + cwarps * B2F_TILE_XS_BYTES + n_slots * (int)slot_bytes;
    m->tile_layout_bytes = (int64_t)layout.size();
    for (bool pk : {false, true}) {
        CUDA_TRY(set_smem_limit(tile_kernel<float>(pk), m->tile_smem_bytes));
        CUDA_TRY(set_smem_limit(tile_kernel<double>(pk), m->tile_smem_bytes));
    }
    m->tile_ok = true;
    /* crossover chosen on the previous GPU generation and kept, not re-measured on the H100: a resident forest ties
     * with the warp kernel from 65 536 rows up (and sums in sklearn's tree order); a streamed forest wins from ~24k rows */
    m->tile_min_rows = (tp.n_pieces <= tp.n_slots) ? 65536 : 24576;
    if (env.tile_min_rows >= 0) m->tile_min_rows = env.tile_min_rows;
    if (env.kernel == KN_TILE) m->tile_min_rows = 1;
    return B2F_OK;
}

/* streams, and the feature-moments kernel's scratch */
static int streams_init(b2f_model *m) {
    for (int s = 0; s < B2F_STREAMS; ++s) CUDA_TRY(cudaStreamCreateWithFlags(&m->slots[s].stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&m->compute, cudaStreamNonBlocking));
    CUDA_TRY(set_smem_limit(k_feature_moments, B2F_MOM_SMEM));
    m->mom_blocks = m->sm_count * 3; /* one full wave: 3 CTAs (3-stage 72 KB ring each) per SM */
    CUDA_TRY(cudaMalloc(&m->d_mom_partials, (size_t)m->mom_blocks * B2F_MOM_PARTIAL_VALUES * sizeof(double)));
    CUDA_TRY(cudaMalloc(&m->d_mom_ticket, sizeof(unsigned int)));
    CUDA_TRY(cudaMemset(m->d_mom_ticket, 0, sizeof(unsigned int)));
    CUDA_TRY(cudaMalloc(&m->d_mom_out, B2F_MOM_VALUES * sizeof(double)));
    return B2F_OK;
}

static int model_init_cuda(b2f_model *m, const uint8_t *blob, size_t nbytes) {
    const EnvHooks env = read_env_hooks();
    CUDA_TRY(cudaSetDevice(m->device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, m->device));
    if (prop.major != 9 || prop.minor != 0)
        return set_err(B2F_ENODEV, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", m->device, prop.major, prop.minor);
    m->sm_count = prop.multiProcessorCount;
    CUDA_TRY(cudaDeviceGetAttribute(&m->max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, m->device));
    CUDA_TRY(cudaMalloc(&m->d_blob, nbytes));
    CUDA_TRY(cudaMemcpy(m->d_blob, blob, nbytes, cudaMemcpyHostToDevice));
    m->forest_bytes = (int64_t)m->hdr.chunks_bytes;
    int rc = warp_init(m, blob, env);
    if (rc == B2F_OK) rc = tile_init(m, blob, env);
    if (rc == B2F_OK) rc = rank_init(m, blob, env);
    if (rc == B2F_OK) rc = streams_init(m);
    return rc;
}

extern "C" b2f_model *b2f_model_create(const void *forest_blob, size_t nbytes, int device) {
    int ndev = b2f_device_count();
    if (ndev < 0) return nullptr;
    if (device < 0 || device >= ndev) {
        set_err(B2F_EINVAL, "device %d out of range (have %d)", device, ndev);
        return nullptr;
    }
    b2f_model *m = new (std::nothrow) b2f_model();
    if (!m) {
        set_err(B2F_ENOMEM, "out of host memory");
        return nullptr;
    }
    m->device = device;
    if (validate_blob(static_cast<const uint8_t *>(forest_blob), nbytes, &m->hdr) != B2F_OK ||
        model_init_cuda(m, static_cast<const uint8_t *>(forest_blob), nbytes) != B2F_OK) {
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        b2f_model_destroy(m);
        memcpy(g_err, keep, sizeof(keep));
        return nullptr;
    }
    return m;
}

extern "C" void b2f_model_destroy(b2f_model *m) {
    if (!m) return;
    cudaSetDevice(m->device);
    cudaDeviceSynchronize();
    if (m->outlier) b2f_model_destroy(m->outlier);
    if (m->ex) explainer_free(m->ex);
    if (m->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(m->comm);
    for (Slot &sl : m->slots) {
        for (DevBuf *b : {&sl.rows, &sl.out, &sl.label, &sl.scratch}) b->release();
        if (sl.stream) cudaStreamDestroy(sl.stream);
    }
    for (DevBuf *b : {&m->scratch, &m->pd.host_spec, &m->pd.device_spec, &m->cf.dev, &m->mom_rows, &m->gather, &m->flush}) b->release();
    for (DevBuf *b : {&m->pair.host_spec, &m->pair.spec_dev, &m->pair.rows, &m->pair.partial, &m->pair.out}) b->release();
    for (DevBuf *b : {&m->ale.spec_dev, &m->ale.rows, &m->ale.psum, &m->ale.pcnt, &m->ale.sums, &m->ale.counts}) b->release();
    for (DevBuf *b : {&m->pi.rows, &m->pi.labels, &m->pi.perm, &m->pi.keys, &m->pi.flags, &m->pi.temp, &m->pi.offsets, &m->pi.segs, &m->pi.scores}) b->release();
    for (EmbeddedRef *e : {&m->mmd.ref, &m->knn.ref})
        for (DevBuf *b : {&e->ref_z, &e->ref_c, &e->rows, &e->z, &e->c}) b->release();
    for (DevBuf *b : {&m->mmd.r_ref, &m->mmd.r, &m->mmd.partial, &m->mmd.sub, &m->mmd.pairs, &m->mmd.out, &m->mmd.hist}) b->release();
    {
        MmdOnline &o = m->mmd.online;
        for (DevBuf *b : {&o.total, &o.rz, &o.rc, &o.carry_z, &o.carry_c, &o.carry_cv, &o.init_z, &o.init_c, &o.init_cv, &o.pos, &o.band,
                          &o.qsum, &o.cv, &o.stats, &o.krr, &o.seq_z, &o.seq_c, &o.out})
            b->release();
    }
    for (DevBuf *b : {&m->knn.orig, &m->knn.cand_d, &m->knn.cand_i, &m->knn.dist, &m->knn.index}) b->release();
    for (auto &t : m->tickets)
        for (auto &e : t.ev)
            if (e) cudaEventDestroy(e);
    if (m->compute) cudaStreamDestroy(m->compute);
    if (m->d_blob) cudaFree(m->d_blob);
    if (m->d_tile_layout) cudaFree(m->d_tile_layout);
    if (m->d_kp) cudaFree(m->d_kp);
    if (m->d_tile_pieces) cudaFree(m->d_tile_pieces);
    if (m->d_rank_layout) cudaFree(m->d_rank_layout);
    if (m->d_mom_partials) cudaFree(m->d_mom_partials);
    if (m->d_mom_ticket) cudaFree(m->d_mom_ticket);
    if (m->d_mom_out) cudaFree(m->d_mom_out);
    delete m;
}

static int pick_rows_per_warp(const b2f_model *m, int64_t n) {
    int r = m->rows_per_warp_max;
    const int64_t warps = (int64_t)m->sm_count * B2F_PREDICT_WARPS;
    while (r > 1 && n / r < warps) r >>= 1; /* small batches: spread rows over more warps */
    return r;
}

extern "C" int b2f_model_info(const b2f_model *m, b2f_info *out) {
    if (!m || !out) return set_err(B2F_EINVAL, "null argument");
    memset(out, 0, sizeof(*out));
    out->device = m->device;
    out->sm_count = m->sm_count;
    out->agg_mode = (int)m->hdr.agg_mode;
    out->walk_mode = m->walk_mode;
    out->n_trees = (int)m->hdr.n_trees;
    out->n_groups = (int)m->hdr.n_groups;
    out->max_depth = (int)m->hdr.max_depth;
    out->n_cat = (int)m->hdr.n_cat;
    out->n_num = (int)m->hdr.n_num;
    out->smem_bytes = m->smem_bytes;
    out->block_threads = B2F_PREDICT_THREADS;
    out->rows_per_warp = m->rows_per_warp_max;
    out->forest_bytes = m->forest_bytes;
    out->launches = m->launches + (m->outlier ? m->outlier->launches : 0);
    out->launches_tile = m->launches_tile + (m->outlier ? m->outlier->launches_tile : 0);
    out->tile_min_rows = m->tile_min_rows;
    out->tile_ok = m->tile_ok ? 1 : 0;
    out->tile_resident = (m->tile_ok && m->tp.n_pieces <= m->tp.n_slots) ? 1 : 0;
    out->packed_ok = m->packed_ok ? 1 : 0;
    out->tile_warps = m->tile_ok ? m->tile_cwarps : 0;
    out->launches_split = m->launches_split;
    out->split_max_rows = m->split_max_rows;
    out->outlier_trees = m->outlier ? (int)m->outlier->hdr.n_trees : 0;
    out->rank_ok = m->rank_ok ? 1 : 0;
    out->launches_rank = m->launches_rank;
    out->rank_smem_bytes = m->rank_ok ? m->rank_smem_bytes : 0;
    out->rank_row_bytes = m->rk.row_bytes;
    out->rank_stream = (m->rank_ok && m->rank_stream) ? 1 : 0;
    return B2F_OK;
}

extern "C" int b2f_model_rank_info(const b2f_model *m, b2f_rank_info *out) {
    if (!m || !out) return set_err(B2F_EINVAL, "null argument");
    fill_rank_info(&m->rk, m->rank_ok, out);
    if (m->rk.ok && !m->rank_ok) snprintf(out->why, sizeof(out->why), "the rank layout (%zu bytes) does not stay resident in shared memory", m->rk.layout.size());
    return B2F_OK;
}

/* ------------------------------------------------------------------ pinned memory */
extern "C" void *b2f_pinned_alloc(size_t nbytes) {
    void *p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, nbytes ? nbytes : 1, cudaHostAllocPortable);
    if (e != cudaSuccess) {
        set_err(B2F_ENOMEM, "cudaHostAlloc(%zu) failed: %s", nbytes, cudaGetErrorString(e));
        return nullptr;
    }
    return p;
}
extern "C" void b2f_pinned_free(void *p) {
    if (p) cudaFreeHost(p);
}

/* ------------------------------------------------------------------ kernel launch */
enum KernelKind { KERN_RANK, KERN_TILE, KERN_SPLIT, KERN_WARP };
struct KernelChoice {
    KernelKind kind;
    int rows_per_warp = 0; /* KERN_WARP */
    bool smem = false;     /* KERN_WARP: the forest is resident in shared memory */
};

/* which kernel scores n rows of format fmt */
static KernelChoice pick_kernel(const b2f_model *m, int64_t n, int fmt) {
    if (fmt == B2F_ROWS_RANKED) return {KERN_RANK}; /* ranked rows have one kernel: integer compares on the rank layout */
    if (m->tile_ok && n >= m->tile_min_rows) return {KERN_TILE};
    if (n <= m->split_max_rows) return {KERN_SPLIT}; /* a handful of rows: spread each row's tree groups over the warps of a CTA */
    return {KERN_WARP, pick_rows_per_warp(m, n), m->walk_mode == B2F_WALK_SMEM};
}

/* persistent kernels: one CTA per `rows_per_cta` rows, at most one per SM */
static unsigned persistent_ctas(const b2f_model *m, int64_t n, int64_t rows_per_cta) {
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>(m->sm_count, (n + rows_per_cta - 1) / rows_per_cta));
}

#ifdef B2F_RANK_PHASES
/* diagnostic build: every rank launch takes the next record of the buffer armed by b2f_rank_phases_arm (tools/rank_phases.py) */
static int32_t g_rank_phase_next = 0;
extern "C" int b2f_rank_phases_arm(b2f_model *m, void *dev_buf, int launches) {
    if (!m || !m->rank_ok) return set_err(B2F_EINVAL, "no rank kernel on this model");
    m->rp.phases = static_cast<unsigned long long *>(dev_buf);
    m->rp.phase_launches = dev_buf ? launches : 0;
    g_rank_phase_next = 0;
    return B2F_OK;
}
#endif

/* The rank kernel goes out with programmatic stream serialization, which relaxes the edge from one such launch to the next
 * on the same stream only: a CTA of launch N + 1 may start as soon as a CTA of launch N retires, and the kernel reads its rows
 * and walks before griddepcontrol.wait.  That is safe because no rank launch writes rows, and everything else that can
 * write them (H2D copies, every other kernel of this library or of the caller) is an ordinary stream predecessor of the
 * first relaxed launch of a chain.  The stores of launch N + 1 follow its wait, so the last launch writing a buffer wins. */
template <typename OutT>
static cudaError_t launch_rank(const b2f_model *m, cudaStream_t st, const void *rows, int64_t n, OutT *proba, int32_t *label, int ostride) {
    const RankKernel<OutT> kernel = rank_kernel<OutT>(m);
    if (!kernel) return cudaErrorInvalidValue;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(persistent_ctas(m, n, 32));
    cfg.blockDim = dim3(B2F_RANK_THREADS);
    cfg.dynamicSmemBytes = (size_t)m->rank_smem_bytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = m->rank_pdl ? 1 : 0;
#ifdef B2F_RANK_PHASES
    RParams rp = m->rp;
    rp.phase_launch = g_rank_phase_next++;
#else
    const RParams &rp = m->rp;
#endif
    return cudaLaunchKernelEx(&cfg, kernel, rp, static_cast<const uint8_t *>(rows), (long long)n, proba, label, ostride);
}

template <typename OutT>
static cudaError_t launch_kernel(const b2f_model *m, const KernelChoice &kc, bool pk, cudaStream_t st, const void *rows, int64_t n, OutT *proba,
                                 int32_t *label, int ostride) {
    const uint32_t *w = static_cast<const uint32_t *>(rows);
    switch (kc.kind) {
    case KERN_RANK:
        return launch_rank(m, st, rows, n, proba, label, ostride);
    case KERN_TILE:
        tile_kernel<OutT>(pk)<<<persistent_ctas(m, n, B2F_TILE_ROWS), (unsigned)(m->tile_cwarps + 1) * 32u, m->tile_smem_bytes, st>>>(m->tp, w, (long long)n, proba, label, ostride);
        break;
    case KERN_SPLIT: /* R = 2 rows per CTA */
        split_kernel<OutT>(pk)<<<(unsigned)((n + 1) / 2), 32u * (unsigned)m->kp.n_groups, 0, st>>>(m->kp, w, (long long)n, proba, label, ostride);
        break;
    case KERN_WARP:
        warp_kernel<OutT>(kc.rows_per_warp, kc.smem, pk)<<<persistent_ctas(m, n, kc.rows_per_warp), B2F_PREDICT_THREADS, kc.smem ? m->smem_bytes : 0, st>>>(
            m->kp, w, (long long)n, proba, label, ostride);
        break;
    }
    return cudaGetLastError();
}

static size_t row_bytes_of(const b2f_model *m, int fmt) {
    return fmt == B2F_ROWS_RANKED ? (size_t)m->rk.row_bytes : (fmt == B2F_ROWS_PACKED64 ? B2F_PACKED_ROW_BYTES : B2F_ROW_BYTES);
}

static int check_row_format(const b2f_model *m, int fmt) {
    if (fmt == B2F_ROWS_WORDS24) return B2F_OK;
    if (fmt == B2F_ROWS_RANKED) {
        if (!m->rank_ok)
            return set_err(B2F_EINVAL, "B2F_ROWS_RANKED is not available for this model (%s)",
                           m->rk.ok ? "its rank layout fits neither shared memory nor the streaming ring" : m->rk.why);
        return B2F_OK;
    }
    if (fmt != B2F_ROWS_PACKED64) return set_err(B2F_EINVAL, "unknown row format %d", fmt);
    if (!m->packed_ok) return set_err(B2F_EINVAL, "this model's schema does not fit the packed 64-byte row (needs exactly 9 categoricals with <= 126 categories, <= 14 numerics)");
    return B2F_OK;
}

static int launch_predict(b2f_model *m, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, bool f64, void *proba_dev, int32_t *label_dev,
                          int ostride = 1) {
    static const char *const names[] = {"k_forest_predict_rank", "k_forest_predict_tile", "k_forest_predict_split", "k_forest_predict"};
    if (n <= 0) return B2F_OK;
    const KernelChoice kc = pick_kernel(m, n, fmt);
    const bool pk = fmt == B2F_ROWS_PACKED64;
    const cudaError_t e = f64 ? launch_kernel(m, kc, pk, st, rows_dev, n, static_cast<double *>(proba_dev), label_dev, ostride)
                              : launch_kernel(m, kc, pk, st, rows_dev, n, static_cast<float *>(proba_dev), label_dev, ostride);
    if (e != cudaSuccess) return set_err(B2F_ECUDA, "%s launch failed: %s", names[kc.kind], cudaGetErrorString(e));
    m->launches++;
    if (kc.kind == KERN_RANK) m->launches_rank++;
    if (kc.kind == KERN_TILE) m->launches_tile++;
    if (kc.kind == KERN_SPLIT) m->launches_split++;
    return B2F_OK;
}

/* ------------------------------------------------------------------ output kinds (B2F_OUT_* in b2f.h)
 * What one output row of a host-buffer call looks like, and which launches write it into a device buffer. */
static size_t out_row_bytes(int kind) {
    switch (kind) {
    case B2F_OUT_F32: return sizeof(float);
    case B2F_OUT_F64: return sizeof(double);
    case B2F_OUT_PAIRS: return sizeof(b2f_scored);
    case B2F_OUT_FULL: return sizeof(b2f_scored_full);
    }
    return 0;
}

/* have_out: the record pointer is not NULL, or there are no rows to write */
static int out_check(const b2f_model *m, int kind, int fmt, bool have_out) {
    if (!out_row_bytes(kind))
        return set_err(B2F_EINVAL, "output kind %d: expected 0 (float), 1 (double), 2 (b2f_scored) or 3 (b2f_scored_full)", kind);
    if (kind >= B2F_OUT_PAIRS && !have_out) return set_err(B2F_EINVAL, "record output requested but the output pointer is NULL");
    if (kind == B2F_OUT_FULL && !m->outlier) return set_err(B2F_ESTATE, "no outlier forest attached (b2f_model_attach_outlier_forest)");
    if (kind == B2F_OUT_FULL && fmt == B2F_ROWS_RANKED)
        return set_err(B2F_EINVAL, "b2f_scored_full records take float32 rows (B2F_ROWS_WORDS24 / B2F_ROWS_PACKED64): ranks are relative to ONE forest's split values");
    return B2F_OK;
}

/* F32 / F64: proba and label arrays (either may be NULL).  PAIRS: {float, int32} records.  FULL: the classifier, then the
 * outlier forest, on the same device rows, into 24-byte records (label_dev is ignored for records). */
static int out_launch(b2f_model *m, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, int kind, void *out_dev, int32_t *label_dev) {
    static_assert(sizeof(b2f_scored_full) == 24 && offsetof(b2f_scored_full, label) == 8 && offsetof(b2f_scored_full, is_outlier) == 12 &&
                      offsetof(b2f_scored_full, outlier_score) == 16,
                  "b2f_scored_full layout");
    uint8_t *rec = static_cast<uint8_t *>(out_dev);
    if (kind == B2F_OUT_PAIRS) return launch_predict(m, st, rows_dev, n, fmt, false, rec, reinterpret_cast<int32_t *>(rec + 4), 2);
    if (kind != B2F_OUT_FULL) return launch_predict(m, st, rows_dev, n, fmt, kind == B2F_OUT_F64, out_dev, label_dev);
    int rc = launch_predict(m, st, rows_dev, n, fmt, true, rec, reinterpret_cast<int32_t *>(rec + 8), B2F_OSTRIDE(3, 6));
    if (rc) return rc;
    return launch_predict(m->outlier, st, rows_dev, n, fmt, false, rec + 16, reinterpret_cast<int32_t *>(rec + 12), B2F_OSTRIDE(6, 6));
}

/* ------------------------------------------------------------------ host-buffer pipeline
 * A host batch is a job: its entry point checks what the job needs and builds this record once per call.  The pipeline
 * (enqueue_host_batch, submit_chunk, timed_host_batch) reads nothing else about what the batch computes. */
struct HostJob {
    size_t row_bytes;   /* bytes of one output row */
    int64_t chunk_rows; /* rows per chunk; 0: the model's chunk size and chunk plan */
    bool label;         /* writes the caller's label array */
    int kind;           /* passed to launch: a B2F_OUT_* kind for scores, the TreeSHAP variant for explanations */
    /* one chunk: n device rows of format fmt on stream st into out_dev (NULL: no output) and label_dev (NULL: no labels), with
     * scratch for partial sums */
    int (*launch)(b2f_model *m, int kind, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, void *out_dev, int32_t *label_dev,
                  DevBuf &scratch);
};

/* the job of a score batch of output kind B2F_OUT_* (checked by out_check) */
static HostJob score_job(int kind) {
    return {out_row_bytes(kind), 0, kind == B2F_OUT_F32 || kind == B2F_OUT_F64, kind,
            [](b2f_model *m, int kind, cudaStream_t st, const void *rows_dev, int64_t n, int fmt, void *out_dev, int32_t *label_dev, DevBuf &) {
                return out_launch(m, st, rows_dev, n, fmt, kind, out_dev, label_dev);
            }};
}

static int score_check(const b2f_model *m, int64_t n, int kind, int fmt, const void *out) {
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    return out_check(m, kind, fmt, out || n == 0);
}

/* One chunk on one slot: rows [lo, lo + cnt) of the caller's host rows -> H2D -> the job's launch -> D2H into the caller's
 * host output(s) at row lo.  marks (B2F_TIMELINE, may be NULL) gets an event before the first chunk's H2D, then one after
 * each of its H2D, launches and D2H. */
static int submit_chunk(b2f_model *m, Slot &sl, const HostJob &job, const void *rows, int fmt, void *out, int32_t *label, int64_t lo, int64_t cnt,
                        std::vector<cudaEvent_t> *marks) {
    if (!job.label) label = nullptr;
    const size_t row_bytes = row_bytes_of(m, fmt), cap = (size_t)std::max<int64_t>(cnt, 1024); /* rows each buffer holds */
    int rc = sl.rows.reserve(sl.stream, (size_t)cnt * B2F_ROW_BYTES, cap * B2F_ROW_BYTES);
    if (rc == B2F_OK && out) rc = sl.out.reserve(sl.stream, (size_t)cnt * job.row_bytes, cap * job.row_bytes);
    if (rc == B2F_OK && label) rc = sl.label.reserve(sl.stream, (size_t)cnt * sizeof(int32_t), cap * sizeof(int32_t));
    if (rc) return rc;
    auto mark = [&] {
        if (!marks) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, sl.stream);
        marks->push_back(e);
    };
    if (marks && marks->empty()) mark();
    CUDA_TRY(cudaMemcpyAsync(sl.rows.p, static_cast<const uint8_t *>(rows) + (size_t)lo * row_bytes, (size_t)cnt * row_bytes, cudaMemcpyHostToDevice,
                             sl.stream));
    mark();
    rc = job.launch(m, job.kind, sl.stream, sl.rows.p, cnt, fmt, out ? sl.out.p : nullptr, label ? static_cast<int32_t *>(sl.label.p) : nullptr,
                    sl.scratch);
    if (rc) return rc;
    mark();
    if (out)
        CUDA_TRY(cudaMemcpyAsync(static_cast<uint8_t *>(out) + (size_t)lo * job.row_bytes, sl.out.p, (size_t)cnt * job.row_bytes,
                                 cudaMemcpyDeviceToHost, sl.stream));
    if (label) CUDA_TRY(cudaMemcpyAsync(label + lo, sl.label.p, (size_t)cnt * sizeof(int32_t), cudaMemcpyDeviceToHost, sl.stream));
    mark();
    return B2F_OK;
}

/* enqueue the whole batch of n >= 0 rows; on return used_mask tells which slot streams carry work.
 * B2F_TIMELINE=1 (debug): record an event after every operation and print the schedule to stderr. */
static int enqueue_host_batch(b2f_model *m, const HostJob &job, const void *rows, int64_t n, int fmt, void *out, int32_t *label,
                              uint32_t *used_mask) {
    *used_mask = 0;
    if (n == 0) return B2F_OK;
    if (!rows) return set_err(B2F_EINVAL, "rows is NULL");
    int rc = check_row_format(m, fmt);
    if (rc) return rc;
    CUDA_TRY(cudaSetDevice(m->device));
    int64_t chunk = job.chunk_rows ? job.chunk_rows : m->chunk_rows;
    if (n <= chunk + chunk / 2) chunk = n; /* small batch: one H2D, one launch */
    static const bool timeline = getenv("B2F_TIMELINE") != nullptr;
    std::vector<cudaEvent_t> tev;
    /* chunk schedule: equal chunks by default; a plan (B2F_CHUNK_PLAN="a,b,c": fractions of the batch in
     * 1/1024ths, the last chunk takes the remainder) front-loads the copies so the un-overlapped tail --
     * the last chunk's kernel and D2H -- is short */
    const bool planned = !job.chunk_rows && !m->chunk_plan.empty() && chunk != n && n >= 2 * m->chunk_rows;
    int c = 0;
    for (int64_t off = 0; off < n; ++c) {
        int64_t cnt = std::min(chunk, n - off);
        if (planned) {
            cnt = (size_t)c < m->chunk_plan.size() ? std::max<int64_t>(1024, (n * m->chunk_plan[c] / 1024 + 1023) / 1024 * 1024) : n - off;
            cnt = std::min(cnt, n - off);
        }
        /* slots rotate ACROSS calls too, so with several batches in flight (async ring, stream dealer) the next
         * batch's H2D does not wait for the previous batch's kernel to release the same staging buffer */
        const int slot_idx = (int)((m->next_slot + (uint64_t)c) % B2F_STREAMS);
        rc = submit_chunk(m, m->slots[slot_idx], job, rows, fmt, out, label, off, cnt, timeline ? &tev : nullptr);
        if (rc) return rc;
        *used_mask |= 1u << slot_idx;
        off += cnt;
    }
    m->next_slot += (uint64_t)c;
    if (timeline) {
        cudaDeviceSynchronize();
        fprintf(stderr, "[b2f timeline] n=%lld chunk=%lld :", (long long)n, (long long)chunk);
        for (size_t i = 1; i < tev.size(); ++i) {
            float ms = 0;
            cudaEventElapsedTime(&ms, tev[0], tev[i]);
            fprintf(stderr, " %s%.1f", (i % 3 == 1) ? "| h2d " : (i % 3 == 2 ? "k " : "d2h "), ms * 1e3f);
        }
        fprintf(stderr, " (us)\n");
        for (auto e : tev) cudaEventDestroy(e);
    }
    return B2F_OK;
}

static int sync_mask(b2f_model *m, uint32_t mask) {
    for (int s = 0; s < B2F_STREAMS; ++s)
        if (mask & (1u << s)) CUDA_TRY(cudaStreamSynchronize(m->slots[s].stream));
    return B2F_OK;
}

static int predict_host(b2f_model *m, const void *rows, int64_t n, int fmt, void *out, int kind, int32_t *label) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    uint32_t mask = 0;
    int rc = score_check(m, n, kind, fmt, out);
    if (rc == B2F_OK) rc = enqueue_host_batch(m, score_job(kind), rows, n, fmt, out, label, &mask);
    int rc2 = sync_mask(m, mask);
    return rc ? rc : rc2;
}

extern "C" int b2f_predict(b2f_model *m, const void *rows, int64_t n, float *proba1, int32_t *label) {
    return predict_host(m, rows, n, B2F_ROWS_WORDS24, proba1, B2F_OUT_F32, label);
}
extern "C" int b2f_predict_f64(b2f_model *m, const void *rows, int64_t n, double *proba1, int32_t *label) {
    return predict_host(m, rows, n, B2F_ROWS_WORDS24, proba1, B2F_OUT_F64, label);
}
extern "C" int b2f_predict_ex(b2f_model *m, const void *rows, int64_t n, int row_format, void *proba1, int proba_is_f64, int32_t *label) {
    return predict_host(m, rows, n, row_format, proba1, proba_is_f64 ? B2F_OUT_F64 : B2F_OUT_F32, label);
}
extern "C" int b2f_predict_pairs(b2f_model *m, const void *rows, int64_t n, int row_format, b2f_scored *out) {
    return predict_host(m, rows, n, row_format, out, B2F_OUT_PAIRS, nullptr);
}

extern "C" int b2f_model_attach_outlier_forest(b2f_model *m, const void *forest_blob, size_t nbytes) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    b2f_blob_header h;
    int rc = validate_blob(static_cast<const uint8_t *>(forest_blob), nbytes, &h);
    if (rc) return rc;
    if (h.agg_mode != B2F_AGG_IFOREST) return set_err(B2F_EINVAL, "outlier forest: agg_mode %u is not B2F_AGG_IFOREST", h.agg_mode);
    if (h.n_cat != m->hdr.n_cat || h.n_num != m->hdr.n_num)
        return set_err(B2F_EINVAL, "outlier forest: row schema (%u categorical, %u numeric) differs from the model's (%u, %u)", h.n_cat, h.n_num,
                       m->hdr.n_cat, m->hdr.n_num);
    b2f_model *child = b2f_model_create(forest_blob, nbytes, m->device);
    if (!child) return B2F_ECUDA; /* message set by b2f_model_create */
    CUDA_TRY(cudaSetDevice(m->device));
    if (m->outlier) {
        CUDA_TRY(cudaDeviceSynchronize());
        b2f_model_destroy(m->outlier);
    }
    m->outlier = child;
    return B2F_OK;
}

extern "C" int b2f_predict_full(b2f_model *m, const void *rows, int64_t n, int row_format, b2f_scored_full *out) {
    return predict_host(m, rows, n, row_format, out, B2F_OUT_FULL, nullptr);
}

/* CUDA events, destroyed on every return path */
struct Events {
    std::vector<cudaEvent_t> e;
    int create(size_t n) {
        e.assign(n, nullptr);
        for (cudaEvent_t &x : e) CUDA_TRY(cudaEventCreate(&x));
        return B2F_OK;
    }
    ~Events() {
        for (cudaEvent_t x : e)
            if (x) cudaEventDestroy(x);
    }
};

/* ------------------------------------------------------------------ helpers of the entry points beside scoring (moments, *_api.cuh) */

/* reserve bytes of b on the compute stream, a failure reported as B2F_ENOMEM and its byte count */
static int compute_reserve(b2f_model *m, DevBuf &b, size_t bytes, const char *who, const char *what) {
    if (b.reserve(m->compute, bytes, bytes) == B2F_OK) return B2F_OK;
    (void)cudaGetLastError(); /* the failed cudaMalloc's error: not left for the next launch check to report */
    return set_err(B2F_ENOMEM, "%s: cannot allocate %zu device bytes for %s", who, bytes, what);
}

/* after a <<< >>> launch (or cudaLaunchKernel): its error, or one more launch counted */
static int launched(b2f_model *m, const char *name) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_err(B2F_ECUDA, "%s launch failed: %s", name, cudaGetErrorString(e));
    m->launches++;
    return B2F_OK;
}

/* device_ms (may be NULL) of a region of the compute stream: start() records its start; finish() records its end, waits for
 * the stream (also without device_ms) and writes the elapsed time */
struct TimedRegion {
    b2f_model *m;
    float *device_ms;
    Events evs;
    int start() {
        if (!device_ms) return B2F_OK;
        const int rc = evs.create(2);
        if (rc) return rc;
        CUDA_TRY(cudaEventRecord(evs.e[0], m->compute));
        return B2F_OK;
    }
    int finish() {
        const cudaStream_t st = m->compute;
        if (device_ms) CUDA_TRY(cudaEventRecord(evs.e[1], st));
        CUDA_TRY(cudaStreamSynchronize(st));
        if (device_ms) CUDA_TRY(cudaEventElapsedTime(device_ms, evs.e[0], evs.e[1]));
        return B2F_OK;
    }
};

/* every analysis reads row values, which ranked rows do not carry; subject: the caller with its verb ("explanations take") */
static int check_value_rows(int fmt, const char *subject) {
    if (fmt == B2F_ROWS_RANKED)
        return set_err(B2F_EINVAL, "%s float32 rows (B2F_ROWS_WORDS24 / B2F_ROWS_PACKED64): ranked rows carry no values", subject);
    return B2F_OK;
}

/* a mask walk holds at most one stack entry per level of the tree; subject: the caller with its verb ("counterfactuals walk") */
static int check_walk_depth(const b2f_model *m, const char *subject) {
    const b2f_blob_header &h = m->hdr;
    if (h.max_depth > B2F_PD_STACK) return set_err(B2F_EINVAL, "%s trees of depth <= %d; this forest has depth %u", subject, B2F_PD_STACK, h.max_depth);
    return B2F_OK;
}

/* a mask-walk spec: the segment table, then the point words */
template <typename Seg>
static void pack_spec(std::vector<uint32_t> &spec, const std::vector<Seg> &segs, const std::vector<uint32_t> &words) {
    spec.assign(segs.size() * (sizeof(Seg) / sizeof(uint32_t)), 0u);
    memcpy(spec.data(), segs.data(), segs.size() * sizeof(Seg));
    spec.insert(spec.end(), words.begin(), words.end());
}

/* a call's spec into buf: synchronously, before a host job's chunks (each host call synchronises, so no earlier call still
 * reads it), or on the compute stream (async), ordered with the launches that read it.  who: the prefix of a failed
 * allocation's B2F_ENOMEM; NULL: DevBuf::reserve's B2F_ECUDA */
static int upload_spec(b2f_model *m, DevBuf &buf, const std::vector<uint32_t> &spec, bool async, const char *who) {
    const size_t bytes = spec.size() * sizeof(uint32_t);
    const int rc = who ? compute_reserve(m, buf, bytes, who, "the point table") : buf.reserve(m->compute, bytes, bytes);
    if (rc) return rc;
    if (async) CUDA_TRY(cudaMemcpyAsync(buf.p, spec.data(), bytes, cudaMemcpyHostToDevice, m->compute));
    else CUDA_TRY(cudaMemcpy(buf.p, spec.data(), bytes, cudaMemcpyHostToDevice));
    return B2F_OK;
}

/* a synchronous host batch of n >= 0 rows of a checked job; device_ms (may be NULL): from the first H2D to the end of the last
 * chunk */
static int timed_host_batch(b2f_model *m, const HostJob &job, const void *rows, int64_t n, int row_format, double *out, float *device_ms) {
    if (device_ms) *device_ms = 0.0f;
    CUDA_TRY(cudaSetDevice(m->device));
    Events evs;
    const int first = (int)(m->next_slot % B2F_STREAMS);
    if (device_ms && n > 0) {
        int rc = evs.create(1 + B2F_STREAMS);
        if (rc) return rc;
        CUDA_TRY(cudaEventRecord(evs.e[0], m->slots[first].stream));
    }
    cudaEvent_t *ev = evs.e.data();
    uint32_t mask = 0;
    int rc = enqueue_host_batch(m, job, rows, n, row_format, out, nullptr, &mask);
    if (device_ms && n > 0 && rc == B2F_OK)
        for (int s = 0; s < B2F_STREAMS && rc == B2F_OK; ++s)
            if ((mask & (1u << s)) && cudaEventRecord(ev[1 + s], m->slots[s].stream) != cudaSuccess)
                rc = set_err(B2F_ECUDA, "cudaEventRecord failed: %s", cudaGetErrorString(cudaGetLastError()));
    int rc2 = sync_mask(m, mask); /* always: the chunks already enqueued write into the caller's output */
    if (rc == B2F_OK) rc = rc2;
    if (device_ms && n > 0)
        for (int s = 0; s < B2F_STREAMS && rc == B2F_OK; ++s)
            if (mask & (1u << s)) {
                float ms = 0.0f;
                CUDA_TRY(cudaEventElapsedTime(&ms, ev[0], ev[1 + s]));
                *device_ms = std::max(*device_ms, ms);
            }
    return rc;
}

extern "C" int b2f_predict_async(b2f_model *m, const void *rows_pinned, int64_t n, void *proba1_pinned, int proba_is_f64,
                                 int32_t *label_pinned, b2f_ticket *ticket) {
    return b2f_predict_async_ex(m, rows_pinned, n, B2F_ROWS_WORDS24, proba1_pinned, proba_is_f64, label_pinned, ticket);
}

extern "C" int b2f_predict_async_ex(b2f_model *m, const void *rows_pinned, int64_t n, int row_format, void *proba1_pinned, int proba_is_f64,
                                    int32_t *label_pinned, b2f_ticket *ticket) {
    if (!m || !ticket) return set_err(B2F_EINVAL, "null argument");
    const uint64_t id = m->next_ticket++;
    TicketRec &t = m->tickets[id % B2F_TICKETS];
    if (t.id != 0) { /* oldest ticket still outstanding in this ring position: retire it */
        for (int s = 0; s < B2F_STREAMS; ++s)
            if (t.used_mask & (1u << s)) CUDA_TRY(cudaEventSynchronize(t.ev[s]));
    }
    uint32_t mask = 0;
    int rc = score_check(m, n, proba_is_f64, row_format, proba1_pinned);
    if (rc == B2F_OK) rc = enqueue_host_batch(m, score_job(proba_is_f64), rows_pinned, n, row_format, proba1_pinned, label_pinned, &mask);
    if (rc) {
        sync_mask(m, mask);
        return rc;
    }
    for (int s = 0; s < B2F_STREAMS; ++s)
        if (mask & (1u << s)) {
            if (!t.ev[s]) CUDA_TRY(cudaEventCreateWithFlags(&t.ev[s], cudaEventDisableTiming));
            CUDA_TRY(cudaEventRecord(t.ev[s], m->slots[s].stream));
        }
    t.id = id;
    t.used_mask = mask;
    *ticket = id;
    return B2F_OK;
}

extern "C" int b2f_wait(b2f_model *m, b2f_ticket ticket) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    TicketRec &t = m->tickets[ticket % B2F_TICKETS];
    if (t.id != ticket) return B2F_OK; /* already retired */
    CUDA_TRY(cudaSetDevice(m->device));
    for (int s = 0; s < B2F_STREAMS; ++s)
        if (t.used_mask & (1u << s)) CUDA_TRY(cudaEventSynchronize(t.ev[s]));
    t.id = 0;
    t.used_mask = 0;
    return B2F_OK;
}

extern "C" int b2f_predict_multi(b2f_model **models, int n_models, const void *rows, int64_t n, void *proba1, int proba_is_f64, int32_t *label) {
    return b2f_predict_multi_ex(models, n_models, rows, n, B2F_ROWS_WORDS24, proba1, proba_is_f64, label);
}

extern "C" int b2f_predict_multi_ex(b2f_model **models, int n_models, const void *rows, int64_t n, int row_format, void *proba1, int proba_is_f64,
                                    int32_t *label) {
    if (!models || n_models <= 0) return set_err(B2F_EINVAL, "no models");
    const size_t row_bytes = row_bytes_of(models[0], row_format);
    if (n < 0) return set_err(B2F_EINVAL, "negative row count");
    std::vector<uint32_t> masks(n_models, 0);
    const size_t out_bytes = out_row_bytes(proba_is_f64);
    int rc = B2F_OK;
    for (int i = 0; i < n_models && rc == B2F_OK; ++i) {
        const int64_t lo = n * i / n_models, hi = n * (i + 1) / n_models;
        if (hi <= lo) continue;
        rc = out_check(models[i], proba_is_f64, row_format, proba1 != nullptr);
        if (rc == B2F_OK)
            rc = enqueue_host_batch(models[i], score_job(proba_is_f64), static_cast<const uint8_t *>(rows) + (size_t)lo * row_bytes, hi - lo, row_format,
                                    proba1 ? static_cast<uint8_t *>(proba1) + (size_t)lo * out_bytes : nullptr, label ? label + lo : nullptr, &masks[i]);
    }
    for (int i = 0; i < n_models; ++i) {
        cudaSetDevice(models[i]->device);
        int rc2 = sync_mask(models[i], masks[i]);
        if (rc == B2F_OK) rc = rc2;
    }
    return rc;
}

static void bind_thread_near(int device); /* scorer.h */

/* Round-robin streaming over the GPUs of one box: batch b (rows [b*batch, (b+1)*batch)) goes to model b % n_models.
 * One host thread per GPU submits that GPU's batches through the asynchronous ring (at most `inflight` batches in
 * flight per GPU), so submission cost is paid in parallel; rows are independent, so there is no inter-GPU traffic. */
extern "C" int b2f_predict_stream(b2f_model **models, int n_models, const void *rows, int64_t n, int64_t batch, int row_format, void *proba1,
                                  int proba_is_f64, int32_t *label, int inflight) {
    if (!models || n_models <= 0 || batch <= 0 || n < 0) return set_err(B2F_EINVAL, "bad argument");
    if (inflight < 1) inflight = 1;
    if (inflight > 8) inflight = 8;
    const size_t row_bytes = row_bytes_of(models[0], row_format), out_bytes = out_row_bytes(proba_is_f64);
    const int64_t n_batches = (n + batch - 1) / batch;
    std::vector<int> rcs(n_models, B2F_OK);
    std::vector<std::string> msgs(n_models);
    auto worker = [&](int d) {
        b2f_model *m = models[d];
        bind_thread_near(m->device); /* submit from the GPU's own NUMA node (scorer.h) */
        std::vector<b2f_ticket> ring;
        int rc = B2F_OK;
        for (int64_t b = d; b < n_batches && rc == B2F_OK; b += n_models) {
            const int64_t lo = b * batch, cnt = std::min(batch, n - lo);
            if ((int)ring.size() >= inflight) {
                rc = b2f_wait(m, ring.front());
                ring.erase(ring.begin());
                if (rc) break;
            }
            b2f_ticket t = 0;
            rc = b2f_predict_async_ex(m, static_cast<const uint8_t *>(rows) + (size_t)lo * row_bytes, cnt, row_format,
                                      proba1 ? static_cast<uint8_t *>(proba1) + (size_t)lo * out_bytes : nullptr, proba_is_f64,
                                      label ? label + lo : nullptr, &t);
            if (rc == B2F_OK) ring.push_back(t);
        }
        for (b2f_ticket t : ring) {
            int rc2 = b2f_wait(m, t);
            if (rc == B2F_OK) rc = rc2;
        }
        rcs[d] = rc;
        if (rc) msgs[d] = b2f_last_error(); /* the message is thread-local: carry it back */
    };
    std::vector<std::thread> threads;
    for (int d = 0; d < n_models; ++d) threads.emplace_back(worker, d); /* every GPU its own thread: the caller's affinity is left alone */
    for (auto &t : threads) t.join();
    for (int d = 0; d < n_models; ++d)
        if (rcs[d]) return set_err(rcs[d], "GPU %d: %s", models[d]->device, msgs[d].c_str());
    return B2F_OK;
}

/* ------------------------------------------------------------------ device-resident interface */
extern "C" void *b2f_device_alloc(b2f_model *m, size_t nbytes) {
    if (!m) return nullptr;
    void *p = nullptr;
    if (cudaSetDevice(m->device) != cudaSuccess || cudaMalloc(&p, nbytes ? nbytes : 1) != cudaSuccess) {
        set_err(B2F_ENOMEM, "cudaMalloc(%zu) failed: %s", nbytes, cudaGetErrorString(cudaGetLastError()));
        return nullptr;
    }
    return p;
}
extern "C" void b2f_device_free(b2f_model *m, void *dptr) {
    if (!m || !dptr) return;
    cudaSetDevice(m->device);
    cudaFree(dptr);
}
extern "C" int b2f_copy_h2d(b2f_model *m, void *dst_dev, const void *src_host, size_t nbytes) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    CUDA_TRY(cudaSetDevice(m->device));
    CUDA_TRY(cudaMemcpyAsync(dst_dev, src_host, nbytes, cudaMemcpyHostToDevice, m->compute));
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    return B2F_OK;
}
extern "C" int b2f_copy_d2h(b2f_model *m, void *dst_host, const void *src_dev, size_t nbytes) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    CUDA_TRY(cudaSetDevice(m->device));
    CUDA_TRY(cudaMemcpyAsync(dst_host, src_dev, nbytes, cudaMemcpyDeviceToHost, m->compute));
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    return B2F_OK;
}
extern "C" int b2f_predict_device(b2f_model *m, const void *rows_dev, int64_t n, void *proba1_dev, int proba_is_f64, int32_t *label_dev) {
    return b2f_predict_device_ex(m, rows_dev, n, B2F_ROWS_WORDS24, proba1_dev, proba_is_f64, label_dev);
}
extern "C" int b2f_predict_device_ex(b2f_model *m, const void *rows_dev, int64_t n, int row_format, void *proba1_dev, int proba_is_f64,
                                     int32_t *label_dev) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    int rcf = check_row_format(m, row_format);
    if (rcf) return rcf;
    CUDA_TRY(cudaSetDevice(m->device));
    return out_launch(m, m->compute, rows_dev, n, row_format, proba_is_f64 ? B2F_OUT_F64 : B2F_OUT_F32, proba1_dev, label_dev);
}
extern "C" int b2f_sync(b2f_model *m) {
    if (!m) return set_err(B2F_EINVAL, "model is NULL");
    CUDA_TRY(cudaSetDevice(m->device));
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    return B2F_OK;
}

/* iters launches on the compute stream, timed by events this function owns.  ms_each: an event pair around each launch, after
 * a memset that flushes L2 when flush_l2 is set.  ms_total: one pair around the whole loop.  Without ms_each nothing is
 * recorded between launches: an event record between two launches keeps them from overlapping (programmatic dependent launch
 * of the rank kernel).  launch(i) enqueues launch i. */
template <typename Launch>
static int timed_launches(b2f_model *m, int iters, bool flush_l2, float *ms_each, float *ms_total, Launch launch) {
    const cudaStream_t st = m->compute;
    int rc = flush_l2 ? m->flush.reserve(st, B2F_FLUSH_BYTES, B2F_FLUSH_BYTES) : B2F_OK;
    Events ev;
    const size_t n_each = ms_each ? 2 * (size_t)iters : 0;
    if (rc == B2F_OK) rc = ev.create(n_each + (ms_total ? 2 : 0));
    if (rc) return rc;
    cudaEvent_t *each = ev.e.data(), *region = each + n_each;
    if (ms_total) CUDA_TRY(cudaEventRecord(region[0], st));
    for (int i = 0; i < iters && rc == B2F_OK; ++i) {
        if (flush_l2) CUDA_TRY(cudaMemsetAsync(m->flush.p, i & 0xff, B2F_FLUSH_BYTES, st));
        if (ms_each) CUDA_TRY(cudaEventRecord(each[2 * i], st));
        rc = launch(i);
        if (ms_each) CUDA_TRY(cudaEventRecord(each[2 * i + 1], st));
    }
    if (ms_total) CUDA_TRY(cudaEventRecord(region[1], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (rc) return rc;
    for (int i = 0; ms_each && i < iters; ++i) CUDA_TRY(cudaEventElapsedTime(&ms_each[i], each[2 * i], each[2 * i + 1]));
    if (ms_total) CUDA_TRY(cudaEventElapsedTime(ms_total, region[0], region[1]));
    return B2F_OK;
}

extern "C" int b2f_predict_device_timed(b2f_model *m, const void *rows_dev, int64_t n, void *proba1_dev, int proba_is_f64, int32_t *label_dev,
                                        int iters, int flush_l2, float *ms_each) {
    if (!m || iters <= 0 || !ms_each) return set_err(B2F_EINVAL, "bad argument");
    CUDA_TRY(cudaSetDevice(m->device));
    const int kind = proba_is_f64 ? B2F_OUT_F64 : B2F_OUT_F32;
    return timed_launches(m, iters, flush_l2, ms_each, nullptr,
                          [&](int) { return out_launch(m, m->compute, rows_dev, n, B2F_ROWS_WORDS24, kind, proba1_dev, label_dev); });
}

/* Streaming measurement: `steps` launches over a pool of `pool` distinct device-resident batches
 * (batch i%pool), so consecutive steps read different HBM lines (pool * n * 96 B should exceed L2).
 * Per-launch events (when ms_each is not NULL) and one region event pair, all on the launching stream. */
extern "C" int b2f_predict_stream_timed(b2f_model *m, const void *rows_dev, int64_t n, int pool, void *proba1_dev, int proba_is_f64,
                                        int32_t *label_dev, int steps, float *ms_each, float *ms_total) {
    return b2f_predict_stream_timed_ex(m, rows_dev, n, B2F_ROWS_WORDS24, pool, proba1_dev, proba_is_f64, label_dev, steps, ms_each, ms_total);
}

extern "C" int b2f_predict_stream_timed_ex(b2f_model *m, const void *rows_dev, int64_t n, int row_format, int pool, void *proba1_dev,
                                           int proba_is_f64, int32_t *label_dev, int steps, float *ms_each, float *ms_total) {
    if (!m || steps <= 0 || pool <= 0 || !ms_total) return set_err(B2F_EINVAL, "bad argument");
    {
        int rcf = check_row_format(m, row_format);
        if (rcf) return rcf;
    }
    const size_t row_bytes = row_bytes_of(m, row_format);
    CUDA_TRY(cudaSetDevice(m->device));
    const int kind = proba_is_f64 ? B2F_OUT_F64 : B2F_OUT_F32;
    const size_t out_bytes = out_row_bytes(kind);
    return timed_launches(m, steps, false, ms_each, ms_total, [&](int i) {
        const size_t b = (size_t)(i % pool);
        return out_launch(m, m->compute, static_cast<const uint8_t *>(rows_dev) + b * (size_t)n * row_bytes, n, row_format, kind,
                          proba1_dev ? static_cast<uint8_t *>(proba1_dev) + b * (size_t)n * out_bytes : nullptr, label_dev ? label_dev + b * (size_t)n : nullptr);
    });
}

/* ------------------------------------------------------------------ moments */
static int launch_moments(b2f_model *m, const void *rows_dev, int64_t n) {
    /* one CTA per 256-row slab up to a full wave of 3 CTAs per SM; small inputs get fewer CTAs so the
     * fixed-order final reduction over block partials stays short */
    const int64_t n_slabs = (n + B2F_MOM_SLAB_ROWS - 1) / B2F_MOM_SLAB_ROWS;
    int64_t blocks = std::min<int64_t>(m->mom_blocks, std::max<int64_t>(std::min<int64_t>(n_slabs, m->sm_count), n_slabs / 4));
    if (blocks < 1) blocks = 1;
    k_feature_moments<<<(unsigned)blocks, B2F_MOM_THREADS, B2F_MOM_SMEM, m->compute>>>(static_cast<const uint4 *>(rows_dev), (long long)n,
                                                                                     (int)m->hdr.n_cat, m->d_mom_partials, m->d_mom_ticket, m->d_mom_out);
    return launched(m, "k_feature_moments");
}

extern "C" int b2f_moments_device(b2f_model *m, const void *rows_dev, int64_t n, double *out) {
    if (!m || !out || n < 0) return set_err(B2F_EINVAL, "bad argument");
    CUDA_TRY(cudaSetDevice(m->device));
    int rc = launch_moments(m, rows_dev, n);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(out, m->d_mom_out, B2F_MOM_VALUES * sizeof(double), cudaMemcpyDeviceToHost, m->compute));
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    return B2F_OK;
}

static int moments_stage(b2f_model *m, const void *rows, int64_t n) {
    int rc = m->mom_rows.reserve(m->compute, (size_t)n * B2F_ROW_BYTES, (size_t)std::max<int64_t>(n, 1024) * B2F_ROW_BYTES);
    if (rc) return rc;
    if (n > 0) CUDA_TRY(cudaMemcpyAsync(m->mom_rows.p, rows, (size_t)n * B2F_ROW_BYTES, cudaMemcpyHostToDevice, m->compute));
    return B2F_OK;
}

extern "C" int b2f_moments(b2f_model *m, const void *rows, int64_t n, double *out) {
    if (!m || !out || n < 0 || (n > 0 && !rows)) return set_err(B2F_EINVAL, "bad argument");
    CUDA_TRY(cudaSetDevice(m->device));
    int rc = moments_stage(m, rows, n);
    if (rc) return rc;
    return b2f_moments_device(m, m->mom_rows.p, n, out);
}

extern "C" int b2f_moments_device_timed(b2f_model *m, const void *rows_dev, int64_t n, int iters, int flush_l2, float *ms_each, double *out) {
    if (!m || iters <= 0 || !ms_each) return set_err(B2F_EINVAL, "bad argument");
    CUDA_TRY(cudaSetDevice(m->device));
    int rc = timed_launches(m, iters, flush_l2, ms_each, nullptr, [&](int) { return launch_moments(m, rows_dev, n); });
    if (rc || !out) return rc;
    CUDA_TRY(cudaMemcpyAsync(out, m->d_mom_out, B2F_MOM_VALUES * sizeof(double), cudaMemcpyDeviceToHost, m->compute));
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    return B2F_OK;
}

/* Chan et al. pairwise merge of (count, mean, M2), in part order */
extern "C" void b2f_moments_merge(const double *parts, int k, double *out) {
    for (int w = 0; w < B2F_ROW_WORDS; ++w) {
        double n = 0.0, mean = 0.0, m2 = 0.0;
        for (int i = 0; i < k; ++i) {
            const double nb = parts[(size_t)i * B2F_MOM_VALUES + w * 3 + 0];
            const double mb = parts[(size_t)i * B2F_MOM_VALUES + w * 3 + 1];
            const double sb = parts[(size_t)i * B2F_MOM_VALUES + w * 3 + 2];
            if (nb <= 0.0) continue;
            if (n == 0.0) {
                n = nb, mean = mb, m2 = sb;
                continue;
            }
            const double tot = n + nb, delta = mb - mean;
            mean += delta * (nb / tot);
            m2 += sb + delta * delta * (n * nb / tot);
            n = tot;
        }
        out[w * 3 + 0] = n;
        out[w * 3 + 1] = mean;
        out[w * 3 + 2] = m2;
    }
}

/* ------------------------------------------------------------------ NCCL plumbing */
extern "C" int b2f_comm_unique_id(void *id_out128) {
    if (!id_out128) return set_err(B2F_EINVAL, "null argument");
    int rc = nccl_load();
    if (rc) return rc;
    ncclUniqueId id;
    NCCL_TRY(g_nccl.GetUniqueId(&id));
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    memcpy(id_out128, &id, 128);
    return B2F_OK;
}

static int comm_buffers(b2f_model *m, int nranks) {
    const size_t bytes = (size_t)(nranks + 1) * B2F_MOM_VALUES * sizeof(double);
    return m->gather.reserve(m->compute, bytes, bytes);
}

extern "C" int b2f_comm_init_rank(b2f_model *m, int nranks, int rank, const void *id128) {
    if (!m || !id128 || nranks <= 0 || rank < 0 || rank >= nranks) return set_err(B2F_EINVAL, "bad argument");
    int rc = nccl_load();
    if (rc) return rc;
    CUDA_TRY(cudaSetDevice(m->device));
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    NCCL_TRY(g_nccl.CommInitRank(&m->comm, nranks, id, rank));
    m->nranks = nranks;
    m->rank = rank;
    return comm_buffers(m, nranks);
}

extern "C" int b2f_comm_init_all(b2f_model **models, int n_models) {
    if (!models || n_models <= 0) return set_err(B2F_EINVAL, "no models");
    int rc = nccl_load();
    if (rc) return rc;
    std::vector<ncclComm_t> comms(n_models);
    std::vector<int> devs(n_models);
    for (int i = 0; i < n_models; ++i) devs[i] = models[i]->device;
    NCCL_TRY(g_nccl.CommInitAll(comms.data(), n_models, devs.data()));
    for (int i = 0; i < n_models; ++i) {
        models[i]->comm = comms[i];
        models[i]->nranks = n_models;
        models[i]->rank = i;
        CUDA_TRY(cudaSetDevice(models[i]->device));
        rc = comm_buffers(models[i], n_models);
        if (rc) return rc;
    }
    return B2F_OK;
}

extern "C" int b2f_moments_allgather(b2f_model *m, const double *local, double *merged) {
    if (!m || !local || !merged) return set_err(B2F_EINVAL, "null argument");
    if (!m->comm) return set_err(B2F_ESTATE, "communicator not initialised (call b2f_comm_init_rank)");
    CUDA_TRY(cudaSetDevice(m->device));
    double *gather = static_cast<double *>(m->gather.p), *send = gather + (size_t)m->nranks * B2F_MOM_VALUES;
    CUDA_TRY(cudaMemcpyAsync(send, local, B2F_MOM_VALUES * sizeof(double), cudaMemcpyHostToDevice, m->compute));
    NCCL_TRY(g_nccl.AllGather(send, gather, B2F_MOM_VALUES, ncclDouble, m->comm, m->compute));
    std::vector<double> parts((size_t)m->nranks * B2F_MOM_VALUES);
    CUDA_TRY(cudaMemcpyAsync(parts.data(), gather, parts.size() * sizeof(double), cudaMemcpyDeviceToHost, m->compute));
    CUDA_TRY(cudaStreamSynchronize(m->compute));
    b2f_moments_merge(parts.data(), m->nranks, merged);
    return B2F_OK;
}

extern "C" int b2f_moments_multi(b2f_model **models, int n_models, const void *rows, int64_t n, double *out) {
    if (!models || n_models <= 0 || !out || n < 0) return set_err(B2F_EINVAL, "bad argument");
    /* 1. every device reduces its contiguous slice */
    int rc = B2F_OK;
    for (int i = 0; i < n_models && rc == B2F_OK; ++i) {
        b2f_model *m = models[i];
        const int64_t lo = n * i / n_models, hi = n * (i + 1) / n_models;
        CUDA_TRY(cudaSetDevice(m->device));
        rc = moments_stage(m, static_cast<const uint8_t *>(rows) + (size_t)lo * B2F_ROW_BYTES, hi - lo);
        if (rc == B2F_OK) rc = launch_moments(m, m->mom_rows.p, hi - lo);
    }
    if (rc) return rc;
    const bool use_nccl = models[0]->comm != nullptr && models[0]->nranks == n_models;
    std::vector<double> parts((size_t)n_models * B2F_MOM_VALUES);
    if (use_nccl) {
        /* 2a. all-gather the 576-byte triples over NVLink; every rank ends up with all partials */
        NCCL_TRY(g_nccl.GroupStart());
        for (int i = 0; i < n_models; ++i) {
            b2f_model *m = models[i];
            ncclResult_t r = g_nccl.AllGather(m->d_mom_out, m->gather.p, B2F_MOM_VALUES, ncclDouble, m->comm, m->compute);
            if (r != ncclSuccess) {
                g_nccl.GroupEnd();
                return set_err(B2F_ENCCL, "ncclAllGather failed: %s", g_nccl.GetErrorString(r));
            }
        }
        NCCL_TRY(g_nccl.GroupEnd());
        CUDA_TRY(cudaSetDevice(models[0]->device));
        CUDA_TRY(cudaMemcpyAsync(parts.data(), models[0]->gather.p, parts.size() * sizeof(double), cudaMemcpyDeviceToHost, models[0]->compute));
        for (int i = 0; i < n_models; ++i) {
            CUDA_TRY(cudaSetDevice(models[i]->device));
            CUDA_TRY(cudaStreamSynchronize(models[i]->compute));
        }
    } else {
        /* 2b. no communicator: gather through the host */
        for (int i = 0; i < n_models; ++i) {
            CUDA_TRY(cudaSetDevice(models[i]->device));
            CUDA_TRY(cudaMemcpyAsync(parts.data() + (size_t)i * B2F_MOM_VALUES, models[i]->d_mom_out, B2F_MOM_VALUES * sizeof(double),
                                     cudaMemcpyDeviceToHost, models[i]->compute));
            CUDA_TRY(cudaStreamSynchronize(models[i]->compute));
        }
    }
    b2f_moments_merge(parts.data(), n_models, out);
    return B2F_OK;
}

/* ------------------------------------------------------------------ columnar request pipeline (encode -> H2D -> kernel -> D2H per chunk) */
#include "scorer.h"

/* ------------------------------------------------------------------ batch drift detector (K3) */
#include "drift_api.cuh"

/* ------------------------------------------------------------------ explanations (K5) */
#include "explain_api.cuh"

/* ------------------------------------------------------------------ partial dependence (K6) */
#include "dependence_api.cuh"

/* ------------------------------------------------------------------ two-way partial dependence (K10) */
#include "pair_dependence_api.cuh"

/* ------------------------------------------------------------------ accumulated local effects (K12) */
#include "ale_api.cuh"

/* ------------------------------------------------------------------ counterfactuals (K7) */
#include "counterfactual_api.cuh"

/* ------------------------------------------------------------------ permutation importance (K8) */
#include "importance_api.cuh"

/* ------------------------------------------------------------------ MMD drift test (K9) */
#include "mmd_api.cuh"

/* ------------------------------------------------------------------ online MMD drift detector (K13) */
#include "mmd_online_api.cuh"

/* ------------------------------------------------------------------ k-nearest reference rows of trust scores (K11) */
#include "knn_api.cuh"
