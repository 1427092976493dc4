/*
 * forest_blob.h -- on-disk / in-HBM layout of a flattened forest ("forest blob", version 2).
 *
 * Written by databricks_kubernetes_mlops_poc_b200/flatten.py from a fitted sklearn Pipeline
 * (the model artefact the reference serves: artifacts/classifier/model/model.pkl, reference
 * databricks/src/02-register-model.ipynb:317-321), read by b2f_model_create().
 *
 * Trees are packed in GROUPS of 32: lane l of a warp walks tree 32*g + l.  Inside a group every
 * per-node array is interleaved by tree, element (slot s, tree l) at index s*32 + l, so that the
 * 32 lanes of a warp -- each at a different node of a different tree -- always touch 32 different
 * shared-memory banks (and, from global memory, 32 consecutive words when the slots coincide).
 *
 * One group chunk, contiguous and 256-byte granular (so a chunk is one TMA bulk copy):
 *     N  : {uint32 T, uint32 M}[n_slots][32]   one 8-byte node per (slot, tree): a single 64-bit
 *                                              shared-memory load per visit, bank-conflict free
 *     LV : float64[n_leaf_slots][32]           leaf payload: RF class-1 fraction, GBDT
 *                                              learning_rate*value, or isolation-forest path length
 *                                              depth(leaf) + c(n_node_samples)
 *   T  threshold word: float32 t' = nextup(floor32(threshold)) for a numeric split, int32 category
 *      code for a one-hot split, leaf_id (row of the leaf's payload in LV) for a leaf
 *   M  meta word: bits 27..31 row word index, bit 26 = categorical test, bits 0..23 = slot of the
 *      FIRST child (second child = first + 1).  The next node's address is one multiply-add:
 *      (M << 8) + lane_base shifts the top byte out and scales the slot by the 256-byte stride.
 *
 * Split semantics (x = row word M.feat of the encoded row, after in-kernel imputation):
 *     numeric      : second child iff x >= t' or unordered     (sklearn: x <= thr -> left, and for
 *                    float32 x:  x <= thr  <=>  x <= floor32(thr)  <=>  x < nextup(floor32(thr)))
 *     categorical  : second child iff int(x) == int(T)         (one-hot column == 1 -> right)
 *   evaluated branch-free as  second = (x ==bits T) or (geu(x, T) and not cat): for a numeric node
 *   bit equality implies x >= t', so the extra term never changes the answer.
 * A leaf slot is a categorical test of row word 23 (the kernel's copy of the row holds 0xFFFFFFFF
 * there) against leaf_id, which never matches, with itself as first child: walking is a fixed
 * `depth`-iteration loop with no leaf branch; leaves simply self-loop.
 */
#ifndef B2F_FOREST_BLOB_H
#define B2F_FOREST_BLOB_H
#include <stdint.h>

#define B2F_BLOB_MAGIC "B2FOREST"
#define B2F_BLOB_VERSION 2u
#define B2F_BLOB_HEADER_BYTES 512u
#define B2F_GROUP_TREES 32u
#define B2F_MAX_GROUPS 32u
#define B2F_SENTINEL_WORD 23u
#define B2F_SENTINEL_BITS 0xFFFFFFFFu
#define B2F_META_SLOT_MASK 0x00FFFFFFu
#define B2F_META_FEAT_SHIFT 27u
#define B2F_NODE_STRIDE 256u /* bytes between consecutive slots of one tree (32 lanes x 8 B) */
#define B2F_META_CAT 0x04000000u
#define B2F_BLOB_HAS_PATH_BOUND 1u

typedef struct b2f_blob_header {
    char magic[8];
    uint32_t version;
    uint32_t header_bytes;
    uint32_t agg_mode;
    uint32_t n_trees;
    uint32_t n_groups;
    uint32_t row_words;
    uint32_t n_cat;
    uint32_t n_num;
    uint32_t max_depth;
    uint32_t flags;  /* B2F_BLOB_HAS_PATH_BOUND */
    double init_raw; /* GBDT: raw prediction of the init estimator; RF: 0; isolation forest: offset_ */
    double denom;    /* RF: n_trees (proba = sum / denom); GBDT: 1; isolation forest: n_trees * c(max_samples) */
    uint64_t groups_off;
    uint64_t chunks_off;
    uint64_t chunks_bytes;
    uint64_t total_bytes;
    float impute[24];  /* per row word: replacement for NaN (numeric words), float32(median) */
    int32_t vocab[24]; /* per row word: vocabulary size (categorical words), else 0 */
    double threshold;  /* isolation forest: is_outlier = score > threshold; other modes: 0 */
    double path_bound; /* isolation forest with B2F_BLOB_HAS_PATH_BOUND: the largest path-length sum whose score numpy puts
                          above `threshold` (flatten.py iforest_path_bound); the kernels flag s <= path_bound */
    uint8_t pad[B2F_BLOB_HEADER_BYTES - 96 - 192 - 16];
} b2f_blob_header;

typedef struct b2f_blob_group {
    uint32_t chunk_off;    /* bytes from chunks_off; multiple of 256 */
    uint32_t chunk_bytes;  /* (n_slots + n_leaf_slots) * 256 */
    uint32_t n_slots;      /* node slots per tree in this group (padded to the group's maximum; < 2^24) */
    uint32_t n_leaf_slots; /* leaf slots per tree (padded) */
    uint32_t depth;        /* walk iterations = deepest leaf in the group */
    uint32_t n_trees;      /* real trees in this group (<= 32; the rest are zero-valued stubs) */
    uint32_t reserved[2];
} b2f_blob_group;

#ifdef __cplusplus
static_assert(sizeof(b2f_blob_header) == B2F_BLOB_HEADER_BYTES, "header size");
static_assert(sizeof(b2f_blob_group) == 32, "group size");
#endif
#endif
