/*
 * forest_paths.h -- layout of a TreeSHAP path table ("explainer", version 1).
 *
 * Written by databricks_kubernetes_mlops_poc_b200/flatten.py (flatten_explainer) from the same fitted Pipeline as the
 * forest blob (forest_blob.h), attached to a model by b2f_model_attach_explainer() and walked by k_tree_shap
 * (tree_shap.cuh).  It holds one path per leaf of every classifier tree; a tree that is a single leaf has no path and
 * moves only base_value.
 *
 *   header  : b2f_paths_header, 256 bytes
 *   paths   : b2f_path[n_paths] at paths_off (= 256)
 *   elements: b2f_path_elem[n_elems] at elems_off (16-byte aligned); path p owns elements [first, first + len)
 *
 * A path's elements are its nodes MERGED BY REQUEST FIELD (GPUTreeShap, Mitchell et al., PeerJ CS 2022).  Element 0 is a
 * bias element (field 0xFF, zero_fraction 1); each other element is one field the path tests, at most once per path:
 *   zero_fraction      product over the path's nodes on that field of cover(child) / cover(parent), with cover =
 *                      tree_.weighted_n_node_samples; inv_zero_fraction = 1 / zero_fraction, so the kernel divides by nothing
 *   condition          what the imputed row word x of that field must satisfy to follow the path at all those nodes:
 *     numeric     : geu(x, lo) and (no HAS_HI flag or x < hi), with lo / hi the float32 t' = nextup(floor32(threshold)) of
 *                   the blob: the prediction kernels' compare (second child iff x >= t' or unordered), so NaN after
 *                   imputation follows right turns only, exactly as it is scored
 *     categorical : bit (code + 1) of mask[4] (bit 0 = unknown / missing, code -1); a code outside [-1, 126] reads bit 0,
 *                   since no node tests it.  Fields of more than 127 categories are refused by the flattener.
 * A field with several one-hot columns is one player: merging its nodes is what makes it so.
 *
 * The leaf payload is the blob's (RF class-1 fraction, GBDT learning_rate * value); phi is the sum over paths divided by
 * denom (RF: n_trees, GBDT: 1), so base_value + sum_f phi[f] is the predicted probability (RF) or raw margin (GBDT).
 * base_value (v of the empty set) is computed on the host in float64.  fingerprint ties the table to one forest blob:
 * sum over the blob's little-endian 64-bit words w_i of splitmix64(w_i ^ i * 0x9E3779B97F4A7C15), mod 2^64.
 */
#ifndef B2F_FOREST_PATHS_H
#define B2F_FOREST_PATHS_H
#include <stdint.h>

#define B2F_PATHS_MAGIC "B2FPATHS"
#define B2F_PATHS_VERSION 1u
#define B2F_PATHS_HEADER_BYTES 256u
#define B2F_PATHS_MAX_LEN 24u /* bias + at most 23 fields (depth 1..24 forests) */
#define B2F_PATH_BIAS_FIELD 0xFFu
#define B2F_PE_BIAS 0u
#define B2F_PE_NUM 1u
#define B2F_PE_CAT 2u
#define B2F_PE_HAS_HI 4u

typedef struct b2f_paths_header {
    char magic[8];
    uint32_t version;
    uint32_t header_bytes;
    uint32_t n_cat;
    uint32_t n_num;
    uint32_t agg_mode; /* B2F_AGG_RF_MEAN or B2F_AGG_GBDT_LOGISTIC */
    uint32_t n_trees;
    uint32_t n_paths;
    uint32_t max_len; /* longest path, elements including the bias */
    uint32_t n_elems;
    uint32_t reserved0;
    double base_value;    /* v(empty set) in the output space: mean expected leaf (RF) or init + sum (GBDT) */
    double denom;         /* RF: n_trees, GBDT: 1 */
    uint64_t fingerprint; /* of the classifier's forest blob */
    uint64_t paths_off;
    uint64_t elems_off;
    uint64_t total_bytes;
    uint8_t pad[B2F_PATHS_HEADER_BYTES - 96];
} b2f_paths_header;

typedef struct b2f_path {
    uint32_t first; /* index of the bias element */
    uint32_t len;   /* elements including the bias, 2 .. max_len */
    uint32_t tree;
    uint32_t reserved;
    double leaf; /* leaf payload, as in the blob */
} b2f_path;

typedef struct b2f_path_elem {
    uint32_t field; /* request field (row word), 0xFF for the bias */
    uint32_t kind;  /* B2F_PE_NUM [| B2F_PE_HAS_HI] | B2F_PE_CAT | B2F_PE_BIAS */
    float lo, hi;   /* numeric condition */
    uint32_t mask[4]; /* categorical condition over code + 1 */
    double zero_fraction;
    double inv_zero_fraction;
} b2f_path_elem;

#ifdef __cplusplus
static_assert(sizeof(b2f_paths_header) == B2F_PATHS_HEADER_BYTES, "paths header size");
static_assert(sizeof(b2f_path) == 24, "path record size");
static_assert(sizeof(b2f_path_elem) == 48, "path element size");
#endif
#endif
