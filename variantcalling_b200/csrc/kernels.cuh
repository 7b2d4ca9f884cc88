// kernels.cuh -- device-side plan view and kernel launch prototypes.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/ugvc_b200.h"
#include "plan.h"

// Device view of a loaded plan (passed to kernels by value).
struct DevPlan {
    PlanHeader h;
    const PlanTag* tags;
    const PlanSlot* slots;
    const PlanDict* dicts;
    const PlanString* strings;
    const PlanFeature* feats;
    const PlanCheck* checks;
    const PlanCombine* combines;
    const double* coef;
    const double* intercept;
    const uint32_t* tree_root;
    const uint8_t* tree_out;
    const PlanNode* nodes;     // blob form (host validation)
    const uint2* dev_nodes;    // device form: x = threshold bits (leaf: quiet NaN | leaf row; categorical node: UGVC_CAT_REF),
                               // y = feature | right_abs << 8 (K3_WALK_CAT: feature | NODE_* flags << 8 | right_abs << 10);
                               // the n_cat_words category bitset words follow the n_nodes nodes
    uint32_t max_depth;        // deepest leaf over all trees
    uint32_t walk;             // K3_WALK_*: which tree walk K3 runs (in what was padding: the layout is unchanged)
    const double* leaves;
    // heap form of the forest (k3_heap): every tree padded to a complete binary tree of depth heap_depth,
    // node i at index i (root 1, children 2i / 2i+1), H = 2^heap_depth entries per tree and array
    const float* heap_thr;     // [n_trees][H] thresholds (+inf below a shallow leaf: every path ends on its row)
    const uint8_t* heap_feat;  // [n_trees][H] feature of the node
    const uint16_t* heap_leaf; // [n_trees][H] leaf row reached from node 2^depth + k
    uint32_t heap_depth;       // 0: the forest has no heap form (too deep / too many leaf rows): k2 + k3_infer
    uint32_t n_cat_words;      // category bitset words (after dev_nodes); K3 stages them all in shared memory
    const uint8_t* htab;       // 256-entry open-addressing table: tag index or 0xFF
    uint32_t first_fixed_slot; // slots [first_fixed_slot, n_slots) are TAG_FIXED
};
// K3's tree walks.  PLAIN: a row goes left when x < / <= threshold (NaN goes right).  CAT (xgboost plans with
// default-left or categorical nodes, plan.h NODE_*): NaN to the default child, categorical sets from the bitsets.
enum : uint32_t { K3_WALK_PLAIN = 0, K3_WALK_CAT = 1 };

// Learned key order ("schedule"): the INFO keys in the order records carry them and the usual
// FORMAT column.  K1 steps through it warp-uniformly, matching "KEY=" word-wise against the
// cursor's look-ahead; keys off the schedule take the generic hash-lookup path.
#define UGVC_MAX_SCHED 128
#define UGVC_MAX_FMT_KEYS 8
enum : uint8_t {
    CLS_SKIP = 0,     // value not needed
    CLS_GENERIC = 1,  // any tag: parse_value()
    CLS_INT = 2,      // n_elem Integer elements (+ element count when SCHED_COUNT_ALL)
    CLS_FLOAT = 3,    // n_elem Float elements
    CLS_DICT1 = 4,    // scalar String looked up in one dictionary
};
#define SCHED_IS_FLAG 1u
#define SCHED_COUNT_ALL 2u
#define SCHED_DICT_INLINE 4u  // UGVC_K1_INLINE_DICT1 builds: one category (<= 7 bytes) of a CLS_DICT1 key held in w1, its length in n_elem
#define SCHED_DICT_INLINE_SECOND 8u  // ... and it is category 1 of 2 (else category 0)
struct alignas(8) SchedEntry {   // 32 bytes
    unsigned long long w0, m0;   // first 8 bytes to match ("KEY=", or "KEY" for a valueless key) and their mask
    unsigned long long w1;       // bytes 8..15, zero padded (len > 8)
    uint8_t len;                 // bytes to match (<= 16; longer keys are not scheduled)
    uint8_t cls;                 // CLS_*
    uint8_t slot0;               // first slot of the tag
    uint8_t n_elem;              // element slots
    uint8_t dict;                // CLS_DICT1
    uint8_t flags;               // SCHED_*
    int16_t tag;                 // plan tag index, or -1
};
struct DevSchedule {
    const SchedEntry* info;      // device array
    int n_info;
    int n_fmt;                   // sub-fields of the expected FORMAT column (0: none learned)
    int fmt_len;                 // its length in bytes
    unsigned long long fmt_w[3]; // its bytes, zero padded
    SchedEntry fmt[UGVC_MAX_FMT_KEYS];  // per sub-field: cls / slot0 / n_elem / dict / flags / tag
};


// ---- K1 fast tier (k1_tok.inc) ------------------------------------------------------------
// The tile kernel identifies INFO keys through a hash table of every key it may meet: the plan's
// tags declared in ##INFO plus the keys ugvc_set_key_order() saw in the data (keys the plan does
// not need decode to nothing).  A record that carries anything else -- an unknown key, a literal
// outside the short decoders, a FORMAT column other than the usual one -- is handed to the
// generic per-record parser (k1_parse over the slow list), which defines the semantics.
#define KF_MAX_KEYS 128
enum : uint8_t {
    FK_SCALAR = 1,     // Number=1 in this header section
    FK_IS_FLAG = 2,    // the data carries the key without a value
    FK_SKIP_FMT = 4,   // the usual FORMAT column has the tag: the sample value overrides the INFO value
    FK_NEEDED = 8,     // the plan has slots for this tag in this section
};
struct alignas(8) FastMeta {   // 8 bytes: how a value of this tag becomes slot words
    uint8_t type;              // KIND_INT / KIND_FLOAT / KIND_STR / KIND_FLAG of this section
    uint8_t flags;             // FK_*
    uint8_t n_elem;            // element slots
    uint8_t slot0;             // first slot of the tag
    uint8_t whole_red;         // RED_* of the whole-value slot, 0xFF if none
    uint8_t whole_slot;
    uint8_t tag;               // plan tag (duplicate-key bitmap), 0xFF if the plan has no such tag
    uint8_t col;               // k1_tok: < KF_COLS column of the window's value table (the tag's values are decoded side by
                               // side for consecutive records), KF_COL_DICT the dictionary queue, KF_COL_NONE decoded where met
};
#define KF_COLS 64
#define KF_COL_DICT 0xFEu
#define KF_COL_NONE 0xFFu
struct alignas(16) FastKey {   // 32 bytes
    uint32_t name[4];          // key bytes, zero padded (keys of up to 15 bytes are matched here)
    FastMeta m;
    uint8_t len;
    uint8_t pad[7];
};
// per-slot byte of the tile kernel: the queue class a value of this slot goes to (bits 0-1: 0 numeric token,
// 1 not on the fast path, 2 dictionary string, 3 small string reducer) and what the decoders need to know
enum : uint8_t { SK_CLS_MASK = 3, SK_CLS_NUM = 0, SK_CLS_BAD = 1, SK_CLS_DICT = 2, SK_CLS_GEN = 3,
                 SK_INT = 4, SK_STRNUM = 8, SK_SCALAR = 16, SK_ZERO_LONG = 32 };
enum { FIX_QUAL = 0, FIX_ALLELE0 = 1, FIX_ALLELE1 = 2, FIX_INDEL = 3, FIX_NALLELES = 4 };
struct DevFast {
    const FastKey* keys;       // device array
    const uint8_t* htab;       // 256-entry open-addressing table: key index or 0xFF
    const uint8_t* slot_kind;  // [n_slots] SK_* bits
    int n_keys;
    int enabled;
    int n_cols;                // columns of the value table in use (FastMeta.col)
    int n_fmt, fmt_len;        // the usual FORMAT column (0: records are expected to end after INFO)
    uint32_t fmt_w[6];
    FastMeta fmt[UGVC_MAX_FMT_KEYS];
    uint8_t fix_slot[8];       // slots of the fixed-column reducers (FIX_*), 0xFF if the plan has none
};
#if defined(__CUDACC__) || defined(UGVC_HOST_EMU)
__host__ __device__
#endif
static inline uint32_t kf_hash(uint32_t k0, uint32_t k1, uint32_t k2, uint32_t k3, uint32_t len) {
    uint32_t h = (k0 * 0x9E3779B1u) ^ (k1 * 0x85EBCA77u) ^ (k2 * 0xC2B2AE3Du) ^ (k3 * 0x27D4EB2Fu) ^ (len * 0x165667B1u);
    h ^= h >> 15;
    h *= 0x2C1B3C6Du;
    return h >> 24;
}

// Error word: smaller is earlier.  (record << 24) | (column << 8) | reason
#define UGVC_NO_ERROR 0xFFFFFFFFFFFFFFFFull
__host__ __device__ inline unsigned long long ugvc_pack_error(long long rec, int col, int reason) {
    return ((unsigned long long)rec << 24) | ((unsigned long long)(col & 0xFFFF) << 8) | (unsigned)(reason & 0xFF);
}

struct LaneBuffers {
    // sizes
    size_t cap_bytes, cap_records;
    // K0 / K1 fast tier scratch: tile ticket, slow-record counter, look-back state words
    uint32_t* chunk_first;
    uint32_t* slow_list;       // [cap_records] records handed to the generic parser
    int64_t* line_start;       // [cap_records + 1]
    int64_t* n_records;        // device scalar
    // K1
    uint32_t* raw;             // [n_slots][cap_records]
    ugvc_recinfo* recinfo;     // [cap_records]
    // K2
    float* feats;              // [n_features][cap_records]
    // K3
    uint8_t* low_score;        // [cap_records]
    float* probs;              // [cap_records][n_classes]
    double* qual;              // [cap_records]
    double* phreds;            // [cap_records][n_classes], only with ugvc_enable_phreds
};

#define K0_TILE_BYTES_HOST 65536  // one 64-bit look-back state word per 64 KiB tile
#ifndef K1_TILE_BYTES_HOST
#define K1_TILE_BYTES_HOST 32768u
#endif
// ... per tile of the K1 tile kernel (32 KiB; more tiles than K0: sizes the scratch)

void launch_k0(const uint8_t* d_text, size_t n_bytes, uint32_t* chunk_first, int64_t* line_start,
               size_t cap_records, int64_t* d_n_records, unsigned long long* d_err, int sm_count,
               cudaStream_t st);
void launch_k1(const DevPlan& plan, const DevSchedule& sched, const uint8_t* d_text, const int64_t* line_start, const int64_t* d_n_records,
               uint32_t* raw, size_t row_stride, ugvc_recinfo* recinfo, unsigned long long* d_err,
               long long* d_counts, int sm_count, cudaStream_t st);
void launch_k2(const DevPlan& plan, const uint32_t* raw, size_t row_stride, const int64_t* d_n_records, float* feats,
               unsigned long long* d_err, int sm_count, cudaStream_t st);
void launch_k1_fast(const DevPlan& plan, const DevFast& fast, const DevSchedule& sched, const uint8_t* d_text, size_t n_bytes,
                    uint32_t* scratch, int64_t* line_start, size_t cap_records, int64_t* d_n_records, uint32_t* raw,
                    size_t row_stride, ugvc_recinfo* recinfo, uint32_t* slow_list, unsigned long long* d_err,
                    long long* d_counts, int sm_count, cudaStream_t st);
// The K3 launch of a plan; ugvc_test_k3_config reports it
enum { K3_KERNEL_HEAP = 0, K3_KERNEL_INFER = 1 };
struct K3Config {
    int kernel;             // K3_KERNEL_HEAP / K3_KERNEL_INFER
    int shape;              // the kernel's instantiation: index into kernels.cu's K3H_SHAPES / K3I_TPB
    int tpb, nbuf, groups;  // threads per CTA, tile buffers per group, independent groups per CTA (records per tile: tpb / groups)
    int nch;                // trees one thread walks at once
    unsigned chunk;         // k3_heap: trees per staged forest chunk; k3_infer: nodes the forest buffer holds (0: linear model)
    bool resident;          // the whole model is staged once (no chunk loop)
    size_t smem;            // dynamic shared memory per CTA
    int grid;               // CTAs of the persistent grid
    int walk;               // K3_WALK_* of the instantiation that runs
};
// The K3 launch of a plan with a model: k3_heap, which assembles the features from K1's raw slots in its tile load,
// when the model has a heap form, else K2 + k3_infer.  tree_root: the host copy of plan.tree_root.  False, with the
// reason in *why, when neither kernel holds the plan.
bool k3_choose(const DevPlan& plan, const uint32_t* tree_root, int sm_count, K3Config* out, std::string* why);
// K3 as c says.  k3_heap reads the raw slots, or the dense feature matrix feats when raw is NULL; k3_infer reads feats.
void launch_k3(const DevPlan& plan, const K3Config& c, const uint32_t* raw, const float* feats, size_t row_stride,
               const int64_t* d_n_records, double threshold, uint8_t* low_score, float* probs, double* qual,
               double* phreds, int phred_mode, long long* d_counts, unsigned long long* d_err, cudaStream_t st);
size_t k1_smem_bytes(const DevPlan& plan);
cudaError_t kernels_configure(const DevPlan& plan);
