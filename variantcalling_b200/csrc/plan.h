// plan.h -- binary layout of the compiled plan blob (host + device).
//
// The Python host (variantcalling_b200/model_compiler.py) lowers
//   (VCF header, fitted ColumnTransformer, model)  ->  this flat blob,
// and ugvc_load_plan() uploads it.  All integers little-endian, every section
// starts 8-byte aligned.  Sections follow the header in the order below.
#pragma once
#include <stdint.h>

#define UGVC_PLAN_MAGIC 0x50564755u /* "UGVP" */
#define UGVC_PLAN_VERSION 9u

#define UGVC_MAX_TAGS 128
#define UGVC_MAX_SLOTS 250
#define UGVC_MAX_FEATURES 250
#define UGVC_MAX_CLASSES 4
#define UGVC_NAME_MAX 32

// ---- value kinds of a tag in one header section (INFO or FORMAT) -----------
enum : uint8_t {
    KIND_NONE = 0,   // tag not declared in this section
    KIND_INT = 1,
    KIND_FLOAT = 2,
    KIND_STR = 3,
    KIND_FLAG = 4,
    KIND_TYPE_MASK = 7,
    KIND_SCALAR = 8, // Number=1 (pysam hands out a scalar, otherwise a tuple)
};

// ---- slot reducers: how K1 turns (an element of) a tag value into one fp32 word
enum : uint8_t {
    RED_NUM = 0,      // numeric element `elem` (Integer/Float per header), "." -> MISSING
    RED_BASE = 1,     // string element `elem`: A,T,G,C -> 1..4 else 0      (transformers.py:72-77)
    RED_INSDEL = 2,   // string element: ins/del/NA -> -1/1/0 else ERR       (transformers.py:101-105)
    RED_DICT = 3,     // string element looked up in dictionary `dict` else ERR (fitted OrdinalEncoder)
    RED_MOTIF_L = 4,  // whole value, base-10 digits right-to-left          (transformers.py:36-47)
    RED_MOTIF_R = 5,  // whole value, base-10 digits left-to-right          (transformers.py:50-60)
    RED_STRNUM = 6,   // scalar string parsed as a number (pd.to_numeric)    (transformers.py:326-333)
    RED_GT_HOM = 7,   // FORMAT/GT == (1,1) -> 1 else 0                      (transformers.py:94-98)
    RED_LEN = 8,      // number of elements of the value
    RED_REGION = 9,   // whole value: subset of the three region names in dictionary `dict` -> 1..8
                      // (transformers.py:108-123), unknown / repeated name -> ERR
    // fixed columns (tag == TAG_FIXED)
    RED_FIX_QUAL = 16,     // QUAL as float32, "." -> MISSING
    RED_FIX_ALLELE0 = 17,  // allele_encode(REF)
    RED_FIX_ALLELE1 = 18,  // allele_encode(first ALT); MISSING when ALT is "."
    RED_FIX_INDEL = 19,    // len({len(a) for a in alleles}) > 1          (vcftools.py:212)
    RED_FIX_NALLELES = 20, // number of alleles
};
#define TAG_FIXED 0xFFu
#define ELEM_WHOLE 0xFFu

// ---- sentinel bit patterns in raw slots (all are NaNs as fp32) -------------
#define RAW_ABSENT 0xFFFFFFFFu   // key not on the line (pysam: defaultdict -> None)
#define RAW_MISSING 0x7FC00002u  // element is "." / vector too short (pysam: None element)
#define RAW_ERR 0x7FC00003u      // the reference would raise on this value (unknown category, bad literal)

// ---- feature policies (K2) -----------------------------------------------------
enum : uint8_t {
    POL_VALUE = 0,  // substitute the given constant
    POL_ERROR = 1,  // the reference raises / produces a null -> UGVC_E_DATA
    POL_NULL = 2,   // keep a null (NaN) for a PlanCombine to resolve
};

// reasons reported by ugvc_last_data_error
enum : int32_t {
    REASON_NONE = 0,
    REASON_NULL_FEATURE = 1,     // _validate_data would assert (variant_filtering_utils.py:128-143)
    REASON_BAD_VALUE = 2,        // unknown category / KeyError / ragged tuple in the reference
    REASON_TOO_MANY_ELEMS = 3,   // e.g. PL wider than the fitted width (transformers.py:171-172)
    REASON_BAD_NUMBER = 4,       // numeric literal outside the supported exact-parse range
    REASON_MALFORMED_LINE = 5,   // fewer than 8 columns
};

enum : uint32_t {
    MODEL_NONE = 0,
    MODEL_LOGISTIC = 1,    // sklearn LogisticRegression: fp64 dot + expit / softmax
    MODEL_GB_SKLEARN = 2,  // sklearn GradientBoostingClassifier: fp64 init + sum(lr*leaf), expit / softmax
    MODEL_RF_SKLEARN = 3,  // sklearn RandomForestClassifier: fp64 mean of per-leaf class fractions
    MODEL_XGB = 4,         // xgboost gbtree: fp32 margin in tree order, fp32 sigmoid / softmax
};

enum : uint32_t {
    CMP_LE = 0,  // go left when x <= thr (sklearn; thr pre-rounded down to fp32)
    CMP_LT = 1,  // go left when x <  thr (xgboost)
};

// All records are naturally aligned so that device code can fetch them with single 32/64-bit
// loads (shared memory copies and __ldg).
struct alignas(8) PlanHeader {
    uint32_t magic, version;
    uint32_t n_tags, n_slots, n_features, n_dicts, n_dict_strings;
    uint32_t model_kind, n_classes, n_outputs; // n_outputs: margins/prob columns the model produces (1 for binary GB/LR/XGB)
    uint32_t n_trees, n_nodes, n_leaf_rows, leaf_width, cmp_mode;
    uint16_t n_checks, n_combines;
    double init[UGVC_MAX_CLASSES]; // GB init raw / XGB base margin / LR intercepts are in their own section
};

struct alignas(8) PlanTag {   // 40 bytes
    char name[32];            // zero padded; compared as four 64-bit words
    uint8_t len;
    uint8_t info_kind;        // KIND_* | KIND_SCALAR, as declared by ##INFO
    uint8_t fmt_kind;         // as declared by ##FORMAT
    uint8_t first_slot;
    uint8_t n_slots;
    uint8_t whole_red;        // RED_* of the tag's whole-value slot, 0xFF if none
    uint8_t whole_slot;       // slot index of that reducer
    uint8_t pad;
};

struct alignas(4) PlanSlot {  // 4 bytes
    uint8_t tag;              // index into tags, or TAG_FIXED
    uint8_t elem;             // element index, or ELEM_WHOLE
    uint8_t reducer;          // RED_*
    uint8_t dict;             // dictionary index for RED_DICT
};

struct alignas(4) PlanDict {  // 4 bytes
    uint16_t first_string;
    uint16_t n_strings;
};

struct alignas(8) PlanString {  // 32 bytes
    char s[24];               // zero padded; compared as three 64-bit words
    uint8_t len;
    uint8_t pad[7];
};

struct alignas(4) PlanFeature {  // 12 bytes
    uint16_t slot;
    uint8_t absent_pol;       // POL_*
    uint8_t missing_pol;
    float absent_val;
    float missing_val;
};

struct alignas(4) PlanCheck {  // 8 bytes: the reference raises unless the slot value satisfies the bound
    uint16_t slot;
    uint8_t kind;             // 0: value <= bound, 1: value >= bound
    uint8_t pad;
    float bound;
};

struct alignas(4) PlanCombine {  // 8 bytes: feature = max(feature, slot_b) skipping nulls (DataFrame.max(axis=1))
    uint16_t feature;
    uint16_t slot_b;
    uint8_t op;               // 0: max, nulls skipped; still null -> the reference's _validate_data asserts
    uint8_t pad[3];
};

struct alignas(8) PlanNode {  // 8 bytes, preorder layout: left child = this + 1
    float value;              // internal: threshold (fp32); categorical: bit pattern of UGVC_CAT_REF(first word, words);
                              // leaf: bit pattern of the int32 leaf row
    int16_t feature;          // < 0 for a leaf
    uint16_t right;           // index of the right child relative to the tree root
};

// ---- per-node flags of a forest (xgboost only; zero for sklearn models and on leaves) -------------
// xgboost 2.1.2's CPU predictor (GetNextNode / common::Decision), restated, PARITY UNPINNED (xgboost is not
// installed where this is built):
//   NaN goes to the default child (left when NODE_DEFAULT_LEFT is set, else right), at every node kind;
//   numeric node: left when fp32 x < threshold;
//   categorical node: left when x < 0 or x >= 2^24 (invalid category), or when int(x) (truncated) is not in the
//   node's category set; right when it is.  The set is a bitset: bit c of word c / 32 of the node's words.
enum : uint8_t {
    NODE_DEFAULT_LEFT = 1,
    NODE_CATEGORICAL = 2,
};
// Categories are codes in [0, UGVC_MAX_CATEGORIES): a node's bitset has at most UGVC_MAX_CATEGORIES / 32 words.
#define UGVC_MAX_CATEGORIES 1024u
#define UGVC_CAT_MAX_WORDS (UGVC_MAX_CATEGORIES / 32u)
#define UGVC_CAT_REF(first, words) ((uint32_t)(first) | ((uint32_t)(words) << 24))  // first word < 2^24
#define UGVC_CAT_FIRST(ref) ((ref) & 0xFFFFFFu)
#define UGVC_CAT_WORDS(ref) ((ref) >> 24)

struct alignas(8) PlanCatHeader {  // 8 bytes: opens the category section of a forest
    uint32_t n_words;              // uint32 bitset words that follow
    uint32_t n_flagged;            // nodes with a non-zero flag byte (0: the plain walk runs)
};
static_assert(sizeof(PlanHeader) == 96 && sizeof(PlanTag) == 40 && sizeof(PlanSlot) == 4 && sizeof(PlanDict) == 4 &&
                  sizeof(PlanString) == 32 && sizeof(PlanFeature) == 12 && sizeof(PlanCheck) == 8 &&
                  sizeof(PlanCombine) == 8 && sizeof(PlanNode) == 8 && sizeof(PlanCatHeader) == 8,
              "plan record layout");

// Hash of a tag name held as four little-endian 64-bit words (+ length); the host builds the
// 256-entry open-addressing table with the same function the device probes it with.
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline unsigned ugvc_key_hash(unsigned long long k0, unsigned long long k1, unsigned long long k2,
                                     unsigned long long k3, int len) {
    unsigned long long h = k0 ^ (k1 * 0x9E3779B97F4A7C15ull) ^ (k2 * 0xC2B2AE3D27D4EB4Full) ^
                           (k3 * 0x165667B19E3779F9ull) ^ (unsigned long long)len;
    h *= 0xFF51AFD7ED558CCDull;
    h ^= h >> 33;
    return (unsigned)(h & 255u);
}

// Section order after PlanHeader (each padded to 8 bytes):
//   PlanTag[n_tags], PlanSlot[n_slots], PlanDict[n_dicts], PlanString[n_dict_strings],
//   PlanFeature[n_features], PlanCheck[n_checks], PlanCombine[n_combines],
//   MODEL_LOGISTIC : double coef[n_outputs * n_features], double intercept[n_outputs]
//   forests        : uint32 tree_root[n_trees + 1], uint8 tree_out[n_trees] (output column of each tree),
//                    PlanNode[n_nodes], double leaves[n_leaf_rows * leaf_width],
//                    uint8 node_flags[n_nodes] (NODE_*), PlanCatHeader, uint32 cat_words[n_words]
//                    (a categorical node's PlanNode.value holds UGVC_CAT_REF of its words in cat_words)
