// capi.cu -- C ABI (include/ugvc_b200.h) over the kernels: context, plan upload,
// batch lanes (stream + device workspace), host-buffer and device-resident entry points.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "kernels.cuh"
#include "inflate.cuh"
#include "deflate.cuh"
#ifndef UGVC_HOST_EMU
#include "fileio.cuh"
#endif

#define UGVC_VERSION 100
#define TEXT_SLACK 64

struct Lane {
    cudaStream_t stream = nullptr;
    uint8_t* d_text = nullptr;
    LaneBuffers b{};
    unsigned long long* d_err = nullptr;
    int64_t* h_n = nullptr;              // pinned
    unsigned long long* h_err = nullptr; // pinned
    std::vector<cudaEvent_t> ev_pool;  // 5 events per timed enqueue
    size_t ev_used = 0;
    size_t n_bytes = 0;
    bool submitted = false;
    int64_t last_n = 0;
    // BGZF input (ugvc_submit_bgzf): compressed bytes + per-block tables on the device, grown on demand
    uint8_t* d_comp = nullptr;
    size_t cap_comp = 0;
    uint64_t* d_blk = nullptr;  // [4][cap_blk]: payload offset, payload bytes, output offset, output bytes
    size_t cap_blk = 0;
    int* d_inf_err = nullptr;
    int* h_inf_err = nullptr;   // pinned
    std::vector<uint64_t> h_blk;
    // device-side record writer + BGZF encoder (ugvc_filter_bgzf), allocated at the first call
    struct FileBufs {
        uint8_t* d_out_text = nullptr;
        size_t cap_out = 0;
        int64_t* d_len = nullptr;     // [cap_records + 1]
        int64_t* d_out_ls = nullptr;  // [cap_records + 1]
        uint8_t* d_score = nullptr;   // [cap_records][16]
        void* d_scan_tmp = nullptr;
        size_t scan_tmp_bytes = 0;
        uint8_t* d_blocks = nullptr;  // [cap_blocks][DEF_BLOCK_STRIDE]
        uint32_t* d_bsize = nullptr;
        uint64_t *d_bwide = nullptr, *d_boff = nullptr;
        size_t cap_blocks = 0;
        uint8_t* d_packed = nullptr;
        int* d_fallback = nullptr;
        int* h_fallback = nullptr;      // pinned
        int64_t* h_total = nullptr;     // pinned
        std::vector<uint32_t> h_bsize;
        cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
        float ms[5] = {0, 0, 0, 0, 0};
    } fb;
};

struct ugvc_ctx {
    int device = 0;
    int sm_count = 132;  // replaced by the device's count when the context opens
    std::string err;
    bool has_plan = false;
    DevPlan plan{};
    K3Config k3{};                 // the K3 launch of the plan's model (k3_choose at load)
    uint8_t* d_plan = nullptr;
    uint8_t* d_htab = nullptr;
    uint2* d_nodes = nullptr;
    float* d_heap_thr = nullptr;     // heap form of the forest (k3_heap)
    uint8_t* d_heap_feat = nullptr;
    uint16_t* d_heap_leaf = nullptr;
    std::vector<PlanTag> h_tags;   // host copies for name lookups / decode classes
    std::vector<PlanSlot> h_slots;
#ifdef UGVC_K1_INLINE_DICT1
    std::vector<PlanDict> h_dicts;
    std::vector<PlanString> h_strings;
#endif
    DevSchedule sched{};           // learned key order (empty: generic path only)
    SchedEntry* d_sched = nullptr;
    DevFast fast{};                // key table / FORMAT column / slot kinds of the tile kernel (k1_tok)
    FastKey* d_fast_keys = nullptr;
    uint8_t* d_fast_htab = nullptr;
    uint8_t* d_slot_kind = nullptr;
    DefTables* d_def_tables = nullptr;  // BGZF encoder tables (ugvc_filter_bgzf)
    std::string learned_info, learned_fmt;  // what ugvc_set_key_order was told
    std::vector<Lane> lanes;
    size_t cap_bytes = 0, cap_records = 0;
    long long* d_counts = nullptr;
    int64_t launches = 0;
    bool timing = false;
    int want_phreds = 0;  // 0: off, 1: per-class phreds, 2: per-class fp64 likelihoods
    float stage_ms[4] = {0, 0, 0, 0};
    int64_t err_record = -1;
    int32_t err_column = -1, err_reason = 0;
};

static std::string g_init_error;

static int fail(ugvc_ctx* ctx, int code, const std::string& msg) {
    if (ctx) ctx->err = msg;
    else g_init_error = msg;
    return code;
}
#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return fail(ctx, UGVC_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e));     \
    } while (0)

extern "C" int ugvc_version(void) { return UGVC_VERSION; }

extern "C" const char* ugvc_last_error(const ugvc_ctx* ctx) { return ctx ? ctx->err.c_str() : g_init_error.c_str(); }

extern "C" int ugvc_init(int device, ugvc_ctx** out) {
    ugvc_ctx* ctx = nullptr;
    if (!out) return fail(nullptr, UGVC_E_ARG, "out is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(nullptr, UGVC_E_CUDA,
                    std::string("no CUDA device available (") + cudaGetErrorString(e) +
                        "); this library has no CPU fallback");
    if (device < 0 || device >= n) return fail(nullptr, UGVC_E_ARG, "device index out of range");
    e = cudaSetDevice(device);
    if (e != cudaSuccess) return fail(nullptr, UGVC_E_CUDA, cudaGetErrorString(e));
    ctx = new ugvc_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    CU(cudaMalloc(&ctx->d_counts, 4 * sizeof(long long)));
    CU(cudaMemset(ctx->d_counts, 0, 4 * sizeof(long long)));
    *out = ctx;
    return UGVC_OK;
}

static void free_lane(Lane& l) {
    if (l.stream) cudaStreamSynchronize(l.stream);
    cudaFree(l.d_text);
    cudaFree(l.b.chunk_first);
    cudaFree(l.b.slow_list);
    cudaFree(l.b.line_start);
    cudaFree(l.b.n_records);
    cudaFree(l.b.raw);
    cudaFree(l.b.recinfo);
    cudaFree(l.b.feats);
    cudaFree(l.b.low_score);
    cudaFree(l.b.probs);
    cudaFree(l.b.qual);
    cudaFree(l.b.phreds);
    cudaFree(l.d_err);
    cudaFree(l.d_comp);
    cudaFree(l.d_blk);
    cudaFree(l.d_inf_err);
    cudaFree(l.fb.d_out_text);
    cudaFree(l.fb.d_len);
    cudaFree(l.fb.d_out_ls);
    cudaFree(l.fb.d_score);
    cudaFree(l.fb.d_scan_tmp);
    cudaFree(l.fb.d_blocks);
    cudaFree(l.fb.d_bsize);
    cudaFree(l.fb.d_bwide);
    cudaFree(l.fb.d_boff);
    cudaFree(l.fb.d_packed);
    cudaFree(l.fb.d_fallback);
    if (l.fb.h_fallback) cudaFreeHost(l.fb.h_fallback);
    if (l.fb.h_total) cudaFreeHost(l.fb.h_total);
    for (auto& e : l.fb.ev)
        if (e) cudaEventDestroy(e);
    if (l.h_inf_err) cudaFreeHost(l.h_inf_err);
    if (l.h_n) cudaFreeHost(l.h_n);
    if (l.h_err) cudaFreeHost(l.h_err);
    for (auto& ev : l.ev_pool)
        if (ev) cudaEventDestroy(ev);
    if (l.stream) cudaStreamDestroy(l.stream);
    l = Lane();
}

extern "C" void ugvc_free(ugvc_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    for (auto& l : ctx->lanes) free_lane(l);
    // from here on the previous plan is gone: no plan is loaded until every step below has succeeded, and the
    // lanes sized for the old slot / feature counts go with it
    ctx->has_plan = false;
    for (auto& l : ctx->lanes) free_lane(l);
    ctx->lanes.clear();
    ctx->cap_bytes = ctx->cap_records = 0;
    cudaFree(ctx->d_plan);
    cudaFree(ctx->d_htab);
    cudaFree(ctx->d_nodes);
    cudaFree(ctx->d_heap_thr);
    cudaFree(ctx->d_heap_feat);
    cudaFree(ctx->d_heap_leaf);
    cudaFree(ctx->d_sched);
    cudaFree(ctx->d_fast_keys);
    cudaFree(ctx->d_fast_htab);
    cudaFree(ctx->d_slot_kind);
    cudaFree(ctx->d_def_tables);
    cudaFree(ctx->d_counts);
    delete ctx;
}

static size_t align8(size_t x) { return (x + 7) & ~(size_t)7; }

static int find_host_tag(const ugvc_ctx* ctx, const std::string& name);
static std::string inf_err_message(int word);

// Tables of the tile kernel (k1_tok): every INFO key it may meet -- the plan's tags declared in ##INFO
// plus the keys seen in the data (`info_keys`, "KEY;KEY!;..." as for the key order; '!' marks a key that
// came without a value) -- the usual FORMAT column, the kind bits of every slot, the fixed-column slots.
static int build_fast(ugvc_ctx* ctx, const std::string& info_keys, const std::string& format_keys) {
    const PlanHeader& h = ctx->plan.h;
    DevFast f{};
    std::vector<int> fmt_tags;
    // ---- the usual FORMAT column
    if (!format_keys.empty() && format_keys.size() <= 24) {
        std::vector<std::string> subs;
        size_t b = 0;
        for (;;) {
            size_t e = format_keys.find(':', b);
            if (e == std::string::npos) e = format_keys.size();
            subs.push_back(format_keys.substr(b, e - b));
            if (e == format_keys.size()) break;
            b = e + 1;
        }
        if (subs.size() <= UGVC_MAX_FMT_KEYS) {
            f.n_fmt = (int)subs.size();
            f.fmt_len = (int)format_keys.size();
            memcpy(f.fmt_w, format_keys.data(), format_keys.size());
            for (size_t i = 0; i < subs.size(); ++i) {
                FastMeta m{};
                m.whole_red = 0xFF;
                m.tag = 0xFF;
                const int t = find_host_tag(ctx, subs[i]);
                if (t >= 0 && ctx->h_tags[t].fmt_kind) {
                    const PlanTag& tg = ctx->h_tags[t];
                    const bool has_whole = tg.whole_red != 0xFF;
                    m.type = tg.fmt_kind & KIND_TYPE_MASK;
                    m.flags = FK_NEEDED | ((tg.fmt_kind & KIND_SCALAR) ? FK_SCALAR : 0);
                    m.n_elem = (uint8_t)(tg.n_slots - (has_whole ? 1 : 0));
                    m.slot0 = tg.first_slot;
                    m.whole_red = tg.whole_red;
                    m.whole_slot = tg.whole_slot;
                    m.tag = (uint8_t)t;
                    fmt_tags.push_back(t);
                }
                f.fmt[i] = m;
            }
        }
    }
    auto in_fmt = [&](int t) {
        for (int x : fmt_tags)
            if (x == t) return true;
        return false;
    };
    // ---- INFO keys
    std::vector<FastKey> keys;
    auto add_key = [&](const std::string& name, int t) {
        if (name.empty() || name.size() > 15 || keys.size() >= KF_MAX_KEYS) return;
        for (const FastKey& k : keys)
            if (k.len == name.size() && memcmp(k.name, name.data(), name.size()) == 0) return;
        FastKey k{};
        memcpy(k.name, name.data(), name.size());
        k.len = (uint8_t)name.size();
        k.m.whole_red = 0xFF;
        k.m.tag = 0xFF;
        if (t >= 0 && ctx->h_tags[t].info_kind) {
            const PlanTag& tg = ctx->h_tags[t];
            const bool has_whole = tg.whole_red != 0xFF;
            k.m.type = tg.info_kind & KIND_TYPE_MASK;
            k.m.flags = FK_NEEDED | ((tg.info_kind & KIND_SCALAR) ? FK_SCALAR : 0) | (in_fmt(t) ? FK_SKIP_FMT : 0);
            k.m.n_elem = (uint8_t)(tg.n_slots - (has_whole ? 1 : 0));
            k.m.slot0 = tg.first_slot;
            k.m.whole_red = tg.whole_red;
            k.m.whole_slot = tg.whole_slot;
            k.m.tag = (uint8_t)t;
        }
        keys.push_back(k);
    };
    for (size_t t = 0; t < ctx->h_tags.size(); ++t)
        if (ctx->h_tags[t].info_kind) add_key(std::string(ctx->h_tags[t].name, ctx->h_tags[t].len), (int)t);
    {
        size_t b = 0;
        while (b < info_keys.size()) {
            size_t e = info_keys.find(';', b);
            if (e == std::string::npos) e = info_keys.size();
            std::string key = info_keys.substr(b, e - b);
            b = e + 1;
            if (!key.empty() && key.back() == '!') key.pop_back();
            if (!key.empty()) add_key(key, find_host_tag(ctx, key));
        }
    }
    uint8_t htab[256];
    memset(htab, 0xFF, sizeof(htab));
    for (size_t i = 0; i < keys.size(); ++i) {
        uint32_t idx = kf_hash(keys[i].name[0], keys[i].name[1], keys[i].name[2], keys[i].name[3], keys[i].len);
        while (htab[idx] != 0xFF) idx = (idx + 1) & 255u;
        htab[idx] = (uint8_t)i;
    }
    // ---- per-slot kind bits, fixed-column slots
    std::vector<uint8_t> kind(h.n_slots ? h.n_slots : 1, 0);
    memset(f.fix_slot, 0xFF, sizeof(f.fix_slot));
    for (uint32_t s = 0; s < h.n_slots; ++s) {
        const PlanSlot& sl = ctx->h_slots[s];
        if (sl.tag == TAG_FIXED) {
            const int which = sl.reducer == RED_FIX_QUAL ? FIX_QUAL : sl.reducer == RED_FIX_ALLELE0 ? FIX_ALLELE0
                              : sl.reducer == RED_FIX_ALLELE1 ? FIX_ALLELE1 : sl.reducer == RED_FIX_INDEL ? FIX_INDEL
                              : sl.reducer == RED_FIX_NALLELES ? FIX_NALLELES : -1;
            if (which >= 0 && f.fix_slot[which] == 0xFF) f.fix_slot[which] = (uint8_t)s;
            continue;
        }
        const PlanTag& tg = ctx->h_tags[sl.tag];
        const unsigned k = (in_fmt(sl.tag) && tg.fmt_kind) ? tg.fmt_kind : (tg.info_kind ? tg.info_kind : tg.fmt_kind);
        const unsigned type = k & KIND_TYPE_MASK;
        uint8_t bits = SK_CLS_BAD;  // region sets, flags, reducers that do not fit the declared type: the generic parser
        if (tg.whole_red != RED_REGION && type != KIND_FLAG) {
            if (sl.reducer == RED_NUM && (type == KIND_INT || type == KIND_FLOAT)) bits = SK_CLS_NUM;
            else if (sl.reducer == RED_STRNUM) bits = SK_CLS_NUM | SK_STRNUM;
            else if (sl.reducer == RED_DICT && type == KIND_STR) bits = SK_CLS_DICT;
            else if ((sl.reducer == RED_INSDEL || sl.reducer == RED_MOTIF_L || sl.reducer == RED_MOTIF_R) && type == KIND_STR) bits = SK_CLS_GEN;
            else if (sl.reducer == RED_BASE && type == KIND_STR) bits = SK_CLS_GEN | SK_ZERO_LONG;
            else if (sl.reducer == RED_GT_HOM) bits = SK_CLS_GEN | SK_ZERO_LONG;
            else if (sl.reducer == RED_LEN) bits = SK_CLS_BAD;  // written directly, never queued
        }
        if (type == KIND_INT && sl.reducer != RED_STRNUM) bits |= SK_INT;
        if (k & KIND_SCALAR) bits |= SK_SCALAR;
        kind[s] = bits;
    }
    // ---- k1_tok: where the values of a tag are decoded.  Numbers and string reducers get a column of the window's
    // value table (same key, same spelling: the lanes of a warp run one path), single categories go through the
    // dictionary queue (mostly sparse annotation flags), everything else is decoded where it is met.
    {
        unsigned next_col = 0;
        auto place = [&](FastMeta& m) {
            m.col = KF_COL_NONE;
            if (!(m.flags & FK_NEEDED) || (m.flags & FK_SKIP_FMT)) return;
            const bool special = m.whole_red != 0xFF && m.whole_red != RED_LEN;
            if (!special && m.n_elem == 0) {  // only the element count is wanted
                if (next_col < KF_COLS) m.col = (uint8_t)next_col++;
                return;
            }
            const unsigned slot = special ? m.whole_slot : m.slot0;
            if (slot >= kind.size()) return;
            const unsigned c = kind[slot] & SK_CLS_MASK;
            if (c == SK_CLS_DICT && (special || m.n_elem == 1)) m.col = KF_COL_DICT;
            else if ((c == SK_CLS_NUM || c == SK_CLS_GEN) && next_col < KF_COLS) m.col = (uint8_t)next_col++;
        };
        for (FastKey& k : keys) place(k.m);
        for (int i = 0; i < f.n_fmt; ++i) place(f.fmt[i]);
        f.n_cols = (int)next_col;
    }
    cudaFree(ctx->d_fast_keys);
    cudaFree(ctx->d_fast_htab);
    cudaFree(ctx->d_slot_kind);
    ctx->d_fast_keys = nullptr;
    ctx->d_fast_htab = nullptr;
    ctx->d_slot_kind = nullptr;
    CU(cudaMalloc(&ctx->d_fast_keys, (keys.size() + 1) * sizeof(FastKey)));
    if (!keys.empty()) CU(cudaMemcpy(ctx->d_fast_keys, keys.data(), keys.size() * sizeof(FastKey), cudaMemcpyHostToDevice));
    CU(cudaMalloc(&ctx->d_fast_htab, 256));
    CU(cudaMemcpy(ctx->d_fast_htab, htab, 256, cudaMemcpyHostToDevice));
    CU(cudaMalloc(&ctx->d_slot_kind, kind.size()));
    CU(cudaMemcpy(ctx->d_slot_kind, kind.data(), kind.size(), cudaMemcpyHostToDevice));
    f.keys = ctx->d_fast_keys;
    f.htab = ctx->d_fast_htab;
    f.slot_kind = ctx->d_slot_kind;
    f.n_keys = (int)keys.size();
    const char* legacy = getenv("UGVC_K1_LEGACY");  // profiling / differential tests: the generic parser alone
    f.enabled = !(legacy && *legacy && *legacy != '0');
    ctx->fast = f;
    return UGVC_OK;
}


extern "C" int ugvc_load_plan(ugvc_ctx* ctx, const void* blob, size_t n_bytes) {
    if (!ctx || !blob) return fail(ctx, UGVC_E_ARG, "null argument");
    CU(cudaSetDevice(ctx->device));
    if (n_bytes < sizeof(PlanHeader)) return fail(ctx, UGVC_E_PLAN, "plan blob too small");
    PlanHeader h;
    memcpy(&h, blob, sizeof(h));
    if (h.magic != UGVC_PLAN_MAGIC) return fail(ctx, UGVC_E_PLAN, "bad plan magic");
    if (h.version != UGVC_PLAN_VERSION) return fail(ctx, UGVC_E_PLAN, "plan version mismatch");
    if (h.n_tags > UGVC_MAX_TAGS || h.n_slots > UGVC_MAX_SLOTS || h.n_features > UGVC_MAX_FEATURES ||
        h.n_checks > 64 || h.n_combines > 16 || h.n_dicts > 64 || h.n_dict_strings > 96 || h.n_classes < 2 || h.n_classes > UGVC_MAX_CLASSES || h.n_outputs < 1 || h.n_outputs > UGVC_MAX_CLASSES)
        return fail(ctx, UGVC_E_PLAN, "plan dimensions out of range");
    size_t off = align8(sizeof(PlanHeader));
    const size_t o_tags = off;
    off = align8(off + (size_t)h.n_tags * sizeof(PlanTag));
    const size_t o_slots = off;
    off = align8(off + (size_t)h.n_slots * sizeof(PlanSlot));
    const size_t o_dicts = off;
    off = align8(off + (size_t)h.n_dicts * sizeof(PlanDict));
    const size_t o_strings = off;
    off = align8(off + (size_t)h.n_dict_strings * sizeof(PlanString));
    const size_t o_feats = off;
    off = align8(off + (size_t)h.n_features * sizeof(PlanFeature));
    const size_t o_checks = off;
    off = align8(off + (size_t)h.n_checks * sizeof(PlanCheck));
    const size_t o_combines = off;
    off = align8(off + (size_t)h.n_combines * sizeof(PlanCombine));
    size_t o_coef = 0, o_icpt = 0, o_root = 0, o_tout = 0, o_nodes = 0, o_leaves = 0, o_flags = 0, o_cat = 0;
    PlanCatHeader cat_h{0, 0};
    if (h.model_kind == MODEL_LOGISTIC) {
        o_coef = off;
        off = align8(off + (size_t)h.n_outputs * h.n_features * sizeof(double));
        o_icpt = off;
        off = align8(off + (size_t)h.n_outputs * sizeof(double));
    } else if (h.model_kind >= MODEL_GB_SKLEARN && h.model_kind <= MODEL_XGB) {
        o_root = off;
        off = align8(off + (size_t)(h.n_trees + 1) * sizeof(uint32_t));
        o_tout = off;
        off = align8(off + (size_t)h.n_trees);
        o_nodes = off;
        off = align8(off + (size_t)h.n_nodes * sizeof(PlanNode));
        o_leaves = off;
        off = align8(off + (size_t)h.n_leaf_rows * h.leaf_width * sizeof(double));
        o_flags = off;
        off = align8(off + (size_t)h.n_nodes);
        if (off + sizeof(PlanCatHeader) > n_bytes) return fail(ctx, UGVC_E_PLAN, "plan blob truncated");
        memcpy(&cat_h, static_cast<const uint8_t*>(blob) + off, sizeof(cat_h));
        off += sizeof(PlanCatHeader);
        if (cat_h.n_words >= (1u << 24)) return fail(ctx, UGVC_E_PLAN, "too many category bitset words");
        o_cat = off;
        off = align8(off + (size_t)cat_h.n_words * sizeof(uint32_t));
    } else if (h.model_kind == MODEL_NONE) {
        if (h.n_features != 0) return fail(ctx, UGVC_E_PLAN, "a plan without a model cannot have features");
    } else {
        return fail(ctx, UGVC_E_PLAN, "unsupported model kind");
    }
    if (off > n_bytes) return fail(ctx, UGVC_E_PLAN, "plan blob truncated");
    const uint8_t* hb = static_cast<const uint8_t*>(blob);
    // validate slot / feature references and build the tag hash table
    const PlanTag* tags = reinterpret_cast<const PlanTag*>(hb + o_tags);
    const PlanSlot* slots = reinterpret_cast<const PlanSlot*>(hb + o_slots);
    const PlanFeature* feats = reinterpret_cast<const PlanFeature*>(hb + o_feats);
    uint8_t htab[256];
    memset(htab, 0xFF, sizeof(htab));
    for (uint32_t t = 0; t < h.n_tags; ++t) {
        if (tags[t].len == 0 || tags[t].len > UGVC_NAME_MAX) return fail(ctx, UGVC_E_PLAN, "bad tag name length");
        if ((uint32_t)tags[t].first_slot + tags[t].n_slots > h.n_slots) return fail(ctx, UGVC_E_PLAN, "tag slots out of range");
        unsigned long long kw[4];
        memcpy(kw, tags[t].name, 32);
        unsigned idx = ugvc_key_hash(kw[0], kw[1], kw[2], kw[3], tags[t].len);
        while (htab[idx] != 0xFF) idx = (idx + 1) & 255u;
        htab[idx] = (uint8_t)t;
    }
    uint32_t first_fixed = h.n_slots;
    for (uint32_t s = 0; s < h.n_slots; ++s) {
        if (slots[s].tag == TAG_FIXED) {
            if (first_fixed == h.n_slots) first_fixed = s;
        } else {
            if (first_fixed != h.n_slots) return fail(ctx, UGVC_E_PLAN, "fixed slots must come last");
            if (slots[s].tag >= h.n_tags) return fail(ctx, UGVC_E_PLAN, "slot tag out of range");
            if (slots[s].reducer == RED_DICT && slots[s].dict >= h.n_dicts) return fail(ctx, UGVC_E_PLAN, "slot dict out of range");
        }
    }
    for (uint32_t f = 0; f < h.n_features; ++f)
        if (feats[f].slot >= h.n_slots) return fail(ctx, UGVC_E_PLAN, "feature slot out of range");
    {
        const PlanCheck* checks = reinterpret_cast<const PlanCheck*>(hb + o_checks);
        for (uint32_t c = 0; c < h.n_checks; ++c)
            if (checks[c].slot >= h.n_slots) return fail(ctx, UGVC_E_PLAN, "check slot out of range");
        const PlanCombine* comb = reinterpret_cast<const PlanCombine*>(hb + o_combines);
        for (uint32_t c = 0; c < h.n_combines; ++c)
            if (comb[c].slot_b >= h.n_slots || comb[c].feature >= h.n_features)
                return fail(ctx, UGVC_E_PLAN, "combine entry out of range");
    }
    if (h.model_kind != MODEL_LOGISTIC && h.model_kind != MODEL_NONE) {
        const uint32_t* root = reinterpret_cast<const uint32_t*>(hb + o_root);
        const PlanNode* nodes = reinterpret_cast<const PlanNode*>(hb + o_nodes);
        const uint8_t* tout = hb + o_tout;
        const uint8_t* nflags = hb + o_flags;
        uint32_t n_flagged = 0;
        for (uint32_t t = 0; t < h.n_trees; ++t) {
            if (root[t] > root[t + 1] || root[t + 1] > h.n_nodes) return fail(ctx, UGVC_E_PLAN, "tree roots not monotone");
            if (tout[t] >= h.n_outputs) return fail(ctx, UGVC_E_PLAN, "tree output out of range");
            const uint32_t n = root[t + 1] - root[t];
            for (uint32_t i = 0; i < n; ++i) {
                const PlanNode& nd = nodes[root[t] + i];
                const uint8_t fl = nflags[root[t] + i];
                if (fl & ~(NODE_DEFAULT_LEFT | NODE_CATEGORICAL)) return fail(ctx, UGVC_E_PLAN, "unknown node flag");
                if (fl && h.model_kind != MODEL_XGB) return fail(ctx, UGVC_E_PLAN, "node flags on a model other than xgboost");
                n_flagged += fl ? 1u : 0u;
                if (nd.feature >= 0) {
                    if ((uint32_t)nd.feature >= h.n_features || nd.right >= n || i + 1 >= n)
                        return fail(ctx, UGVC_E_PLAN, "tree node out of range");
                    if (fl & NODE_CATEGORICAL) {  // the node's bitset lies inside the category section
                        uint32_t ref;
                        memcpy(&ref, &nd.value, 4);
                        const uint32_t words = UGVC_CAT_WORDS(ref);
                        if (words == 0 || words > UGVC_CAT_MAX_WORDS || UGVC_CAT_FIRST(ref) + words > cat_h.n_words)
                            return fail(ctx, UGVC_E_PLAN, "category bitset reference out of range");
                    }
                } else {
                    if (fl) return fail(ctx, UGVC_E_PLAN, "node flags on a leaf");
                    int32_t leaf;
                    memcpy(&leaf, &nd.value, 4);
                    if (leaf < 0 || (uint32_t)leaf >= h.n_leaf_rows) return fail(ctx, UGVC_E_PLAN, "leaf row out of range");
                }
            }
        }
        if (n_flagged != cat_h.n_flagged) return fail(ctx, UGVC_E_PLAN, "flagged node count does not match the node flags");
    }
    // walk variant, chosen once here: the plain walks unless a node routes by a flag
    const uint32_t walk = cat_h.n_flagged ? K3_WALK_CAT : K3_WALK_PLAIN;
    // device form of the forest: leaves become absorbing nodes (threshold = quiet NaN carrying the
    // leaf row, right child = itself) so a fixed-depth, branch-free walk ends on them; right
    // children are absolute indices.  Also the depth of the deepest leaf.
    std::vector<uint2> dev_nodes;
    uint32_t max_depth = 0;
    if (h.model_kind != MODEL_LOGISTIC && h.model_kind != MODEL_NONE) {
        const uint32_t* root = reinterpret_cast<const uint32_t*>(hb + o_root);
        const PlanNode* nodes = reinterpret_cast<const PlanNode*>(hb + o_nodes);
        const uint8_t* nflags = hb + o_flags;
        // the categorical walk keeps the node flags in bits 8-9 of y: right children take 22 bits there
        const unsigned rsh = walk == K3_WALK_CAT ? 10u : 8u;
        if (h.n_nodes >= (1u << (32 - rsh)) || h.n_leaf_rows >= (1u << 22) || h.n_features > 255)
            return fail(ctx, UGVC_E_PLAN, "forest too large for the device node format");
        // the category bitset words follow the nodes in the same device allocation
        dev_nodes.resize(h.n_nodes + (cat_h.n_words + 1) / 2);
        if (cat_h.n_words) memcpy(dev_nodes.data() + h.n_nodes, hb + o_cat, (size_t)cat_h.n_words * sizeof(uint32_t));
        std::vector<uint32_t> depth(h.n_nodes, 0);
        for (uint32_t t = 0; t < h.n_trees; ++t) {
            const uint32_t r0 = root[t], n = root[t + 1] - root[t];
            if (n) depth[r0] = 0;
            for (uint32_t i = 0; i < n; ++i) {  // preorder: parents precede children
                const PlanNode& nd = nodes[r0 + i];
                if (nd.feature >= 0) {
                    uint32_t thr;
                    memcpy(&thr, &nd.value, 4);
                    dev_nodes[r0 + i] = make_uint2(thr, (uint32_t)nd.feature | ((uint32_t)nflags[r0 + i] << 8) | ((r0 + nd.right) << rsh));
                    depth[r0 + i + 1] = depth[r0 + i] + 1;
                    depth[r0 + nd.right] = depth[r0 + i] + 1;
                } else {
                    int32_t leaf;
                    memcpy(&leaf, &nd.value, 4);
                    dev_nodes[r0 + i] = make_uint2(0x7FC00000u | (uint32_t)leaf, (r0 + i) << rsh);
                    if (depth[r0 + i] > max_depth) max_depth = depth[r0 + i];
                }
            }
        }
    }

    // heap form for k3_heap: every tree padded to a complete binary tree (breadth-first, root at index 1);
    // below a shallow leaf every node is (+inf, feature 0, no flags) and every leaf slot carries its row, so a row
    // reaches it whichever way it goes there (NaN included).  The categorical walk's node flags follow the features
    // in the same array (heap_feat[n_trees * H + i]); a categorical node's threshold word is its bitset reference.
    std::vector<float> heap_thr;
    std::vector<uint8_t> heap_feat;
    std::vector<uint16_t> heap_leaf;
    uint32_t heap_depth = 0;
    if (!dev_nodes.empty() && max_depth <= 8 && h.n_leaf_rows < 65536 && h.n_features <= 255) {
        const uint32_t* root = reinterpret_cast<const uint32_t*>(hb + o_root);
        const PlanNode* nodes = reinterpret_cast<const PlanNode*>(hb + o_nodes);
        heap_depth = max_depth ? max_depth : 1;
        const uint32_t H = 1u << heap_depth;
        const float inf = __builtin_huge_valf();
        heap_thr.assign((size_t)h.n_trees * H, inf);
        heap_feat.assign((size_t)h.n_trees * H * (walk == K3_WALK_CAT ? 2 : 1), 0);
        const uint8_t* nflags = hb + o_flags;
        heap_leaf.assign((size_t)h.n_trees * H, 0);
        struct Item { uint32_t node, heap, level; int32_t leaf; };  // leaf >= 0: inside a padded subtree
        std::vector<Item> stack;
        for (uint32_t t = 0; t < h.n_trees; ++t) {
            const uint32_t r0 = root[t];
            float* thr = heap_thr.data() + (size_t)t * H;
            uint8_t* ft = heap_feat.data() + (size_t)t * H;
            uint16_t* lf = heap_leaf.data() + (size_t)t * H;
            stack.clear();
            stack.push_back({0, 1, 0, -1});
            while (!stack.empty()) {
                const Item it = stack.back();
                stack.pop_back();
                int32_t leaf = it.leaf;
                if (leaf < 0) {
                    const PlanNode& nd = nodes[r0 + it.node];
                    if (nd.feature >= 0) {
                        thr[it.heap] = nd.value;
                        ft[it.heap] = (uint8_t)nd.feature;
                        if (walk == K3_WALK_CAT) ft[(size_t)h.n_trees * H + it.heap] = nflags[r0 + it.node];
                        stack.push_back({it.node + 1, 2 * it.heap, it.level + 1, -1});
                        stack.push_back({nd.right, 2 * it.heap + 1, it.level + 1, -1});
                        continue;
                    }
                    memcpy(&leaf, &nd.value, 4);
                }
                if (it.level == heap_depth) {
                    lf[it.heap - H] = (uint16_t)leaf;
                } else {  // thr stays +inf, feature 0
                    stack.push_back({0, 2 * it.heap, it.level + 1, leaf});
                    stack.push_back({0, 2 * it.heap + 1, it.level + 1, leaf});
                }
            }
        }
    }
    // from here on the previous plan is gone: no plan is loaded until every step below has succeeded, and the
    // lanes sized for the old slot / feature counts go with it
    ctx->has_plan = false;
    for (auto& l : ctx->lanes) free_lane(l);
    ctx->lanes.clear();
    ctx->cap_bytes = ctx->cap_records = 0;
    cudaFree(ctx->d_plan);
    cudaFree(ctx->d_htab);
    cudaFree(ctx->d_nodes);
    cudaFree(ctx->d_heap_thr);
    cudaFree(ctx->d_heap_feat);
    cudaFree(ctx->d_heap_leaf);
    ctx->d_heap_thr = nullptr;
    ctx->d_heap_feat = nullptr;
    ctx->d_heap_leaf = nullptr;
    if (heap_depth) {
        CU(cudaMalloc(&ctx->d_heap_thr, heap_thr.size() * sizeof(float)));
        CU(cudaMemcpy(ctx->d_heap_thr, heap_thr.data(), heap_thr.size() * sizeof(float), cudaMemcpyHostToDevice));
        CU(cudaMalloc(&ctx->d_heap_feat, heap_feat.size()));
        CU(cudaMemcpy(ctx->d_heap_feat, heap_feat.data(), heap_feat.size(), cudaMemcpyHostToDevice));
        CU(cudaMalloc(&ctx->d_heap_leaf, heap_leaf.size() * sizeof(uint16_t)));
        CU(cudaMemcpy(ctx->d_heap_leaf, heap_leaf.data(), heap_leaf.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
    }
    ctx->d_plan = nullptr;
    ctx->d_htab = nullptr;
    ctx->d_nodes = nullptr;
    if (!dev_nodes.empty()) {
        CU(cudaMalloc(&ctx->d_nodes, dev_nodes.size() * sizeof(uint2)));
        CU(cudaMemcpy(ctx->d_nodes, dev_nodes.data(), dev_nodes.size() * sizeof(uint2), cudaMemcpyHostToDevice));
    }
    CU(cudaMalloc(&ctx->d_plan, off));
    CU(cudaMemcpy(ctx->d_plan, blob, off, cudaMemcpyHostToDevice));
    CU(cudaMalloc(&ctx->d_htab, 256));
    CU(cudaMemcpy(ctx->d_htab, htab, 256, cudaMemcpyHostToDevice));
    DevPlan& p = ctx->plan;
    p.h = h;
    const uint8_t* d = ctx->d_plan;
    p.tags = reinterpret_cast<const PlanTag*>(d + o_tags);
    p.slots = reinterpret_cast<const PlanSlot*>(d + o_slots);
    p.dicts = reinterpret_cast<const PlanDict*>(d + o_dicts);
    p.strings = reinterpret_cast<const PlanString*>(d + o_strings);
    p.feats = reinterpret_cast<const PlanFeature*>(d + o_feats);
    p.checks = reinterpret_cast<const PlanCheck*>(d + o_checks);
    p.combines = reinterpret_cast<const PlanCombine*>(d + o_combines);
    p.coef = reinterpret_cast<const double*>(d + o_coef);
    p.intercept = reinterpret_cast<const double*>(d + o_icpt);
    p.tree_root = reinterpret_cast<const uint32_t*>(d + o_root);
    p.tree_out = d + o_tout;
    p.nodes = reinterpret_cast<const PlanNode*>(d + o_nodes);
    p.dev_nodes = ctx->d_nodes;
    p.max_depth = max_depth;
    p.walk = walk;
    p.n_cat_words = cat_h.n_words;
    p.heap_thr = ctx->d_heap_thr;
    p.heap_feat = ctx->d_heap_feat;
    p.heap_leaf = ctx->d_heap_leaf;
    p.heap_depth = heap_depth;
    p.leaves = reinterpret_cast<const double*>(d + o_leaves);
    p.htab = ctx->d_htab;
    p.first_fixed_slot = first_fixed;
    if (k1_smem_bytes(p) > 227 * 1024)
        return fail(ctx, UGVC_E_PLAN, "plan needs more shared memory than one sm_90 CTA has (K1 field parse)");
    if (h.model_kind != MODEL_NONE) {
        std::string why;
        if (!k3_choose(p, reinterpret_cast<const uint32_t*>(hb + o_root), ctx->sm_count, &ctx->k3, &why))
            return fail(ctx, UGVC_E_PLAN, why);
    }
    CU(kernels_configure(p));
    ctx->h_tags.assign(tags, tags + h.n_tags);
    ctx->h_slots.assign(slots, slots + h.n_slots);
#ifdef UGVC_K1_INLINE_DICT1
    {
        const PlanDict* dd = reinterpret_cast<const PlanDict*>(hb + o_dicts);
        const PlanString* ss = reinterpret_cast<const PlanString*>(hb + o_strings);
        ctx->h_dicts.assign(dd, dd + h.n_dicts);
        ctx->h_strings.assign(ss, ss + h.n_dict_strings);
    }
#endif
    cudaFree(ctx->d_sched);  // a key order belongs to a plan
    ctx->d_sched = nullptr;
    ctx->sched = DevSchedule{};
    ctx->learned_info.clear();
    ctx->learned_fmt.clear();
    {
        const int rc = build_fast(ctx, "", "");
        if (rc) return rc;
    }
    ctx->has_plan = true;
    // a new plan changes the slot/feature counts: lanes must be re-reserved
    for (auto& l : ctx->lanes) free_lane(l);
    ctx->lanes.clear();
    ctx->cap_bytes = ctx->cap_records = 0;
    return UGVC_OK;
}

static int find_host_tag(const ugvc_ctx* ctx, const std::string& name) {
    for (size_t t = 0; t < ctx->h_tags.size(); ++t)
        if (ctx->h_tags[t].len == name.size() && memcmp(ctx->h_tags[t].name, name.data(), name.size()) == 0) return (int)t;
    return -1;
}

// decode class of a tag in one header section, from the plan's slot layout
static void classify(const ugvc_ctx* ctx, int tag, bool format, SchedEntry& se) {
    se.tag = (int16_t)tag;
    se.cls = CLS_SKIP;
    if (tag < 0) return;
    const PlanTag& tg = ctx->h_tags[tag];
    const unsigned kind = format ? tg.fmt_kind : tg.info_kind;
    if (!kind) return;  // not declared in this section: the value is skipped
    se.cls = CLS_GENERIC;
    const unsigned type = kind & KIND_TYPE_MASK;
    const bool scalar = (kind & KIND_SCALAR) != 0;
    const bool has_whole = tg.whole_red != 0xFF;
    const int n_elem = (int)tg.n_slots - (has_whole ? 1 : 0);
    se.slot0 = tg.first_slot;
    se.n_elem = (uint8_t)n_elem;
    bool all_num = true;
    for (int e = 0; e < n_elem; ++e) all_num &= ctx->h_slots[tg.first_slot + e].reducer == RED_NUM;
    if (type == KIND_INT && all_num && (!has_whole || tg.whole_red == RED_LEN)) {
        se.cls = CLS_INT;
        if (has_whole) se.flags |= SCHED_COUNT_ALL;
    } else if (type == KIND_FLOAT && all_num && !has_whole) {
        se.cls = CLS_FLOAT;
    } else if (type == KIND_STR && scalar && n_elem == 1 && !has_whole &&
               ctx->h_slots[tg.first_slot].reducer == RED_DICT) {
        se.cls = CLS_DICT1;
        se.dict = ctx->h_slots[tg.first_slot].dict;
#ifdef UGVC_K1_INLINE_DICT1
        // a single short category and a key that leaves w1 free: K1 compares the value in the schedule loop itself
        // (for the default annotation encoder the categories are {FALSE, TRUE} and the file only ever spells TRUE:
        // the last category is the one compared inline, any other spelling takes the full decoder)
        if (!format && se.dict < ctx->h_dicts.size() && ctx->h_dicts[se.dict].n_strings >= 1 &&
            ctx->h_dicts[se.dict].n_strings <= 2) {
            const int pick = ctx->h_dicts[se.dict].n_strings - 1;
            const PlanString& ps = ctx->h_strings[ctx->h_dicts[se.dict].first_string + pick];
            if (ps.len >= 1 && ps.len <= 7) {
                se.flags |= SCHED_DICT_INLINE | (pick ? SCHED_DICT_INLINE_SECOND : 0u);
                se.n_elem = ps.len;
                se.w1 = 0;
                memcpy(&se.w1, &ps, ps.len);
            }
        }
#endif
    }
}

extern "C" int ugvc_set_key_order(ugvc_ctx* ctx, const char* info_keys, const char* format_keys) {
    if (!ctx) return UGVC_E_ARG;
    if (!ctx->has_plan) return fail(ctx, UGVC_E_STATE, "set_key_order: load a plan first");
    CU(cudaSetDevice(ctx->device));
    CU(cudaDeviceSynchronize());
    std::vector<SchedEntry> entries;
    if (info_keys) {
        const char* p = info_keys;
        while (*p && entries.size() < UGVC_MAX_SCHED) {
            const char* e = p;
            while (*e && *e != ';') ++e;
            std::string key(p, e);
            p = *e ? e + 1 : e;
            if (key.empty()) continue;
            SchedEntry se;
            memset(&se, 0, sizeof(se));
            const bool is_flag = key.back() == '!';
            if (is_flag) key.pop_back();
            const std::string bytes = key + (is_flag ? "" : "=");
            if (key.empty() || bytes.size() > 16) continue;  // longer keys simply take the generic path
            if (is_flag) se.flags |= SCHED_IS_FLAG;
            classify(ctx, find_host_tag(ctx, key), false, se);
            se.len = (uint8_t)bytes.size();
            unsigned char buf[16] = {0};
            memcpy(buf, bytes.data(), bytes.size());
            memcpy(&se.w0, buf, 8);
#ifdef UGVC_K1_INLINE_DICT1
            if ((se.flags & SCHED_DICT_INLINE) && bytes.size() > 8) se.flags &= ~SCHED_DICT_INLINE;  // w1 is needed for the key
            if (!(se.flags & SCHED_DICT_INLINE))
#endif
            memcpy(&se.w1, buf + 8, 8);
            se.m0 = bytes.size() >= 8 ? ~0ull : ((1ull << (8 * bytes.size())) - 1ull);
            entries.push_back(se);
        }
    }
    DevSchedule sc{};
    cudaFree(ctx->d_sched);
    ctx->d_sched = nullptr;
    if (!entries.empty()) {
        CU(cudaMalloc(&ctx->d_sched, entries.size() * sizeof(SchedEntry)));
        CU(cudaMemcpy(ctx->d_sched, entries.data(), entries.size() * sizeof(SchedEntry), cudaMemcpyHostToDevice));
        sc.info = ctx->d_sched;
        sc.n_info = (int)entries.size();
    }
    if (format_keys && *format_keys) {
        const std::string f(format_keys);
        if (f.size() <= 24) {
            int n = 0;
            size_t b = 0;
            bool ok = true;
            for (;;) {
                size_t e = f.find(':', b);
                if (e == std::string::npos) e = f.size();
                if (n >= UGVC_MAX_FMT_KEYS) {
                    ok = false;
                    break;
                }
                memset(&sc.fmt[n], 0, sizeof(SchedEntry));
                classify(ctx, find_host_tag(ctx, f.substr(b, e - b)), true, sc.fmt[n]);
                ++n;
                if (e == f.size()) break;
                b = e + 1;
            }
            if (ok) {
                sc.n_fmt = n;
                sc.fmt_len = (int)f.size();
                memcpy(sc.fmt_w, f.data(), f.size());
            }
        }
    }
    ctx->sched = sc;
    ctx->learned_info = info_keys ? info_keys : "";
    ctx->learned_fmt = format_keys ? format_keys : "";
    return build_fast(ctx, ctx->learned_info, ctx->learned_fmt);
}

extern "C" int ugvc_plan_info(const ugvc_ctx* ctx, int32_t* n_features, int32_t* n_classes, int32_t* n_slots) {
    if (!ctx || !ctx->has_plan) return UGVC_E_STATE;
    if (n_features) *n_features = (int32_t)ctx->plan.h.n_features;
    if (n_classes) *n_classes = (int32_t)ctx->plan.h.n_classes;
    if (n_slots) *n_slots = (int32_t)ctx->plan.h.n_slots;
    return UGVC_OK;
}

extern "C" int ugvc_reserve(ugvc_ctx* ctx, size_t max_bytes, size_t max_records, int n_pipeline) {
    if (!ctx) return UGVC_E_ARG;
    if (!ctx->has_plan) return fail(ctx, UGVC_E_STATE, "ugvc_reserve: load a plan first");
    if (n_pipeline < 1 || n_pipeline > 8 || max_bytes == 0 || max_records == 0)
        return fail(ctx, UGVC_E_ARG, "ugvc_reserve: bad sizes");
    CU(cudaSetDevice(ctx->device));
    for (auto& l : ctx->lanes) free_lane(l);
    ctx->lanes.clear();
    max_records = (max_records + 127) & ~(size_t)127;  // rows stay 512-byte aligned
    ctx->cap_bytes = max_bytes;
    ctx->cap_records = max_records;
    ctx->lanes.resize(n_pipeline);
    const size_t n_chunks = 2 * ((max_bytes + K1_TILE_BYTES_HOST - 1) / K1_TILE_BYTES_HOST + 4);  // uint32 words
    const DevPlan& p = ctx->plan;
    for (auto& l : ctx->lanes) {
        CU(cudaStreamCreateWithFlags(&l.stream, cudaStreamNonBlocking));
        CU(cudaMalloc(&l.d_text, max_bytes + TEXT_SLACK));
        l.b.cap_bytes = max_bytes;
        l.b.cap_records = max_records;
        CU(cudaMalloc(&l.b.chunk_first, n_chunks * sizeof(uint32_t)));
        CU(cudaMalloc(&l.b.slow_list, max_records * sizeof(uint32_t)));
        CU(cudaMalloc(&l.b.line_start, (max_records + 1) * sizeof(int64_t)));
        CU(cudaMalloc(&l.b.n_records, sizeof(int64_t)));
        CU(cudaMalloc(&l.b.raw, (size_t)p.h.n_slots * max_records * sizeof(uint32_t)));
        CU(cudaMalloc(&l.b.recinfo, max_records * sizeof(ugvc_recinfo)));
        CU(cudaMalloc(&l.b.feats, (size_t)p.h.n_features * max_records * sizeof(float)));
        CU(cudaMalloc(&l.b.low_score, max_records));
        CU(cudaMalloc(&l.b.probs, max_records * p.h.n_classes * sizeof(float)));
        CU(cudaMalloc(&l.b.qual, max_records * sizeof(double)));
        if (ctx->want_phreds) CU(cudaMalloc(&l.b.phreds, max_records * p.h.n_classes * sizeof(double)));
        CU(cudaMalloc(&l.d_err, sizeof(unsigned long long)));
        CU(cudaHostAlloc(&l.h_n, sizeof(int64_t), cudaHostAllocDefault));
        CU(cudaHostAlloc(&l.h_err, sizeof(unsigned long long), cudaHostAllocDefault));
    }
    return UGVC_OK;
}

// enqueue K0..K3 for text already on the device
static int enqueue_kernels(ugvc_ctx* ctx, Lane& l, const uint8_t* d_text, size_t n_bytes, double threshold,
                           uint8_t* d_low, float* d_probs, double* d_qual, ugvc_recinfo* d_recinfo,
                           int64_t* d_line_start, size_t line_cap, int64_t* d_n_records, cudaStream_t st) {
    const DevPlan& p = ctx->plan;
    const bool timing = ctx->timing;
    cudaEvent_t* ev = nullptr;
    if (timing) {
        if (l.ev_used + 5 > l.ev_pool.size()) {
            const size_t old = l.ev_pool.size();
            l.ev_pool.resize(old + 5 * 64, nullptr);
            for (size_t i = old; i < l.ev_pool.size(); ++i) CU(cudaEventCreate(&l.ev_pool[i]));
        }
        ev = &l.ev_pool[l.ev_used];
        l.ev_used += 5;
    }
    CU(cudaMemsetAsync(l.d_err, 0xFF, sizeof(unsigned long long), st));
    if (timing) CU(cudaEventRecord(ev[0], st));
    const bool fast = ctx->fast.enabled && p.h.n_slots <= 250 && line_cap <= 0xFFFFFFFFull;
    if (!fast) launch_k0(d_text, n_bytes, l.b.chunk_first, d_line_start, line_cap, d_n_records, l.d_err, ctx->sm_count, st);
    if (timing) CU(cudaEventRecord(ev[1], st));
    if (fast)  // line index, field parse and the slow tier in one stage
        launch_k1_fast(p, ctx->fast, ctx->sched, d_text, n_bytes, l.b.chunk_first, d_line_start, line_cap, d_n_records,
                       l.b.raw, l.b.cap_records, d_recinfo, l.b.slow_list, l.d_err, ctx->d_counts, ctx->sm_count, st);
    else
        launch_k1(p, ctx->sched, d_text, d_line_start, d_n_records, l.b.raw, l.b.cap_records, d_recinfo, l.d_err,
                  ctx->d_counts, ctx->sm_count, st);
    if (timing) CU(cudaEventRecord(ev[2], st));
    const bool has_model = p.h.model_kind != MODEL_NONE;
    const bool fused = has_model && ctx->k3.kernel == K3_KERNEL_HEAP;  // features assembled in k3_heap's tile load
    if (has_model && !fused) launch_k2(p, l.b.raw, l.b.cap_records, d_n_records, l.b.feats, l.d_err, ctx->sm_count, st);
    if (timing) CU(cudaEventRecord(ev[3], st));
    if (has_model)
        launch_k3(p, ctx->k3, l.b.raw, l.b.feats, l.b.cap_records, d_n_records, threshold, d_low, d_probs, d_qual,
                  d_low == l.b.low_score ? l.b.phreds : nullptr, ctx->want_phreds, ctx->d_counts, l.d_err, st);
    if (timing) CU(cudaEventRecord(ev[4], st));
    ctx->launches += (has_model ? (fused ? 1 : 2) : 0) + (fast ? 2 : 2 + (p.h.n_slots ? 1 : 0));
    CU(cudaGetLastError());
    return UGVC_OK;
}

extern "C" int ugvc_submit_batch(ugvc_ctx* ctx, int lane, const uint8_t* vcf_text, size_t n_bytes, double threshold) {
    if (!ctx) return UGVC_E_ARG;
    if (!ctx->has_plan || ctx->lanes.empty()) return fail(ctx, UGVC_E_STATE, "submit: load a plan and reserve first");
    if (lane < 0 || lane >= (int)ctx->lanes.size()) return fail(ctx, UGVC_E_ARG, "submit: lane out of range");
    if (n_bytes > ctx->cap_bytes) return fail(ctx, UGVC_E_ARG, "submit: batch larger than the reserved max_bytes");
    if (n_bytes && (!vcf_text || vcf_text[n_bytes - 1] != '\n'))
        return fail(ctx, UGVC_E_ARG, "submit: the batch must be whole lines ending with a newline");
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[lane];
    if (l.submitted) return fail(ctx, UGVC_E_STATE, "submit: lane already has a batch in flight");
    if (n_bytes) CU(cudaMemcpyAsync(l.d_text, vcf_text, n_bytes, cudaMemcpyHostToDevice, l.stream));
    CU(cudaMemsetAsync(l.d_text + n_bytes, '\n', TEXT_SLACK, l.stream));
    int rc = enqueue_kernels(ctx, l, l.d_text, n_bytes, threshold, l.b.low_score, l.b.probs, l.b.qual, l.b.recinfo,
                             l.b.line_start, l.b.cap_records, l.b.n_records, l.stream);
    if (rc) return rc;
    CU(cudaMemcpyAsync(l.h_n, l.b.n_records, sizeof(int64_t), cudaMemcpyDeviceToHost, l.stream));
    CU(cudaMemcpyAsync(l.h_err, l.d_err, sizeof(unsigned long long), cudaMemcpyDeviceToHost, l.stream));
    l.n_bytes = n_bytes;
    l.submitted = true;
    return UGVC_OK;
}

static int decode_error(ugvc_ctx* ctx, unsigned long long e) {
    if (e == UGVC_NO_ERROR) return UGVC_OK;
    ctx->err_record = (int64_t)(e >> 24);
    const int col = (int)((e >> 8) & 0xFFFF);
    ctx->err_column = col == 0xFFFF ? -1 : col;
    ctx->err_reason = (int32_t)(e & 0xFF);
    static const char* names[] = {"none",
                                  "null feature value (the reference's _validate_data asserts)",
                                  "value the reference transformer raises on (unknown category / ragged or absent tuple)",
                                  "more elements than the fitted width / more records than reserved",
                                  "numeric literal outside the exact-parse range",
                                  "malformed line (fewer than 8 columns or batch not newline-terminated)"};
    char buf[256];
    snprintf(buf, sizeof(buf), "data error at record %lld, feature column %d: %s", (long long)ctx->err_record,
             ctx->err_column, names[ctx->err_reason < 6 ? ctx->err_reason : 0]);
    ctx->err = buf;
    return UGVC_E_DATA;
}

extern "C" int ugvc_collect_batch(ugvc_ctx* ctx, int lane, uint8_t* out_low_score, float* out_probs, double* out_qual,
                                  ugvc_recinfo* out_recinfo, int64_t* out_line_start, size_t capacity_records,
                                  int64_t* out_n_records) {
    if (!ctx) return UGVC_E_ARG;
    if (lane < 0 || lane >= (int)ctx->lanes.size()) return fail(ctx, UGVC_E_ARG, "collect: lane out of range");
    Lane& l = ctx->lanes[lane];
    if (!l.submitted) return fail(ctx, UGVC_E_STATE, "collect: nothing submitted on this lane");
    CU(cudaSetDevice(ctx->device));
    l.submitted = false;
    CU(cudaStreamSynchronize(l.stream));
    const int64_t n = *l.h_n;
    l.last_n = n;
    if (out_n_records) *out_n_records = n;
    if (l.h_inf_err && *l.h_inf_err) {
        const int code = *l.h_inf_err;
        *l.h_inf_err = 0;
        return fail(ctx, UGVC_E_IO, inf_err_message(code));
    }
    const int rc = decode_error(ctx, *l.h_err);
    if (rc) return rc;
    if ((size_t)n > capacity_records) return fail(ctx, UGVC_E_ARG, "collect: output capacity smaller than the record count");
    const int K = ctx->plan.h.n_classes;
    if (n > 0) {
        if (out_low_score) CU(cudaMemcpyAsync(out_low_score, l.b.low_score, (size_t)n, cudaMemcpyDeviceToHost, l.stream));
        if (out_probs) CU(cudaMemcpyAsync(out_probs, l.b.probs, (size_t)n * K * sizeof(float), cudaMemcpyDeviceToHost, l.stream));
        if (out_qual) CU(cudaMemcpyAsync(out_qual, l.b.qual, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, l.stream));
        if (out_recinfo) CU(cudaMemcpyAsync(out_recinfo, l.b.recinfo, (size_t)n * sizeof(ugvc_recinfo), cudaMemcpyDeviceToHost, l.stream));
    }
    if (out_line_start) CU(cudaMemcpyAsync(out_line_start, l.b.line_start, (size_t)(n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, l.stream));
    CU(cudaStreamSynchronize(l.stream));
    return UGVC_OK;
}

extern "C" int ugvc_filter_batch(ugvc_ctx* ctx, const uint8_t* vcf_text, size_t n_bytes, double threshold,
                                 uint8_t* out_low_score, float* out_probs, double* out_qual,
                                 ugvc_recinfo* out_recinfo, int64_t* out_line_start, size_t capacity_records,
                                 int64_t* out_n_records) {
    int rc = ugvc_submit_batch(ctx, 0, vcf_text, n_bytes, threshold);
    if (rc) return rc;
    return ugvc_collect_batch(ctx, 0, out_low_score, out_probs, out_qual, out_recinfo, out_line_start,
                              capacity_records, out_n_records);
}

extern "C" int ugvc_filter_device_lane(ugvc_ctx* ctx, int lane, const uint8_t* d_text, size_t n_bytes, double threshold,
                                       uint8_t* d_low_score, float* d_probs, double* d_qual, ugvc_recinfo* d_recinfo,
                                       int64_t* d_line_start, size_t capacity_records, int64_t* d_n_records, void* stream) {
    if (!ctx) return UGVC_E_ARG;
    if (!ctx->has_plan || ctx->lanes.empty()) return fail(ctx, UGVC_E_STATE, "filter_device: load a plan and reserve first");
    if (lane < 0 || lane >= (int)ctx->lanes.size()) return fail(ctx, UGVC_E_ARG, "filter_device: lane out of range");
    if (n_bytes > ctx->cap_bytes) return fail(ctx, UGVC_E_ARG, "filter_device: batch larger than the reserved max_bytes");
    if (!d_text || !d_low_score || !d_probs || !d_qual) return fail(ctx, UGVC_E_ARG, "filter_device: null device pointer");
    if (reinterpret_cast<uintptr_t>(d_text) & 15u) return fail(ctx, UGVC_E_ARG, "filter_device: d_text must be 16-byte aligned");
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[lane];
    if (capacity_records == 0 || capacity_records > l.b.cap_records)
        return fail(ctx, UGVC_E_ARG, "filter_device: capacity_records must be in (0, reserved max_records]");
    const size_t line_cap = capacity_records;
    if (!d_line_start) d_line_start = l.b.line_start;
    if (!d_recinfo) d_recinfo = l.b.recinfo;
    if (!d_n_records) d_n_records = l.b.n_records;
    cudaStream_t st = stream ? (cudaStream_t)stream : l.stream;
    return enqueue_kernels(ctx, l, d_text, n_bytes, threshold, d_low_score, d_probs, d_qual, d_recinfo, d_line_start,
                           line_cap, d_n_records, st);
}

extern "C" int ugvc_filter_device(ugvc_ctx* ctx, const uint8_t* d_text, size_t n_bytes, double threshold,
                                  uint8_t* d_low_score, float* d_probs, double* d_qual, ugvc_recinfo* d_recinfo,
                                  int64_t* d_line_start, size_t capacity_records, int64_t* d_n_records, void* stream) {
    return ugvc_filter_device_lane(ctx, 0, d_text, n_bytes, threshold, d_low_score, d_probs, d_qual, d_recinfo, d_line_start,
                                   capacity_records, d_n_records, stream);
}

extern "C" int ugvc_device_status_lane(ugvc_ctx* ctx, int lane, void* stream) {
    // blocking: surfaces data errors of the last ugvc_filter_device_lane call on `lane`
    if (!ctx || lane < 0 || lane >= (int)ctx->lanes.size()) return UGVC_E_STATE;
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[lane];
    cudaStream_t st = stream ? (cudaStream_t)stream : l.stream;
    CU(cudaStreamSynchronize(st));
    unsigned long long e;
    CU(cudaMemcpy(&e, l.d_err, sizeof(e), cudaMemcpyDeviceToHost));
    return decode_error(ctx, e);
}

extern "C" int ugvc_device_status(ugvc_ctx* ctx, void* stream) {
    // blocking: surfaces data errors of the last ugvc_filter_device call
    if (!ctx || ctx->lanes.empty()) return UGVC_E_STATE;
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[0];
    cudaStream_t st = stream ? (cudaStream_t)stream : l.stream;
    CU(cudaStreamSynchronize(st));
    unsigned long long e;
    CU(cudaMemcpy(&e, l.d_err, sizeof(e), cudaMemcpyDeviceToHost));
    return decode_error(ctx, e);
}

// ------------------------------------------------------------------------------------------
// BGZF input: inflate on the device (inflate.cuh), then K0..K3 as usual
// ------------------------------------------------------------------------------------------
// The error word of an inflate launch: 0 when every block decoded, else the lowest failing block and its INF_* code
// (atomicMax over the word keeps the lowest block: blocks are counted down from INF_ERR_BLOCKS).
#define INF_ERR_BLOCKS 0x7FFFFF
__host__ __device__ inline int inf_err_word(int b, int rc) { return ((INF_ERR_BLOCKS - b) << 8) | rc; }
static std::string inf_err_message(int word) {
    return "BGZF inflate failed on the device (block " + std::to_string(INF_ERR_BLOCKS - (word >> 8)) + ", code " +
           std::to_string(word & 0xFF) + ")";
}

// block_rc: nullptr, or the INF_* code of every block (ugvc_test_device_inflate)
__global__ void __launch_bounds__(64) bgzf_inflate_blocks(const uint8_t* __restrict__ comp, const uint64_t* __restrict__ blk,
                                                          size_t cap_blk, int n_blocks, uint8_t* __restrict__ out,
                                                          const DefTables* __restrict__ dt, int* __restrict__ err,
                                                          int* __restrict__ block_rc) {
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < n_blocks; b += gridDim.x * blockDim.x) {
        const int rc = inf_block(comp + blk[b], (uint32_t)blk[cap_blk + b], out + blk[2 * cap_blk + b],
                                 (uint32_t)blk[3 * cap_blk + b], *dt);
        if (rc != INF_OK) atomicMax(err, inf_err_word(b, rc));
        if (block_rc) block_rc[b] = rc;
    }
}

#ifndef UGVC_HOST_EMU
#define INFW_WARPS 16
__global__ void __launch_bounds__(INFW_WARPS * 32) bgzf_inflate_warps(const uint8_t* __restrict__ comp, const uint64_t* __restrict__ blk,
                                                                      size_t cap_blk, int n_blocks, uint8_t* __restrict__ out,
                                                                      const DefTables* __restrict__ dt, int* __restrict__ err,
                                                                      int* __restrict__ block_rc) {
    extern __shared__ __align__(16) uint8_t infw_smem[];
    InfWarpTables& T = reinterpret_cast<InfWarpTables*>(infw_smem)[threadIdx.x >> 5];
    const int warp = (int)(blockIdx.x * INFW_WARPS + (threadIdx.x >> 5)), n_warps = (int)(gridDim.x * INFW_WARPS);
    for (int b = warp; b < n_blocks; b += n_warps) {
        const int rc = inf_block_warp(comp + blk[b], (uint32_t)blk[cap_blk + b], out + blk[2 * cap_blk + b],
                                      (uint32_t)blk[3 * cap_blk + b], T, *dt);
        if ((threadIdx.x & 31) == 0) {
            if (rc != INF_OK) atomicMax(err, inf_err_word(b, rc));
            if (block_rc) block_rc[b] = rc;
        }
        __syncwarp();
    }
}
#endif

// walk the BGZF block headers of host bytes: payload offset / size, output offset / size per block
static int scan_bgzf(ugvc_ctx* ctx, const uint8_t* p, size_t n, std::vector<uint64_t>& coff, std::vector<uint64_t>& clen,
                     std::vector<uint64_t>& uoff, std::vector<uint64_t>& ulen, size_t* total_out) {
    size_t at = 0, total = 0;
    while (at < n) {
        if (n - at < 18 + 8 || p[at] != 0x1f || p[at + 1] != 0x8b || p[at + 2] != 8 || !(p[at + 3] & 4))
            return fail(ctx, UGVC_E_IO, "not a BGZF block at byte " + std::to_string(at));
        const size_t xlen = p[at + 10] | ((size_t)p[at + 11] << 8);
        size_t bsize = 0, x = at + 12;
        const size_t xend = x + xlen;
        if (xend > n) return fail(ctx, UGVC_E_IO, "truncated BGZF header");
        while (x + 4 <= xend) {
            const size_t slen = p[x + 2] | ((size_t)p[x + 3] << 8);
            if (p[x] == 'B' && p[x + 1] == 'C' && slen == 2 && x + 6 <= xend) bsize = (p[x + 4] | ((size_t)p[x + 5] << 8)) + 1;
            x += 4 + slen;
        }
        if (bsize < 12 + xlen + 8 || at + bsize > n) return fail(ctx, UGVC_E_IO, "bad BGZF block size at byte " + std::to_string(at));
        const uint8_t* tail = p + at + bsize - 4;
        const size_t isize = tail[0] | ((size_t)tail[1] << 8) | ((size_t)tail[2] << 16) | ((size_t)tail[3] << 24);
        if (isize > 65536) return fail(ctx, UGVC_E_IO, "BGZF block larger than 64 KiB");
        if (isize) {  // the empty EOF block carries nothing
            coff.push_back(at + 12 + xlen);
            clen.push_back(bsize - 12 - xlen - 8);
            uoff.push_back(total);
            ulen.push_back(isize);
        }
        total += isize;
        at += bsize;
    }
    *total_out = total;
    return UGVC_OK;
}

// The CRC32 tables of the BGZF decoder and encoder (deflate.cuh), uploaded once per context
static int def_tables(ugvc_ctx* ctx) {
    static std::mutex tables_mu;  // lanes may take their first BGZF call on different host threads
    std::lock_guard<std::mutex> lock(tables_mu);
    if (!ctx->d_def_tables) {
        DefTables* t = new DefTables();
        def_build_tables(*t);
        CU(cudaMalloc(&ctx->d_def_tables, sizeof(DefTables)));
        const cudaError_t e = cudaMemcpy(ctx->d_def_tables, t, sizeof(DefTables), cudaMemcpyHostToDevice);
        delete t;
        CU(e);
    }
    return UGVC_OK;
}

enum { INF_DEC_WARP = 0, INF_DEC_THREAD = 1 };

// UGVC_INFLATE_THREADS=1: the thread-per-block decoder instead of the warp-per-block one (A/B)
static int inflate_decoder() {
    static const int dec = [] {
        const char* e = getenv("UGVC_INFLATE_THREADS");
        return e && *e != '0' ? INF_DEC_THREAD : INF_DEC_WARP;
    }();
    return dec;
}

// compressed bytes -> lane device buffers -> inflate into l.d_text with `decoder` (INF_DEC_*); *n_text = uncompressed
// size.  d_block_rc: nullptr, or room for the INF_* code of every block with ISIZE > 0.  The host emulation runs
// inf_block whatever the decoder.
static int stage_bgzf(ugvc_ctx* ctx, Lane& l, const uint8_t* bgzf, size_t n_bytes, int decoder, size_t* n_text,
                      size_t out_shift = 0, int* d_block_rc = nullptr) {
    std::vector<uint64_t> coff, clen, uoff, ulen;
    size_t total = 0;
    int rc = scan_bgzf(ctx, bgzf, n_bytes, coff, clen, uoff, ulen, &total);
    if (rc) return rc;
    if (total + out_shift > ctx->cap_bytes) return fail(ctx, UGVC_E_ARG, "bgzf: the inflated batch is larger than the reserved max_bytes");
    for (auto& u : uoff) u += out_shift;
    const size_t nb = coff.size();
    if (nb > INF_ERR_BLOCKS) return fail(ctx, UGVC_E_ARG, "bgzf: too many blocks in one call");
    rc = def_tables(ctx);
    if (rc) return rc;
    if (n_bytes + 8 > l.cap_comp) {
        cudaFree(l.d_comp);
        l.d_comp = nullptr;
        l.cap_comp = n_bytes + n_bytes / 4 + 4096;
        CU(cudaMalloc(&l.d_comp, l.cap_comp));
    }
    if (nb > l.cap_blk) {
        cudaFree(l.d_blk);
        l.d_blk = nullptr;
        l.cap_blk = nb + nb / 4 + 64;
        CU(cudaMalloc(&l.d_blk, 4 * l.cap_blk * sizeof(uint64_t)));
    }
    if (!l.d_inf_err) {
        CU(cudaMalloc(&l.d_inf_err, sizeof(int)));
        CU(cudaHostAlloc(&l.h_inf_err, sizeof(int), cudaHostAllocDefault));
        *l.h_inf_err = 0;
    }
    *n_text = total;
    cudaStream_t st = l.stream;
    CU(cudaMemsetAsync(l.d_inf_err, 0, sizeof(int), st));
    if (nb == 0) return UGVC_OK;
    l.h_blk.resize(4 * l.cap_blk);  // kept in the lane: the copy below is asynchronous
    for (size_t i = 0; i < nb; ++i) {
        l.h_blk[i] = coff[i];
        l.h_blk[l.cap_blk + i] = clen[i];
        l.h_blk[2 * l.cap_blk + i] = uoff[i];
        l.h_blk[3 * l.cap_blk + i] = ulen[i];
    }
    CU(cudaMemcpyAsync(l.d_comp, bgzf, n_bytes, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(l.d_blk, l.h_blk.data(), 4 * l.cap_blk * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
#ifdef UGVC_HOST_EMU
    (void)decoder;
    for (size_t i = 0; i < nb; ++i) {
        const int e = inf_block(l.d_comp + coff[i], (uint32_t)clen[i], l.d_text + uoff[i], (uint32_t)ulen[i], *ctx->d_def_tables);
        if (e != INF_OK && *l.d_inf_err < inf_err_word((int)i, e)) *l.d_inf_err = inf_err_word((int)i, e);
        if (d_block_rc) d_block_rc[i] = e;
    }
#else
    if (decoder == INF_DEC_THREAD) {
        const int threads = 64;
        int grid = (int)((nb + threads - 1) / threads);
        if (grid > ctx->sm_count * 16) grid = ctx->sm_count * 16;
        bgzf_inflate_blocks<<<grid, threads, 0, st>>>(l.d_comp, l.d_blk, l.cap_blk, (int)nb, l.d_text, ctx->d_def_tables,
                                                      l.d_inf_err, d_block_rc);
    } else {  // one warp per block, tables in shared memory
        const size_t smem = INFW_WARPS * sizeof(InfWarpTables);
        // per call: a function attribute belongs to the current device, and lanes are driven from several host threads
        CU(cudaFuncSetAttribute(bgzf_inflate_warps, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int grid = (int)((nb + INFW_WARPS - 1) / INFW_WARPS);
        if (grid > ctx->sm_count * 3) grid = ctx->sm_count * 3;
        bgzf_inflate_warps<<<grid, INFW_WARPS * 32, smem, st>>>(l.d_comp, l.d_blk, l.cap_blk, (int)nb, l.d_text,
                                                                 ctx->d_def_tables, l.d_inf_err, d_block_rc);
    }
    CU(cudaGetLastError());
#endif
    ctx->launches += 1;
    CU(cudaMemcpyAsync(l.h_inf_err, l.d_inf_err, sizeof(int), cudaMemcpyDeviceToHost, st));
    return UGVC_OK;
}

extern "C" int ugvc_submit_bgzf(ugvc_ctx* ctx, int lane, const uint8_t* bgzf, size_t n_bytes, double threshold) {
    if (!ctx) return UGVC_E_ARG;
    if (!ctx->has_plan || ctx->lanes.empty()) return fail(ctx, UGVC_E_STATE, "submit_bgzf: load a plan and reserve first");
    if (lane < 0 || lane >= (int)ctx->lanes.size()) return fail(ctx, UGVC_E_ARG, "submit_bgzf: lane out of range");
    if (n_bytes && !bgzf) return fail(ctx, UGVC_E_ARG, "submit_bgzf: NULL input");
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[lane];
    if (l.submitted) return fail(ctx, UGVC_E_STATE, "submit_bgzf: lane already has a batch in flight");
    size_t n_text = 0;
    int rc = stage_bgzf(ctx, l, bgzf, n_bytes, inflate_decoder(), &n_text);
    if (rc) return rc;
    CU(cudaMemsetAsync(l.d_text + n_text, '\n', TEXT_SLACK, l.stream));
    rc = enqueue_kernels(ctx, l, l.d_text, n_text, threshold, l.b.low_score, l.b.probs, l.b.qual, l.b.recinfo,
                         l.b.line_start, l.b.cap_records, l.b.n_records, l.stream);
    if (rc) return rc;
    CU(cudaMemcpyAsync(l.h_n, l.b.n_records, sizeof(int64_t), cudaMemcpyDeviceToHost, l.stream));
    CU(cudaMemcpyAsync(l.h_err, l.d_err, sizeof(unsigned long long), cudaMemcpyDeviceToHost, l.stream));
    l.n_bytes = n_text;
    l.submitted = true;
    return UGVC_OK;
}

extern "C" int ugvc_bgzf_inflate_device(ugvc_ctx* ctx, const uint8_t* bgzf, size_t n_bytes, uint8_t* out_host,
                                        size_t capacity, size_t* out_n) {
    if (!ctx) return UGVC_E_ARG;
    if (ctx->lanes.empty()) return fail(ctx, UGVC_E_STATE, "bgzf_inflate_device: reserve first (the text lands in lane 0)");
    if (n_bytes && !bgzf) return fail(ctx, UGVC_E_ARG, "bgzf_inflate_device: NULL input");
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[0];
    if (l.submitted) return fail(ctx, UGVC_E_STATE, "bgzf_inflate_device: lane 0 has a batch in flight");
    size_t n_text = 0;
    int rc = stage_bgzf(ctx, l, bgzf, n_bytes, inflate_decoder(), &n_text);
    if (rc) return rc;
    if (out_n) *out_n = n_text;
    CU(cudaStreamSynchronize(l.stream));
    if (l.h_inf_err && *l.h_inf_err) {
        const int code = *l.h_inf_err;
        *l.h_inf_err = 0;
        return fail(ctx, UGVC_E_IO, inf_err_message(code));
    }
    if (out_host) {
        if (n_text > capacity) return fail(ctx, UGVC_E_ARG, "bgzf_inflate_device: output capacity too small");
        CU(cudaMemcpy(out_host, l.d_text, n_text, cudaMemcpyDeviceToHost));
    }
    return UGVC_OK;
}

extern "C" int ugvc_test_device_inflate(ugvc_ctx* ctx, const uint8_t* bgzf, size_t n_bytes, int decoder, uint8_t* out,
                                        size_t capacity, size_t* out_n, int32_t* block_rc, size_t block_capacity,
                                        size_t* out_n_blocks) {
    // test hook: ugvc_bgzf_inflate_device with the decoder named, reporting the INF_* code of every block instead of
    // the lowest failing one
    if (!ctx || (n_bytes && !bgzf) || !out_n || !out_n_blocks || (decoder != INF_DEC_WARP && decoder != INF_DEC_THREAD))
        return UGVC_E_ARG;
#ifdef UGVC_HOST_EMU
    if (decoder == INF_DEC_WARP) return fail(ctx, UGVC_E_STATE, "the warp-per-block decoder is not part of the host emulation");
#endif
    if (ctx->lanes.empty()) return fail(ctx, UGVC_E_STATE, "test_device_inflate: reserve first (the text lands in lane 0)");
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[0];
    if (l.submitted) return fail(ctx, UGVC_E_STATE, "test_device_inflate: lane 0 has a batch in flight");
    std::vector<uint64_t> coff, clen, uoff, ulen;
    size_t n_text = 0;
    int rc = scan_bgzf(ctx, bgzf, n_bytes, coff, clen, uoff, ulen, &n_text);
    if (rc) return rc;
    const size_t nb = coff.size();
    if (nb > block_capacity || (nb && !block_rc)) return fail(ctx, UGVC_E_ARG, "test_device_inflate: more blocks than block_capacity");
    if (n_text > capacity || (n_text && !out)) return fail(ctx, UGVC_E_ARG, "test_device_inflate: output capacity too small");
    struct DevFree {
        int* p = nullptr;
        ~DevFree() { cudaFree(p); }
    } d_rc;
    CU(cudaMalloc(&d_rc.p, (nb ? nb : 1) * sizeof(int)));
    rc = stage_bgzf(ctx, l, bgzf, n_bytes, decoder, &n_text, 0, d_rc.p);
    if (rc) return rc;
    CU(cudaStreamSynchronize(l.stream));
    if (l.h_inf_err) *l.h_inf_err = 0;  // reported through block_rc
    if (nb) CU(cudaMemcpy(block_rc, d_rc.p, nb * sizeof(int), cudaMemcpyDeviceToHost));
    if (n_text) CU(cudaMemcpy(out, l.d_text, n_text, cudaMemcpyDeviceToHost));
    *out_n = n_text;
    *out_n_blocks = nb;
    return UGVC_OK;
}


// ------------------------------------------------------------------------------------------
// file to file on the device: inflate -> K1..K3 -> record writer -> deflate (fileio.cu)
// ------------------------------------------------------------------------------------------
#ifdef UGVC_HOST_EMU
extern "C" int ugvc_filter_bgzf(ugvc_ctx* ctx, int, const uint8_t*, size_t, uint32_t, uint64_t, double, int, uint8_t*, size_t, size_t*,
                                uint32_t*, size_t, size_t*, ugvc_recinfo*, int64_t*, uint8_t*, size_t, int64_t*) {
    return fail(ctx, UGVC_E_FALLBACK, "the device-side record writer is not part of the host emulation");
}
extern "C" int ugvc_filter_bgzf_stage_ms(ugvc_ctx*, int, float*) { return UGVC_E_STATE; }
extern "C" int ugvc_filter_bgzf_first_records(ugvc_ctx*, int, const uint64_t*, int, int64_t*) { return UGVC_E_STATE; }
extern "C" int ugvc_test_device_deflate(ugvc_ctx* ctx, const uint8_t*, size_t, int, uint8_t*, size_t, uint32_t*, size_t, size_t*,
                                        size_t*) {
    return fail(ctx, UGVC_E_STATE, "the device BGZF encoder is not part of the host emulation");
}
#else
static int file_bufs(ugvc_ctx* ctx, Lane& l) {
    Lane::FileBufs& f = l.fb;
    if (f.d_out_text) return UGVC_OK;
    const size_t cap_rec = l.b.cap_records;
    f.cap_out = ctx->cap_bytes + cap_rec * 64 + 4096;
    f.cap_blocks = f.cap_out / DEF_CHUNK + 2;
    CU(cudaMalloc(&f.d_out_text, f.cap_out + 64));
    CU(cudaMalloc(&f.d_len, (cap_rec + 1) * sizeof(int64_t)));
    CU(cudaMalloc(&f.d_out_ls, (cap_rec + 1) * sizeof(int64_t)));
    CU(cudaMalloc(&f.d_score, cap_rec * 16));
    size_t t1 = 0, t2 = 0;
    CU(fio_scan_i64(nullptr, t1, f.d_len, f.d_out_ls, (int64_t)cap_rec + 1, nullptr));
    CU(fio_scan_u64(nullptr, t2, nullptr, nullptr, (int)f.cap_blocks + 1, nullptr));
    f.scan_tmp_bytes = (t1 > t2 ? t1 : t2) + 256;
    CU(cudaMalloc(&f.d_scan_tmp, f.scan_tmp_bytes));
    CU(cudaMalloc(&f.d_blocks, f.cap_blocks * (size_t)DEF_BLOCK_STRIDE));
    CU(cudaMalloc(&f.d_bsize, (f.cap_blocks + 1) * sizeof(uint32_t)));
    CU(cudaMalloc(&f.d_bwide, (f.cap_blocks + 1) * sizeof(uint64_t)));
    CU(cudaMalloc(&f.d_boff, (f.cap_blocks + 1) * sizeof(uint64_t)));
    CU(cudaMalloc(&f.d_packed, f.cap_blocks * (size_t)DEF_BLOCK_STRIDE));
    CU(cudaMalloc(&f.d_fallback, sizeof(int)));
    CU(cudaHostAlloc(&f.h_fallback, sizeof(int), cudaHostAllocDefault));
    CU(cudaHostAlloc(&f.h_total, sizeof(int64_t), cudaHostAllocDefault));
    for (auto& e : f.ev) CU(cudaEventCreate(&e));
    return def_tables(ctx);
}

// UGVC_DEFLATE_THREADS=1: the thread-per-block encoder instead of the warp-per-block one (A/B)
static int deflate_encoder() {
    static const int enc = [] {
        const char* e = getenv("UGVC_DEFLATE_THREADS");
        return e && e[0] == '1' ? FIO_ENC_THREAD : FIO_ENC_WARP;
    }();
    return enc;
}

// The encoder of the file path: f.d_out_text[0, n_text) (16 zero bytes after it: the encoder reads whole words) ->
// n_blocks BGZF blocks (deflate), their sizes widened and scanned into offsets, the blocks packed back to back into
// f.d_packed.  The sizes stay in f.d_bsize.
static int encode_blocks(ugvc_ctx* ctx, Lane::FileBufs& f, size_t n_text, int n_blocks, int encoder, cudaStream_t st) {
    CU(cudaGetLastError());
    CU(fio_launch_deflate(f.d_out_text, n_text, ctx->d_def_tables, f.d_blocks, f.d_bsize, n_blocks, encoder, st));
    fio_launch_widen(f.d_bsize, f.d_bwide, n_blocks, st);
    CU(cudaGetLastError());
    CU(cudaMemsetAsync(f.d_bwide + n_blocks, 0, sizeof(uint64_t), st));
    size_t tmp = f.scan_tmp_bytes;
    CU(fio_scan_u64(f.d_scan_tmp, tmp, f.d_bwide, f.d_boff, n_blocks + 1, st));
    fio_launch_pack(f.d_blocks, f.d_bsize, f.d_bwide, f.d_boff, n_blocks, f.d_packed, ctx->sm_count, st);
    CU(cudaGetLastError());
    return UGVC_OK;
}

extern "C" int ugvc_filter_bgzf(ugvc_ctx* ctx, int lane, const uint8_t* bgzf, size_t n_bytes, uint32_t skip_head, uint64_t take_bytes,
                                double threshold, int flags, uint8_t* out_bgzf, size_t out_capacity, size_t* out_bytes,
                                uint32_t* out_block_csize, size_t block_capacity, size_t* out_n_blocks, ugvc_recinfo* out_recinfo,
                                int64_t* out_line_start, uint8_t* out_low_score, size_t capacity_records, int64_t* out_n_records) {
    if (!ctx) return UGVC_E_ARG;
    if (!ctx->has_plan || ctx->lanes.empty()) return fail(ctx, UGVC_E_STATE, "filter_bgzf: load a plan and reserve first");
    if (ctx->plan.h.model_kind == MODEL_NONE) return fail(ctx, UGVC_E_STATE, "filter_bgzf: the plan carries no model");
    if (lane < 0 || lane >= (int)ctx->lanes.size()) return fail(ctx, UGVC_E_ARG, "filter_bgzf: lane out of range");
    if (!bgzf || !n_bytes || !out_bgzf || !out_bytes || !out_n_records) return fail(ctx, UGVC_E_ARG, "filter_bgzf: NULL argument");
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[lane];
    if (l.submitted) return fail(ctx, UGVC_E_STATE, "filter_bgzf: lane already has a batch in flight");
    int rc = file_bufs(ctx, l);
    if (rc) return rc;
    Lane::FileBufs& f = l.fb;
    cudaStream_t st = l.stream;
    (void)cudaGetLastError();  // nothing stale from this host thread's earlier calls
    CU(cudaEventRecord(f.ev[0], st));
    // ---- compressed blocks -> text on the device, the range's first byte 16-byte aligned
    const size_t shift = (16 - (skip_head & 15u)) & 15u;
    size_t total = 0;
    rc = stage_bgzf(ctx, l, bgzf, n_bytes, inflate_decoder(), &total, shift);
    if (rc) return rc;
    if (skip_head > total) return fail(ctx, UGVC_E_ARG, "filter_bgzf: skip_head beyond the inflated blocks");
    const size_t n_text = take_bytes ? (size_t)take_bytes : total - skip_head;
    if (skip_head + n_text > total) return fail(ctx, UGVC_E_ARG, "filter_bgzf: the range is longer than the inflated blocks");
    const uint8_t* d_text = l.d_text + shift + skip_head;
    CU(cudaEventRecord(f.ev[1], st));
    // ---- K1..K3
    rc = enqueue_kernels(ctx, l, d_text, n_text, threshold, l.b.low_score, l.b.probs, l.b.qual, l.b.recinfo, l.b.line_start,
                         l.b.cap_records, l.b.n_records, st);
    if (rc) return rc;
    CU(cudaMemcpyAsync(l.h_n, l.b.n_records, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(l.h_err, l.d_err, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(f.ev[2], st));
    CU(cudaStreamSynchronize(st));
    if (l.h_inf_err && *l.h_inf_err) {
        const int code = *l.h_inf_err;
        *l.h_inf_err = 0;
        return fail(ctx, UGVC_E_IO, inf_err_message(code));
    }
    rc = decode_error(ctx, *l.h_err);
    if (rc) return rc;
    const int64_t n = *l.h_n;
    l.last_n = n;
    *out_n_records = n;
    if ((size_t)n > capacity_records) return fail(ctx, UGVC_E_ARG, "filter_bgzf: output capacity smaller than the record count");
    // ---- record writer
    CU(cudaMemsetAsync(f.d_fallback, 0, sizeof(int), st));
    CU(cudaMemsetAsync(f.d_len + n, 0, sizeof(int64_t), st));
    fio_launch_splice_len(d_text, l.b.line_start, l.b.recinfo, l.b.low_score, l.b.qual, n, flags, f.d_len, f.d_score, f.d_fallback,
                          ctx->sm_count, st);
    size_t tmp = f.scan_tmp_bytes;
    CU(fio_scan_i64(f.d_scan_tmp, tmp, f.d_len, f.d_out_ls, n + 1, st));
    CU(cudaMemcpyAsync(f.h_total, f.d_out_ls + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(f.h_fallback, f.d_fallback, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (*f.h_fallback) return UGVC_E_FALLBACK;
    const size_t out_text = (size_t)*f.h_total;
    if (out_text > f.cap_out) return fail(ctx, UGVC_E_ARG, "filter_bgzf: the edited text exceeds the writer's buffer");
    fio_launch_splice_copy(d_text, l.b.line_start, l.b.recinfo, l.b.low_score, n, flags, f.d_out_ls, f.d_score, f.d_out_text,
                           f.d_fallback, ctx->sm_count, st);
    CU(cudaMemsetAsync(f.d_out_text + out_text, 0, 16, st));  // the encoder reads whole words
    CU(cudaMemcpyAsync(f.h_fallback, f.d_fallback, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(f.ev[3], st));
    // ---- deflate, pack
    const int n_blocks = (int)((out_text + DEF_CHUNK - 1) / DEF_CHUNK);
    if ((size_t)n_blocks > f.cap_blocks || (out_block_csize && (size_t)n_blocks > block_capacity))
        return fail(ctx, UGVC_E_ARG, "filter_bgzf: more output blocks than room for them");
    rc = encode_blocks(ctx, f, out_text, n_blocks, deflate_encoder(), st);
    if (rc) return rc;
    f.h_bsize.resize((size_t)n_blocks + 1);
    if (n_blocks) CU(cudaMemcpyAsync(f.h_bsize.data(), f.d_bsize, (size_t)n_blocks * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(f.ev[4], st));
    CU(cudaStreamSynchronize(st));
    if (*f.h_fallback) return UGVC_E_FALLBACK;
    size_t packed = 0;
    for (int b = 0; b < n_blocks; ++b) packed += f.h_bsize[b];
    if (packed > out_capacity)  // the caller sized out_bgzf for text that compresses; it can take its host writer instead
        return fail(ctx, UGVC_E_FALLBACK, "filter_bgzf: out_capacity smaller than the compressed output");
    ctx->launches += 6;
    // ---- results to the host
    if (packed) CU(cudaMemcpyAsync(out_bgzf, f.d_packed, packed, cudaMemcpyDeviceToHost, st));
    if (out_block_csize && n_blocks) memcpy(out_block_csize, f.h_bsize.data(), (size_t)n_blocks * sizeof(uint32_t));
    if (out_recinfo && n) CU(cudaMemcpyAsync(out_recinfo, l.b.recinfo, (size_t)n * sizeof(ugvc_recinfo), cudaMemcpyDeviceToHost, st));
    if (out_line_start) CU(cudaMemcpyAsync(out_line_start, f.d_out_ls, (size_t)(n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    if (out_low_score && n) CU(cudaMemcpyAsync(out_low_score, l.b.low_score, (size_t)n, cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(f.ev[5], st));
    CU(cudaStreamSynchronize(st));
    *out_bytes = packed;
    if (out_n_blocks) *out_n_blocks = (size_t)n_blocks;
    for (int k = 0; k < 5; ++k) cudaEventElapsedTime(&f.ms[k], f.ev[k], f.ev[k + 1]);
    return UGVC_OK;
}

extern "C" int ugvc_filter_bgzf_stage_ms(ugvc_ctx* ctx, int lane, float out_ms[5]) {
    if (!ctx || !out_ms || lane < 0 || lane >= (int)ctx->lanes.size()) return UGVC_E_ARG;
    for (int k = 0; k < 5; ++k) out_ms[k] = ctx->lanes[lane].fb.ms[k];
    return UGVC_OK;
}

extern "C" int ugvc_filter_bgzf_first_records(ugvc_ctx* ctx, int lane, const uint64_t* text_offsets, int n, int64_t* out_first_record) {
    if (!ctx || lane < 0 || lane >= (int)ctx->lanes.size() || n < 0 || (n && (!text_offsets || !out_first_record))) return UGVC_E_ARG;
    Lane& l = ctx->lanes[lane];
    if (!l.fb.d_out_text || l.last_n < 0) return fail(ctx, UGVC_E_STATE, "filter_bgzf_first_records: no ugvc_filter_bgzf call on this lane yet");
    if (n == 0) return UGVC_OK;
    if ((size_t)n * 16 > l.fb.scan_tmp_bytes) return fail(ctx, UGVC_E_ARG, "filter_bgzf_first_records: too many offsets");
    CU(cudaSetDevice(ctx->device));
    uint64_t* d_off = reinterpret_cast<uint64_t*>(l.fb.d_scan_tmp);
    int64_t* d_out = reinterpret_cast<int64_t*>(d_off + n);
    CU(cudaMemcpyAsync(d_off, text_offsets, (size_t)n * sizeof(uint64_t), cudaMemcpyHostToDevice, l.stream));
    fio_launch_first_records(l.b.line_start, l.last_n, d_off, n, d_out, l.stream);
    CU(cudaMemcpyAsync(out_first_record, d_out, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost, l.stream));
    CU(cudaStreamSynchronize(l.stream));
    return UGVC_OK;
}

extern "C" int ugvc_test_device_deflate(ugvc_ctx* ctx, const uint8_t* data, size_t n, int encoder, uint8_t* out, size_t capacity,
                                        uint32_t* out_block_csize, size_t block_capacity, size_t* out_bytes, size_t* out_n_blocks) {
    // test hook: the file path's encoder (encode_blocks) on the caller's bytes, staged in lane 0's writer buffer the way
    // ugvc_filter_bgzf stages the edited text
    if (!ctx || (n && !data) || !out_bytes || !out_n_blocks || (encoder != FIO_ENC_WARP && encoder != FIO_ENC_THREAD))
        return UGVC_E_ARG;
    if (ctx->lanes.empty()) return fail(ctx, UGVC_E_STATE, "test_device_deflate: reserve first (the bytes go to lane 0)");
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[0];
    if (l.submitted) return fail(ctx, UGVC_E_STATE, "test_device_deflate: lane 0 has a batch in flight");
    int rc = file_bufs(ctx, l);
    if (rc) return rc;
    Lane::FileBufs& f = l.fb;
    if (n > f.cap_out) return fail(ctx, UGVC_E_ARG, "test_device_deflate: more bytes than the writer's buffer holds");
    const int n_blocks = (int)((n + DEF_CHUNK - 1) / DEF_CHUNK);
    if ((size_t)n_blocks > block_capacity || (n_blocks && !out_block_csize))
        return fail(ctx, UGVC_E_ARG, "test_device_deflate: more output blocks than room for them");
    cudaStream_t st = l.stream;
    (void)cudaGetLastError();
    if (n) CU(cudaMemcpyAsync(f.d_out_text, data, n, cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(f.d_out_text + n, 0, 16, st));
    rc = encode_blocks(ctx, f, n, n_blocks, encoder, st);
    if (rc) return rc;
    f.h_bsize.resize((size_t)n_blocks + 1);
    if (n_blocks) CU(cudaMemcpyAsync(f.h_bsize.data(), f.d_bsize, (size_t)n_blocks * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    size_t packed = 0;
    for (int b = 0; b < n_blocks; ++b) packed += f.h_bsize[b];
    if (packed > capacity || (packed && !out)) return fail(ctx, UGVC_E_ARG, "test_device_deflate: capacity smaller than the compressed output");
    if (packed) CU(cudaMemcpyAsync(out, f.d_packed, packed, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (n_blocks) memcpy(out_block_csize, f.h_bsize.data(), (size_t)n_blocks * sizeof(uint32_t));
    *out_bytes = packed;
    *out_n_blocks = (size_t)n_blocks;
    return UGVC_OK;
}
#endif  // !UGVC_HOST_EMU

// K3 alone on a dense feature matrix assembled by the caller (row-major, n x n_features, leading
// dimension ld): the model-apply step of variant_filtering_utils.apply_model / the other model-apply
// tools, without the VCF front end.  Features are staged feature-major in lane 0's K3 input buffer.
extern "C" int ugvc_predict_features(ugvc_ctx* ctx, const float* x, size_t n, size_t ld, double threshold,
                                     uint8_t* out_low_score, float* out_probs, double* out_qual) {
    if (!ctx) return UGVC_E_ARG;
    if (!ctx->has_plan || ctx->lanes.empty()) return fail(ctx, UGVC_E_STATE, "predict_features: load a plan and reserve first");
    const DevPlan& p = ctx->plan;
    const size_t F = p.h.n_features;
    if (p.h.model_kind == MODEL_NONE || F == 0) return fail(ctx, UGVC_E_STATE, "predict_features: the plan carries no model");
    if ((n && !x) || ld < F) return fail(ctx, UGVC_E_ARG, "predict_features: bad matrix arguments");
    if (n > ctx->cap_records) return fail(ctx, UGVC_E_ARG, "predict_features: more rows than the reserved max_records");
    Lane& l = ctx->lanes[0];
    if (l.submitted) return fail(ctx, UGVC_E_STATE, "predict_features: lane 0 has a batch in flight");
    CU(cudaSetDevice(ctx->device));
    l.last_n = (int64_t)n;
    if (n == 0) return UGVC_OK;
    // feature-major staging copy; +-inf is refused like the reference's estimators do ("Input X contains NaN /
    // infinity"), NaN too unless the model is xgboost's: there it is a missing value that K3 sends to the default child
    const bool nan_ok = p.h.model_kind == MODEL_XGB;
    std::vector<float> cols(F * n);
    for (size_t r0 = 0; r0 < n; r0 += 256) {
        const size_t r1 = r0 + 256 < n ? r0 + 256 : n;
        for (size_t f = 0; f < F; ++f)
            for (size_t r = r0; r < r1; ++r) {
                const float v = x[r * ld + f];
                if (!(v - v == 0.0f) && !(nan_ok && v != v)) {  // +-inf, or NaN where it is not a missing value
                    ctx->err_record = (int64_t)r;
                    ctx->err_column = (int32_t)f;
                    ctx->err_reason = REASON_NULL_FEATURE;
                    return fail(ctx, UGVC_E_DATA, "predict_features: non-finite value at row " + std::to_string(r) +
                                                      ", column " + std::to_string(f));
                }
                cols[f * n + r] = v;
            }
    }
    cudaStream_t st = l.stream;
    CU(cudaMemcpy2DAsync(l.b.feats, l.b.cap_records * sizeof(float), cols.data(), n * sizeof(float), n * sizeof(float), F,
                         cudaMemcpyHostToDevice, st));
    const int64_t n64 = (int64_t)n;
    CU(cudaMemcpyAsync(l.b.n_records, &n64, sizeof(n64), cudaMemcpyHostToDevice, st));
    launch_k3(p, ctx->k3, nullptr, l.b.feats, l.b.cap_records, l.b.n_records, threshold, l.b.low_score, l.b.probs, l.b.qual,
              l.b.phreds, ctx->want_phreds, ctx->d_counts, l.d_err, st);
    ctx->launches += 1;
    CU(cudaGetLastError());
    if (out_low_score) CU(cudaMemcpyAsync(out_low_score, l.b.low_score, n, cudaMemcpyDeviceToHost, st));
    if (out_probs) CU(cudaMemcpyAsync(out_probs, l.b.probs, n * p.h.n_classes * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (out_qual) CU(cudaMemcpyAsync(out_qual, l.b.qual, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));  // also keeps `cols` and n64 alive until the copies are done
    return UGVC_OK;
}

extern "C" int ugvc_enable_phreds(ugvc_ctx* ctx, int on) {
    // takes effect at the next ugvc_reserve
    if (!ctx) return UGVC_E_ARG;
    if (on < 0 || on > 2) return fail(ctx, UGVC_E_ARG, "enable_phreds: mode must be 0, 1 or 2");
    ctx->want_phreds = on;
    return UGVC_OK;
}

extern "C" int ugvc_collect_phreds(ugvc_ctx* ctx, int lane, double* out, size_t capacity_records) {
    if (!ctx || !out || lane < 0 || lane >= (int)ctx->lanes.size()) return UGVC_E_ARG;
    Lane& l = ctx->lanes[lane];
    if (!l.b.phreds) return fail(ctx, UGVC_E_STATE, "collect_phreds: call ugvc_enable_phreds before ugvc_reserve");
    if ((size_t)l.last_n > capacity_records) return fail(ctx, UGVC_E_ARG, "collect_phreds: capacity too small");
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(l.stream));
    if (l.last_n)
        CU(cudaMemcpy(out, l.b.phreds, (size_t)l.last_n * ctx->plan.h.n_classes * sizeof(double), cudaMemcpyDeviceToHost));
    return UGVC_OK;
}

extern "C" int ugvc_counts_reset(ugvc_ctx* ctx) {
    if (!ctx) return UGVC_E_ARG;
    CU(cudaSetDevice(ctx->device));
    CU(cudaDeviceSynchronize());
    CU(cudaMemset(ctx->d_counts, 0, 4 * sizeof(long long)));
    return UGVC_OK;
}

extern "C" int ugvc_counts_get(ugvc_ctx* ctx, ugvc_counts* out) {
    if (!ctx || !out) return UGVC_E_ARG;
    CU(cudaSetDevice(ctx->device));
    CU(cudaDeviceSynchronize());
    long long c[4];
    CU(cudaMemcpy(c, ctx->d_counts, sizeof(c), cudaMemcpyDeviceToHost));
    out->n_records = c[0];
    out->n_low_score = c[1];
    out->n_pass = c[2];
    out->n_cg = c[3];
    return UGVC_OK;
}

extern "C" int ugvc_counts_device_ptr(ugvc_ctx* ctx, int64_t** d_counts) {
    if (!ctx || !d_counts) return UGVC_E_ARG;
    *d_counts = reinterpret_cast<int64_t*>(ctx->d_counts);
    return UGVC_OK;
}

extern "C" int ugvc_debug_raw(ugvc_ctx* ctx, int lane, uint32_t* out, size_t capacity_words) {
    if (!ctx || lane < 0 || lane >= (int)ctx->lanes.size()) return UGVC_E_ARG;
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[lane];
    const size_t n = (size_t)l.last_n, S = ctx->plan.h.n_slots;
    if (capacity_words < n * S) return fail(ctx, UGVC_E_ARG, "debug_raw: capacity too small");
    CU(cudaStreamSynchronize(l.stream));
    if (n) CU(cudaMemcpy2D(out, n * 4, l.b.raw, l.b.cap_records * 4, n * 4, S, cudaMemcpyDeviceToHost));
    return UGVC_OK;
}

extern "C" int ugvc_debug_features(ugvc_ctx* ctx, int lane, float* out, size_t capacity_floats) {
    if (!ctx || lane < 0 || lane >= (int)ctx->lanes.size()) return UGVC_E_ARG;
    CU(cudaSetDevice(ctx->device));
    Lane& l = ctx->lanes[lane];
    const size_t n = (size_t)l.last_n, F = ctx->plan.h.n_features;
    if (capacity_floats < n * F) return fail(ctx, UGVC_E_ARG, "debug_features: capacity too small");
    CU(cudaStreamSynchronize(l.stream));
    if (n && F) {
        // the product path assembles features inside the inference kernel; this diagnostic runs the stand-alone
        // assembly kernel (same k2_apply) on the lane's raw slots, into the lane's feature buffer
        unsigned long long* d_scratch_err = nullptr;
        CU(cudaMalloc(&d_scratch_err, sizeof(unsigned long long)));
        CU(cudaMemset(d_scratch_err, 0xFF, sizeof(unsigned long long)));
        launch_k2(ctx->plan, l.b.raw, l.b.cap_records, l.b.n_records, l.b.feats, d_scratch_err, ctx->sm_count, l.stream);
        CU(cudaStreamSynchronize(l.stream));
        cudaFree(d_scratch_err);
    }
    if (n) CU(cudaMemcpy2D(out, n * 4, l.b.feats, l.b.cap_records * 4, n * 4, F, cudaMemcpyDeviceToHost));
    return UGVC_OK;
}

extern "C" int ugvc_last_data_error(const ugvc_ctx* ctx, int64_t* record, int32_t* column, int32_t* reason) {
    if (!ctx) return UGVC_E_ARG;
    if (record) *record = ctx->err_record;
    if (column) *column = ctx->err_column;
    if (reason) *reason = ctx->err_reason;
    return UGVC_OK;
}

extern "C" int64_t ugvc_debug_slow_records(ugvc_ctx* ctx, int lane) {
    // records of the lane's last batch that the tile kernel handed to the generic parser (blocking)
    if (!ctx || lane < 0 || lane >= (int)ctx->lanes.size()) return UGVC_E_ARG;
    Lane& l = ctx->lanes[lane];
    if (cudaSetDevice(ctx->device) != cudaSuccess || cudaStreamSynchronize(l.stream) != cudaSuccess) return UGVC_E_CUDA;
    uint32_t w[2] = {0, 0};
    if (cudaMemcpy(w, l.b.chunk_first, sizeof(w), cudaMemcpyDeviceToHost) != cudaSuccess) return UGVC_E_CUDA;
    return ctx->fast.enabled ? (int64_t)w[1] : -1;
}

#ifndef UGVC_HOST_EMU
void launch_test_sigmoid(const float* d_m, int n, float* d_p1, float* d_e, cudaStream_t st);
extern "C" int ugvc_test_device_sigmoid(ugvc_ctx* ctx, const float* margins, int n, float* out_p1, float* out_e) {
    // test hook: K3's fp32 sigmoid (xgboost flavour) on the device, for comparison with the restatement
    if (!ctx || !margins || !out_p1 || !out_e || n <= 0) return UGVC_E_ARG;
    CU(cudaSetDevice(ctx->device));
    float *d_m = nullptr, *d_p = nullptr, *d_e = nullptr;
    CU(cudaMalloc(&d_m, n * sizeof(float)));
    CU(cudaMalloc(&d_p, n * sizeof(float)));
    CU(cudaMalloc(&d_e, n * sizeof(float)));
    CU(cudaMemcpy(d_m, margins, n * sizeof(float), cudaMemcpyHostToDevice));
    launch_test_sigmoid(d_m, n, d_p, d_e, nullptr);
    CU(cudaMemcpy(out_p1, d_p, n * sizeof(float), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(out_e, d_e, n * sizeof(float), cudaMemcpyDeviceToHost));
    cudaFree(d_m);
    cudaFree(d_p);
    cudaFree(d_e);
    return UGVC_OK;
}
extern "C" int ugvc_test_format_g(ugvc_ctx* ctx, const float* v, int64_t n, uint8_t* out) {
    // test hook: the record writer's "%g" (fileio.cu: fio_format_g) on the device, for comparison with a correctly
    // rounded formatter; 16 bytes per value as splice_len stores them
    if (!ctx || !v || !out || n <= 0) return UGVC_E_ARG;
    CU(cudaSetDevice(ctx->device));
    float* d_v = nullptr;
    uint8_t* d_out = nullptr;
    CU(cudaMalloc(&d_v, (size_t)n * sizeof(float)));
    CU(cudaMalloc(&d_out, (size_t)n * 16));
    CU(cudaMemcpy(d_v, v, (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
    fio_launch_test_format_g(d_v, n, d_out, ctx->sm_count, nullptr);
    CU(cudaGetLastError());
    CU(cudaMemcpy(out, d_out, (size_t)n * 16, cudaMemcpyDeviceToHost));
    cudaFree(d_v);
    cudaFree(d_out);
    return UGVC_OK;
}
#else
extern "C" int ugvc_test_device_sigmoid(ugvc_ctx*, const float*, int, float*, float*) { return UGVC_E_CUDA; }
extern "C" int ugvc_test_format_g(ugvc_ctx*, const float*, int64_t, uint8_t*) { return UGVC_E_CUDA; }
#endif

extern "C" int ugvc_test_k3_config(ugvc_ctx* ctx, int32_t out[9]) {
    // test hook: the K3 launch the loaded plan gets
    if (!ctx || !out) return UGVC_E_ARG;
    if (!ctx->has_plan || ctx->plan.h.model_kind == MODEL_NONE)
        return fail(ctx, UGVC_E_STATE, "test_k3_config: load a plan with a model first");
    const K3Config& c = ctx->k3;
    const int32_t v[9] = {c.kernel, c.tpb, c.nbuf, c.groups, c.nch, (int32_t)c.chunk, c.resident ? 1 : 0, c.grid, c.walk};
    memcpy(out, v, sizeof(v));
    return UGVC_OK;
}

extern "C" int64_t ugvc_launch_count(const ugvc_ctx* ctx) { return ctx ? ctx->launches : 0; }

extern "C" int ugvc_enable_stage_timing(ugvc_ctx* ctx, int on) {
    if (!ctx) return UGVC_E_ARG;
    ctx->timing = on != 0;
    for (auto& l : ctx->lanes) l.ev_used = 0;  // (re)start accumulation
    return UGVC_OK;
}

extern "C" int ugvc_stage_ms(ugvc_ctx* ctx, float out_ms[4], int64_t* out_n_calls) {
    // Sum of the device-side durations of K0..K3 over every enqueue since
    // ugvc_enable_stage_timing(ctx, 1); blocks until those enqueues finished.
    if (!ctx || !out_ms) return UGVC_E_ARG;
    CU(cudaSetDevice(ctx->device));
    CU(cudaDeviceSynchronize());
    double sum[4] = {0, 0, 0, 0};
    int64_t calls = 0;
    for (auto& l : ctx->lanes) {
        for (size_t i = 0; i + 5 <= l.ev_used; i += 5) {
            for (int k = 0; k < 4; ++k) {
                float ms = 0.f;
                CU(cudaEventElapsedTime(&ms, l.ev_pool[i + k], l.ev_pool[i + k + 1]));
                sum[k] += ms;
            }
            ++calls;
        }
    }
    for (int k = 0; k < 4; ++k) out_ms[k] = (float)sum[k];
    if (out_n_calls) *out_n_calls = calls;
    return UGVC_OK;
}

extern "C" int ugvc_bind_thread(ugvc_ctx* ctx) {
    // make the context's device current on the calling host thread (helper threads that allocate pinned memory)
    if (!ctx) return UGVC_E_ARG;
    CU(cudaSetDevice(ctx->device));
    return UGVC_OK;
}

extern "C" int ugvc_host_alloc(void** out, size_t n_bytes) {
    // pinned host memory for the host-buffer API (H2D/D2H at full PCIe rate)
    ugvc_ctx* ctx = nullptr;
    if (!out) return UGVC_E_ARG;
    CU(cudaHostAlloc(out, n_bytes, cudaHostAllocDefault));
    return UGVC_OK;
}

extern "C" int ugvc_host_free(void* p) {
    ugvc_ctx* ctx = nullptr;
    CU(cudaFreeHost(p));
    return UGVC_OK;
}

// used by synth_kernel.cu
int ugvc_ctx_device(const ugvc_ctx* ctx) { return ctx->device; }
int ugvc_ctx_sm_count(const ugvc_ctx* ctx) { return ctx->sm_count; }
void ugvc_ctx_count_launches(ugvc_ctx* ctx, int n) { ctx->launches += n; }
cudaStream_t ugvc_ctx_default_stream(ugvc_ctx* ctx) { return ctx->lanes.empty() ? nullptr : ctx->lanes[0].stream; }
int ugvc_ctx_fail(ugvc_ctx* ctx, int code, const char* msg) { return fail(ctx, code, msg); }
