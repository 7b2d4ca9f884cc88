/*
 * ugvc_b200.h -- C ABI of the H100-native (sm_90a) filter_variants_pipeline hot path.
 *
 * The reference (Ultimagen/VariantCalling, 100 % Python) has no FFI for this
 * path; its boundary is the CLI, the model pickle and the Python functions
 * below.  Each entry point here replaces the native work behind one of them and
 * is what a ctypes / cgo / JNI stub binds (see INTEGRATION.md).  All pointers
 * are plain host or device pointers; no torch / C++ types cross the boundary.
 *
 * Reference interfaces replaced (paths under ugbio_utils/src/):
 *   get_vcf_df            core/ugbio_core/vcfbed/vcftools.py:16-217      -> K0 + K1 (line index, field parse)
 *   transformer.transform filtering/ugbio_filtering/transformers.py:144-369
 *                         (called at variant_filtering_utils.py:116-121)   -> K2 (feature assembly)
 *   model.predict_proba   filtering/ugbio_filtering/variant_filtering_utils.py:123-124
 *   score math + decision filtering/ugbio_filtering/filter_variants_pipeline.py:170-195
 *                         core/ugbio_core/math_utils.py:28-44              -> K3 (inference + phred/qual/FILTER)
 *   record writer         filtering/ugbio_filtering/filter_variants_pipeline.py:188-228
 *                         (+ htslib BGZF / `bcftools index -t` at :115,:231) -> ugvc_bgzf_* / ugvc_splice_*
 *
 * Conventions: every function returns 0 on success or a negative UGVC_E_* code;
 * ugvc_last_error() gives the message.  The caller owns all host buffers; the
 * context owns device memory and streams.  One context per GPU; a context is
 * not thread-safe, different contexts are independent.
 */
#ifndef UGVC_B200_H
#define UGVC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UGVC_OK 0
#define UGVC_E_CUDA (-1)      /* CUDA runtime error (no device, launch failure, ...) */
#define UGVC_E_ARG (-2)       /* bad argument / capacity exceeded */
#define UGVC_E_PLAN (-3)      /* malformed or unsupported plan blob */
#define UGVC_E_DATA (-4)      /* the reference would raise on this input (null feature, unknown category, ...) */
#define UGVC_E_IO (-5)        /* file / BGZF error */
#define UGVC_E_STATE (-6)     /* call order (no plan loaded, nothing submitted, ...) */

typedef struct ugvc_ctx ugvc_ctx;

/* Per-record writer support emitted by K1 (16 bytes, one 128-bit store).
 * Offsets are relative to the start of the record's line; 0xFFFF = saturated
 * (line longer than 64 KiB: the host re-scans that line). */
typedef struct ugvc_recinfo {
    int32_t pos;          /* 1-based POS */
    uint16_t qual_off;    /* offset of the QUAL column */
    uint16_t filter_off;  /* offset of the FILTER column */
    uint16_t info_off;    /* offset of the INFO column */
    uint16_t format_off;  /* offset one past the tab after INFO (== line length + 1 when there is no FORMAT column) */
    uint32_t flags;       /* bit0: an allele equals GGC or CCG (blacklist_cg_insertions, blacklist.py:85-101);
                             bits 1..7: number of alleles (saturating at 127), for --recalibrate_genotype;
                             bits 8..31: length of REF (saturating), for the tabix index of the output */
} ugvc_recinfo;

/* Counters of one batch / one run (what the single NCCL all-reduce sums). */
typedef struct ugvc_counts {
    int64_t n_records;
    int64_t n_low_score;  /* records with quals <= threshold (filter_variants_pipeline.py:192) */
    int64_t n_pass;       /* n_records - n_low_score */
    int64_t n_cg;         /* records flagged by the CG-insertion rule */
} ugvc_counts;

/* ---- lifetime ---------------------------------------------------------- */
int ugvc_init(int device, ugvc_ctx** out);
void ugvc_free(ugvc_ctx* ctx);
const char* ugvc_last_error(const ugvc_ctx* ctx); /* ctx may be NULL: error of a failed ugvc_init */
int ugvc_version(void);

/* Load the compiled plan: tag table built from the VCF header (Number/Type per
 * INFO/FORMAT tag, replaces pysam's typed decode at vcftools.py:63-89), the
 * fitted transformer lowered to slot/feature ops (transformers.py:221-344) and
 * the model (sklearn LR / GB / RF natively, xgboost via its JSON dump;
 * variant_filtering_utils.py:70-89).  Layout: variantcalling_b200/csrc/plan.h. */
int ugvc_load_plan(ugvc_ctx* ctx, const void* blob, size_t n_bytes);
int ugvc_plan_info(const ugvc_ctx* ctx, int32_t* n_features, int32_t* n_classes, int32_t* n_slots);

/* Optional: the order in which records carry their INFO keys (';'-separated key names, a
 * trailing '!' marks a key that appears without a value) and the usual FORMAT column (e.g.
 * "GT:AD:DP:GQ:PL"), learned by the host from the first records of the file.  K1 then steps
 * through that order warp-uniformly; records that deviate fall back to the generic key lookup,
 * results are identical either way.  NULL / "" clears.  Belongs to the loaded plan. */
int ugvc_set_key_order(ugvc_ctx* ctx, const char* info_keys, const char* format_keys);

/* Size the context's device workspace: n_pipeline independent batch lanes, each
 * for up to max_bytes of VCF text and max_records records. */
int ugvc_reserve(ugvc_ctx* ctx, size_t max_bytes, size_t max_records, int n_pipeline);

/* ---- the hot path: host buffers in, host buffers out -------------------- */
/* One batch of whole VCF data lines (no header lines; must end with '\n').
 * Copies the text to the device, runs K0..K3, copies results back, blocks.
 * out_low_score[i] = 1 iff quals[i] <= threshold; out_probs is N x n_classes
 * fp32 row-major; out_qual is the fp64 TREE_SCORE; out_recinfo may be NULL. */
int ugvc_filter_batch(ugvc_ctx* ctx, const uint8_t* vcf_text, size_t n_bytes, double threshold,
                      uint8_t* out_low_score, float* out_probs, double* out_qual,
                      ugvc_recinfo* out_recinfo, int64_t* out_line_start,
                      size_t capacity_records, int64_t* out_n_records);

/* Pipelined form of the same call: submit on lane `lane` (0 <= lane <
 * n_pipeline), collect later; copies and kernels of different lanes overlap. */
int ugvc_submit_batch(ugvc_ctx* ctx, int lane, const uint8_t* vcf_text, size_t n_bytes, double threshold);
int ugvc_collect_batch(ugvc_ctx* ctx, int lane, uint8_t* out_low_score, float* out_probs, double* out_qual,
                       ugvc_recinfo* out_recinfo, int64_t* out_line_start,
                       size_t capacity_records, int64_t* out_n_records);

/* ---- the hot path: device-resident text (bench `value`, multi-GPU shards) - */
/* d_* are device pointers sized for capacity_records (d_recinfo / d_line_start
 * may be NULL -> context scratch).  Runs on `stream` (a cudaStream_t, NULL =
 * the context's lane-0 stream) without any host synchronisation; the record
 * count lands in *d_n_records (device int64).  d_text must be 16-byte aligned (K0 streams the
 * text with 16-byte loads), hold whole lines ending with '\n', and have at least 16 readable
 * bytes after n_bytes (K1 reads aligned 8-byte words one word ahead of its cursor). */
int ugvc_filter_device(ugvc_ctx* ctx, const uint8_t* d_text, size_t n_bytes, double threshold,
                       uint8_t* d_low_score, float* d_probs, double* d_qual, ugvc_recinfo* d_recinfo,
                       int64_t* d_line_start, size_t capacity_records, int64_t* d_n_records, void* stream);

/* The same call on lane `lane` (0 <= lane < n_pipeline of ugvc_reserve): every lane has its own scratch (raw slots,
 * line index, error word), so device-resident batches submitted on different lanes and streams may overlap;
 * ugvc_filter_device is lane 0.  ugvc_device_status_lane reports the lane's data errors (blocking). */
int ugvc_filter_device_lane(ugvc_ctx* ctx, int lane, const uint8_t* d_text, size_t n_bytes, double threshold,
                            uint8_t* d_low_score, float* d_probs, double* d_qual, ugvc_recinfo* d_recinfo,
                            int64_t* d_line_start, size_t capacity_records, int64_t* d_n_records, void* stream);
int ugvc_device_status_lane(ugvc_ctx* ctx, int lane, void* stream);

/* BGZF input, inflated on the device (csrc/inflate.cuh): the host ships the compressed bytes, so the
 * PCIe traffic of the end-to-end path shrinks by the compression ratio (htslib's BGZF reader behind
 * pysam.VariantFile, filter_variants_pipeline.py:106,115).  `bgzf` = consecutive whole BGZF blocks in
 * host memory whose uncompressed bytes are whole VCF data lines (<= the max_bytes of ugvc_reserve).
 * ugvc_submit_bgzf is ugvc_submit_batch for such input (results through ugvc_collect_batch as usual);
 * ugvc_bgzf_inflate_device only inflates into lane 0's text buffer and optionally copies the text
 * back (out_host may be NULL).  A block is refused (UGVC_E_IO, the message names the lowest such block) when its
 * DEFLATE stream is one zlib refuses or does not end inside the payload, when it inflates to other than ISIZE bytes,
 * or when their CRC32 differs from the footer's -- htslib's rule. */
int ugvc_submit_bgzf(ugvc_ctx* ctx, int lane, const uint8_t* bgzf, size_t n_bytes, double threshold);
int ugvc_bgzf_inflate_device(ugvc_ctx* ctx, const uint8_t* bgzf, size_t n_bytes, uint8_t* out_host, size_t capacity,
                             size_t* out_n);

/* The model-apply step alone (variant_filtering_utils.py:95-125 after the transform; the other
 * model-apply tools' predict_proba): K3 on a dense row-major float32 matrix x[n][ld] whose first
 * n_features columns are the features of a plan compiled with model_compiler.compile_plan_model_only
 * (or any plan with a model).  n <= the max_records of ugvc_reserve; outputs may be NULL; with
 * ugvc_enable_phreds(ctx, 2) the fp64 class probabilities are fetched with ugvc_collect_phreds(ctx, 0, ...).
 * An infinite input value is UGVC_E_DATA, and so is NaN unless the plan's model is xgboost (the reference's sklearn
 * estimators raise on it).  For an xgboost model NaN is a missing value: every node sends it to its default child
 * (default_left), as xgboost's predictor does; the row and column of a refused value come from ugvc_last_data_error. */
int ugvc_predict_features(ugvc_ctx* ctx, const float* x, size_t n, size_t ld, double threshold,
                          uint8_t* out_low_score, float* out_probs, double* out_qual);

/* --recalibrate_genotype (filter_variants_pipeline.py:203-215): ask K3 to keep the per-class
 * phreds -10*log10(p + 1e-10) of the host-buffer lanes (takes effect at the next ugvc_reserve)
 * and fetch them (N x n_classes fp64) after ugvc_collect_batch.  on = 2 keeps the fp64 class
 * likelihoods themselves instead (--treat_multiallelics merges the likelihoods of split rows on
 * the host before the phred step, variant_filtering_utils.py:346-408). */
int ugvc_enable_phreds(ugvc_ctx* ctx, int on);
int ugvc_collect_phreds(ugvc_ctx* ctx, int lane, double* out, size_t capacity_records);

/* Blocking: waits for `stream` and surfaces a data error (UGVC_E_DATA) of the last
 * ugvc_filter_device call. */
int ugvc_device_status(ugvc_ctx* ctx, void* stream);

/* Make the context's device current on the calling host thread (a helper thread that is about to allocate pinned
 * memory with ugvc_host_alloc: the allocation belongs to the current device's context). */
int ugvc_bind_thread(ugvc_ctx* ctx);
/* Pinned host memory for the host-buffer API (full-rate PCIe copies). */
int ugvc_host_alloc(void** out, size_t n_bytes);
int ugvc_host_free(void* p);

/* Counters accumulated since the last reset (device-side, summed over batches). */
int ugvc_counts_reset(ugvc_ctx* ctx);
int ugvc_counts_get(ugvc_ctx* ctx, ugvc_counts* out);
/* Device address of the int64[4] counter block {n_records, n_low_score, n_pass,
 * n_cg}: this is the buffer the one NCCL all-reduce of the path sums in place
 * (the host passes it to torch.distributed / ncclAllReduce). */
int ugvc_counts_device_ptr(ugvc_ctx* ctx, int64_t** d_counts);
/* The single collective of the path (SURVEY.md 8b/8e; the reference's only precedent for combining shards is
 * `bcftools concat` of per-contig parts, ugbio_core/vcfbed/variant_annotation.py:96-110): NCCL sum all-reduce of
 * that block, in place, on `stream` (NULL: the context's lane-0 stream after a device synchronise).  `nccl_comm`
 * is an ncclComm_t of this rank -- the host's own, or one made by ugvc_nccl_comm_init (rank 0 draws the 128-byte
 * id with ugvc_nccl_unique_id and hands it to the other ranks by whatever channel it has).  out_counts (may be
 * NULL) receives the reduced counters; then the call blocks until the collective is done.  NCCL is bound at run
 * time (the process's own libnccl if one is loaded, else libnccl.so.2): UGVC_E_STATE when there is none. */
#define UGVC_NCCL_ID_BYTES 128
int ugvc_nccl_unique_id(uint8_t id[UGVC_NCCL_ID_BYTES]);
int ugvc_nccl_comm_init(ugvc_ctx* ctx, const uint8_t id[UGVC_NCCL_ID_BYTES], int world_size, int rank, void** out_comm);
int ugvc_nccl_comm_destroy(void* nccl_comm);
int ugvc_counts_allreduce(ugvc_ctx* ctx, void* nccl_comm, int64_t out_counts[4], void* stream);

/* ---- introspection for the parity tests --------------------------------- */
/* Raw slot columns (K1 output, n_slots x n_records fp32 bit patterns) and the
 * feature matrix (K2 output, n_features x n_records fp32, column-major) of the
 * last batch on `lane`. */
int ugvc_debug_raw(ugvc_ctx* ctx, int lane, uint32_t* out, size_t capacity_words);
int ugvc_debug_features(ugvc_ctx* ctx, int lane, float* out, size_t capacity_floats);
/* Error detail of the last UGVC_E_DATA: record index within the batch, feature
 * column (or -1) and a reason code. */
int ugvc_last_data_error(const ugvc_ctx* ctx, int64_t* record, int32_t* column, int32_t* reason);

/* Records of the last batch on `lane` that K1's tile kernel handed to the generic per-record parser
 * (unknown INFO key, unusual literal or FORMAT column ...); -1 when the tile kernel is switched off
 * (UGVC_K1_LEGACY=1).  Blocking; a diagnostic, the results do not depend on it. */
int64_t ugvc_debug_slow_records(ugvc_ctx* ctx, int lane);
/* Number of kernel launches issued by this context since ugvc_init. */
int64_t ugvc_launch_count(const ugvc_ctx* ctx);
/* Stage timing: while enabled every enqueue brackets K0,K1,K2,K3 with CUDA events on
 * the launching stream; ugvc_stage_ms blocks and returns the summed device time (ms) of
 * each stage over all enqueues since ugvc_enable_stage_timing(ctx, 1), and their count. */
int ugvc_enable_stage_timing(ugvc_ctx* ctx, int on);
int ugvc_stage_ms(ugvc_ctx* ctx, float out_ms[4], int64_t* out_n_calls);

/* ---- synthetic input (bench / tests) ------------------------------------ */
/* Generate `n_records` synthetic single-sample VCF data lines (SURVEY.md 8d
 * schema, n_custom custom annotations) for global record indices
 * [first_record, first_record + n_records) of a job of total_records, straight
 * into device memory.  Returns bytes written in *out_bytes. */
int ugvc_synth_device(ugvc_ctx* ctx, uint64_t seed, int64_t first_record, int64_t n_records,
                      int64_t total_records, int n_custom, uint8_t* d_text, size_t capacity_bytes,
                      size_t* out_bytes, void* stream);
/* The matching header text (host). Returns its length, or negative on error. */
int64_t ugvc_synth_header(int n_custom, char* out, size_t capacity);

/* ---- container formats either side of the path (host, multi-threaded) ---- */
/* Inflate a whole BGZF file (or a virtual-offset range) into `out`; returns
 * bytes produced in *out_bytes.  Replaces htslib's reader behind
 * pysam.VariantFile (filter_variants_pipeline.py:106,117). */
int ugvc_bgzf_inflate_file(const char* path, uint64_t voff_begin, uint64_t voff_end, uint8_t* out,
                           size_t capacity, size_t* out_bytes, int n_threads);
int64_t ugvc_bgzf_uncompressed_size(const char* path);
/* The blocks that hold the virtual-offset range [voff_begin, voff_end) of a BGZF file: their compressed byte range
 * [c_begin, c_end), the bytes of the first block before the range and the range's uncompressed length -- the
 * arguments of ugvc_filter_bgzf for one contig of a tabix-indexed call set. */
int ugvc_bgzf_range_info(const char* path, uint64_t voff_begin, uint64_t voff_end, uint64_t* c_begin, uint64_t* c_end,
                         uint32_t* skip_head, uint64_t* take_bytes);
/* Per-contig summary of a tabix index (`data`: the inflated .tbi): out_lo / out_hi = smallest chunk begin / largest chunk
 * end over the contig's bins (~0 / 0 when it has none), out_linear_offset / out_linear_count = where its linear index
 * (uint64 virtual offsets) sits in `data`; the contig names are the NUL-separated bytes at out_names_offset.  What
 * pysam's fetch(contig) (filter_variants_pipeline.py:130) gets from htslib's index loader. */
int ugvc_tbi_summary(const uint8_t* data, size_t n, int32_t n_ref_capacity, uint64_t* out_lo, uint64_t* out_hi,
                     int64_t* out_linear_offset, int32_t* out_linear_count, int32_t* out_n_ref, int64_t* out_names_offset,
                     int32_t* out_names_bytes);
/* Append `n_bytes` as BGZF blocks to `path` (mode 'w' truncates, 'a' appends;
 * write_eof != 0 adds the 28-byte EOF block).  Every block but the last holds
 * 0xff00 bytes of input; out_block_csize (may be NULL) receives the compressed
 * size of each block so the caller can build the tabix index that the reference
 * obtains from `bcftools index -t` (filter_variants_pipeline.py:231).  Replaces
 * htslib's writer (filter_variants_pipeline.py:115,228). */
int ugvc_bgzf_deflate_to_file(const char* path, const char* mode, const uint8_t* data, size_t n_bytes,
                              int level, int write_eof, int n_threads, uint64_t* out_compressed_bytes,
                              uint32_t* out_block_csize, size_t block_capacity, size_t* out_n_blocks);
/* Number of bytes equal to `byte` in data[0, n) (the record count of inflated VCF text), threaded. */
int64_t ugvc_count_byte(const uint8_t* data, size_t n, int byte, int n_threads);
/* INFO/END of every record of a batch (0 where there is none): the end of a record's tabix interval when it lies beyond
 * POS, as htslib takes it for the index `bcftools index -t` writes (filter_variants_pipeline.py:231).  line_start /
 * recinfo are the batch's outputs of ugvc_filter_batch.  Returns the number of records that carry the tag. */
int64_t ugvc_info_end(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo, int64_t n_records,
                      int64_t* out_end, int n_threads);
/* Build the edited output text of a batch: for each record copy the original
 * line with FILTER rewritten (PASS removed / LOW_SCORE appended / empty -> PASS)
 * and TREE_SCORE (and optionally QUAL, BLACKLST) spliced in, exactly the rules of
 * filter_variants_pipeline.py:188-228.  blacklist_code (may be NULL) selects,
 * per record, one ';'-joined annotation string of blacklist_table (string c is
 * bytes [table_off[c], table_off[c+1])) as the BLACKLST value.  phreds != NULL selects the
 * --recalibrate_genotype rules instead of TREE_SCORE (:203-215): GQ = int(2nd smallest - smallest
 * phred), PL = int(phreds[:n_genotypes]), GT = genotype of the smallest PL, QUAL = GQ (float) when
 * overwrite_qual, all on the first sample.  out_line_start (may be
 * NULL, n_records + 1 entries) receives the offset of every output line.
 * Returns bytes written. */
int64_t ugvc_splice_records(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo,
                            const uint8_t* low_score, const double* qual, int64_t n_records,
                            int overwrite_qual, int with_model, const int32_t* blacklist_code,
                            const char* blacklist_table, const int64_t* blacklist_table_off,
                            const double* phreds, int n_classes,
                            uint8_t* out, size_t capacity, int64_t* out_line_start, int n_threads);

/* ---- file to file on the device: compressed bytes in, compressed bytes out ---------------------------------
 * One range of whole VCF data lines (a contig of an indexed call set) per call: `bgzf` = the consecutive BGZF blocks
 * that hold it (host memory), `skip_head` = bytes of the first block before the range (the low 16 bits of the tabix
 * virtual offset), `take_bytes` = uncompressed bytes of the range (0: to the end of the blocks).  The blocks are
 * inflated on the device, the records filtered and scored (K1..K3 with the loaded plan), the edited records --
 * FILTER (LOW_SCORE / PASS rules), INFO ";TREE_SCORE=<%g>", with UGVC_FILE_BLACKLIST_CG ";BLACKLST=CG_NON_HMER_INDEL"
 * on flagged records, with UGVC_FILE_OVERWRITE_QUAL the QUAL column (filter_variants_pipeline.py:188-228) -- are
 * written and BGZF-compressed there too: out_bgzf receives complete BGZF blocks of 57344 uncompressed bytes each (the
 * last one shorter), no EOF block.  For the tabix index of the output (the reference runs `bcftools index -t`,
 * filter_variants_pipeline.py:231): out_block_csize[b] = compressed size of block b, out_line_start[i] =
 * uncompressed offset of record i in this call's output (n + 1 entries), out_recinfo[i].pos / flags >> 8 = POS and
 * len(REF).  Returns UGVC_E_FALLBACK (nothing written) when a record needs the general writer of ugvc_splice_records
 * (an INFO column that is ".", has empty pieces or already carries TREE_SCORE / BLACKLST; a score that prints in
 * exponent form; a line longer than 64 KiB): the caller then takes the host-buffer path for this range.
 * Needs a plan with a model and ugvc_reserve() sized for the range.  Replaces htslib's reader / writer either side
 * of the path (filter_variants_pipeline.py:106,115,228). */
#define UGVC_E_FALLBACK (-7)
#define UGVC_FILE_OVERWRITE_QUAL 1
#define UGVC_FILE_BLACKLIST_CG 2
int ugvc_filter_bgzf(ugvc_ctx* ctx, int lane, const uint8_t* bgzf, size_t n_bytes, uint32_t skip_head, uint64_t take_bytes,
                     double threshold, int flags, uint8_t* out_bgzf, size_t out_capacity, size_t* out_bytes,
                     uint32_t* out_block_csize, size_t block_capacity, size_t* out_n_blocks, ugvc_recinfo* out_recinfo,
                     int64_t* out_line_start, uint8_t* out_low_score, size_t capacity_records, int64_t* out_n_records);
/* ugvc_filter_bgzf with the rest of the tool's record edits (ugvc_filter_bgzf is this call with with_model = 1 and
 * everything else zero; --treat_multiallelics runs through ugvc_filter_bgzf_split, which writes the same way):
 *   with_model = 0     a model-less plan (FILTER keeps its non-empty pieces, PASS when none is left; no TREE_SCORE;
 *                      QUAL untouched; out_low_score all 0)
 *   recalibrate_genotype  --recalibrate_genotype (filter_variants_pipeline.py:203-215): GQ = int(second smallest -
 *                      smallest phred), PL = int() of the first min(n_classes, n_alleles (n_alleles + 1) / 2) phreds,
 *                      GT = genotype of the first smallest PL ('|' when the input GT is phased), on the first sample only,
 *                      missing keys appended in the order GQ, PL, GT; no TREE_SCORE; UGVC_FILE_OVERWRITE_QUAL writes
 *                      %g of the GQ difference to QUAL.  Needs a model and ugvc_enable_phreds(ctx, 1) before ugvc_reserve.
 *   blacklists         Blacklist.apply with selection_fcn = ALL for the range's contig: blacklist k is the sorted POS
 *                      array blacklist_pos[blacklist_pos_off[k], blacklist_pos_off[k + 1]) and the annotation
 *                      blacklist_names[blacklist_name_off[k], ..[k + 1]).  INFO gets BLACKLST= and the non-PASS
 *                      annotations of the record joined with ',', the CG flag (UGVC_FILE_BLACKLIST_CG) first, then the
 *                      blacklists in order.  At most UGVC_MAX_BLACKLISTS blacklists, UGVC_MAX_BLACKLIST_POSITIONS
 *                      positions and UGVC_MAX_BLACKLIST_NAME_BYTES of annotations a call (UGVC_E_ARG beyond).
 *   out_end            (may be NULL; capacity_records entries) INFO/END of every record, 0 where there is none: the
 *                      rule of ugvc_info_end, read while the INFO column is copied.
 *   n_blacklisted      (out) records with at least one annotation, CG included.
 * UGVC_E_FALLBACK as for ugvc_filter_bgzf, and also for a recalibrated record whose phreds are not finite or whose int()
 * leaves int32 (or a model with fewer than two classes), for a GQ that %g prints in exponent form under
 * UGVC_FILE_OVERWRITE_QUAL, and for edited text that outgrows the writer's buffer (long annotations).  Output bytes
 * equal ugvc_splice_records' on the same records. */
#define UGVC_MAX_BLACKLISTS 31
#define UGVC_MAX_BLACKLIST_POSITIONS (1ll << 28)
#define UGVC_MAX_BLACKLIST_NAME_BYTES 4096
typedef struct ugvc_file_edits {
    int with_model;
    int recalibrate_genotype;
    int n_blacklists;
    const int64_t* blacklist_pos;
    const int64_t* blacklist_pos_off;   /* n_blacklists + 1 entries, from 0 */
    const char* blacklist_names;
    const int64_t* blacklist_name_off;  /* n_blacklists + 1 entries, from 0 */
    int64_t* out_end;
    int64_t n_blacklisted;
} ugvc_file_edits;
int ugvc_filter_bgzf_edits(ugvc_ctx* ctx, int lane, const uint8_t* bgzf, size_t n_bytes, uint32_t skip_head, uint64_t take_bytes,
                           double threshold, int flags, ugvc_file_edits* edits, uint8_t* out_bgzf, size_t out_capacity,
                           size_t* out_bytes, uint32_t* out_block_csize, size_t block_capacity, size_t* out_n_blocks,
                           ugvc_recinfo* out_recinfo, int64_t* out_line_start, uint8_t* out_low_score, size_t capacity_records,
                           int64_t* out_n_records);
/* Test hook: the record writer of ugvc_filter_bgzf_edits alone, on the caller's records (text, line_start and recinfo as
 * ugvc_filter_batch returns them), scores (low_score / qual, with_model) and phreds ([n][n_classes],
 * recalibrate_genotype), staged in lane 0.  Returns the bytes of the edited text written to out (out_line_start: n + 1
 * entries; edits->out_end filled when given), UGVC_E_FALLBACK when the device writer hands the records back. */
int64_t ugvc_test_write_records(ugvc_ctx* ctx, const uint8_t* text, size_t n_bytes, const int64_t* line_start,
                                const ugvc_recinfo* recinfo, int64_t n, const uint8_t* low_score, const double* qual,
                                const double* phreds, int n_classes, int flags, ugvc_file_edits* edits, uint8_t* out,
                                size_t capacity, int64_t* out_line_start);
/* Stage seconds of the last ugvc_filter_bgzf call on `lane`: H2D + inflate, K1..K3, record writer, deflate + pack,
 * D2H (device-timed with CUDA events). */
int ugvc_filter_bgzf_stage_ms(ugvc_ctx* ctx, int lane, float out_ms[5]);
/* After ugvc_filter_bgzf on `lane`: for each of `n` byte offsets into the range's text (0 = its first byte), the index of the
 * first record that starts at or after it.  A caller that hands several contigs to one call (adjacent in the file) gives
 * the offsets where each contig's text begins and gets back where its records begin: what the per-contig tabix
 * bookkeeping of the writer (filter_variants_pipeline.py:231, `bcftools index -t`) needs. */
int ugvc_filter_bgzf_first_records(ugvc_ctx* ctx, int lane, const uint64_t* text_offsets, int n, int64_t* out_first_record);

/* ---- concordance metrics (BASELINE configs[4]: evaluate_concordance on the filtered set) ----
 * Precision / recall of calls against truth labels, per variant group, replacing the array work
 * of ugbio_core/concordance/concordance_utils.py:11-188,346-458 and stats_utils.py:141-210 (which
 * wraps sklearn.metrics.precision_recall_curve).  Group g: 0..6 = the selection functions of
 * concordance_utils.py:266-275 in order (SNP, Non-hmer INDEL, HMER indel <= 4, (4,8), [8,10],
 * 11,12, > 12), 7 = INDELS, 8 = H-INDELS.  Per record: scores (tree_score, fp64), pred (1 when
 * the final FILTER is PASS), cls (0 fp, 1 tp, 2 fn, 3 tn: the classify / classify_gt column), indel,
 * hmer_len (hmer_indel_length, < 0 for null), group (NULL = derive from indel / hmer_len, else the
 * caller's group id per record, -1 = none).  Inputs are host arrays, or device arrays when
 * inputs_on_device != 0.  A group id outside -1..6 or a cls code above 3 anywhere in the input makes the
 * call return UGVC_E_ARG with every output zero.
 *   out_counts[g][8]   = tp, fp, missed (call < truth), initial_tp, n_called (not fn), n_fn,
 *                        n_nan, n_inf (called records whose score is NaN / +-inf: where sklearn's
 *                        assert_all_finite raises, the Python mirror raises; the curve is still drawn)
 *   out_curve_len[g]   = points of the raw precision/recall curve kept on the device (0 for g = 8)
 *   out_cutoff[g]      = the 20th largest score of the group (stats_utils.py:202-207)
 *   out_selected[g][2] = number of called records, number of true ones among them
 * ugvc_conc_curve copies group g's raw curve: precision = tps/(tps+fps), recall = tps/tps[-1] at each
 * distinct score, in increasing-threshold order (sklearn's order, without its final (1, 0) point).  The
 * threshold of a run of equal scores is its first score in input order, so a run of -0.0 and +0.0 reports
 * the sign of its first zero (scikit-learn 1.5, the reference's pin). */
#define UGVC_CONC_GROUPS 9
#define UGVC_CONC_COUNTERS 8
typedef struct ugvc_conc ugvc_conc;
int ugvc_conc_create(int device, ugvc_conc** out);
void ugvc_conc_free(ugvc_conc* h);
const char* ugvc_conc_last_error(const ugvc_conc* h);
long long ugvc_conc_launch_count(const ugvc_conc* h);
int ugvc_conc_run(ugvc_conc* h, int64_t n, const double* scores, const uint8_t* pred, const uint8_t* cls,
                  const uint8_t* indel, const int32_t* hmer_len, const int8_t* group, int inputs_on_device,
                  int want_curves, int64_t* out_counts, int64_t* out_curve_len, double* out_cutoff,
                  int64_t* out_selected);
/* The per-record rules that produce the `classify` / `classify_gt` columns the metrics consume (vcf2concordance,
 * ugbio_comparison/comparison_utils.py:153-229): gt_ultima / gt_truth hold two int8 per record (allele index, -1 for
 * None, -2 when the genotype tuple has a single element), base_fn (may be NULL) is 1 where vcfeval's BASE is FN or
 * FN_CA.  Outputs: 0 = tp, 1 = fp, 2 = fn. */
int ugvc_conc_classify(ugvc_conc* h, int64_t n, const int8_t* gt_ultima, const int8_t* gt_truth, const uint8_t* base_fn,
                       uint8_t* out_classify, uint8_t* out_classify_gt);
int ugvc_conc_curve(ugvc_conc* h, int group, double* precision, double* recall, double* thresholds,
                    size_t capacity);
/* Annotation of a concordance frame (comparison_utils.annotate_concordance, ugbio_comparison/comparison_utils.py:
 * 321-380; DESIGN.md 4b).  Contigs are uploaded once and stay on the handle: ugvc_conc_annot_add_contig copies one
 * contig's raw FASTA bytes (case kept) and returns its id; ugvc_conc_annot_clear drops them all.
 * ugvc_conc_annotate: per record the contig id (-1 = not in the FASTA), 1-based pos, indel (0/1), REF as bytes at
 * ref_bytes[ref_off[i] .. ref_off[i+1]), and the alleles k in [rec_allele_off[i], rec_allele_off[i+1]) at
 * allele_bytes[allele_off[k] .. allele_off[k+1]) (every record has at least one allele).  flow_order is a NUL-terminated
 * string, or NULL for no cycle-skip column.  Outputs, per record: class (0 None, 1 ins, 2 del), indel length, hmer indel
 * length and base (0 = None), the upper-cased motifs (motif_size bytes per record, zero-padded, lengths apart), the GC fraction
 * (fp64) and the cycle-skip code (0 NA, 1 cycle-skip, 2 possible-cycle-skip, 3 non-skip).  Where the reference raises,
 * the call returns UGVC_E_DATA and ugvc_conc_annot_error gives the record it raises at and a UGVC_ANNOT_E_* reason. */
#define UGVC_ANNOT_E_INDEX 1          /* IndexError: an insertion whose alleles all equal REF */
#define UGVC_ANNOT_E_KEY 2            /* KeyError: the record's contig is not in the FASTA */
#define UGVC_ANNOT_E_ZERO_DIVISION 3  /* ZeroDivisionError: an empty GC window */
int ugvc_conc_annot_add_contig(ugvc_conc* h, const uint8_t* seq, int64_t len, int32_t* out_id);
int ugvc_conc_annot_clear(ugvc_conc* h);
int ugvc_conc_annotate(ugvc_conc* h, int64_t n, const int32_t* contig, const int64_t* pos, const uint8_t* indel,
                       const uint8_t* ref_bytes, const int64_t* ref_off, const uint8_t* allele_bytes,
                       const int64_t* allele_off, const int64_t* rec_allele_off, const char* flow_order, int motif_size,
                       int gc_window, int8_t* out_class, int32_t* out_indel_len, int32_t* out_hmer_len,
                       uint8_t* out_hmer_nuc, uint8_t* out_left, uint8_t* out_right, uint8_t* out_left_len,
                       uint8_t* out_right_len, double* out_gc, int8_t* out_cycleskip);
int ugvc_conc_annot_error(const ugvc_conc* h, int64_t* row, int* reason);
/* CUDA-event time in ms of the kernel of the last ugvc_conc_annotate call (uploads and downloads excluded). */
double ugvc_conc_annot_kernel_ms(const ugvc_conc* h);

/* ---- --treat_multiallelics on the device (SURVEY.md 8 row f2) -------------
 * Replaces, per contig, the frame surgery of training_prep.process_multiallelic_spandel
 * (ugbio_filtering/training_prep.py:226-287: select_overlapping_variants multiallelics.py:13-62,
 * split_multiallelic_variants :65-127, split_multiallelic_variants_with_spandel spandel.py:11-63,
 * extract_allele_subset_from_multiallelic(_spanning_deletion) multiallelics.py:130-177 / spandel.py:66-128,
 * classify_hmer_indel_relative :385-465, cleanup_multiallelics :503-559) and the merge of
 * variant_filtering_utils.combine_multiallelic_spandel / merge_and_assign_pls (:309-408).
 *   ugvc_ma_set_rules  per-tag rules derived from the VCF header by the host (variantcalling_b200/multiallelics.py:
 *                      rules_blob): how the values of every loaded per-allele tag are sub-sampled
 *   ugvc_ma_build      host text of one contig + line_start / recinfo of the index pass (ugvc_filter_batch with the
 *                      model-less plan) + the contig's reference sequence -> groups, split rows, scored text.
 *                      out[0..6] = n_singles, n_cluster_records, n_kept_records, n_split_rows, kept_bytes,
 *                      rows_bytes, entries of the widest two-row group's genotype vector.
 *                      UGVC_E_DATA: the reference raises on a group (ugvc_ma_data_error: group index in processing
 *                      order -- multi-allelic singles first, then cluster records -- and the reason code:
 *                      1 AssertionError (GT without the selected alleles), 2 / 3 RuntimeError (Number=G / Number=n tag),
 *                      4 RuntimeError ('*' without its deletion), 5 ValueError (flow key of a non-ACGT sequence),
 *                      6 IndexError, 7 TypeError, 8 ValueError (not an integer), 9 limits, 10 IndexError (2-class merge))
 *   ugvc_ma_fetch      the text of the scored pass (untouched lines in input order, then the split rows: singles,
 *                      then clusters -- the row order of the reference's frame) and the group table
 *   ugvc_ma_merge      fp64 class likelihoods of the scored pass (row-major n_kept + n_split_rows by n_classes) ->
 *                      out[n_records][width] in input record order, zero padded, width = max(n_classes, out[6])
 * One handle per GPU and host thread (not thread-safe per handle); it keeps its device buffers from contig to contig. */
typedef struct ugvc_ma ugvc_ma;
int ugvc_ma_create(int device, ugvc_ma** out);
void ugvc_ma_free(ugvc_ma* h);
const char* ugvc_ma_last_error(const ugvc_ma* h);
long long ugvc_ma_launch_count(const ugvc_ma* h);
int ugvc_ma_set_rules(ugvc_ma* h, const void* blob, size_t n_bytes);
int ugvc_ma_build(ugvc_ma* h, const uint8_t* text, size_t n_bytes, const int64_t* line_start, const ugvc_recinfo* recinfo,
                  int64_t n_records, const uint8_t* ref_seq, size_t ref_len, int64_t out[8]);
int ugvc_ma_data_error(const ugvc_ma* h, int64_t* group, int32_t* code);
int ugvc_ma_fetch(ugvc_ma* h, uint8_t* out_text, size_t capacity, int32_t* out_origin, uint8_t* out_n_rows,
                  uint8_t* out_n_alleles, size_t capacity_groups);
int ugvc_ma_merge(ugvc_ma* h, const double* lik, int64_t n_rows, int n_classes, double* out, int width);
/* --treat_multiallelics on the file path: ugvc_filter_bgzf_edits for one whole contig a call (overlap clusters must not
 * be cut), with the split branch between the inflate and the record writer, every stage on `lane`'s stream and device
 * pointers: the blocks are inflated (skip_head / take_bytes as for ugvc_filter_bgzf), indexed by K1 of the model-less
 * plan of `index_ctx` (its lane `lane` keeps the line starts / recinfo), split by `ma` (ugvc_ma_build on the device text,
 * ref_seq = the contig's reference sequence, host memory), the scored pass (K1..K3 of ctx, fp64 likelihoods) runs on
 * the split text, ugvc_ma_merge folds the likelihoods into N x W (W = max(n_classes, widest group)), and the score
 * math of filter_variants_pipeline.py:174-180,192 runs on the device (phreds = -10 log10(lik + 1e-10) over all W
 * columns, qual = max(30 + ph0 - min(ph[1:]), 0), LOW_SCORE = qual <= threshold; exactly 100 where lik + 1e-10 rounds
 * to 1e-10).  The records of the original text are then written with those scores (recalibrate_genotype: PL / GQ / GT
 * from the W phreds) and BGZF-compressed; the outputs are those of ugvc_filter_bgzf_edits (edits->with_model must be 1).
 * out_split[0..6] = out[0..6] of ugvc_ma_build; out_split[7] = 0, or with UGVC_E_DATA where the reference raises:
 * 1 = the split build (a group, see ugvc_ma_data_error, or a contig without multi-allelic sites (out_split[0] = 0) or
 * without deletion clusters (out_split[1] = 0)), 2 = the merge (a 2-class model).  UGVC_E_DATA with out_split[7] = 0
 * is a data error of K1 (ugvc_last_data_error).  UGVC_E_FALLBACK (nothing written) where ugvc_filter_bgzf_edits falls
 * back, and for a contig beyond the path's limits: text of 4 GiB or more, or larger than the reserved lanes of ctx /
 * index_ctx.  Needs ugvc_enable_phreds(ctx, 2) before ugvc_reserve, and ctx, index_ctx and ma on one device. */
int ugvc_filter_bgzf_split(ugvc_ctx* ctx, ugvc_ctx* index_ctx, ugvc_ma* ma, int lane, const uint8_t* bgzf, size_t n_bytes,
                           uint32_t skip_head, uint64_t take_bytes, const uint8_t* ref_seq, size_t ref_len, double threshold, int flags,
                           ugvc_file_edits* edits, uint8_t* out_bgzf, size_t out_capacity, size_t* out_bytes, uint32_t* out_block_csize,
                           size_t block_capacity, size_t* out_n_blocks, ugvc_recinfo* out_recinfo, int64_t* out_line_start,
                           uint8_t* out_low_score, size_t capacity_records, int64_t* out_n_records, int64_t out_split[8]);
/* Stage times of the last ugvc_filter_bgzf_split call on `lane`, ms between CUDA events on its stream: H2D + inflate,
 * index K1, split build, scored K1..K3, merge + score, record writer, deflate + pack, D2H.  The split build and the
 * merge wait on the stream for their counts, so their stages include that host round trip. */
int ugvc_filter_bgzf_split_stage_ms(ugvc_ctx* ctx, int lane, float out_ms[8]);
/* Test hook: the score kernel of ugvc_filter_bgzf_split (ma_score) on n caller rows of `width` (>= 2) likelihoods:
 * out_phreds[n][width], out_qual[n], out_low[n]. */
int ugvc_test_ma_score(ugvc_ctx* ctx, const double* lik, int64_t n, int width, double threshold, double* out_phreds,
                       double* out_qual, uint8_t* out_low);

/* ---- filter_low_af_ratio_to_background on the device (DESIGN.md 4c) -------
 * Replaces ugbio_filtering/filter_low_af_ratio_to_background.py:35-65 and process_record (:75-114): per record, unless
 * FILTER holds RefCall, the AF-ratio rule over every sample (GT / VAF / BG_VAF typed by the header as pysam does) and the
 * FILTER edit of pysam's record.filter.clear() / add() (htslib bcf_add_filter): new_filter is removed from the list, and
 * added back when the rule fails the record.  Every byte outside FILTER is kept as read.
 *   variant_type_kind  1: INFO/VARIANT_TYPE is declared Number=1 String/Character (compared with "h-indel"); 0: never equal
 *   vaf_kind / bg_vaf_kind  UGVC_AFR_KIND_*; *_integer: Type=Integer (else Float) */
#define UGVC_AFR_KIND_NONE 0    /* absent from the header: the value is None */
#define UGVC_AFR_KIND_SCALAR 1  /* Number=1: a scalar, whose len() raises TypeError */
#define UGVC_AFR_KIND_TUPLE 2   /* any other Number */
#define UGVC_AFR_MAX_FILTER_BYTES 63
#define UGVC_AFR_E_LITERAL 1    /* a GT / VAF / BG_VAF literal the parser refuses (numparse.h) */
#define UGVC_AFR_E_TYPE 2       /* TypeError: len() of a Number=1 VAF / BG_VAF */
#define UGVC_AFR_FAILED 1
#define UGVC_AFR_REWRITTEN 2
#define UGVC_AFR_NEW_CONTIG 4
typedef struct ugvc_afr_params {
    double af_ratio_threshold;
    double af_ratio_threshold_h_indels;
    double t_vaf_threshold;
    const char* new_filter;  /* 1..UGVC_AFR_MAX_FILTER_BYTES bytes, not NUL-terminated */
    int32_t new_filter_len;
    int32_t variant_type_kind;
    int32_t vaf_kind, vaf_integer;
    int32_t bg_vaf_kind, bg_vaf_integer;
} ugvc_afr_params;
/* One range of whole VCF data lines per call, in the shape of ugvc_filter_bgzf: `data` = consecutive BGZF blocks
 * (skip_head / take_bytes as there) or, with is_text != 0, the plain text itself (skip_head must be 0).  The text is
 * inflated on the device, indexed by K1 of the context's plan (load the model-less plan), decided, written with its new
 * FILTER column and BGZF-compressed there; outputs as ugvc_filter_bgzf: out_bgzf (blocks of 57344 uncompressed bytes),
 * out_block_csize, out_line_start (n + 1 entries, offsets in this call's output), out_recinfo (POS, len(REF) in
 * flags >> 8), plus out_end (INFO/END of each record, 0 where none; may be NULL), out_flags (may be NULL; per record
 * UGVC_AFR_FAILED | UGVC_AFR_REWRITTEN | UGVC_AFR_NEW_CONTIG: CHROM differs from the previous line's, or the first record
 * of the call) and *out_n_filtered (records that get new_filter).  UGVC_E_DATA where the reference raises: ugvc_afr_error gives the record (index in this call) and the
 * UGVC_AFR_E_* reason (-1 / 0 for a data error of the index pass, see ugvc_last_data_error). */
int ugvc_afr_bgzf(ugvc_ctx* ctx, int lane, const uint8_t* data, size_t n_bytes, uint32_t skip_head, uint64_t take_bytes,
                  int is_text, const ugvc_afr_params* params, uint8_t* out_bgzf, size_t out_capacity, size_t* out_bytes,
                  uint32_t* out_block_csize, size_t block_capacity, size_t* out_n_blocks, ugvc_recinfo* out_recinfo,
                  int64_t* out_line_start, int64_t* out_end, uint8_t* out_flags, size_t capacity_records,
                  int64_t* out_n_records, int64_t* out_n_filtered);
int ugvc_afr_error(const ugvc_ctx* ctx, int lane, int64_t* out_record, int32_t* out_reason);
/* ms of the last ugvc_afr_bgzf call on `lane` between CUDA events: H2D + inflate, index K1, decide + scan + copy,
 * deflate + pack, D2H. */
int ugvc_afr_stage_ms(ugvc_ctx* ctx, int lane, float out_ms[5]);
/* Test hook: decide, scan and copy on the caller's records (line_start: n + 1 entries, every line ending with '\n'),
 * without a context.  Returns the bytes written to out, UGVC_E_DATA with *out_err_record / *out_err_reason where the
 * reference raises (nothing written). */
int64_t ugvc_test_afr(const uint8_t* text, size_t n_bytes, const int64_t* line_start, int64_t n, const ugvc_afr_params* params,
                      uint8_t* out, size_t capacity, int64_t* out_line_start, uint8_t* out_failed, int64_t* out_end,
                      int64_t* out_n_filtered, int64_t* out_err_record, int32_t* out_err_reason);

/* ---- calibrate_bridging_snvs on the device (DESIGN.md 4d) ------------------
 * Replaces the per-record loop of ugvc/pipelines/vcfbed/calibrate_bridging_snvs.py (run, :91-130; is_homopolymer_snp,
 * :9-66): a non-PASS single-base SNV with QUAL >= min_initial_qual whose ALT base extends a reference homopolymer to at
 * least min_query_hmer_size (not a tandem repeat, both sides at least min_distance_from_edge long) and whose sample 0
 * has sum(AD[1:]) / DP >= min_tumor_vaf, sum(BG_AD[1:]) / max(0.01, BG_DP) <= max_normal_vaf and
 * BG_DP > min_normal_depth is rescued: QUAL becomes qual_text and FILTER "PASS".  Every other byte is kept as read.
 * The FASTA window is read from the context's contig table (ugvc_bsn_add_contig), bytes compared as stored.
 *   *_kind  UGVC_BSN_KIND_*: how the header declares AD / DP / BG_AD / BG_DP; *_integer: Type=Integer (else Float) */
#define UGVC_BSN_KIND_NONE 0    /* not declared: reading it raises KeyError */
#define UGVC_BSN_KIND_SCALAR 1  /* Number=1 */
#define UGVC_BSN_KIND_TUPLE 2   /* any other Number */
#define UGVC_BSN_MAX_QUAL_BYTES 31
#define UGVC_BSN_E_LITERAL 1        /* a QUAL / AD / DP / BG_AD / BG_DP literal the parser refuses (numparse.h) */
#define UGVC_BSN_E_TYPE 2           /* TypeError: None or a tuple where a number is needed, a slice of a scalar, ALT "." */
#define UGVC_BSN_E_ZERO_DIVISION 3  /* ZeroDivisionError: DP is 0 */
#define UGVC_BSN_E_KEY 4            /* KeyError: a rescue key missing from the header or the record's FORMAT / sample */
#define UGVC_BSN_E_FETCH 5          /* ValueError of FastaFile.fetch: negative window start or contig not in the FASTA */
#define UGVC_BSN_RESCUED 1
#define UGVC_BSN_NEW_CONTIG 4
typedef struct ugvc_bsn_params {
    int32_t min_query_hmer_size;     /* >= 0 */
    int32_t min_distance_from_edge;
    double min_initial_qual;
    double min_tumor_vaf;
    double max_normal_vaf;
    double min_normal_depth;
    const char* qual_text;           /* the rescued QUAL column, 1..UGVC_BSN_MAX_QUAL_BYTES bytes, not NUL-terminated */
    int32_t qual_len;
    int32_t ad_kind, ad_integer;
    int32_t dp_kind, dp_integer;
    int32_t bg_ad_kind, bg_ad_integer;
    int32_t bg_dp_kind, bg_dp_integer;
} ugvc_bsn_params;
/* Contigs of the FASTA stay on the context until ugvc_bsn_clear_contigs or ugvc_free: one copy of the raw bytes (case
 * kept) per name; adding a name again replaces its bytes. */
int ugvc_bsn_add_contig(ugvc_ctx* ctx, const char* name, const uint8_t* seq, int64_t len);
int ugvc_bsn_clear_contigs(ugvc_ctx* ctx);
/* One range of whole VCF data lines per call, in the shape and with the outputs of ugvc_afr_bgzf; out_flags holds
 * UGVC_BSN_RESCUED | UGVC_BSN_NEW_CONTIG, out_hmer (may be NULL) the hmer_size of each record whose window was walked
 * (0 elsewhere), out_src_line_start (may be NULL; n + 1 entries) the line starts in the range's input text, and
 * *out_n_rescued the rescued count.  UGVC_E_DATA where the reference raises: ugvc_bsn_error gives the record (index in
 * this call) and the UGVC_BSN_E_* reason (-1 / 0 for a data error of the index pass, see ugvc_last_data_error). */
int ugvc_bsn_bgzf(ugvc_ctx* ctx, int lane, const uint8_t* data, size_t n_bytes, uint32_t skip_head, uint64_t take_bytes,
                  int is_text, const ugvc_bsn_params* params, uint8_t* out_bgzf, size_t out_capacity, size_t* out_bytes,
                  uint32_t* out_block_csize, size_t block_capacity, size_t* out_n_blocks, ugvc_recinfo* out_recinfo,
                  int64_t* out_line_start, int64_t* out_src_line_start, int64_t* out_end, uint8_t* out_flags,
                  int32_t* out_hmer, size_t capacity_records, int64_t* out_n_records, int64_t* out_n_rescued);
int ugvc_bsn_error(const ugvc_ctx* ctx, int lane, int64_t* out_record, int32_t* out_reason);
/* ms of the last ugvc_bsn_bgzf call on `lane` between CUDA events: H2D + inflate, index K1, decide + scan + copy,
 * deflate + pack, D2H. */
int ugvc_bsn_stage_ms(ugvc_ctx* ctx, int lane, float out_ms[5]);
/* Test hook: decide, scan and copy on the caller's records (line_start: n + 1 entries, every line ending with '\n')
 * and contigs (n_contigs names at names[name_off[k] .. name_off[k+1]), bytes at seq[seq_off[k] .. seq_off[k+1])), without
 * a context.  Returns the bytes written to out, UGVC_E_DATA with *out_err_record / *out_err_reason where the reference
 * raises (nothing written). */
int64_t ugvc_test_bsn(const uint8_t* text, size_t n_bytes, const int64_t* line_start, int64_t n, const uint8_t* names,
                      const int64_t* name_off, const uint8_t* seq, const int64_t* seq_off, int32_t n_contigs,
                      const ugvc_bsn_params* params, uint8_t* out, size_t capacity, int64_t* out_line_start,
                      uint8_t* out_rescued, int32_t* out_hmer, int64_t* out_end, int64_t* out_n_rescued,
                      int64_t* out_err_record, int32_t* out_err_reason);

/* ---- gvcf_hcr on the device (DESIGN.md 4e) ---------------------------------
 * Replaces ugvc/joint/gvcf_bed.py:gvcf_to_bed and the bedtools merge of ugvc/pipelines/vcfbed/gvcf_hcr_main.py: each
 * record's interval [POS - 1, end) (end = INFO/END under the index rule, else POS - 1 + len(REF); a RefCall deletion --
 * len(REF) > 1 and sample 0 without GQ, or with GT (0, 0) or (None, None) -- ends at POS), records that start before the
 * end of the last kept record of their contig skipped, kept records selected by sample 0's GQ (gt: GQ >= threshold,
 * else GQ absent or < threshold) and written as BED lines "CHROM\tstart\tend\n" (merge: book-ended selected records
 * joined into one line).  The output is plain text. */
#define UGVC_HCR_GQ_STRING 0   /* GQ undeclared or of Type String / Character: comparing it raises TypeError */
#define UGVC_HCR_GQ_SCALAR 1   /* Number=1, Integer or Float */
#define UGVC_HCR_GQ_TUPLE 2    /* any other Number: comparing it raises TypeError */
#define UGVC_HCR_E_LITERAL 1   /* a GQ / GT literal the parser refuses (numparse.h) */
#define UGVC_HCR_E_TYPE 2      /* TypeError: a kept record's GQ is None, a tuple or a string */
#define UGVC_HCR_E_KEY 3       /* KeyError: a RefCall candidate whose FORMAT has GQ but not GT */
#define UGVC_HCR_E_UNSORTED 4  /* POS decreases within a contig: the file cannot carry a tabix index */
#define UGVC_HCR_SELECTED 1    /* flags: selected if the record is kept */
#define UGVC_HCR_GQ_ERROR 2    /* flags: comparing the record's GQ raises TypeError */
#define UGVC_HCR_NEW_CONTIG 4  /* flags: the record starts a contig run of the call */
#define UGVC_HCR_RESET 8       /* flags: the record starts at or after every earlier end of its contig (kept for sure) */
#define UGVC_HCR_KEPT 16       /* flags: not skipped */
#define UGVC_HCR_LINE 32       /* flags: the record starts an output line */
typedef struct ugvc_hcr_params {
    int64_t gq_threshold;
    int32_t gt;          /* 1: GQ >= threshold; 0: GQ absent or GQ < threshold */
    int32_t merge;       /* 1: one line per merged (book-ended) run of selected records; 0: one per selected record */
    int32_t info_end;    /* the header declares INFO/END */
    int32_t gq_kind;     /* UGVC_HCR_GQ_*: how the header declares FORMAT/GQ */
    int32_t gq_integer;  /* Type=Integer (else Float) */
} ugvc_hcr_params;
/* First half of one range of whole gVCF data lines (BGZF blocks, skip_head / take_bytes as for ugvc_afr_bgzf): inflate,
 * the index K1 pass of the model-less plan, then per record the interval, the selection and the GQ / GT checks, and the
 * per-contig prefix maximum of the ends.  The piece stays on the lane for ugvc_hcr_emit.  out_stats = {contig runs that
 * start in the range, the first record > 0 that starts one (n: none), POS - 1 of the first and of the last record};
 * out_run_starts (2 * capacity_records entries) a (record, line start) pair for each record that starts a contig run,
 * in no order. */
int ugvc_hcr_scan(ugvc_ctx* ctx, int lane, const uint8_t* data, size_t n_bytes, uint32_t skip_head, uint64_t take_bytes,
                  const ugvc_hcr_params* params, size_t capacity_records, int64_t* out_n_records, int64_t out_stats[4],
                  int64_t* out_run_starts);
/* Second half, in file order: the kept flags from the entry state (continues_contig: the range's first record is on the
 * contig of the previous range's last one, whose kept records end at entry_extent), selection, merge and the BED text
 * (*out_bytes bytes at out_bed).  out_stats = {output lines, skipped records, the exit extent (end of the last kept
 * record; entry_extent or -1 when none), longest reset-to-reset segment}.  UGVC_E_DATA where the reference raises:
 * ugvc_hcr_error gives the record (index in the range) and the UGVC_HCR_E_* reason. */
int ugvc_hcr_emit(ugvc_ctx* ctx, int lane, const ugvc_hcr_params* params, int continues_contig, int64_t entry_extent,
                  uint8_t* out_bed, size_t out_capacity, size_t* out_bytes, int64_t out_stats[4]);
int ugvc_hcr_error(const ugvc_ctx* ctx, int lane, int64_t* out_record, int32_t* out_reason);
/* ms of the last scan + emit on `lane` between CUDA events: H2D + inflate, index K1, decide + prefix max, emit kernels,
 * D2H. */
int ugvc_hcr_stage_ms(ugvc_ctx* ctx, int lane, float out_ms[5]);
/* Test hook: scan and emit kernels on the caller's records (line_start: n + 1 entries, every line ending with '\n') with
 * the given entry state, without a context.  seg_bound: records a thread walks before a segment takes the parallel form
 * (0: the build's bound).  out_flags (n bytes) the UGVC_HCR_* flags, out_stats as ugvc_hcr_emit's.  Returns the bytes
 * written to out, UGVC_E_DATA with *out_err_record / *out_err_reason where the reference raises. */
int64_t ugvc_test_hcr(const uint8_t* text, size_t n_bytes, const int64_t* line_start, int64_t n, const ugvc_hcr_params* params,
                      int continues_contig, int64_t entry_extent, int64_t seg_bound, uint8_t* out, size_t capacity,
                      uint8_t* out_flags, int64_t out_stats[4], int64_t* out_err_record, int32_t* out_err_reason);

/* ---- test hook ------------------------------------------------------------ */
/* K1's numeric-literal parser (csrc/numparse.h) compiled for the host: parses one token of
 * `text` (NUL-terminated); returns 0 ok / 1 missing (".") / 2 not exactly parseable. */
/* Test hook: K3's xgboost-flavoured fp32 sigmoid evaluated on the device for an array of margins (p1 and the
 * exponential it used). */
int ugvc_test_device_sigmoid(ugvc_ctx* ctx, const float* margins, int n, float* out_p1, float* out_e);
/* Test hook: the record writer's "%g" (csrc/fileio.cu: fio_format_g) on the device for n float32 values.  out receives
 * 16 bytes per value, the slot layout of the writer: the text in bytes 0..14 (zero padded), its length in byte 15;
 * length 0 = a value the device writer leaves to the host writer (exponent form, negative, inf, NaN). */
int ugvc_test_format_g(ugvc_ctx* ctx, const float* v, int64_t n, uint8_t* out);
/* Test hook: the BGZF encoder of ugvc_filter_bgzf (deflate, block offsets, pack) on the caller's n bytes, staged in
 * lane 0's writer buffer (needs ugvc_reserve; n at most what that buffer holds).  encoder 0 = one warp per block (the
 * default), 1 = one thread per block (UGVC_DEFLATE_THREADS=1).  out receives the packed blocks (*out_bytes bytes),
 * out_block_csize the size of each of the *out_n_blocks blocks of 57344 input bytes (none for n = 0). */
int ugvc_test_device_deflate(ugvc_ctx* ctx, const uint8_t* data, size_t n, int encoder, uint8_t* out, size_t capacity,
                             uint32_t* out_block_csize, size_t block_capacity, size_t* out_bytes, size_t* out_n_blocks);
/* Test hook: ugvc_bgzf_inflate_device (lane 0, same staging and kernels) with the decoder named: 0 = one warp per block
 * (the default), 1 = one thread per block (UGVC_INFLATE_THREADS=1).  *out_n = the summed ISIZE; out receives the
 * inflated bytes (a failed block's range is unspecified), block_rc the INF_* code (csrc/inflate.cuh; 0 = accepted,
 * 9 = CRC32 mismatch) of each of the *out_n_blocks blocks with ISIZE > 0, in file order.  The host emulation has
 * decoder 1 only (0 is UGVC_E_STATE there). */
int ugvc_test_device_inflate(ugvc_ctx* ctx, const uint8_t* bgzf, size_t n_bytes, int decoder, uint8_t* out, size_t capacity,
                             size_t* out_n, int32_t* block_rc, size_t block_capacity, size_t* out_n_blocks);
/* Test hook: the K3 launch the loaded plan gets (also in the host emulation, which runs the same chunking).
 * out = {kernel (0 k3_heap, 1 k3_infer), threads per CTA, tile buffers per group, groups per CTA, trees one thread
 * walks at once, forest chunk (k3_heap: trees, k3_infer: nodes; 0 for a linear model), 1 when the whole model is staged
 * once, CTAs of the persistent grid, tree walk (0 plain; 1 default-left / categorical routing of an xgboost model with
 * such nodes), threads per record (2: k3_heap_split)}.  Records per tile: threads / groups / threads per record.
 * UGVC_E_STATE without a model. */
int ugvc_test_k3_config(ugvc_ctx* ctx, int32_t out[10]);
int ugvc_test_parse_float(const char* text, float* out_f32, double* out_f64, int* out_consumed);
/* Test hook: the device BGZF encoder (csrc/deflate.cuh) run on the host on one block of at most 57344 bytes (4 readable
 * bytes after n); out receives a complete BGZF block (<= 65536 bytes), the size is returned. */
int64_t ugvc_test_deflate_block(const uint8_t* in, uint32_t n, uint8_t* out);
/* Test hook: the host model of the warp-per-block encoder (fileio.cu: fio_deflate_warp) -- same windows, candidate
 * rule, token bits and slice-wise CRC, the 32 lanes as a loop.  Same contract as ugvc_test_deflate_block. */
int64_t ugvc_test_deflate_block_lanes(const uint8_t* in, uint32_t n, uint8_t* out);

#ifdef __cplusplus
}
#endif
#endif /* UGVC_B200_H */
