/*
 * gnm.h -- C ABI of libgnm.so: the H100 (sm_90a) implementation of geNomad's
 * nn-classification hot path.
 *
 * The reference has no FFI: its hot path is Python calling TensorFlow/Keras and numba
 * (reference genomad/modules/nn_classification.py, genomad/neural_network/{model,igloo}.py,
 * genomad/sequence.py).  Each entry point below replaces one reference call site; the
 * ctypes binding a geNomad maintainer would add is shown in INTEGRATION.md.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; gnm_last_error() returns a
 *     thread-local message.  No C++ exception crosses this boundary.
 *   - pointers prefixed d_ are DEVICE pointers on the handle's device, h_ are HOST pointers.
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream).  Calls are
 *     asynchronous with respect to the host unless stated otherwise; the caller owns all
 *     input/output buffers and the stream.
 *   - one handle per (device, stream user); calls on one handle are not thread-safe.
 *   - there is NO CPU fallback: every compute entry point fails if no sm_90 device is present.
 */
#ifndef GNM_H_
#define GNM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GNM_WINDOW 6000   /* nucleotides per window     (nn_classification.py:68)  */
#define GNM_TOKENS 5997   /* 4-mer tokens per window    (sequence.py:172; model.py:15) */
#define GNM_CLASSES 3     /* chromosome, plasmid, virus (model.py:44) */

typedef struct gnm_handle gnm_handle;

/* One IGLOO1D_kernel's weights, Keras layouts (reference igloo.py:117-188). */
typedef struct gnm_igloo_weights {
  const float*   w_mult;    /* [1][2100][4][128] */
  const float*   w_summer;  /* [1][512][1]       */
  const float*   w_bias;    /* [1][2100]         */
  const float*   w_qk;      /* [2100][749]       */
  const float*   w_v;       /* [1][128][128]     */
  const int32_t* patches;   /* [2100][4][1], values in [0, 5997) */
} gnm_igloo_weights;

typedef struct gnm_bn_weights {   /* keras BatchNormalization, epsilon = 1e-3 */
  const float* gamma; const float* beta; const float* moving_mean; const float* moving_variance;  /* [512] each */
} gnm_bn_weights;

/*
 * All weights of create_classifier() (reference model.py:34-45) as HOST pointers in the exact
 * layouts stored in genomad/data/nn_classifier.h5 (Keras: Conv1D kernel [k][in][out], Dense
 * kernel [in][out]).  Replaces nn_model.load_weights(...) (nn_classification.py:310).
 */
typedef struct gnm_weights {
  const float* conv1_kernel;  /* [6][257][128]  /model/conv1d   */
  const float* conv1_bias;    /* [128] */
  const float* conv2_kernel;  /* [6][128][128]  /model/conv1d_1 */
  const float* conv2_bias;
  const float* conv3_kernel;  /* [6][128][128]  /model/conv1d_2 */
  const float* conv3_bias;
  gnm_igloo_weights igloo[2]; /* [0] on conv1 output, [1] on conv3 output (igloo.py:54-82) */
  const float* dense0_kernel; /* [256][512]  /model/dense */
  const float* dense0_bias;   /* [512] */
  gnm_bn_weights bn0;         /* /model/batch_normalization */
  const float* dense1_kernel; /* [512][512]  /dense_1 */
  const float* dense1_bias;
  gnm_bn_weights bn1;         /* /batch_normalization_1 */
  const float* dense2_kernel; /* [512][3]    /dense_2 */
  const float* dense2_bias;   /* [3] */
} gnm_weights;

/* Thread-local description of the last failure on the calling thread. */
const char* gnm_last_error(void);

/* Library / build information, e.g. "libgnm 0.4 (sm_90a; ...)". */
const char* gnm_version(void);

/*
 * Create a classifier on CUDA device `device`.  Copies and re-packs the weights (fp16 hi/lo
 * operand splits, folded patch weights, batch-norm scale/shift) and allocates a workspace able
 * to process `max_batch` windows per internal step.  Synchronous.
 * Replaces create_classifier() + load_weights() (nn_classification.py:309-310).
 */
int gnm_create(int device, const gnm_weights* weights, int max_batch, gnm_handle** out);
int gnm_destroy(gnm_handle* h);

/*
 * ASCII windows -> 4-mer tokens.  d_ascii: uint8 [n][6000] (upper-cased, N-padded by the caller,
 * as nn_classification.py:72 does); d_tokens: uint16 [n][5997], 0 = k-mer containing a non-ACGT
 * byte, else 1 + base-4 value.  Bit-exact replacement of sequence.tokenize_dna(seq, 4)
 * (sequence.py:170-193).
 */
int gnm_encode(gnm_handle* h, const uint8_t* d_ascii, int n, uint16_t* d_tokens, void* stream);

/*
 * Per-window class probabilities from ASCII windows (encode fused with the first layer).
 * d_probs: float [n][3] (chromosome, plasmid, virus).  Replaces the TFRecord round trip +
 * nn_model.predict(batch) (nn_classification.py:73,316-317).  n may exceed max_batch (processed
 * in steps).
 */
int gnm_forward_ascii(gnm_handle* h, const uint8_t* d_ascii, int n, float* d_probs, void* stream);

/* Same, from tokens (uint16 [n][5997], values 0..256): nn_model.predict on an int64[B,5997] batch. */
int gnm_forward_tokens(gnm_handle* h, const uint16_t* d_tokens, int n, float* d_probs, void* stream);

/*
 * Per-contig reduction of window probabilities.  d_offsets: int32 [n_contigs + 1], window range
 * of contig c is [offsets[c], offsets[c+1]) (contig ids are sorted, nn_classification.py:66-75).
 * gnm_segment_mean replaces tf.math.segment_mean (nn_classification.py:320): fp32 running sum in
 * window order, divided by the count; empty segments give zeros.
 * gnm_segment_sum writes float [n_contigs][4] = (sum p0, sum p1, sum p2, count) -- the partial
 * a rank contributes when a contig's windows span several GPUs.
 */
int gnm_segment_mean(gnm_handle* h, const float* d_probs, const int32_t* d_offsets, int n_contigs,
                     float* d_mean, void* stream);
int gnm_segment_sum(gnm_handle* h, const float* d_probs, const int32_t* d_offsets, int n_contigs,
                    float* d_sum4, void* stream);

/*
 * Synchronise `stream` and report device-side failures of the steps queued so far: an mbarrier time-out (protocol bug),
 * or an ACTIVATION RANGE OVERFLOW -- the tensor-core convs carry activations as fp16 + e4m3 correction planes scaled for
 * |y| <= 3.5 (csrc/common.cuh); weights that drive a layer-1 or conv output beyond that (fp16: 2047) would silently lose the
 * 1e-4 parity, so the producing kernels raise a flag and the library fails loudly instead.  gnm_forward_* are asynchronous
 * and only see the flag at the start of the NEXT call; gnm_classify_host checks before it returns.
 */
int gnm_check_status(gnm_handle* h, void* stream);

/*
 * Host-buffer convenience path (what a drop-in module calls): h_ascii uint8 [n][6000] in host
 * memory (pinned or pageable) -> h_probs float [n][3].  Copies in steps of max_batch on two
 * internal streams so the copy of step i+1 overlaps the compute of step i.  Synchronous.
 */
int gnm_classify_host(gnm_handle* h, const uint8_t* h_ascii, int n, float* h_probs);

/* ---- host-side FASTA front end (no GPU involved) ------------------------------------------ */

/*
 * FASTA -> windows, INDEX then STREAM (csrc/fasta.cpp).  Replaces the Python loop read_fasta(strip_n=True) ->
 * seq_windows(6000, 2500) -> N rule -> upper-case + pad (sequence.py:96-167, nn_classification.py:65-72).
 *   gnm_fasta_open   : plain (uncompressed) FASTA file; the file is mmap'ed, never copied into anonymous memory.
 *   gnm_fasta_open_gz: gzip / BGZF FASTA: inflated into library-owned memory (BGZF block-parallel on `threads` threads, plain gzip
 *                      sequentially by zlib), then indexed like the others.
 *   gnm_fasta_parse  : FASTA text in caller memory (decompressed input; `len` bytes, must stay alive until gnm_fasta_free).
 *                      Both build the same multi-threaded index: O(records) state, no copy of the sequences.
 *   gnm_fasta_info   : n_records_nonempty / has_duplicate_ids are what check_fasta() tests (sequence.py:124-131);
 *                      n_contigs = records kept after stripping n/N; header_bytes = size of the headers export.
 *   gnm_fasta_export : windows uint8 [n_windows][6000] (may be pinned memory), offsets int32 [n_contigs + 1],
 *                      headers = the kept records' header lines joined with '\n' (header_bytes bytes); any pointer
 *                      may be NULL to skip that output.
 *   gnm_fasta_export_windows : windows [first, first + count) of the GLOBAL window list -> dst uint8 [count][6000], straight
 *                      from the text (any block, any order, `threads` threads): what a rank calls for its shard, chunk by chunk.
 *   gnm_fasta_release_before : mmap mode only -- drop the mapped pages that lie before the record holding window `upto`
 *                      from the resident set (they stay in the page cache).
 */
typedef struct gnm_fasta gnm_fasta;
const char* gnm_fasta_last_error(void);
int gnm_fasta_open(const char* path, int single_window, int threads, gnm_fasta** out);
int gnm_fasta_open_gz(const char* path, int single_window, int threads, gnm_fasta** out);
int gnm_fasta_parse(const uint8_t* text, size_t len, int single_window, int threads, gnm_fasta** out);
int gnm_fasta_info(const gnm_fasta* f, int64_t* n_records_nonempty, int* has_duplicate_ids, int64_t* n_contigs,
                   int64_t* n_windows, int64_t* header_bytes);
int gnm_fasta_export(const gnm_fasta* f, uint8_t* windows, int32_t* offsets, char* headers, int threads);
int gnm_fasta_export_windows(const gnm_fasta* f, int64_t first, int64_t count, uint8_t* dst, int threads);
int gnm_fasta_release_before(const gnm_fasta* f, int64_t upto);
void gnm_fasta_free(gnm_fasta* f);

/* ---- TFRecord files of tokenised windows (host side, no GPU involved; off by default) ------ */

/*
 * Byte-compatible with the reference's encoding-stage intermediates: one tf.train.Example per window with
 * features {"sequence": Int64List(5997 tokens)} in TFRecord framing -- what write_tfrecord produces
 * (nn_classification.py:43-52) and parse_tfrecord reads (:87-91).  Nothing downstream reads these files
 * (SURVEY.md §8f rank 4); they exist for directory-level compatibility with the reference.
 *   gnm_tfrecord_write : tokens uint16 [n][5997] (host) -> one .tfrec file at `path` (overwritten); records are
 *                        serialised on `threads` threads and written in window order.
 *   gnm_tfrecord_read  : verifies both masked CRC-32C of every record; tokens may be NULL to only count records;
 *                        fails if a record is not exactly that Example layout or if there are more than `capacity`.
 *   gnm_crc32c         : CRC-32C (Castagnoli) of a buffer -- exposed for the known-answer tests.
 */
const char* gnm_tfrecord_last_error(void);
int gnm_tfrecord_write(const char* path, const uint16_t* tokens, int64_t n, int threads);
int gnm_tfrecord_read(const char* path, uint16_t* tokens, int64_t capacity, int64_t* n_records);
uint32_t gnm_crc32c(const void* data, size_t n);

/* ---- introspection / test hooks (not needed by a drop-in caller) ------------------------- */

/* Options: "conv_impl" 0 = wgmma tensor-core path (default), 1 = fp32 CUDA-core validation
 * kernels (test hook: lets the tensor-core path be checked on the GPU at large batch);
 * "debug_stop" 0 = full pipeline, 1 = stop after layer 1 + gather#0, 2 = after conv2, 3 = after conv3;
 * "profile_stages" 1 = record a CUDA event between stages (see gnm_stage_times);
 * "conv_experiment" bit mask for timing experiments on the conv kernel: 2 = skip the epilogue's global stores (results
 * become wrong), 4 / 8 = collect per-CTA cycle counters of conv3 / conv2 (gnm_debug_fetch "conv_dbg");
 * "fuse_l1" 1 = run layer 1 and the first IGLOO kernel's value projection as ONE kernel (csrc/layer1_wv.cuh: SIMT producers
 * write the tensor core's B operand straight into swizzled shared memory; bit-identical results, 17 instead of 18 launches
 * per step; measured slower than the two separate kernels at the end of round 1, hence 0 by default);
 * "fuse_gather" 1 (default) = IGLOO value projection + patch gather in one pass over the activations (csrc/wv_gather.cuh),
 * 0 = the round-1 pair conv_t_kernel<true> + patch_stream_kernel (A/B baseline and cross-check);
 * "tail_overlap" 1 (default) = calls that span several internal steps run each step's tail (logits, attention, head) on a
 * second stream next to the next step's main part; 0 = strictly in order (bitwise identical results);
 * "conv_cluster" 1 (default), 2, 4, 8 = thread-block cluster size of the conv kernel's launch (experiment, measured slower);
 * "wv_cost_group" per-mille weight of a band's position groups in the fused IGLOO kernel's unit split (default 100; experiment);
 * further "conv_experiment" bits for wv_gather_kernel: 32 = no gather, 64 = no part_t stores, 128 = no q stores, 256 = gather
 * reads only, 512 = cycle counters (gnm_debug_fetch "conv_dbg"), 1024 = no weight loads, 2048 = no ldmatrix. */
int gnm_set_option(gnm_handle* h, const char* name, int value);
int gnm_get_option(gnm_handle* h, const char* name, int* value);

/*
 * Host-only test hook (no GPU needed): how gnm_create lays out one IGLOO layer's patch set for the gather kernels
 * (csrc/api.cu pack_patches; reference semantics igloo.py:192-206: gather_nd(patches) * w_mult, reshaped, @ w_summer).
 *   layout[4]   (out, optional): {positions per band, bands, entry slots, max entries per position group}
 *   patches [2100][4], w_mult [2100][4][128], w_summer [512] as in gnm_igloo_weights; with all three NULL only `layout` is filled
 *   slot_of [8400]            entry slot of (patch, k); slots are sorted by position
 *   ent_pos [slots]           position of every slot;  ent_w [slots][128] folded weights w_mult * w_summer / 32
 *   groups [*n_groups][2]     {first slot, row inside the band | entries << 8}: the entries (<= 4) on one position; *n_groups is
 *                             the capacity on input and the number of groups on output
 *   band_first_group [bands + 1]
 *   frag [slots][128] words   the folded weights * 2^k as mma.m16n8k16 B fragments: per slot [K-half 2][k-step 4][tig 4] x
 *                             {hi b0, hi b1, lo b0, lo b1}, each word two fp16: b0 = channels (k0, k0 + 1), b1 = (k0 + 8, k0 + 9),
 *                             k0 = 64 K-half + 16 k-step + 2 tig; hi = fp16(w 2^k), lo = fp16(w 2^k - hi)
 *   unscale                   2^-k
 * Any output pointer may be NULL.
 */
int gnm_pack_patches(const int32_t* patches, const float* w_mult, const float* w_summer, int32_t* slot_of, int32_t* ent_pos,
                     float* ent_w, int32_t* groups, int* n_groups, int32_t* band_first_group, uint32_t* frag, float* unscale,
                     int* layout);

/* Number of kernels this library has launched through handle h (monotonic). */
long long gnm_kernel_launches(gnm_handle* h);

/* Per-stage device times (CUDA events recorded on the caller's stream between the stages of every
 * gnm_forward_* / gnm_classify_host step) since option "profile_stages" was last set to 1.
 * names/ms: arrays of capacity *count on input; *count on output = number of (stage, ms) records
 * written, in execution order, one per stage per step.  Synchronises on the last recorded event. */
int gnm_stage_times(gnm_handle* h, const char** names, float* ms, int* count);

/*
 * Copy an intermediate of the most recent forward step (first n <= max_batch windows) to a device
 * buffer as fp32.  which: "buf0","buf1" = the two activation buffers [n][5997][128] (after a full
 * step buf0 = y3, buf1 = y2; with debug_stop = 1, buf0 = y1); "q0","q1" [n][749][128];
 * "mpi0","mpi1" [n][2100]; "logits" [n][752]; "h0" [n][256]; "conv_dbg" [num_sms][16] (int64 counters viewed as
 * float pairs).  Used by the per-kernel parity tests and tools/gpu_experiment.py.
 */
int gnm_debug_fetch(gnm_handle* h, const char* which, int n, float* d_dst, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GNM_H_ */
