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
#define GNM_EMBED 512     /* encoder output: Dense(512) + BatchNorm + ReLU, model.py:28-30 */

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
 * to process `max_batch` windows per internal step.  Synchronous.  Fails, naming the IGLOO layer, if its w_v or its folded
 * patch weights w_mult * w_summer / 32 are not all finite (no fp16 operand split carries them); any finite ones are accepted.
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

/* Same, from tokens (uint16 [n][5997]): nn_model.predict on an int64[B,5997] batch.  Any uint16 is accepted, and the
 * tokens need not come from gnm_encode: as in tf.one_hot(x, 257), a value above 256 contributes nothing. */
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

/* ---- contigs in memory -> windows, on the GPU ---------------------------------------------- */

/*
 * The windowing of read_fasta(strip_n=True) -> seq_windows(6000, 2500) -> N rule -> upper-case + pad
 * (sequence.py:96-167, nn_classification.py:65-72) for contigs already in device memory; the same rules as the FASTA
 * reader below, byte for byte (csrc/contigs.cuh).
 *
 * Input: d_seq holds the contigs' bytes back to back; contig c is d_seq[d_seq_offsets[c] .. d_seq_offsets[c+1]), int64
 * offsets, n_contigs + 1 of them, non-decreasing, any start address.  A contig is its sequence as read_fasta joins its
 * lines: no header, no line terminators, NOT yet stripped of leading / trailing n/N.
 *
 * gnm_contig_windows: plans the kept windows of every contig.
 *   d_win_start [capacity]    absolute byte offset in d_seq of each kept window's first byte
 *   d_win_len   [capacity]    1..6000 bytes of sequence; the rest of the window is 'N' padding
 *   d_win_offsets [n_contigs + 1]  CSR: the windows of contig c are [off[c], off[c+1]), in order
 *   *h_n_windows              number of kept windows (also set when the call fails for lack of capacity)
 *   A contig that is empty after stripping gets ZERO windows; the reference drops such a contig entirely, so a caller that
 *   mirrors its outputs drops the rows whose window count is 0 (gnm_segment_mean writes zeros for them).
 *   capacity >= n_contigs + total_bytes / 6000 is always enough.  If the plan needs more than `capacity` windows, or more
 *   than 2^31 - 1, or the offsets decrease, the call fails with a message and writes nothing to d_win_start / d_win_len.
 *   d_win_offsets doubles as the planning scratch: no other memory is used or allocated.
 *   Synchronous: one device-to-host copy of the count; the start / length arrays are written in `stream` order after it.
 *
 * gnm_contig_windows_stride: the same plan with a window every `stride` nt (1 <= stride <= 6000) instead of every 6000: the
 *   overlapping windows of a score profile, always over the whole contig (no single_window).  Candidate k of a stripped contig
 *   of L nt starts at k * stride and is min(6000, L - k * stride) long; candidate 0 is always kept, any other one if it has
 *   >= 2500 nt and <= 4000 'N' -- 1 + max(0, (L - 2500) / stride) candidates.  At stride 6000 this is gnm_contig_windows
 *   (same kernels, bitwise the same plan).  capacity >= n_contigs + total_bytes / stride is always enough; the failures and
 *   their messages are those of gnm_contig_windows.  Each candidate's N count reads its own 6000 bytes, ~6000 / stride reads
 *   per byte.
 *
 * gnm_gather_windows: kept windows -> d_ascii uint8 [n][6000] (16-byte aligned), ASCII-upper-cased ('a'..'z' only) and
 *   'N'-padded: exactly the bytes gnm_forward_ascii takes, and gnm_fasta_export gives for the same contigs as FASTA text.
 *   Asynchronous.
 *
 * gnm_forward_windows: per-window probabilities float [n][3] straight from the sequence buffer.  Each internal step
 *   gathers its <= max_batch windows into the staging buffers gnm_classify_host copies into (two, alternated by step), then
 *   runs the same forward step as gnm_forward_ascii: bitwise the same probabilities.  Asynchronous like gnm_forward_ascii;
 *   synchronise `stream` before calling gnm_classify_host on the same handle.
 *
 * Per-contig scores: gnm_segment_mean(h, d_probs, d_win_offsets, n_contigs, d_mean, stream).
 *
 * The reverse strand.  rc(S) is the reference's Sequence.rc() (sequence.py:41-43): ACTGNactgn -> TGACNtgacn, every other byte
 * unchanged, then reversed; stripping n/N commutes with it.
 * gnm_contig_windows_rc: the windows of every contig's reverse complement, i.e. what gnm_contig_windows (single_window) or
 *   gnm_contig_windows_stride (stride) plans for rc(S), with the same arguments, capacity rule, failures and messages.
 *   Candidate k is laid from the stripped end: it covers the forward segment [L - k stride - len_k, L - k stride) of the
 *   stripped contig, len_k = min(6000, L - k stride), and d_win_start / d_win_len name that segment (so a start is still an
 *   offset in d_seq).  Its N count is the segment's 'N' count.  single_window: the last <= 6000 nt.  At L = 10000 and stride
 *   6000 the windows are [4000, 10000) and [0, 4000), not the forward ones in reverse order.
 * gnm_gather_windows_rc: planned reverse windows -> d_ascii rows, row byte j = upper(comp(seg[len - 1 - j])), 'N' past len:
 *   the rows gnm_gather_windows gives for rc(S).
 * gnm_forward_windows_rc / gnm_embed_windows_rc: gnm_forward_windows / gnm_embed_windows with that gather: the same staging and
 *   the same forward step, so bitwise gnm_forward_ascii / gnm_embed_ascii on gnm_gather_windows_rc's rows.
 */
int gnm_contig_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_seq_offsets, int n_contigs, int single_window,
                       int64_t* d_win_start, int32_t* d_win_len, int64_t capacity, int32_t* d_win_offsets,
                       int64_t* h_n_windows, void* stream);
int gnm_contig_windows_stride(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_seq_offsets, int n_contigs, int stride,
                              int64_t* d_win_start, int32_t* d_win_len, int64_t capacity, int32_t* d_win_offsets,
                              int64_t* h_n_windows, void* stream);
int gnm_contig_windows_rc(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_seq_offsets, int n_contigs, int single_window,
                          int stride, int64_t* d_win_start, int32_t* d_win_len, int64_t capacity, int32_t* d_win_offsets,
                          int64_t* h_n_windows, void* stream);
int gnm_gather_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                       uint8_t* d_ascii, void* stream);
int gnm_gather_windows_rc(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                          uint8_t* d_ascii, void* stream);
int gnm_forward_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                        float* d_probs, void* stream);
int gnm_forward_windows_rc(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                           float* d_probs, void* stream);

/* ---- encoder embeddings ------------------------------------------------------------------- */

/*
 * The output of the reference's encoder sub-model, create_encoder() (model.py:14-31): relu(BN(h0 @ dense0 + b0)), float
 * [n][GNM_EMBED] per window -- the "vector representation" the classifier head is trained on (docs nn_classification.md).  The
 * reference computes it inside nn_model.predict and never hands it out; Keras users rebuild it with nn_model.get_layer("model").
 * Each gnm_embed_* is the matching gnm_forward_* / gnm_classify_host call with d_embed threaded through: the same steps, the
 * same kernels, bitwise the same probabilities; dense layer 0's epilogue also stores its rows to d_embed (no extra launch),
 * so the embeddings are bitwise what gnm_debug_fetch("h1") shows for the last step.
 *   d_embed  DEVICE float [n][GNM_EMBED], caller-owned, may not be NULL; row offsets are 64-bit (n * 2 KB may exceed 2^31 B).
 *   d_probs / h_probs  may be NULL: then the head stops after the encoder (device calls) or the probabilities are not copied
 *            back (gnm_embed_host).
 * gnm_embed_tokens / gnm_embed_ascii / gnm_embed_windows: asynchronous, like gnm_forward_*.
 * gnm_embed_host: host windows in, host probabilities out, embeddings stay on the device; synchronous, like gnm_classify_host.
 *
 * gnm_segment_sum_rows: per-segment sums of 512-wide rows, d_rows float [rows][512], d_offsets int32 [k + 1] with offsets[0] = 0
 *   (segment c = rows [offsets[c], offsets[c+1])), d_sums float [k][512].  Each column is a plain fp32 running sum in row order
 *   (no FMA, no tree: gnm_segment_mean's rule).  Segment 0 starts from d_carry_in [512] when it is not NULL; the running sum of
 *   segment k-1 is written to d_carry_out [512] when it is not NULL (it may alias d_carry_in).  Summing the rows in several calls,
 *   each seeded with the previous call's carry, gives the same bits as one call over all rows: what a caller that streams chunks,
 *   or a rank that continues a contig begun on an earlier rank, needs.  d_rows, d_sums and d_carry_in 16-byte aligned.
 *   Asynchronous.  Per-contig mean embedding = sums / count in fp32 (empty contig: zeros).
 */
int gnm_embed_tokens(gnm_handle* h, const uint16_t* d_tokens, int n, float* d_probs, float* d_embed, void* stream);
int gnm_embed_ascii(gnm_handle* h, const uint8_t* d_ascii, int n, float* d_probs, float* d_embed, void* stream);
int gnm_embed_windows(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                      float* d_probs, float* d_embed, void* stream);
int gnm_embed_windows_rc(gnm_handle* h, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len, int n,
                         float* d_probs, float* d_embed, void* stream);
int gnm_embed_host(gnm_handle* h, const uint8_t* h_ascii, int n, float* h_probs, float* d_embed);
int gnm_segment_sum_rows(gnm_handle* h, const float* d_rows, const int32_t* d_offsets, int k, const float* d_carry_in,
                         float* d_sums, float* d_carry_out, void* stream);

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
 *
 * Window lists at any stride (score profiles): the list above is the stride-6000 case of one enumeration over the index --
 * candidate k of a kept record starts k * stride nt into its stripped sequence, is min(6000, L - k * stride) long, and is kept
 * if it is the first or has >= 2500 nt and <= 4000 'N' (the rules of gnm_contig_windows_stride).
 *   gnm_fasta_windows_plan   : the list at `stride` (1..6000; single_window keeps only the first window of each record) over the
 *                      index of f, records on `threads` threads; f must outlive it.  ~16 B per record, plus 8 B per candidate
 *                      window of records with irregular lines and 4 B per window of records that lost one to the N rule.
 *                      Fails, before anything is built, if the list could have more than 2^31 - 1 windows (its
 *                      candidates before the N rule, a closed form).  Each list releases the pages behind its own
 *                      export cursor (gnm_fasta_windows_release_before), so a second pass over the file stays bounded too.
 *   gnm_fasta_windows_plan_rc: the list gnm_fasta_windows_plan makes from every kept record's reverse complement rc(S)
 *                      (gnm_contig_windows_rc's windows); its export reverse-complements and upper-cases, its spans name each
 *                      window's forward segment.  N counts come from the same one-walk running count.
 *   gnm_fasta_windows_info   : kept records (= contigs) and windows of the list.
 *   gnm_fasta_windows_spans  : offsets int32 [n_contigs + 1] (CSR: the windows of contig c), starts int64 [n_windows] (0-based,
 *                      in the record's sequence BEFORE stripping, i.e. its joined lines), lengths int32 [n_windows] (1..6000,
 *                      padding excluded); any pointer may be NULL.
 *   gnm_fasta_windows_export / _release_before : gnm_fasta_export_windows / gnm_fasta_release_before on this list.
 *   gnm_fasta_spans          : starts / lengths, as gnm_fasta_windows_spans gives them, of the list gnm_fasta_export serves.
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
typedef struct gnm_fasta_windows gnm_fasta_windows;
int gnm_fasta_windows_plan(const gnm_fasta* f, int stride, int single_window, int threads, gnm_fasta_windows** out);
int gnm_fasta_windows_plan_rc(const gnm_fasta* f, int stride, int single_window, int threads, gnm_fasta_windows** out);
int gnm_fasta_windows_info(const gnm_fasta_windows* w, int64_t* n_contigs, int64_t* n_windows);
int gnm_fasta_windows_spans(const gnm_fasta_windows* w, int32_t* offsets, int64_t* starts, int32_t* lengths);
int gnm_fasta_windows_export(const gnm_fasta_windows* w, int64_t first, int64_t count, uint8_t* dst, int threads);
int gnm_fasta_windows_release_before(const gnm_fasta_windows* w, int64_t upto);
void gnm_fasta_windows_free(gnm_fasta_windows* w);
int gnm_fasta_spans(const gnm_fasta* f, int64_t* starts, int32_t* lengths);

/* ---- per-window score table (host side, no GPU involved) ----------------------------------- */

/*
 * gnm_write_window_tsv: writes `header`, then one line per window w of contig c,
 *   "<name c>\t<starts[w] + 1>\t<starts[w] + lengths[w]>\t<p0>\t<p1>\t<p2>\n"  (1-based start, inclusive end),
 *   to `path` (overwritten).  names: the contigs' names back to back, name c = names[name_offsets[c] .. name_offsets[c+1]);
 *   win_offsets int32 [n_contigs + 1] (CSR); probs float [win_offsets[n_contigs]][3].  Scores carry exactly the digits of
 *   Python's f"{float(x):.4f}" (the float value rounded half to even at the fourth decimal; no locale).  Rows are formatted on
 *   `threads` threads and written in order.
 * gnm_write_window_tsv_cols: the same table with n_cols scores per row (1 <= n_cols <= 32; probs float
 *   [win_offsets[n_contigs]][n_cols]): the per-window scores of a C-class head.  gnm_write_window_tsv is its n_cols = 3 case.
 * gnm_format_scores: the same score formatting, one value per line into out (<= 49 bytes per value); *out_len = bytes written.
 */
const char* gnm_tsv_last_error(void);
int gnm_write_window_tsv(const char* path, const char* header, const char* names, const int64_t* name_offsets, int64_t n_contigs,
                         const int32_t* win_offsets, const int64_t* starts, const int32_t* lengths, const float* probs,
                         int threads);
int gnm_write_window_tsv_cols(const char* path, const char* header, const char* names, const int64_t* name_offsets,
                              int64_t n_contigs, const int32_t* win_offsets, const int64_t* starts, const int32_t* lengths,
                              const float* probs, int n_cols, int threads);
int gnm_format_scores(const float* x, int64_t n, char* out, int64_t* out_len);

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
 *   unscale                   2^-k, k = 14 - (exponent of max |w|) clamped to [-126, 121]: max |w| 2^k in [2^13, 2^14)
 * Any output pointer may be NULL.  Fails if a folded weight is not finite (as gnm_create does).
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
 * "mpi0","mpi1" [n][2100]; "logits" [n][752] (of the second IGLOO kernel after a full step); "h0" [n][256];
 * "h1","h2" [n][512] = the outputs of the two Dense(512) + BatchNorm + ReLU layers of the head (h1 is the encoder output, the
 * embedding gnm_embed_* return);
 * "conv_dbg" [num_sms][16] (int64 counters viewed as float pairs).  Used by the per-kernel parity tests and tools/gpu_experiment.py.
 *   conv_t_kernel's counters, per CTA, in clock64 cycles: [0] first consumer warpgroup's total, [1] its MMA phases (first
 *   barrier wait of a unit to its last wgmma's completion), [2] its waits on a_full, [3] its waits on w_full, [4] units,
 *   [5] the second consumer warpgroup's MMA phases, [6] the first's epilogues, [7] the second's epilogues.
 *   wv_gather_kernel's counters ("conv_experiment" bit 512, second IGLOO launch), per CTA, in clock64 cycles: [0] the first
 *   gather warp's total, [1] its waits on a_full, [2] its gather work (reads, mma, part_t stores, release), [3] the first MMA
 *   warpgroup's MMA phases (first a_full wait of a unit to its last wgmma's completion, waits included), [4] that warpgroup's
 *   waits on a_full, [5] units, [6] that warpgroup's epilogues (max-pool and q stores), [7] the producer's waits on a_empty.
 * After an attribution call (gnm_attribute_*), for its last chunk (n <= the context's max_batch, checked): "route0","route1" = uint8
 * [n][749][128], the row 0..7 inside each max-pool window of the pooled maximum (first row on ties) -- n * 749 * 128 BYTES are
 * written to d_dst; "routeq0","routeq1" [n][749][128] = the maxima the routing pass found (bitwise "q0","q1"); "attr_y1"
 * [n][5997][128] = its layer-1 copy (y1, bitwise what the forward's layer 1 wrote).  An attribution
 * call re-runs IGLOO#0's logits, so "logits" then holds the first IGLOO kernel's.  The backward pass's intermediates, same
 * conditions, positions in natural order: "attr_g_out" [n][256] = d log p_c / d h0 (unscaled; d D_c / d h0 after a novelty
 * attribution call); "attr_g_h1" [n][512] = d D_c / d h1 of the last novelty attribution chunk (fp32); "attr_s_w" [n] = the per-window
 * power of two s_w; "attr_s2" [n] = the power of two of conv3's backward output (max |s_w g_z2| s2 in [1, 2)); "attr_gz3",
 * "attr_gz2" [n][5997][128] = s_w g_z3 and s2 s_w g_z2 as the next conv reads them (the joined hi16 + lo8 of the operand rows);
 * "attr_gy1" [n][5997][128] = IGLOO#0's part of g_y1 (fp32, unscaled); "attr_gz1" [n][5997][128] = s_w g_z1 (fp32).  After an
 * integrated-gradients call they hold the last chunk's rows, except "attr_gy1", which then holds the layer-1 IG rows.
 */
int gnm_debug_fetch(gnm_handle* h, const char* which, int n, float* d_dst, void* stream);

/*
 * Attributions: the input gradient of a class's log-probability, per 4-mer position of a window (gradient x input on the
 * one-hot tokens).  For a window with tokens tok[0..5996] (the tokenizer's output, 0..256) and a target class c (0 chromosome,
 * 1 plasmid, 2 virus):
 *
 *     attr[t] = d log p_c / d x[t, tok[t]]
 *
 * with x the one-hot input of the first Conv1D (reference model.py:9-11), at the window's own input, for the unchanged model.
 * Token position t covers bases t .. t+3 of the window.  Token 0 (a 4-mer with a non-ACGT base) is a real one-hot row, so the
 * N-padded tail of a short window gets attributions too.  log p_c rather than p_c: a saturated class still has a gradient.
 * Max-pool gradients go to the first row of a tie (ties are exact and common inside N runs).  DESIGN.md, "Attributions".
 *
 * gnm_attr_create: the attribution workspace for up to max_batch windows per chunk (1 <= max_batch <= the handle's), allocated
 *   here, not by gnm_create: gnm_attr_bytes_per_window() bytes per window (~21 MB) plus ~14 MB of re-packed weights (W2^T, W3^T packs
 *   0.8 MB, w_v^T 0.1 MB, w_qk^T 12.6 MB, patch index 0.06 MB).  The
 *   context belongs to the handle; destroy it before the handle.
 * gnm_attribute_ascii / gnm_attribute_windows: n windows (ASCII rows as for gnm_forward_ascii, or planned windows of a sequence
 *   buffer as for gnm_forward_windows) in chunks of the context's max_batch.  Each chunk runs the unchanged forward step, strictly
 *   in order (no tail overlap), then the backward pass over what that step left on the device.
 *   d_attr  DEVICE float [n][5997], caller-owned.
 *   d_probs DEVICE float [n][3] or NULL; when given, bitwise what gnm_forward_ascii / gnm_forward_windows return.
 *   Asynchronous on `stream`.  The gradient rows the two backward convs read carry per-window powers of two (s_w, s2) that put
 *   their maxima in the operand format's range whatever the weights' scale; only a gradient that is not finite is reported, as
 *   a gradient range overflow by the next call or gnm_check_status, like act_overflow.  Fails with conv_impl = 1: the fp32
 *   validation kernels have no backward pass.
 */
typedef struct gnm_attr gnm_attr;
int gnm_attr_create(gnm_handle* h, int max_batch, gnm_attr** out);
int gnm_attr_destroy(gnm_attr* a);
long long gnm_attr_bytes_per_window(void);
int gnm_attribute_ascii(gnm_handle* h, gnm_attr* a, const uint8_t* d_ascii, int n, int target, float* d_probs, float* d_attr,
                        void* stream);
int gnm_attribute_windows(gnm_handle* h, gnm_attr* a, const uint8_t* d_seq, const int64_t* d_win_start, const int32_t* d_win_len,
                          int n, int target, float* d_probs, float* d_attr, void* stream);

/*
 * Integrated gradients (IG): attributions that add up to the change in log p_c from a baseline input x' to the window x, so that
 * windows classified confidently as the target (where gradient x input scales as e^-margin and reaches exactly 0) get
 * attributions too.  With m steps and the midpoint rule alpha_k = (k + 1/2) / m, k = 0..m-1, and g_k the gradient of log p_c
 * with respect to the one-hot input at x' + alpha_k (x - x'):
 *
 *   GNM_IG_BASELINE_ZERO  x' = all-zero one-hot rows (the model's causal padding):   IG[t] = (1/m) sum_k g_k[t, tok[t]]
 *   GNM_IG_BASELINE_N     x' = the all-N window (token 0 everywhere, a real input):  IG[t] = (1/m) sum_k (g_k[t, tok[t]] - g_k[t, 0]),
 *                         and 0 where tok[t] = 0
 *
 *   sum_t IG[t] -> log p_c(x) - log p_c(x') as m grows (completeness; the gap at a given m is measured in
 *   profiles/integrated_gradients_h100.md).
 *
 * Layer 1 at an interpolated input is lrelu(b1 + alpha S_tok + (1 - alpha) S_base) (Conv1D #1 is linear in its one-hot input);
 * everything after it is the unchanged model, and each (window, alpha_k) row goes through the gnm_attribute_* backward pass
 * (routing, LeakyReLU branches, head gradient, s_w: per row).  The mean over k is taken in fp32, k ascending, no atomics: the
 * result does not depend on the batch, the chunking, fuse_l1 or tail_overlap.  DESIGN.md, "Integrated gradients".
 *
 * gnm_attribute_ig_ascii / gnm_attribute_ig_windows: windows as for gnm_attribute_ascii / gnm_attribute_windows (the same
 *   bytes: no case folding for ASCII rows), in chunks of floor(max_batch / steps) windows of the context.
 *   steps     1 <= steps <= the context's max_batch.
 *   baseline  GNM_IG_BASELINE_ZERO or GNM_IG_BASELINE_N.
 *   d_attr    DEVICE float [n][5997], caller-owned.
 *   d_probs   DEVICE float [n][3] or NULL: bitwise what gnm_forward_ascii / gnm_forward_windows return.
 *   d_logp    DEVICE float [n][2] or NULL: log p_c(x), log p_c(x') (the second column is the same in every row), from fp32
 *             probabilities without cancellation: -log1p(sum_{i != c} p_i) when p_c is the largest, log p_c otherwise,
 *             evaluated in fp64 and rounded to fp32.
 *   Cost: per window one forward (when d_probs or d_logp is given) plus `steps` attribution rows, ~1 + 4.2 steps forwards;
 *   one more one-row forward per call for log p_c(x').  No memory beyond the context's.
 *   After the call, "route*", "routeq*", "attr_y1", "buf0", "buf1", "h2" of gnm_debug_fetch hold the last chunk's ROWS, row
 *   w * steps + k = window w at alpha_k.  Asynchronous on `stream`; range overflows are reported as for gnm_attribute_*.
 */
#define GNM_IG_BASELINE_ZERO 0
#define GNM_IG_BASELINE_N    1
int gnm_attribute_ig_ascii(gnm_handle* h, gnm_attr* a, const uint8_t* d_ascii, int n, int target, int steps, int baseline,
                           float* d_probs, float* d_logp, float* d_attr, void* stream);
int gnm_attribute_ig_windows(gnm_handle* h, gnm_attr* a, const uint8_t* d_seq, const int64_t* d_win_start,
                             const int32_t* d_win_len, int n, int target, int steps, int baseline, float* d_probs, float* d_logp,
                             float* d_attr, void* stream);

/*
 * Head attributions: the same attributions and integrated gradients for a class of a trained head (gnm_head_create, below),
 * so that a sequence scored as one of the user's classes can be explained.  For a head with C classes, a target c in [0, C)
 * and the head's inference-mode forward on the window's encoder output h1 (dense layer 0's output, gnm_embed_*):
 *
 *     z = h1 W1 + b1;  a = scale * z + shift (BN folded as gnm_head_create folds it);  hh = relu(a);
 *     logits = hh W2 + b2;  p = softmax(logits) (the sequence of gnm_head_forward)
 *     attr[t] = d log p_c / d x[t, tok[t]]
 *
 * at the window's own input, with the routing rule (first row on ties) and LeakyReLU branches of gnm_attribute_*.  The head
 * gradient keeps the shipped rule for all C classes: g_i = -p_i for i != c and g_c = sum_{i != c} p_i in ascending i, never
 * 1 - p_c.  IG uses the same midpoint rule and baselines, and log p_c(x), log p_c(x') the same no-cancellation form, over the
 * head's C probabilities.  A head with the shipped tail's own weights (C = 3) gives bitwise the attributions of gnm_attribute_*.
 *
 * gnm_attribute_head_ascii / _windows, gnm_attribute_head_ig_ascii / _ig_windows: arguments as gnm_attribute_* and
 *   gnm_attribute_ig_*, plus
 *   head          a head created on h (gnm_head_create).
 *   target        in [0, C); any other value is refused.
 *   d_probs       DEVICE float [n][3] or NULL: the shipped probabilities, bitwise those of gnm_forward_*.
 *   d_head_probs  DEVICE float [n][C] or NULL: the head's probabilities, bitwise those of gnm_head_forward on the gnm_embed_*
 *                 output of the same windows.
 *   d_logp        (IG) DEVICE float [n][2] or NULL: log p_c(x), log p_c(x') of the head's class.
 *   Per chunk, one dense_1 GEMM on the tensor cores and one softmax more than gnm_attribute_*; no memory beyond the context's
 *   (the head's hidden rows use the handle's h2, its probabilities the context's scratch).  Refused under conv_impl = 1 or a
 *   debug_stop, as gnm_attribute_*.  Asynchronous on `stream`.
 */
typedef struct gnm_head gnm_head;
int gnm_attribute_head_ascii(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_ascii, int n, int target,
                             float* d_probs, float* d_head_probs, float* d_attr, void* stream);
int gnm_attribute_head_windows(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_seq, const int64_t* d_win_start,
                               const int32_t* d_win_len, int n, int target, float* d_probs, float* d_head_probs, float* d_attr,
                               void* stream);
int gnm_attribute_head_ig_ascii(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_ascii, int n, int target,
                                int steps, int baseline, float* d_probs, float* d_head_probs, float* d_logp, float* d_attr,
                                void* stream);
int gnm_attribute_head_ig_windows(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_seq,
                                  const int64_t* d_win_start, const int32_t* d_win_len, int n, int target, int steps, int baseline,
                                  float* d_probs, float* d_head_probs, float* d_logp, float* d_attr, void* stream);

/*
 * Novelty attributions: the same passes for a head's novelty distance (gnm_head_set_novelty, below) to a target class, so that
 * a window flagged as novel can be explained.  For a window's encoder output h1 (gnm_embed_*) and its target class c:
 *
 *     r = P (h1 - center) - m_c;   D_c = ||r||^2 / 512;   g_h1 = dD_c / dh1 = (2 / 512) P^T r
 *     attr[t] = d D_c / d x[t, tok[t]]     (D_c itself, not its log)
 *
 * r and g_h1 are computed in fp64 on the tensor cores (r's Y as gnm_head_novelty computes it; P^T r over the tiles where P is
 * not zero, k ascending) and g_h1 is rounded to fp32 once; from there the pass is gnm_attribute_head_*'s from dense layer 0
 * down, with the same routing rule and LeakyReLU branches.  No atomics: a window's row does not depend on its batch, its
 * position in it, n or the chunking.  IG uses the same midpoint rule and baselines; sum_t IG[t] -> D_c(x) - D_c(x').
 *
 * gnm_attribute_novelty_ascii / _windows, gnm_attribute_novelty_ig_ascii / _ig_windows: arguments as gnm_attribute_head_*, except
 *   head           a head created on h that carries a novelty model; one without is refused.
 *   h_target       HOST int32 [n]: each window's target class.  Every entry is checked before any launch; one outside [0, C)
 *                  is refused, naming its index.
 *   d_probs        DEVICE float [n][3] or NULL: bitwise what gnm_forward_* returns.
 *   d_dist         DEVICE float [n][C] or NULL: the windows' distances, bitwise gnm_head_novelty on the gnm_embed_* output of the
 *                  same windows.
 *   d_dist_target  (IG) DEVICE float [n][2] or NULL: D_c(x), bitwise d_dist[w][c], and D_c(x') from one one-row forward of the
 *                  baseline per call.
 *   Per chunk, three fp64 kernels (~1 MFLOP per window; 1.02x the time of gnm_attribute_head_* on an H100) instead of the
 *   head's forward and backward; the context's memory holds
 *   4 KB of r and 2 KB of g_h1 per window.  A gradient that is not finite is reported as for gnm_attribute_*.  Refused under
 *   conv_impl = 1 or a debug_stop.  gnm_debug_fetch "attr_g_h1" [n][512] holds the last chunk's fp32 g_h1 rows.  Work is queued
 *   on `stream`, but the call is not fully asynchronous: each chunk's targets are copied from pageable host memory, which can
 *   make the host wait for the previous chunk's kernels before it issues the next chunk.
 */
int gnm_attribute_novelty_ascii(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_ascii, int n,
                                const int32_t* h_target, float* d_probs, float* d_dist, float* d_attr, void* stream);
int gnm_attribute_novelty_windows(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_seq,
                                  const int64_t* d_win_start, const int32_t* d_win_len, int n, const int32_t* h_target,
                                  float* d_probs, float* d_dist, float* d_attr, void* stream);
int gnm_attribute_novelty_ig_ascii(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_ascii, int n,
                                   const int32_t* h_target, int steps, int baseline, float* d_probs, float* d_dist,
                                   float* d_dist_target, float* d_attr, void* stream);
int gnm_attribute_novelty_ig_windows(gnm_handle* h, gnm_attr* a, const gnm_head* head, const uint8_t* d_seq,
                                     const int64_t* d_win_start, const int32_t* d_win_len, int n, const int32_t* h_target,
                                     int steps, int baseline, float* d_probs, float* d_dist, float* d_dist_target, float* d_attr,
                                     void* stream);

/*
 * Embedding neighbours: for each query row, the k reference rows nearest in cosine similarity.  Rows are GNM_EMBED (512) fp32
 * values (the encoder embeddings of gnm_embed_*), finite, contiguous, row pitch 2 KB.  No handle, no allocation: the calls run on
 * the current device and `stream`, and use only the caller's workspace.  DESIGN.md, "Embedding neighbours".
 *
 *   similarity   s(q, r) = <q / |q|, r / |r|>, |x| the fp32 norm summed in a fixed order; a row of norm 0 becomes the zero row,
 *                so its similarity with every row is 0.  Computed on the tensor cores as three TF32 products of the split rows
 *                (hi * hi + lo * hi + hi * lo) in one fp32 accumulator, K ascending: |s - exact| is about 1e-6, and a pair's s
 *                is bitwise the same whatever call, chunk, tile or offset computes it.
 *   order        (s descending, global reference index ascending): ties, such as duplicate rows, go to the lower index.
 *   result       d_sim [n_query][k] float, d_idx [n_query][k] int64 (DEVICE): row q holds query q's k first references under
 *                that order; global index = ref_index0 + reference row.  When fewer than k references qualify, the list is
 *                padded with index -1 and similarity -inf.
 *   self         self_index0 >= 0: query q never returns global index self_index0 + q (all-vs-all: pass the same rows as
 *                query and reference with self_index0 = ref_index0).  -1: no exclusion.
 *
 * gnm_neighbours_workspace_bytes: the bytes of d_work a call with these sizes needs on the current device (0 on invalid
 *   arguments, see gnm_last_error): the normalised rows of both sets as TF32 halves (4 KB per row) and the partial lists of the
 *   reference splits (8 k bytes per query and split).
 * gnm_embedding_neighbours: 1 <= k <= 64; 0 <= n_query, n_ref <= 2^30 (more reference rows: call once per chunk with its
 *   ref_index0 and merge); d_query, d_ref 16-byte aligned, d_work 256-byte aligned.  n_ref = 0 gives padded lists.
 * gnm_neighbours_merge: merges the lists (d_sim_b, d_idx_b) into (d_sim, d_idx), in place, under the same order: the result of a
 *   call over references A followed by a merge of the result over a disjoint set B is bitwise the result of one call over A + B.
 *   Both inputs must be lists of this form (sorted, padded at the end).
 */
size_t gnm_neighbours_workspace_bytes(int64_t n_query, int64_t n_ref, int k);
int gnm_embedding_neighbours(const float* d_query, int64_t n_query, const float* d_ref, int64_t n_ref, int64_t ref_index0,
                             int64_t self_index0, int k, float* d_sim, int64_t* d_idx, void* d_work, size_t work_bytes,
                             void* stream);
int gnm_neighbours_merge(float* d_sim, int64_t* d_idx, const float* d_sim_b, const int64_t* d_idx_b, int64_t n_query, int k,
                         void* stream);

/*
 * Embedding index: an inverted-file (IVF) search over reference rows split into L lists by spherical k-means.  s(q, r) is the
 * similarity gnm_embedding_neighbours returns for query q and reference r; "the total order" is its (s descending, index
 * ascending).  DESIGN.md, "Embedding index".
 *
 * Build (spherical k-means, Dhillon & Modha 2001; engine.ivf_build drives it with the calls below), from n reference rows, L lists
 * (1 <= L <= n), I iterations and a seed:
 *   training rows   the first min(n, 256 L) rows in the order of (mix32(key ^ row), row) ascending, mix32 the lowbias32 hash and
 *                   key = (seed * 0x9E3779B1 + 0x7F4A7C15) mod 2^32 (gnm_map_init's key);
 *   initial         centroid l = training row l of that order, normalised (gnm_ivf_normalize);
 *   each iteration  every training row is assigned its k = 1 centroid under s, the row as the query (gnm_embedding_neighbours);
 *                   the normalised training rows are stably sorted by list and centroid l = normalise(sum of its rows in that
 *                   order) (gnm_ivf_centroids); then, in ascending list order, each empty list takes as its centroid the
 *                   normalised training row, not yet taken, of lowest best similarity (ties: the lowest row);
 *   layout          every reference row is assigned as above; rows [n] int64 = the rows in (list, row) order, offsets [L + 1].
 * The same rows, L, I and seed give a bitwise identical index.
 *
 * Search: probes(q) = q's top-nprobe centroids under the total order (gnm_embedding_neighbours of the queries against the
 * centroids, 1 <= nprobe <= min(64, L)); the result is the top-k under the total order of {(s(q, r), r) : r in a probed list,
 * r not q's self index}, padded with (-inf, -1).  At nprobe = L it is bitwise gnm_embedding_neighbours; it does not depend on the
 * query order, the query or reference chunking, or the GPU count.
 *
 * gnm_ivf_normalize: d_out [n][512] = each row / its fp64 norm, rounded to fp32 (a zero row stays zero), as gnm_map_pca's x^.
 * gnm_ivf_centroids: d_centroids [lists][512] = the normalised fp32 sums (row order) of the rows d_xhat[d_offsets[l] ..
 *   d_offsets[l + 1]) (int32 offsets [lists + 1]); an empty list gives the zero row.  d_sums [lists][512] is scratch.
 * gnm_ivf_prepare: d_hi, d_lo [n][512] = the TF32 halves of gnm_embedding_neighbours' operands (the row normalised by its fp32
 *   norm, then split), row by row: a reference chunk's halves, made once and searched by any number of gnm_ivf_search calls.
 * gnm_ivf_search: one reference chunk of an index against the live (query, list) pairs of some queries.
 *   d_ref_hi / d_ref_lo [n_ref][512]   gnm_ivf_prepare of reference rows in list order, list l at rows [h_offsets[l],
 *                                      h_offsets[l + 1]) (h_offsets: HOST int64 [lists + 1] from 0 to n_ref, checked before any
 *                                      launch), with global indices d_ref_index [n_ref] (DEVICE int64) ascending within each list;
 *   d_pair_query, d_pair_list [n_pairs] DEVICE int32: pair e asks for the rows of list d_pair_list[e] for query d_pair_query[e],
 *                                      in ascending query order; each (query, list) at most once.  A pair whose list is outside
 *                                      [0, lists) or whose query is outside [0, n_query) is dropped.
 *   result  d_sim / d_idx [n_query][k]: for query q of d_query [n_query][512], the top-k under the total order of the rows of its
 *           pairs' lists, global indices from d_ref_index, excluding global index self_index0 + q when self_index0 >= 0; a query
 *           without pairs gets a padded list.
 *   1 <= k <= 64, n_pairs, n_query, n_ref <= 2^30.  Asynchronous; d_work 256-byte aligned.
 * gnm_ivf_search_workspace_bytes: the bytes of d_work a call with n_pairs pairs needs (0 on invalid arguments): each pair's query
 *   row and halves (6 KB) and a partial list of 8 k bytes per 1,536-row range of the longest list, whatever the pairs are.
 */
int gnm_ivf_normalize(const float* d_rows, int64_t n, float* d_out, void* stream);
int gnm_ivf_centroids(const float* d_xhat, const int32_t* d_offsets, int lists, float* d_sums, float* d_centroids, void* stream);
int gnm_ivf_prepare(const float* d_rows, int64_t n, float* d_hi, float* d_lo, void* stream);
size_t gnm_ivf_search_workspace_bytes(int64_t n_pairs, int64_t n_ref, const int64_t* h_offsets, int lists, int k);
int gnm_ivf_search(const float* d_query, int64_t n_query, const int32_t* d_pair_query, const int32_t* d_pair_list, int64_t n_pairs,
                   const float* d_ref_hi, const float* d_ref_lo, int64_t n_ref, const int64_t* h_offsets, int lists,
                   const int64_t* d_ref_index, int64_t self_index0, int k, float* d_sim, int64_t* d_idx, void* d_work,
                   size_t work_bytes, void* stream);

/*
 * Growing lists: the search of a clustering through an index (embedding-clusters --index), whose lists of representatives grow
 * block by block.  The representatives live in slots laid out like the index: list l owns slots [h_offsets[l], h_offsets[l + 1])
 * (HOST int64 [lists + 1] from 0 to n_slots, the index offsets: the capacities), and holds at any time the prefix
 * [h_offsets[l], d_end[l]) (DEVICE int64 [lists], clamped to the list's slots), filled in ascending global index.  Appending
 * writes only the new slots' halves (gnm_ivf_prepare): nothing placed earlier moves.
 * gnm_ivf_search_ranges: gnm_ivf_search with list l read as [h_offsets[l], d_end[l]) and no self-exclusion; d_slot_hi / d_slot_lo
 *   [n_slots][512] are the slots' halves, d_slot_index [n_slots] their global indices (read only inside the prefixes).  Same
 *   pairs, order, padding and bitwise similarities as gnm_ivf_search; it runs the same kernels, instantiated to read d_end.
 * gnm_ivf_search_ranges_workspace_bytes: as gnm_ivf_search_workspace_bytes, sized from the capacities, so it holds for any d_end
 *   and the caller needs no device-to-host copy of the ends.
 */
size_t gnm_ivf_search_ranges_workspace_bytes(int64_t n_pairs, int64_t n_slots, const int64_t* h_offsets, int lists, int k);
int gnm_ivf_search_ranges(const float* d_query, int64_t n_query, const int32_t* d_pair_query, const int32_t* d_pair_list,
                          int64_t n_pairs, const float* d_slot_hi, const float* d_slot_lo, int64_t n_slots, const int64_t* h_offsets,
                          const int64_t* d_end, int lists, const int64_t* d_slot_index, int k, float* d_sim, int64_t* d_idx,
                          void* d_work, size_t work_bytes, void* stream);

/*
 * Embedding clusters: one block step of greedy clustering at a cosine threshold t.  Rows are processed in file order, block by
 * block; row j is a representative iff s(j, i) < t for every representative i < j, where s(a, b) is the similarity
 * gnm_embedding_neighbours returns for QUERY row a and REFERENCE row b (s is not bitwise symmetric: the row being placed is
 * always the query, the candidate representative always the reference).  Same rules as the neighbour calls: no handle, no
 * allocation, the current device and `stream`.  DESIGN.md, "Embedding clusters".
 *
 * The caller finds the covered rows of the block, those whose best representative of earlier blocks has s >= t, with
 * gnm_embedding_neighbours at k = 1 against those representatives; this call decides the rest against the block itself:
 *   d_rows          DEVICE float [n_block][512], 16-byte aligned: the block's rows in file order.
 *   d_covered       DEVICE uint8 [n_block]: nonzero = covered by a representative of an earlier block.
 *   min_similarity  t in (0, 1] (fp32).
 *   d_new_reps      DEVICE int32 [n_block]: the block's new representatives, block-local rows, ascending; row j is one iff it is
 *                   not covered and s(j, i) < t for every new representative i < j of the block.
 *   d_n_new         DEVICE int32 [1]: their count.
 * Each in-block comparison s(j, i) >= t is computed by the search's own tensor-core mainloop, so it is bitwise the comparison of
 * the similarity gnm_embedding_neighbours returns for that pair.  A zero row has s = 0 with every row, so it is never covered
 * and never covers.
 *
 * gnm_cluster_block_workspace_bytes: the bytes of d_work (256-byte aligned) a block of n_block rows needs (0 on invalid
 *   arguments, and for n_block = 0): TF32 halves of the rows (4 KB per row) and the threshold mask (n_block * ceil(n_block / 32)
 *   words; 8 MB at the largest block).  0 <= n_block <= 8192.
 */
size_t gnm_cluster_block_workspace_bytes(int64_t n_block);
int gnm_cluster_block(const float* d_rows, int64_t n_block, const uint8_t* d_covered, float min_similarity, int32_t* d_new_reps,
                      int32_t* d_n_new, void* d_work, size_t work_bytes, void* stream);

/*
 * Clustering through an index (embedding-clusters --index; DESIGN.md, "Embedding clusters through the index").  With home(i) the
 * list the index places row i in and P(j) row j's nprobe nearest centroids under the total order (P(j)[0] = home(j)):
 *   row j is a representative iff s(j, i) < t for every representative i < j with home(i) in P(j);
 *   every other row joins the first representative under the total order among the representatives i with home(i) in P(j).
 * At nprobe = L this is the exact greedy clustering above.  The caller finds the covered rows with gnm_ivf_search_ranges at k = 1
 * against the earlier blocks' representatives in the row's probed lists.
 * gnm_cluster_block_probed: gnm_cluster_block, except that the in-block comparison (j, i) counts only when home(i) is one of j's
 *   probes: d_probes DEVICE int32 [n_block][nprobe] (row j's probes), d_home DEVICE int32 [n_block], 1 <= nprobe <= 64.  The
 *   threshold mask is the same; a filter kernel clears its other bits before the rows are decided.  Workspace:
 *   gnm_cluster_block_workspace_bytes.
 */
int gnm_cluster_block_probed(const float* d_rows, int64_t n_block, const uint8_t* d_covered, float min_similarity,
                             const int32_t* d_probes, int nprobe, const int32_t* d_home, int32_t* d_new_reps, int32_t* d_n_new,
                             void* d_work, size_t work_bytes, void* stream);

/*
 * Embedding map: the stages of a 2-D UMAP layout (McInnes, Healy & Melville 2018) of n rows, 2 <= n <= 2^30, as umap-learn
 * computes it with min_dist = 0.1 and spread = 1 (a = 1.57694346, b = 0.89506088), except where marked (dev).  DESIGN.md,
 * "Embedding map".  No handle, no allocation: the current device, `stream` and the caller's buffers, all DEVICE.  Asynchronous.
 *
 * gnm_map_membership: from the all-vs-all lists of gnm_embedding_neighbours at k (1 <= k <= min(64, n - 1)), d_sim [n][k] and
 *   d_idx [n][k], with d = 1 - s in fp64 (a zero row has s = 0 with every row, so its d is 1 everywhere and its list is the
 *   lowest indices):
 *     d_mean_d [1]     the mean d over all n k entries, summed in a fixed order;
 *     d_rho [n]        the smallest d > 0 of the row, 0 if none;
 *     d_sigma [n]      umap-learn's smooth_knn_dist bisection (64 steps, exit at |sum - target| < 1e-5, sigma doubled while the
 *                      upper end is infinite) for sum_p f(d_ip - rho_i) = log2(k + 1), f(x) = exp(-x / sigma) for x > 0, else 1;
 *                      then at least 1e-3 x the row's mean d, or x mean_d when rho_i = 0;
 *     d_w [n][k]       w_ip = f(d_ip - rho_i) (fp64);
 *     d_union [n][k]   for j = idx[i][p]: a + b - a b with a = w_ip and b = w_jq where idx[j][q] = i (0 if i is not in j's list),
 *                      at the entry that emits the unordered pair {i, j} (the lower index when the entries are mutual, else the
 *                      row that holds it), and -1 at every other entry.
 * gnm_map_pca: (dev: a PCA initialisation, not spectral) d_xhat [n][512] fp32 = each row / its fp64 norm (a zero row stays
 *   zero); d_center [512] and d_S [512][512] (fp64), the mean and covariance (1/n) sum (x^ - center)(x^ - center)^T from the
 *   novelty fit's kernels at one class; d_V [2][512] (fp64), the top-2 eigenvectors of S by a fixed-step subspace iteration
 *   from a fixed start, each signed so its largest-magnitude component is positive.  S = 0 leaves V at the start vectors.
 *   gnm_map_pca_workspace_bytes(n): the bytes of d_work (256-byte aligned) it needs; 0 on invalid n.
 * gnm_map_init: d_Y [n][2] fp32, the initial layout: p = (x^ - center) . v_c in fp64 (workspace bytes [0, 16 n)), scaled by
 *   10 / max |p| (skipped when max |p| = 0) and rounded to fp32, plus (dev) the fp32 noise
 *   (mix32(mix32(key ^ row) + axis) - 2^31 + 0.5) * 1e-4 / 2^31 with mix32 the lowbias32 hash and key = (seed * 0x9E3779B1 +
 *   0x7F4A7C15) mod 2^32; then each axis mapped to [0, 10] by 10 (y - min) / (max - min) in fp32.
 *   gnm_map_init_workspace_bytes(n): the bytes of d_work (256-byte aligned) it needs; 0 on invalid n.
 * gnm_map_epochs: epochs e_begin .. e_end - 1 of `epochs` (dev: synchronous) on the CSR graph d_row_ptr [n + 1] int64,
 *   d_col [nnz] int32 (both directions of every edge, each row sorted by column) and d_eps [nnz] fp64, the epochs per sample
 *   max w / w.  Epoch e reads Y and writes the next Y: vertex i adds, in fp32 per term and in a fixed order, over each entry
 *   (i, j) at CSR position p sampled at e (e >= 1 and floor(e / eps) > floor((e - 1) / eps) in fp64):
 *     twice the attraction clip(-2ab d^(2(b-1)) / (1 + a d^2b) (y_i - y_j), +-4) (0 when d = 0), and
 *     (dev) for s = 0..4 the repulsion of vertex m = mix32(mix32(mix32(key ^ e) + p mod 2^32) + s) mod n, skipped when m = i:
 *     clip(2b / ((0.001 + d^2)(1 + a d^2b)) (y_i - y_m), +-4) (0 when d = 0);
 *   then y_i += (1 - e / epochs) x the sum.  No atomics: the result is bitwise reproducible.  Epoch 0 samples nothing.  d_Y
 *   holds the result; d_Y_tmp [n][2] is the second buffer.
 */
int gnm_map_membership(const float* d_sim, const int64_t* d_idx, int64_t n, int k, double* d_mean_d, double* d_rho,
                       double* d_sigma, double* d_w, double* d_union, void* stream);
size_t gnm_map_pca_workspace_bytes(int64_t n);
int gnm_map_pca(const float* d_rows, int64_t n, float* d_xhat, double* d_center, double* d_S, double* d_V, void* d_work,
                size_t work_bytes, void* stream);
size_t gnm_map_init_workspace_bytes(int64_t n);
int gnm_map_init(const float* d_xhat, int64_t n, const double* d_center, const double* d_V, uint64_t seed, float* d_Y,
                 void* d_work, size_t work_bytes, void* stream);
int gnm_map_epochs(const int64_t* d_row_ptr, const int32_t* d_col, const double* d_eps, int64_t n, int epochs, int e_begin,
                   int e_end, uint64_t seed, float* d_Y, float* d_Y_tmp, void* stream);

/*
 * Window regions: an HMM decode of each sequence's window-score profile (nn-classification --write-window-scores, or a head's)
 * into class regions.  No handle, no allocation: the current device and `stream`, the caller's workspace.  Asynchronous.
 * DESIGN.md, "Window regions" states the model; in short, for sequence windows w = 0..n-1 with scores p_w in R^C, starts a_w,
 * lengths l_w, stride s and mean region length L:
 *   states      one per class, uniform start;  emission eps_w(k) = (s / 6000) ln max(p_w(k), 1e-30)
 *   transition  rho = s / L, lambda = 1 - rho C / (C - 1), g_w = (a_w - a_{w-1}) / s;  stay T_g = 1/C + (1 - 1/C) lambda^g,
 *               move to a given other class (1 - T_g) / (C - 1)
 *   outputs     forward-backward posteriors gamma_w(k) and the Viterbi path (ties: stay, then the lowest class; the final state
 *               the lowest class); a region is a maximal run of equal path states, from a_0 or the floor of the midpoint of the
 *               neighbouring window centres c = a + floor(l / 2), to the next such midpoint or a_{n-1} + l_{n-1}.
 * All recursions run in fp64.  A sequence's results depend only on its own windows: bitwise the same in any call or order.
 *
 *   d_scores       DEVICE float [n_windows][C], finite (not checked: the caller validates)
 *   d_offsets      DEVICE int32 [n_seqs + 1], non-decreasing: sequence i has the rows [d_offsets[i], d_offsets[i+1]) - d_offsets[0]
 *                  of every per-window buffer, so a call can take any run of whole sequences of a larger CSR
 *   d_start        DEVICE int64 [n_windows]: 0-based first base; within a sequence increasing by positive multiples of `stride`
 *                  (not checked: a violation gives wrong results, never an out-of-bounds access)
 *   d_length       DEVICE int32 [n_windows]: bases of sequence in the window, >= 1
 *   d_posterior    DEVICE float [n_windows][C]: gamma;  d_state DEVICE int32 [n_windows]: the Viterbi path
 *   d_region_first DEVICE uint8 [n_windows]: 1 at the first window of each region, 0 elsewhere.  At those rows only:
 *                  d_region_start / d_region_end DEVICE int64 (0-based, end exclusive), d_region_windows DEVICE int32 (window
 *                  count), d_region_posterior DEVICE float (mean gamma of the region's class, an fp64 sum in window order),
 *                  d_region_scores DEVICE float [n_windows][C] (mean score of every class, fp64 sums in window order); the
 *                  region's class is d_state at that row.  Compacting the flagged rows in order gives the region table.
 *   2 <= C <= 32, 1 <= stride <= 6000, mean_region_length >= 12000 (so rho <= 0.5), 0 <= n_windows < 2^31; any other value or a
 *   null buffer (when n_windows > 0) fails without launching.
 *
 * gnm_window_regions_workspace_bytes: the bytes of d_work (256-byte aligned) a call with n_windows windows of C classes needs
 *   (0 on invalid arguments): 8 C + 6 bytes per window, each part rounded up to 256 bytes.
 */
size_t gnm_window_regions_workspace_bytes(int64_t n_windows, int C);
int gnm_window_regions(const float* d_scores, int64_t n_windows, int C, const int32_t* d_offsets, int n_seqs,
                       const int64_t* d_start, const int32_t* d_length, int stride, double mean_region_length, float* d_posterior,
                       int32_t* d_state, uint8_t* d_region_first, int64_t* d_region_start, int64_t* d_region_end,
                       int32_t* d_region_windows, float* d_region_posterior, float* d_region_scores, void* d_work,
                       size_t work_bytes, void* stream);

/*
 * Classifier heads: the layers the reference trains on the frozen encoder (create_classifier, model.py:34-45), with C classes
 * instead of 3.  DESIGN.md, "Classifier heads".  Host pointers, Keras layouts; 2 <= n_classes <= 32.
 */
typedef struct gnm_head_weights {
  int n_classes;               /* C */
  const float* dense1_kernel;  /* [512][512] */
  const float* dense1_bias;    /* [512] */
  gnm_bn_weights bn1;          /* batch_normalization_1 (epsilon 1e-3) */
  const float* dense2_kernel;  /* [512][C] */
  const float* dense2_bias;    /* [C] */
} gnm_head_weights;
typedef struct gnm_head_train gnm_head_train;   /* gnm_head: declared with the head attributions */

/*
 * Upload a head for inference on handle h's device.  BN is folded into scale and shift and dense_1 split into TF32 halves with
 * the host code gnm_create uses for the shipped head.  Refuses (naming the array and index) an array that is not finite, and a
 * moving variance with var + 1e-3 <= 0 in fp32, where the folded scale 1 / sqrt(var + 1e-3) would be NaN or infinite;
 * gnm_head_train_create refuses the same.  Synchronous.
 */
int gnm_head_create(gnm_handle* h, const gnm_head_weights* w, gnm_head** out);
int gnm_head_destroy(gnm_head* head);

/*
 * Encoder embeddings DEVICE float [n][512] (gnm_embed_*) -> probabilities DEVICE float [n][C].  Steps of max_batch rows on the
 * handle's head workspace, in `stream` order (so not concurrently with other calls on h), following h's conv_impl: 0 splits
 * the rows into TF32 halves (the bits the forward pass writes for its dense_1) and runs the forward pass's 3 x TF32 dense_1
 * GEMM + BN + ReLU; 1 runs the FFMA dense_1 kernel.  Both end in a C-class softmax with dense3's k order, shuffle tree and
 * max / exp / sum / multiply sequence, so the shipped head at C = 3 gives bitwise the probabilities of gnm_forward_*.
 */
int gnm_head_forward(gnm_handle* h, const gnm_head* head, const float* d_embed, int n, float* d_probs, void* stream);

/*
 * gnm_segment_mean / gnm_segment_sum for rows of C columns (1 <= C <= 32): float [n_contigs][C] means, or [n_contigs][C + 1]
 * = (sums, count).  One fp32 running sum per column in window order, so C = 3 gives the bits of gnm_segment_*.
 */
int gnm_head_segment_mean(gnm_handle* h, const float* d_probs, int C, const int32_t* d_offsets, int n_contigs, float* d_mean,
                          void* stream);
int gnm_head_segment_sum(gnm_handle* h, const float* d_probs, int C, const int32_t* d_offsets, int n_contigs, float* d_sum,
                         void* stream);

/*
 * Head novelty: a Gaussian model of the embeddings a head was trained on, one mean per class and one shared covariance (Lee et
 * al. 2018).  DESIGN.md, "Head novelty".  All of it in fp64, in a fixed order without atomics: a fit is bitwise reproducible
 * for the same rows, and a row's distances do not depend on the batch it is scored in, its position there or n.
 *   fit rows      x_i = d_X[d_idx[r]] (float [512], the gnm_embed_* rows), label y_i = d_labels[d_idx[r]] in [0, C), r < n_fit
 *   means         mu_c = mean of class c's rows (block sums of 4096 rows, combined in block order);  N_c = 0 is an error
 *                 center = (sum over c, in class order, of the class sums) / N
 *   scatter       S = (1/N) sum_i (x_i - mu_{y_i})(x_i - mu_{y_i})^T, two-pass (x - mu centred in fp64 as the DMMA operand is
 *                 loaded); lower 64 x 64 tiles only, K in chunks of 8192 rows combined in chunk order; S exactly symmetric
 *   shrinkage     Sigma = (1 - 0.01) S + 0.01 (tr S / 512) I;  tr S = 0 is an error ("no within-class variation"), and so
 *                 is a non-finite tr S ("a fit row has a non-finite value": a NaN or an infinity in a fit row)
 *   whitening     Sigma = L L^T (Cholesky, right-looking, one CTA; a pivot that is not > 0 is an error naming its column);
 *                 P = L^-1 (lower triangular, forward substitution per column, k ascending)
 *   whitened means  m_c = P (mu_c - center)
 *   distance      D_c(x) = || P (x - center) - m_c ||^2 / 512 = || P (x - mu_c) ||^2 / 512 (about 1 for a typical training
 *                 row), fp64, stored as float
 *
 * gnm_novelty_fit_workspace_bytes: bytes of d_work (256-byte aligned) for n_fit rows and C classes (0 on bad arguments);
 *   about n_fit * (C * 512 * 8 / 4096 + 36 * 4096 * 8 / 8192) bytes + 6.3 MB.
 * gnm_novelty_fit: d_X DEVICE float [n_rows][512], d_idx DEVICE int64 [n_fit] (rows of d_X), d_labels DEVICE int32 [n_rows]
 *   (the d_idx / d_labels form of gnm_head_train_step).  Waits for `stream` and writes HOST fp64 arrays (any may be NULL):
 *   h_center [512], h_whitening [512][512] = P (zeros above the diagonal), h_means [C][512] = m_c, h_min_pivot = the smallest
 *   Cholesky pivot (a diagonal of Sigma after the earlier columns' updates, before its square root), and, for tests,
 *   h_class_means [C][512] = mu_c and h_scatter [512][512] = S.  An index outside [0, n_rows), a label outside [0, C) or a
 *   NaN or infinity in a fit row fails, each with its own message; the handle stays usable.
 * gnm_head_set_novelty: attach a model (HOST fp64 center [512], whitening [512][512] lower triangular with a positive diagonal,
 *   means [C][512] whitened) to a head; refuses non-finite values and a malformed whitening, naming the index.  Synchronous.
 * gnm_head_novelty: embeddings DEVICE float [n][512] -> D DEVICE float [n][C] for the head's model.  One CTA per 64 rows:
 *   Y = (x - center) P^T by DMMA in 64-column tiles in order (the k tiles above the diagonal skipped), each followed by an
 *   epilogue adding sum_j (Y_j - m_cj)^2 over the tile's columns in order into a per-(row, class) fp64 sum; divided by 512.
 *   Asynchronous on `stream`.  Per-sequence values: gnm_head_segment_mean of the rows.
 */
size_t gnm_novelty_fit_workspace_bytes(int64_t n_fit, int C);
int gnm_novelty_fit(gnm_handle* h, const float* d_X, int64_t n_rows, const int64_t* d_idx, int64_t n_fit, const int32_t* d_labels,
                    int C, double* h_center, double* h_whitening, double* h_means, double* h_min_pivot, double* h_class_means,
                    double* h_scatter, void* d_work, size_t work_bytes, void* stream);
int gnm_head_set_novelty(gnm_handle* h, gnm_head* head, const double* center, const double* whitening, const double* means);
int gnm_head_novelty(gnm_handle* h, const gnm_head* head, const float* d_embed, int n, float* d_dist, void* stream);

/*
 * Head training on cached embeddings (no encoder gradients).  Semantics, Keras 3 defaults with the reference's stack:
 *   training forward  z1 = x W1 + b1;  mu, var = batch mean and biased batch variance of z1 (per column);
 *                     y = gamma (z1 - mu) / sqrt(var + 1e-3) + beta;  h = relu(y) * keep / 0.8;  logits = h W2 + b2
 *   dropout           keep(seed, step, row, col) = mix32(mix32(mix32(K(seed) ^ step) + row) + col) >= ceil(0.2 * 2^32),
 *                     mix32 = lowbias32, K(seed) = (seed * 0x9E3779B1 + 0x7F4A7C15) mod 2^32 (genomad_b200/synth.py),
 *                     step = the 0-based global step, row = the position in the batch; arithmetic mod 2^32
 *   loss              sum_i w[y_i] * (-log softmax(logits_i)[y_i]) / B  (log-softmax from the logits, max-shifted:
 *                     -log softmax_y = (max - l_y) + log1p(sum_{c != a} exp(l_c - max)), a the lowest class at the max; the
 *                     gradient's target component is -sum_{c != y} p_c, never p_y - 1, so neither cancels when p_y is near 1)
 *   Adam              t = step + 1; m += (g - m)(1 - 0.9); v += (g^2 - v)(1 - 0.999);
 *                     p -= (m * lr sqrt(1 - 0.999^t) / (1 - 0.9^t)) / (sqrt(v) + 1e-7), over W1, b1, gamma, beta, W2, b2; no decay
 *   moving stats      mean = 0.99 mean + 0.01 mu;  var = 0.99 var + 0.01 var_batch (biased)
 * Every reduction (over the batch or over k) runs in a fixed order without atomics: a run is bitwise reproducible for a seed
 * on one device model.
 *
 * gnm_head_train_create: `init` holds the initial parameters and moving statistics (the caller draws them); seed keys the
 *   dropout; max_batch in [1, 65536] bounds B.  Adam moments start at zero.  Synchronous.
 * gnm_head_train_step: one step on the batch rows d_idx (DEVICE int64 [B], indices into d_X) of d_X (DEVICE float
 *   [n_rows][512], the embeddings of the whole training set); d_labels DEVICE int32 [n_rows] (label of each row of d_X, in
 *   [0, C)); d_class_weights DEVICE float [C]; 1 <= B <= max_batch.  Writes the batch loss to d_loss (DEVICE float [1]).
 *   Asynchronous on `stream`.  An index outside [0, n_rows) or a label outside [0, C) is not read: the step flags it (and uses
 *   row 0 / class 0), and the next gnm_head_train_step or gnm_head_train_read fails naming which; the trainer is then spent.
 * gnm_head_train_read: waits for `stream` and copies the parameters to HOST buffers (any may be NULL): h_params float
 *   [512*512 + 3*512 + 512*C + C] flat = W1, b1, gamma, beta, W2, b2; moving mean and variance [512]; the step count.
 * gnm_head_train_fetch (tests): HOST copy of the last step's "grad" (float, flat like h_params), "adam_m" and "adam_v" (the
 *   Adam moments after the step, float, flat like h_params), "mask" (uint8 [B][512], 1 = kept) or "batch_stats" (float [3][512]
 *   = mu, 1 / sqrt(var + 1e-3), var).  Waits for `stream`.
 */
int gnm_head_train_create(int device, const gnm_head_weights* init, int max_batch, uint64_t seed, float learning_rate,
                          gnm_head_train** out);
int gnm_head_train_destroy(gnm_head_train* tr);
int gnm_head_train_step(gnm_head_train* tr, const float* d_X, int64_t n_rows, const int64_t* d_idx, const int32_t* d_labels,
                        const float* d_class_weights, int B, float* d_loss, void* stream);
int gnm_head_train_read(gnm_head_train* tr, float* h_params, float* h_moving_mean, float* h_moving_variance, long long* h_step,
                        void* stream);
int gnm_head_train_fetch(gnm_head_train* tr, const char* which, void* h_dst, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GNM_H_ */
