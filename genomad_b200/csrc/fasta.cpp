// Native, streaming FASTA -> window front end of the nn-classification path (host code, part of libgnm.so).
//
// Behavioural mirror (not a translation) of what the reference does per record in Python:
//   read_fasta(strip_n=True)   genomad/sequence.py:96-121   text mode => universal newlines: "\r\n" and "\r" end a
//                              line like "\n"; text before the first line starting with '>' is ignored; the record's
//                              sequence is every byte of its lines except the line terminators; leading/trailing
//                              'n'/'N' of the whole contig are stripped; records that are then empty are dropped
//   seq_windows(6000, 2500)    genomad/sequence.py:150-167   consecutive 6000-nt slices; a shorter last slice is kept
//                              only if >= 2500 nt, except that the first window is always kept; max_windows=1 for
//                              --single-window
//   N rule / pad / upper-case  genomad/modules/nn_classification.py:70-72   a window other than the first is skipped if
//                              its RAW text holds more than 4000 upper-case 'N'; windows are upper-cased (ASCII) and
//                              right-padded with 'N' to 6000 bytes
// Golden vectors produced with the real reference code pin all of this (tests/golden/encoder_golden.json,
// tests/test_host_cpu.py::test_native_fasta_*).
//
// Round-2 design: INDEX, then STREAM.  Nothing is copied or compacted up front and the file is never held in
// anonymous memory:
//   * the text is either an mmap of the file (gnm_fasta_open: plain FASTA; pages come from the page cache and are
//     released behind the export cursor with madvise) or caller memory (gnm_fasta_parse: decompressed input);
//   * the index pass is multi-threaded twice over: header lines ('>' at a line start) are found per byte range,
//     then records are indexed in parallel -- line layout (nucleotides per line + stride, or "irregular"), leading /
//     trailing n/N strip, sequence length, window count incl. the N rule.  It keeps O(records) state: ~100 bytes per
//     record, plus 8 bytes per window only for records whose lines are irregular and 4 bytes per window only for
//     records that lost a window to the N rule;
//   * gnm_fasta_export_windows(first, count) produces any block of the GLOBAL window list straight from the text into
//     caller memory (a pinned chunk): binary search for the record, file offset of the window start by arithmetic,
//     line-by-line copy, upper-case, pad.  Under torchrun every rank builds the same index (cheap, deterministic,
//     no communication) and extracts only its own contiguous block of windows.
//   * a window list (gnm_fasta_windows) is one enumeration over the index: candidate k of a record starts k * step nt into
//     its stripped sequence and is min(6000, L - k * step) long; the first is always kept, every other one if it has >= 2500 nt
//     and <= 4000 'N'.  The index pass builds the reference's list (step 6000, --single-window or not); gnm_fasta_windows_plan
//     builds a list at any step in [1, 6000] (overlapping windows of a score profile) over the same index.  A list keeps
//     ~16 bytes per record, 8 bytes per candidate window only for records whose lines are irregular and 4 bytes per window
//     only for records that lost a window to the N rule: at most 12 bytes per window, 12 MB for a 1 Gbp input at step 1000.
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cerrno>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include "../../include/gnm.h"

#if defined(__has_include)
#if __has_include(<zlib.h>)
#include <zlib.h>
#define GNM_HAVE_ZLIB 1
#endif
#endif

namespace {

constexpr int64_t kWin = GNM_WINDOW, kMinTail = 2500, kMaxN = 4000;

struct Record {
  int64_t hdr_begin, hdr_end;      // header text (without '>' and terminator)
  int64_t body_begin, body_end;    // raw body bytes (with terminators)
  int64_t raw_len;                 // nucleotides (non-terminator bytes) in the body
  int64_t lead;                    // leading n/N stripped
  int64_t seq_len;                 // length after stripping both ends (0 => record dropped)
  int64_t line_len, stride;        // regular layout: every line but the last holds line_len nucleotides and starts
                                   // stride bytes after the previous one; stride == 0 => irregular (see win_off)
  uint8_t has_cr;                  // body contains '\r' (byte-wise line walking)
};

inline bool is_eol(uint8_t c) { return c == '\n' || c == '\r'; }

template <class F>
void parallel_for(int64_t n, int threads, F fn) {
  threads = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(threads, n)));
  if (threads == 1) { for (int64_t i = 0; i < n; ++i) fn(i); return; }
  std::atomic<int64_t> next{0};
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&] { for (int64_t i; (i = next.fetch_add(1)) < n;) fn(i); });
  for (auto& th : pool) th.join();
}

inline int64_t count_N(const uint8_t* p, int64_t n) {
  int64_t c = 0;
  for (int64_t i = 0; i < n; ++i) c += (p[i] == 'N');
  return c;
}

// Calls fn(line_start, line_end) for every line of the record's body (terminators excluded; "\r\n" is one terminator).
template <class F>
void walk_lines(const uint8_t* t, const Record& R, F&& fn) {
  const int64_t b0 = R.body_begin, b1 = R.body_end;
  int64_t i = b0;
  if (!R.has_cr) {
    while (i < b1) {
      const void* q = std::memchr(t + i, '\n', static_cast<size_t>(b1 - i));
      const int64_t j = q ? static_cast<const uint8_t*>(q) - t : b1;
      fn(i, j);
      i = j + 1;
    }
  } else {
    while (i < b1) {
      int64_t j = i;
      while (j < b1 && !is_eol(t[j])) ++j;
      fn(i, j);
      if (j < b1 && t[j] == '\r' && j + 1 < b1 && t[j + 1] == '\n') ++j;      // "\r\n" is one terminator
      i = j + 1;
    }
  }
}

}  // namespace

// One window list over the index (see the top of the file).  Kept records are numbered in file order.
struct gnm_fasta_windows {
  const gnm_fasta* f = nullptr;
  int64_t step = kWin;
  int single_window = 0;
  int reverse = 0;                              // windows of the reverse complement (see reverse_begin)
  int64_t n_windows = 0;
  std::vector<int64_t> first;                   // per kept record: its first window in the list (sorted: window -> record)
  std::vector<int32_t> off_idx, kept_idx;       // per kept record: index into win_off / kept_wins, or -1
  std::vector<std::vector<int64_t>> win_off;    // irregular records: file offset of the start of every candidate window
  std::vector<std::vector<int32_t>> kept_wins;  // records that lost windows to the N rule: candidate numbers kept
  // bytes of the mapping this list's stream has handed back (madvise): each list streams the file from its start, so each
  // keeps its own mark (a second pass re-faults the pages a first pass released, and must release them again)
  mutable std::atomic<int64_t> released{0};
};

struct gnm_fasta {
  const uint8_t* text = nullptr;
  int64_t len = 0;
  int single_window = 0;
  void* map_base = nullptr;        // mmap'ed file (gnm_fasta_open) or nullptr (caller memory)
  size_t map_len = 0;
  std::unique_ptr<uint8_t[]> owned;   // inflated text of a gzip input (gnm_fasta_open_gz)
  std::vector<Record> recs;        // every record found (before dropping empties)
  std::vector<int64_t> kept;       // indices of records whose stripped sequence is non-empty
  gnm_fasta_windows windows;       // the reference's window list (step 6000, single_window)
  int64_t n_nonempty_raw = 0;      // records with a non-empty sequence before stripping (what check_fasta counts)
  int has_dup = 0;
};

static thread_local std::string g_fasta_err;
extern "C" const char* gnm_fasta_last_error(void) { return g_fasta_err.c_str(); }

// ------------------------------------------------------------------------------------------------ index pass
// One record: walk its lines once.  Everything the reference derives from the joined, stripped string is derived here
// from the line structure without building that string.
static void index_record(gnm_fasta* f, Record& R) {
  const uint8_t* t = f->text;
  const int64_t b0 = R.body_begin, b1 = R.body_end;
  R.has_cr = std::memchr(t + b0, '\r', static_cast<size_t>(b1 - b0)) != nullptr;
  // ---- one pass over the lines: raw length, regularity, leading strip
  int64_t raw = 0, lead = 0;
  bool in_lead = true, regular = true;
  int64_t line_len = -1, stride = 0, nlines = 0, prev_start = -1, prev_len = -1;
  int64_t last_nonstrip_raw = -1;          // raw index of the last byte that is not n/N
  walk_lines(t, R, [&](int64_t ls, int64_t le) {   // one line [ls, le), possibly empty
    const int64_t n = le - ls;
    if (nlines == 0) { line_len = n; }
    else {
      if (nlines == 1) stride = ls - prev_start;
      if (prev_len != line_len || ls - prev_start != stride) regular = false;   // only the LAST line may be shorter
    }
    if (n > line_len && nlines > 0) regular = false;
    if (in_lead) {
      int64_t k = 0;
      while (k < n && (t[ls + k] == 'n' || t[ls + k] == 'N')) ++k;
      lead += k;
      if (k < n) in_lead = false;
    }
    for (int64_t k = n - 1; k >= 0; --k)       // cheap: stops at the first non-N from the right
      if (t[ls + k] != 'n' && t[ls + k] != 'N') { last_nonstrip_raw = raw + k; break; }
    raw += n;
    prev_start = ls; prev_len = n; ++nlines;
  });
  R.raw_len = raw;
  if (last_nonstrip_raw < 0) { R.lead = raw; R.seq_len = 0; }       // nothing but n/N (or empty)
  else { R.lead = lead; R.seq_len = last_nonstrip_raw + 1 - lead; }
  if (line_len <= 0 || nlines <= 1) { regular = regular && line_len > 0; stride = line_len > 0 ? line_len + 1 : 0; }
  if (regular && stride < line_len) regular = false;
  R.line_len = regular ? line_len : 0;
  R.stride = regular ? stride : 0;
}

// Candidate windows of a stripped record of L > 0 nt at window step `step`: 1 + max(0, (L - 2500) / step); at step 6000 this
// is seq_windows(6000, 2500) (sequence.py:150-167).
static inline int64_t candidate_windows(int64_t L, int64_t step, int single_window) {
  return single_window ? 1 : 1 + (L > kMinTail ? (L - kMinTail) / step : 0);
}

// Reverse lists: candidate k is window k of rc(S) -- rc(S)[k step, k step + len_k) with len_k = min(6000, L - k step) -- and
// that is the forward segment [L - k step - len_k, L - k step) of the stripped sequence, read backwards and complemented.
// reverse_begin is that segment's first position (forward lists: k step).  rc maps 'N' to 'N', so the N rule counts the
// segment's 'N' bytes.
static inline int64_t window_len(int64_t L, int64_t step, int64_t k) { return std::min(kWin, L - k * step); }
static inline int64_t segment_begin(int64_t L, int64_t step, int reverse, int64_t k) {
  return reverse ? L - k * step - window_len(L, step, k) : k * step;
}

// One kept record's windows in list p: returns how many are kept; fills *offs (irregular records: file offset of every
// candidate's first byte) and *keptw (only if the N rule dropped one: the candidate numbers kept).  The N count of candidate w
// is the running count of 'N' at its end minus the one at its start; both are taken in one walk over the lines, so
// overlapping windows cost no re-reading.  Only the windows open at one position (<= 6000 / step + 1) keep their start count,
// in a ring, so the walk needs no memory per candidate; a window is kept or dropped as soon as its end is reached.
// The walk takes the candidates in the order of their forward segments: k = 0, 1, .. for a forward list, k = ncand - 1, .., 0
// for a reverse one (both starts and ends then ascend, and window j - ring has still ended before window j starts).
static int64_t plan_record(const gnm_fasta* f, const Record& R, int64_t step, int single_window, int reverse,
                           std::vector<int64_t>* offs, std::vector<int32_t>* keptw) {
  const int64_t L = R.seq_len;
  if (L == 0) return 0;
  const int64_t ncand = candidate_windows(L, step, single_window);
  if (ncand == 1 && R.stride != 0) return 1;   // one window (exempt from the N rule) of a regular record: nothing to walk
  auto cand = [&](int64_t j) { return reverse ? ncand - 1 - j : j; };     // walk position -> candidate number
  auto wbeg = [&](int64_t j) { return segment_begin(L, step, reverse, cand(j)); };
  auto wend = [&](int64_t j) { return wbeg(j) + window_len(L, step, cand(j)); };   // in the stripped sequence
  const bool need_n = ncand > 1;            // the first window is exempt from the N rule
  const bool need_off = R.stride == 0;
  // ring of the running 'N' count at the start of the open windows: window j - ring has ended before window j starts
  // (ring * step > 6000 >= any window's length)
  const int64_t ring = kWin / step + 2;
  std::vector<int64_t> n_start(need_n ? static_cast<size_t>(std::min(ring, ncand)) : 0);
  if (need_off) offs->assign(static_cast<size_t>(ncand), -1);
  std::vector<int32_t> drops;               // candidates the N rule dropped (rare)
  auto decide = [&](int64_t j, int64_t n_count) {
    const int64_t k = cand(j);
    if (k > 0 && n_count > kMaxN) drops.push_back(static_cast<int32_t>(k));
  };
  const uint8_t* t = f->text;
  const int64_t s0 = R.lead, s1 = R.lead + wend(ncand - 1);
  int64_t pos = 0, cnt = 0, ws = 0, we = 0;   // raw index of the line's first byte; running 'N' count; next start / end event
  walk_lines(t, R, [&](int64_t ls, int64_t le) {
    const int64_t n = le - ls;
    int64_t a = std::max(pos, s0) - s0;
    const int64_t e = std::min(pos + n, s1) - s0;    // part of this line inside the windows, in the stripped sequence
    const int64_t base = ls + s0 - pos;              // file offset of stripped position 0 on this line's terms
    if (a < e) {
      for (;;) {                                     // window starts in [a, e) and ends in (a, e], in order
        const int64_t qs = ws < ncand ? wbeg(ws) : INT64_MAX;
        const int64_t qe = need_n && we < ncand ? wend(we) : INT64_MAX;
        const bool is_start = qs < e && qs <= qe;
        if (!is_start && qe > e) break;
        const int64_t q = is_start ? qs : qe;
        if (need_n) cnt += count_N(t + base + a, q - a);
        a = q;
        if (is_start) {
          if (need_n) n_start[static_cast<size_t>(ws % ring)] = cnt;
          if (need_off) (*offs)[static_cast<size_t>(cand(ws))] = base + q;
          ++ws;
        } else {
          decide(we, cnt - n_start[static_cast<size_t>(we % ring)]);
          ++we;
        }
      }
      if (need_n) cnt += count_N(t + base + a, e - a);
    }
    pos += n;
  });
  if (!drops.empty()) {                     // the kept candidate numbers, ascending
    std::sort(drops.begin(), drops.end());
    keptw->reserve(static_cast<size_t>(ncand) - drops.size());
    size_t d = 0;
    for (int64_t k = 0; k < ncand; ++k) {
      if (d < drops.size() && drops[d] == k) ++d;
      else keptw->push_back(static_cast<int32_t>(k));
    }
  }
  return ncand - static_cast<int64_t>(drops.size());
}

// Windows of a stripped record of L nt at `step`, before the N rule (closed form): what a list can hold at most.
static int64_t candidate_total(const gnm_fasta* f, int64_t step, int single_window) {
  int64_t total = 0;
  for (int64_t r : f->kept) total += candidate_windows(f->recs[static_cast<size_t>(r)].seq_len, step, single_window);
  return total;
}

// The window list of every kept record at p->step, records in parallel.
static void build_windows(const gnm_fasta* f, gnm_fasta_windows* p, int threads) {
  const size_t nk = f->kept.size();
  std::vector<std::vector<int64_t>> offs(nk);
  std::vector<std::vector<int32_t>> keptw(nk);
  std::vector<int64_t> nw(nk);
  parallel_for(static_cast<int64_t>(nk), threads, [&](int64_t i) {
    nw[i] = plan_record(f, f->recs[static_cast<size_t>(f->kept[i])], p->step, p->single_window, p->reverse, &offs[i],
                        &keptw[i]);
  });
  p->f = f;
  p->n_windows = 0;
  p->first.resize(nk);
  p->off_idx.assign(nk, -1);
  p->kept_idx.assign(nk, -1);
  for (size_t i = 0; i < nk; ++i) {
    p->first[i] = p->n_windows;
    p->n_windows += nw[i];
    if (!offs[i].empty()) { p->off_idx[i] = static_cast<int32_t>(p->win_off.size()); p->win_off.push_back(std::move(offs[i])); }
    if (!keptw[i].empty()) { p->kept_idx[i] = static_cast<int32_t>(p->kept_wins.size()); p->kept_wins.push_back(std::move(keptw[i])); }
  }
}

static int build_index(gnm_fasta* f, int threads) {
  const uint8_t* text = f->text;
  const int64_t len = f->len;
  threads = std::max(1, threads);
  // ---- header lines: '>' at offset 0 or right after a line terminator, found per byte range
  const int64_t nblk = std::max<int64_t>(1, std::min<int64_t>(threads * 4, (len + (1 << 20) - 1) >> 20));
  std::vector<std::vector<int64_t>> blk_starts(static_cast<size_t>(nblk));
  parallel_for(nblk, threads, [&](int64_t b) {
    const int64_t lo = len * b / nblk, hi = len * (b + 1) / nblk;
    int64_t pos = lo;
    while (pos < hi) {
      const void* p = std::memchr(text + pos, '>', static_cast<size_t>(hi - pos));
      if (!p) break;
      const int64_t i = static_cast<const uint8_t*>(p) - text;
      if (i == 0 || is_eol(text[i - 1])) blk_starts[static_cast<size_t>(b)].push_back(i);
      pos = i + 1;
    }
  });
  std::vector<int64_t> starts;
  for (auto& v : blk_starts) starts.insert(starts.end(), v.begin(), v.end());
  f->recs.resize(starts.size());
  for (size_t r = 0; r < starts.size(); ++r) {
    Record& R = f->recs[r];
    const int64_t rec_end = r + 1 < starts.size() ? starts[r + 1] : len;
    int64_t e = starts[r] + 1;
    const void* q = std::memchr(text + e, '\n', static_cast<size_t>(rec_end - e));
    int64_t nl = q ? static_cast<const uint8_t*>(q) - text : rec_end;
    const void* c = std::memchr(text + e, '\r', static_cast<size_t>(nl - e));      // a lone '\r' also ends the header line
    e = c ? static_cast<const uint8_t*>(c) - text : nl;
    R.hdr_begin = starts[r] + 1; R.hdr_end = e;
    if (e < rec_end && text[e] == '\r' && e + 1 < rec_end && text[e + 1] == '\n') ++e;   // "\r\n" is one terminator
    R.body_begin = std::min(e + 1, rec_end); R.body_end = rec_end;
  }
  // ---- records in parallel
  const size_t nrec = f->recs.size();
  parallel_for(static_cast<int64_t>(nrec), threads, [&](int64_t r) { index_record(f, f->recs[r]); });
  // ---- bookkeeping: kept records, duplicate identifiers (first whitespace-delimited token)
  std::unordered_set<std::string> ids;
  ids.reserve(nrec * 2);
  for (size_t r = 0; r < nrec; ++r) {
    Record& R = f->recs[r];
    if (R.raw_len > 0) {
      ++f->n_nonempty_raw;
      int64_t a = R.hdr_begin, e = R.hdr_end;
      auto ws = [](uint8_t ch) { return ch == ' ' || (ch >= 9 && ch <= 13) || (ch >= 28 && ch <= 31); };
      while (a < e && ws(text[a])) ++a;
      int64_t b = a;
      while (b < e && !ws(text[b])) ++b;
      if (!ids.emplace(reinterpret_cast<const char*>(text + a), static_cast<size_t>(b - a)).second) f->has_dup = 1;
    }
    if (R.seq_len > 0) f->kept.push_back(static_cast<int64_t>(r));
  }
  // ---- the reference's window list
  f->windows.single_window = f->single_window;
  build_windows(f, &f->windows, threads);
  return 0;
}

extern "C" int gnm_fasta_parse(const uint8_t* text, size_t len_, int single_window, int threads, gnm_fasta** out) {
  if (!out || (!text && len_)) { g_fasta_err = "gnm_fasta_parse: null argument"; return 1; }
  gnm_fasta* f = new gnm_fasta();
  f->text = text; f->len = static_cast<int64_t>(len_); f->single_window = single_window;
  build_index(f, threads);
  *out = f;
  return 0;
}

// Plain (uncompressed) FASTA file: mmap + index.  The file is never read into anonymous memory.
extern "C" int gnm_fasta_open(const char* path, int single_window, int threads, gnm_fasta** out) {
  if (!out || !path) { g_fasta_err = "gnm_fasta_open: null argument"; return 1; }
  const int fd = ::open(path, O_RDONLY);
  if (fd < 0) { g_fasta_err = std::string("gnm_fasta_open: cannot open ") + path + ": " + std::strerror(errno); return 1; }
  struct stat st;
  if (::fstat(fd, &st) != 0) { g_fasta_err = "gnm_fasta_open: fstat failed"; ::close(fd); return 1; }
  gnm_fasta* f = new gnm_fasta();
  f->single_window = single_window;
  if (st.st_size > 0) {
    void* m = ::mmap(nullptr, static_cast<size_t>(st.st_size), PROT_READ, MAP_PRIVATE, fd, 0);
    if (m == MAP_FAILED) { g_fasta_err = std::string("gnm_fasta_open: mmap failed: ") + std::strerror(errno); ::close(fd); delete f; return 1; }
    ::madvise(m, static_cast<size_t>(st.st_size), MADV_WILLNEED);
    f->map_base = m; f->map_len = static_cast<size_t>(st.st_size);
    f->text = static_cast<const uint8_t*>(m); f->len = static_cast<int64_t>(st.st_size);
  }
  ::close(fd);
  build_index(f, threads);
  // the index pass touched every page: drop them from the resident set (they stay in the page cache); the streaming phase
  // faults in only what this rank extracts, and gnm_fasta_release_before lets go of it again behind the cursor
  if (f->map_base) ::madvise(f->map_base, f->map_len, MADV_DONTNEED);
  *out = f;
  return 0;
}

// ------------------------------------------------------------------------------------------------ gzip input
// gzip / BGZF FASTA -> text in memory -> index.  A gzip stream cannot be entered in the middle, so compressed input is
// inflated completely (the reference does the same through Python's gzip module, utils.py:155-171); what is native here:
//   * BGZF files (bgzip, the block-compressed gzip dialect of htslib: every <= 64 KB block is its own gzip member and carries
//     its compressed size in a "BC" extra field, its inflated size in its trailer) are inflated block-parallel on `threads`
//     threads straight into their final positions;
//   * plain gzip (single or concatenated members) is inflated sequentially by zlib with the output pre-sized from the trailer.
extern "C" int gnm_fasta_open_gz(const char* path, int single_window, int threads, gnm_fasta** out) {
  if (!out || !path) { g_fasta_err = "gnm_fasta_open_gz: null argument"; return 1; }
#ifndef GNM_HAVE_ZLIB
  g_fasta_err = "gnm_fasta_open_gz: libgnm was built without zlib";
  return 1;
#else
  const int fd = ::open(path, O_RDONLY);
  if (fd < 0) { g_fasta_err = std::string("gnm_fasta_open_gz: cannot open ") + path + ": " + std::strerror(errno); return 1; }
  struct stat st;
  if (::fstat(fd, &st) != 0 || st.st_size < 18) { g_fasta_err = "gnm_fasta_open_gz: not a gzip file"; ::close(fd); return 1; }
  const size_t clen = static_cast<size_t>(st.st_size);
  void* m = ::mmap(nullptr, clen, PROT_READ, MAP_PRIVATE, fd, 0);
  ::close(fd);
  if (m == MAP_FAILED) { g_fasta_err = std::string("gnm_fasta_open_gz: mmap failed: ") + std::strerror(errno); return 1; }
  const uint8_t* c = static_cast<const uint8_t*>(m);
  struct Unmap { void* p; size_t n; ~Unmap() { ::munmap(p, n); } } unmap{m, clen};
  if (c[0] != 0x1f || c[1] != 0x8b) { g_fasta_err = "gnm_fasta_open_gz: not a gzip file"; return 1; }
  auto rd16 = [&](size_t o) { return static_cast<uint32_t>(c[o]) | (static_cast<uint32_t>(c[o + 1]) << 8); };
  auto rd32 = [&](size_t o) { return rd16(o) | (rd16(o + 2) << 16); };
  // ---- BGZF?  header: 1f 8b 08 04 .. XLEN=6 'B' 'C' 02 00 BSIZE(2)
  std::vector<size_t> blk_off, blk_out;
  std::vector<uint32_t> blk_clen, blk_ulen;
  bool bgzf = true;
  {
    size_t o = 0, total = 0;
    while (o < clen) {
      if (o + 18 > clen || c[o] != 0x1f || c[o + 1] != 0x8b || c[o + 2] != 8 || !(c[o + 3] & 4) || rd16(o + 10) != 6 ||
          c[o + 12] != 'B' || c[o + 13] != 'C' || rd16(o + 14) != 2) { bgzf = false; break; }
      const size_t bsize = static_cast<size_t>(rd16(o + 16)) + 1;
      if (bsize < 26 || o + bsize > clen) { bgzf = false; break; }
      const uint32_t ulen = rd32(o + bsize - 4);
      blk_off.push_back(o); blk_clen.push_back(static_cast<uint32_t>(bsize)); blk_ulen.push_back(ulen); blk_out.push_back(total);
      total += ulen;
      o += bsize;
    }
    if (bgzf) blk_out.push_back(total);
  }
  gnm_fasta* f = new gnm_fasta();
  f->single_window = single_window;
  if (bgzf && !blk_off.empty()) {
    const size_t total = blk_out.back();
    f->owned.reset(new uint8_t[total + 1]);
    std::atomic<int> bad{0};
    parallel_for(static_cast<int64_t>(blk_off.size()), threads, [&](int64_t b) {
      if (blk_ulen[b] == 0) return;                        // the empty end-of-file marker block
      z_stream zs;
      std::memset(&zs, 0, sizeof zs);
      if (inflateInit2(&zs, -15) != Z_OK) { bad = 1; return; }
      zs.next_in = const_cast<Bytef*>(c + blk_off[b] + 18);
      zs.avail_in = blk_clen[b] - 18 - 8;
      zs.next_out = f->owned.get() + blk_out[b];
      zs.avail_out = blk_ulen[b];
      const int rc = inflate(&zs, Z_FINISH);
      if (rc != Z_STREAM_END || zs.avail_out != 0) bad = 1;
      inflateEnd(&zs);
    });
    if (bad) { delete f; g_fasta_err = "gnm_fasta_open_gz: corrupt BGZF block"; return 1; }
    f->len = static_cast<int64_t>(total);
  } else {
    // plain gzip, possibly several concatenated members; zlib's counters are 32-bit, so input and output are fed in <= 1 GiB pieces
    size_t cap = std::max<size_t>(static_cast<size_t>(rd32(clen - 4)) + 64, clen * 3), n = 0, in_off = 0;
    std::unique_ptr<uint8_t[]> buf(new uint8_t[cap]);
    z_stream zs;
    std::memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, 15 + 32) != Z_OK) { delete f; g_fasta_err = "gnm_fasta_open_gz: inflateInit2 failed"; return 1; }
    bool ok = true, done = false;
    constexpr size_t kPiece = size_t(1) << 30;
    while (!done) {
      if (zs.avail_in == 0 && in_off < clen) {
        const size_t piece = std::min(kPiece, clen - in_off);
        zs.next_in = const_cast<Bytef*>(c + in_off);
        zs.avail_in = static_cast<uInt>(piece);
        in_off += piece;
      }
      if (n == cap) {                                        // grow the output geometrically
        const size_t ncap = cap * 2;
        std::unique_ptr<uint8_t[]> nb(new uint8_t[ncap]);
        std::memcpy(nb.get(), buf.get(), n);
        buf.swap(nb); cap = ncap;
      }
      const size_t room = std::min(kPiece, cap - n);
      zs.next_out = buf.get() + n;
      zs.avail_out = static_cast<uInt>(room);
      const uInt in_before = zs.avail_in;
      const int rc = inflate(&zs, Z_NO_FLUSH);
      const size_t produced = room - zs.avail_out;
      n += produced;
      if (rc == Z_STREAM_END) {                              // one member finished: another one may follow
        const bool more = zs.avail_in > 0 || in_off < clen;
        const uint8_t next = zs.avail_in > 0 ? *zs.next_in : (in_off < clen ? c[in_off] : 0);
        if (more && next == 0x1f) inflateReset(&zs); else done = true;
      } else if (rc == Z_OK || rc == Z_BUF_ERROR) {
        if (produced == 0 && zs.avail_in == in_before && zs.avail_in == 0 && in_off >= clen) { ok = false; done = true; }   // truncated
      } else { ok = false; done = true; }
    }
    inflateEnd(&zs);
    if (!ok) { delete f; g_fasta_err = "gnm_fasta_open_gz: corrupt or truncated gzip stream"; return 1; }
    f->owned.swap(buf);
    f->len = static_cast<int64_t>(n);
  }
  f->text = f->owned.get();
  build_index(f, threads);
  *out = f;
  return 0;
#endif
}

extern "C" int gnm_fasta_info(const gnm_fasta* f, int64_t* n_records_nonempty, int* has_duplicate_ids, int64_t* n_contigs,
                              int64_t* n_windows, int64_t* header_bytes) {
  if (!f) { g_fasta_err = "gnm_fasta_info: null handle"; return 1; }
  if (n_records_nonempty) *n_records_nonempty = f->n_nonempty_raw;
  if (has_duplicate_ids) *has_duplicate_ids = f->has_dup;
  if (n_contigs) *n_contigs = static_cast<int64_t>(f->kept.size());
  if (n_windows) *n_windows = f->windows.n_windows;
  if (header_bytes) {
    int64_t b = 0;
    for (int64_t r : f->kept) b += f->recs[r].hdr_end - f->recs[r].hdr_begin + 1;
    *header_bytes = b;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ window extraction
// file offset of raw nucleotide index `a` of a regular record
static inline int64_t regular_offset(const Record& R, int64_t a) {
  return R.body_begin + (a / R.line_len) * R.stride + a % R.line_len;
}

// upper(comp(c)) for every byte: comp is the reference's Sequence.rc() table (sequence.py:41-43), ACTGNactgn -> TGACNtgacn and
// every other byte unchanged; upper() changes 'a'..'z' only
struct RcUpperTable {
  uint8_t v[256];
  RcUpperTable() {
    for (int c = 0; c < 256; ++c) v[c] = static_cast<uint8_t>(c);
    const char* from = "ACTGNactgn";
    const char* to = "TGACNtgacn";
    for (int i = 0; i < 10; ++i) v[static_cast<uint8_t>(from[i])] = static_cast<uint8_t>(to[i]);
    for (int c = 0; c < 256; ++c) if (v[c] >= 'a' && v[c] <= 'z') v[c] = static_cast<uint8_t>(v[c] - 32);
  }
};

// window wdx of list p -> dst[6000]
static void extract_window(const gnm_fasta_windows* p, int64_t wdx, uint8_t* dst) {
  const gnm_fasta* f = p->f;
  const size_t ki = static_cast<size_t>(std::upper_bound(p->first.begin(), p->first.end(), wdx) - p->first.begin()) - 1;
  const Record& R = f->recs[static_cast<size_t>(f->kept[ki])];
  int64_t cand = wdx - p->first[ki];
  if (p->kept_idx[ki] >= 0) cand = p->kept_wins[static_cast<size_t>(p->kept_idx[ki])][static_cast<size_t>(cand)];
  const int64_t n = window_len(R.seq_len, p->step, cand);
  const uint8_t* t = f->text;
  int64_t got = 0;
  if (R.stride > 0) {
    const int64_t a = R.lead + segment_begin(R.seq_len, p->step, p->reverse, cand);
    int64_t off = regular_offset(R, a), in_line = R.line_len - a % R.line_len;
    while (got < n) {
      const int64_t c = std::min(n - got, in_line);
      std::memcpy(dst + got, t + off, static_cast<size_t>(c));
      got += c; off += c + (R.stride - R.line_len); in_line = R.line_len;
    }
  } else {
    int64_t i = p->win_off[static_cast<size_t>(p->off_idx[ki])][static_cast<size_t>(cand)];
    while (got < n && i < R.body_end) {
      int64_t j = i;
      if (!R.has_cr) {
        const void* q = std::memchr(t + i, '\n', static_cast<size_t>(R.body_end - i));
        j = q ? static_cast<const uint8_t*>(q) - t : R.body_end;
      } else {
        while (j < R.body_end && !is_eol(t[j])) ++j;
      }
      const int64_t c = std::min(n - got, j - i);
      std::memcpy(dst + got, t + i, static_cast<size_t>(c));
      got += c;
      i = j + 1;                      // a "\r\n" pair leaves an empty line behind: harmless
    }
  }
  if (p->reverse) {                   // rc, then ASCII upper(): byte j = upper(comp(segment[n - 1 - j]))
    static const RcUpperTable tab;
    for (int64_t i = 0, j = n - 1; i <= j; ++i, --j) {
      const uint8_t c = dst[i];
      dst[i] = tab.v[dst[j]];
      dst[j] = tab.v[c];
    }
  } else {
    for (int64_t k = 0; k < n; ++k) {   // ASCII upper(), as bytes.upper()
      const uint8_t c = dst[k];
      dst[k] = (c >= 'a' && c <= 'z') ? static_cast<uint8_t>(c - 32) : c;
    }
  }
  if (n < kWin) std::memset(dst + n, 'N', static_cast<size_t>(kWin - n));
}

static int export_windows(const gnm_fasta_windows* p, int64_t first, int64_t count, uint8_t* dst, int threads,
                          const char* fn) {
  if (first < 0 || count < 0 || first + count > p->n_windows) { g_fasta_err = std::string(fn) + ": range out of bounds"; return 1; }
  constexpr int64_t kBlock = 32;                            // windows per work item
  parallel_for((count + kBlock - 1) / kBlock, threads, [&](int64_t b) {
    const int64_t lo = first + b * kBlock, hi = std::min(first + count, lo + kBlock);
    for (int64_t wdx = lo; wdx < hi; ++wdx) extract_window(p, wdx, dst + (wdx - first) * kWin);
  });
  return 0;
}

static int release_before(const gnm_fasta_windows* p, int64_t upto) {
  const gnm_fasta* f = p->f;
  if (!f->map_base || f->kept.empty()) return 0;
  int64_t byte_end;
  if (upto >= p->n_windows) byte_end = f->len;
  else if (upto <= 0) return 0;
  else {
    const size_t ki = static_cast<size_t>(std::upper_bound(p->first.begin(), p->first.end(), upto) - p->first.begin()) - 1;
    byte_end = f->recs[static_cast<size_t>(f->kept[ki])].hdr_begin - 1;      // start of the record that holds window `upto`
  }
  const int64_t page = 4096;
  const int64_t aligned = byte_end / page * page;
  int64_t done = p->released.load();
  if (aligned > done) {
    ::madvise(static_cast<uint8_t*>(f->map_base) + done, static_cast<size_t>(aligned - done), MADV_DONTNEED);
    p->released.store(aligned);
  }
  return 0;
}

extern "C" int gnm_fasta_export(const gnm_fasta* f, uint8_t* windows, int32_t* offsets, char* headers, int threads) {
  if (!f) { g_fasta_err = "gnm_fasta_export: null handle"; return 1; }
  if (f->windows.n_windows > INT32_MAX) { g_fasta_err = "gnm_fasta_export: more than 2^31-1 windows"; return 1; }
  const int64_t nk = static_cast<int64_t>(f->kept.size());
  if (offsets) {
    for (int64_t i = 0; i < nk; ++i) offsets[i] = static_cast<int32_t>(f->windows.first[static_cast<size_t>(i)]);
    offsets[nk] = static_cast<int32_t>(f->windows.n_windows);
  }
  if (headers) {
    char* h = headers;
    for (int64_t i = 0; i < nk; ++i) {
      const Record& R = f->recs[f->kept[i]];
      const int64_t n = R.hdr_end - R.hdr_begin;
      std::memcpy(h, f->text + R.hdr_begin, static_cast<size_t>(n));
      h[n] = '\n';
      h += n + 1;
    }
  }
  if (windows) return gnm_fasta_export_windows(f, 0, f->windows.n_windows, windows, threads);
  return 0;
}

// windows [first, first + count) of the global window list -> dst [count][6000]  (streaming export: the driver fills one
// pinned chunk while the GPU classifies the previous one)
extern "C" int gnm_fasta_export_windows(const gnm_fasta* f, int64_t first, int64_t count, uint8_t* dst, int threads) {
  if (!f || (!dst && count)) { g_fasta_err = "gnm_fasta_export_windows: null argument"; return 1; }
  return export_windows(&f->windows, first, count, dst, threads, "gnm_fasta_export_windows");
}

// Hand the pages of the mapping that lie entirely before window `upto` back to the kernel (they stay in the page
// cache; the process' resident set stops growing with the file).  No-op for caller-memory text.
extern "C" int gnm_fasta_release_before(const gnm_fasta* f, int64_t upto) {
  if (!f) { g_fasta_err = "gnm_fasta_release_before: null handle"; return 1; }
  return release_before(&f->windows, upto);
}

// ------------------------------------------------------------------------------------------------ window lists at any step
static int plan_windows(const char* fn, const gnm_fasta* f, int stride, int single_window, int reverse, int threads,
                        gnm_fasta_windows** out) {
  const std::string name(fn);
  if (!f || !out) { g_fasta_err = name + ": null argument"; return 1; }
  if (stride < 1 || stride > kWin) {
    g_fasta_err = name + ": stride must be in [1, 6000], not " + std::to_string(stride);
    return 1;
  }
  // checked before anything is built: the candidate count has a closed form, and the kept windows are at most that many
  if (candidate_total(f, stride, single_window) > INT32_MAX) {
    g_fasta_err = name + ": more than 2^31-1 windows (before the N rule)";
    return 1;
  }
  std::unique_ptr<gnm_fasta_windows> p(new gnm_fasta_windows());
  p->step = stride;
  p->single_window = single_window;
  p->reverse = reverse;
  build_windows(f, p.get(), std::max(1, threads));
  *out = p.release();
  return 0;
}

extern "C" int gnm_fasta_windows_plan(const gnm_fasta* f, int stride, int single_window, int threads, gnm_fasta_windows** out) {
  return plan_windows("gnm_fasta_windows_plan", f, stride, single_window, 0, threads, out);
}

// The windows of every kept record's reverse complement: the list gnm_fasta_windows_plan makes from rc(S), with starts and
// lengths naming each window's forward segment
extern "C" int gnm_fasta_windows_plan_rc(const gnm_fasta* f, int stride, int single_window, int threads,
                                         gnm_fasta_windows** out) {
  return plan_windows("gnm_fasta_windows_plan_rc", f, stride, single_window, 1, threads, out);
}

extern "C" int gnm_fasta_windows_info(const gnm_fasta_windows* p, int64_t* n_contigs, int64_t* n_windows) {
  if (!p) { g_fasta_err = "gnm_fasta_windows_info: null handle"; return 1; }
  if (n_contigs) *n_contigs = static_cast<int64_t>(p->first.size());
  if (n_windows) *n_windows = p->n_windows;
  return 0;
}

static void window_spans(const gnm_fasta_windows* p, int32_t* offsets, int64_t* starts, int32_t* lengths) {
  const size_t nk = p->first.size();
  if (offsets) {
    for (size_t i = 0; i < nk; ++i) offsets[i] = static_cast<int32_t>(p->first[i]);
    offsets[nk] = static_cast<int32_t>(p->n_windows);
  }
  if (!starts && !lengths) return;
  for (size_t i = 0; i < nk; ++i) {
    const Record& R = p->f->recs[static_cast<size_t>(p->f->kept[i])];
    const int64_t w0 = p->first[i], w1 = i + 1 < nk ? p->first[i + 1] : p->n_windows;
    const std::vector<int32_t>* kw = p->kept_idx[i] >= 0 ? &p->kept_wins[static_cast<size_t>(p->kept_idx[i])] : nullptr;
    for (int64_t w = w0; w < w1; ++w) {
      const int64_t cand = kw ? (*kw)[static_cast<size_t>(w - w0)] : w - w0;
      if (starts) starts[w] = R.lead + segment_begin(R.seq_len, p->step, p->reverse, cand);
      if (lengths) lengths[w] = static_cast<int32_t>(window_len(R.seq_len, p->step, cand));
    }
  }
}

extern "C" int gnm_fasta_windows_spans(const gnm_fasta_windows* p, int32_t* offsets, int64_t* starts, int32_t* lengths) {
  if (!p) { g_fasta_err = "gnm_fasta_windows_spans: null handle"; return 1; }
  if (p->n_windows > INT32_MAX) { g_fasta_err = "gnm_fasta_windows_spans: more than 2^31-1 windows"; return 1; }
  window_spans(p, offsets, starts, lengths);
  return 0;
}

extern "C" int gnm_fasta_spans(const gnm_fasta* f, int64_t* starts, int32_t* lengths) {
  if (!f) { g_fasta_err = "gnm_fasta_spans: null handle"; return 1; }
  window_spans(&f->windows, nullptr, starts, lengths);
  return 0;
}

extern "C" int gnm_fasta_windows_export(const gnm_fasta_windows* p, int64_t first, int64_t count, uint8_t* dst, int threads) {
  if (!p || (!dst && count)) { g_fasta_err = "gnm_fasta_windows_export: null argument"; return 1; }
  return export_windows(p, first, count, dst, threads, "gnm_fasta_windows_export");
}

extern "C" int gnm_fasta_windows_release_before(const gnm_fasta_windows* p, int64_t upto) {
  if (!p) { g_fasta_err = "gnm_fasta_windows_release_before: null handle"; return 1; }
  return release_before(p, upto);
}

extern "C" void gnm_fasta_windows_free(gnm_fasta_windows* p) { delete p; }

extern "C" void gnm_fasta_free(gnm_fasta* f) {
  if (!f) return;
  if (f->map_base) ::munmap(f->map_base, f->map_len);
  delete f;
}
