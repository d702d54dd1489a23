// Per-window score table of nn-classification --write-window-scores (host code, part of libgnm.so).
//
// One line per window: "<seq_name>\t<start>\t<end>\t<chromosome>\t<plasmid>\t<virus>\n", start 1-based and end inclusive (the
// convention of geNomad's provirus table); a classifier head's table (gnm_write_window_tsv_cols) has one score column per
// class.  Scores carry the digits Python's f"{float(x):.4f}" gives, which is what the contig table uses: the float32 value,
// exactly, rounded half to even at the fourth decimal.  That rounding is done here in integer arithmetic (no printf, so no
// locale and no libc rounding mode is involved).  A table can have hundreds of millions
// of rows: blocks of rows are formatted on `threads` threads and written in order.
#include <algorithm>
#include <atomic>
#include <cerrno>
#include <charconv>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/gnm.h"

namespace {

thread_local std::string g_tsv_err;

// f"{float(x):.4f}" of a float32 x -> o (at most 48 bytes); returns the number of bytes written
int format_score(float x, char* o) {
  uint32_t b;
  std::memcpy(&b, &x, 4);
  const bool neg = b >> 31;
  const uint32_t ex = (b >> 23) & 0xffu, man = b & 0x7fffffu;
  char* p = o;
  if (ex == 0xffu) {                                      // Python prints nan without a sign
    const char* s = man ? "nan" : neg ? "-inf" : "inf";
    const size_t n = std::strlen(s);
    std::memcpy(o, s, n);
    return static_cast<int>(n);
  }
  if (ex >= 127 + 24) {                                   // |x| >= 2^24: an integer; never a probability
    return std::snprintf(o, 48, "%.0f.0000", static_cast<double>(x));
  }
  if (neg) *p++ = '-';
  const uint64_t m = ex ? (man | 0x800000u) : man;        // |x| = m * 2^e2, m < 2^24, e2 <= 0 here
  const int sh = ex ? 150 - static_cast<int>(ex) : 149;
  const uint64_t v = m * 10000u;                          // < 2^38
  uint64_t q = 0;                                         // round_half_even(|x| * 10^4)
  if (sh <= 0) {
    q = v << -sh;
  } else if (sh < 64) {
    q = v >> sh;
    const uint64_t rem = v & ((uint64_t(1) << sh) - 1), half = uint64_t(1) << (sh - 1);
    if (rem > half || (rem == half && (q & 1))) ++q;
  }
  p = std::to_chars(p, p + 24, q / 10000).ptr;
  const unsigned frac = static_cast<unsigned>(q % 10000);
  *p++ = '.';
  p[0] = static_cast<char>('0' + frac / 1000);
  p[1] = static_cast<char>('0' + frac / 100 % 10);
  p[2] = static_cast<char>('0' + frac / 10 % 10);
  p[3] = static_cast<char>('0' + frac % 10);
  return static_cast<int>(p + 4 - o);
}

}  // namespace

extern "C" const char* gnm_tsv_last_error(void) { return g_tsv_err.c_str(); }

extern "C" int gnm_format_scores(const float* x, int64_t n, char* out, int64_t* out_len) {
  if ((!x || !out) && n) { g_tsv_err = "gnm_format_scores: null argument"; return 1; }
  char* p = out;
  for (int64_t i = 0; i < n; ++i) { p += format_score(x[i], p); *p++ = '\n'; }
  if (out_len) *out_len = p - out;
  return 0;
}

extern "C" int gnm_write_window_tsv_cols(const char* path, const char* header, const char* names,
                                         const int64_t* name_offsets, int64_t n_contigs, const int32_t* win_offsets,
                                         const int64_t* starts, const int32_t* lengths, const float* probs, int n_cols,
                                         int threads) {
  if (!path || !header || !name_offsets || !win_offsets || n_contigs < 0) { g_tsv_err = "gnm_write_window_tsv: null argument"; return 1; }
  if (n_cols < 1 || n_cols > 32) { g_tsv_err = "gnm_write_window_tsv: n_cols must be in [1, 32]"; return 1; }
  const int64_t n = win_offsets[n_contigs];
  if (n < 0 || (n > 0 && (!names || !starts || !lengths || !probs))) { g_tsv_err = "gnm_write_window_tsv: null argument"; return 1; }
  for (int64_t c = 0; c < n_contigs; ++c)
    if (win_offsets[c + 1] < win_offsets[c] || name_offsets[c + 1] < name_offsets[c]) {
      g_tsv_err = "gnm_write_window_tsv: offsets are not non-decreasing";
      return 1;
    }
  FILE* fh = std::fopen(path, "wb");
  if (!fh) { g_tsv_err = std::string("gnm_write_window_tsv: cannot open ") + path + ": " + std::strerror(errno); return 1; }
  bool ok = std::fputs(header, fh) >= 0;
  constexpr int64_t kRows = 1 << 16;                      // rows per block
  threads = std::max(1, threads);
  const int64_t n_blocks = (n + kRows - 1) / kRows;
  // a row is at most nl + row_max bytes: name, 3 tabs + two 20-character coordinates, n_cols x (tab + <= 45-character score +
  // snprintf's terminator), newline
  const size_t row_max = 44 + 47 * static_cast<size_t>(n_cols);
  std::vector<std::string> buf(static_cast<size_t>(threads));
  for (int64_t b0 = 0; ok && b0 < n_blocks; b0 += threads) {
    const int nb = static_cast<int>(std::min<int64_t>(threads, n_blocks - b0));
    auto work = [&](int t) {
      const int64_t lo = (b0 + t) * kRows, hi = std::min(n, lo + kRows);
      std::string& s = buf[static_cast<size_t>(t)];
      s.resize(static_cast<size_t>(hi - lo) * (152 + 16 * static_cast<size_t>(n_cols)));   // grown below for long rows
      size_t at = 0;
      int64_t c = std::upper_bound(win_offsets, win_offsets + n_contigs + 1, static_cast<int32_t>(lo)) - win_offsets - 1;
      for (int64_t w = lo; w < hi; ++w) {
        while (win_offsets[c + 1] <= w) ++c;
        const size_t nl = static_cast<size_t>(name_offsets[c + 1] - name_offsets[c]);
        if (s.size() < at + nl + row_max + 64) s.resize((at + nl + row_max + 64) * 2);
        char* p = &s[at];
        std::memcpy(p, names + name_offsets[c], nl);
        p += nl;
        *p++ = '\t';
        p = std::to_chars(p, p + 24, starts[w] + 1).ptr;
        *p++ = '\t';
        p = std::to_chars(p, p + 24, starts[w] + lengths[w]).ptr;
        for (int k = 0; k < n_cols; ++k) { *p++ = '\t'; p += format_score(probs[static_cast<int64_t>(n_cols) * w + k], p); }
        *p++ = '\n';
        at = static_cast<size_t>(p - s.data());
      }
      s.resize(at);
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < nb; ++t) pool.emplace_back(work, t);
    work(0);
    for (auto& th : pool) th.join();
    for (int t = 0; t < nb && ok; ++t) ok = std::fwrite(buf[static_cast<size_t>(t)].data(), 1, buf[static_cast<size_t>(t)].size(), fh) == buf[static_cast<size_t>(t)].size();
  }
  if (std::fclose(fh) != 0) ok = false;
  if (!ok) { g_tsv_err = std::string("gnm_write_window_tsv: write to ") + path + " failed"; return 1; }
  return 0;
}

extern "C" int gnm_write_window_tsv(const char* path, const char* header, const char* names, const int64_t* name_offsets,
                                    int64_t n_contigs, const int32_t* win_offsets, const int64_t* starts,
                                    const int32_t* lengths, const float* probs, int threads) {
  return gnm_write_window_tsv_cols(path, header, names, name_offsets, n_contigs, win_offsets, starts, lengths, probs, 3,
                                   threads);
}
