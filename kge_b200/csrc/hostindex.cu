// hostindex.cu — host-side (CPU) label plumbing next to the scoring path: the key -> all-values index that
// KvsAll training and filtered entity ranking build their label / filter coordinates from.
//
// Replaces the reference's KvsAllIndex (indexing.py:10-194: numpy argsort + np.unique + a numba dict) and the
// Python collate loops that walk it (train_KvsAll.py:116-203, util.py:6-30) with plain C++: a sort, a unique
// pass and binary searches; results are returned in CSR form (row offsets + column ids), which is what the
// device epilogues consume instead of `coord_to_sparse_tensor(...).to_dense()` (util.py:32-60).
// No device code here; the functions run without a GPU.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <numeric>
#include <vector>
#include "common.cuh"

namespace b200kge {
namespace {

inline bool col_ok(int c) { return c >= 0 && c <= 2; }

// index of (k0, k1) in the sorted unique key list, or -1
inline int64_t find_key(const int64_t* keys, int64_t num_keys, int64_t k0, int64_t k1) {
  int64_t lo = 0, hi = num_keys;
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo) / 2;
    const int64_t a = keys[2 * mid], b = keys[2 * mid + 1];
    if (a < k0 || (a == k0 && b < k1)) lo = mid + 1;
    else hi = mid;
  }
  if (lo < num_keys && keys[2 * lo] == k0 && keys[2 * lo + 1] == k1) return lo;
  return -1;
}

// Frequency weights quantised at scale 2^s: q_x = c_x * 2^s + round(alpha * 2^s), rounded half to even.  True if
// Q = sum q_x <= 2^62; then cdf (when given, [vocab + 1]) receives the exclusive prefix of q, cdf[vocab] = Q.
bool quantised_total(const int64_t* counts, int64_t vocab, double alpha, int s, uint64_t* cdf) {
  constexpr uint64_t LIM = 1ull << 62;
  const double qa = std::nearbyint(std::ldexp(alpha, s));
  if (!(qa <= (double)LIM)) return false;
  const uint64_t ua = (uint64_t)qa;
  uint64_t total = 0;
  if (cdf) cdf[0] = 0;
  for (int64_t x = 0; x < vocab; ++x) {
    const uint64_t c = (uint64_t)counts[x];
    if (c > 0 && (s > 62 || c > (LIM >> s))) return false;
    const uint64_t q = (c << (s > 62 ? 0 : s)) + ua;   // <= 2^63: no wrap
    if (q > LIM - total) return false;
    total += q;
    if (cdf) cdf[x + 1] = total;
  }
  return true;
}

}  // namespace
}  // namespace b200kge

using namespace b200kge;

extern "C" {

int b200kge_kvsall_index_build(const int64_t* triples, int64_t n, int key_col0, int key_col1, int value_col,
                               int64_t* keys_out, int64_t* offsets_out, int64_t* values_out, int64_t* num_keys) {
  if ((!triples && n > 0) || !offsets_out || !num_keys || (n > 0 && (!keys_out || !values_out))) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  if (n < 0 || !col_ok(key_col0) || !col_ok(key_col1) || !col_ok(value_col) || key_col0 == key_col1 ||
      value_col == key_col0 || value_col == key_col1) {
    set_error("key/value columns must be a permutation of (0,1,2)");
    return B200KGE_ERR_INVALID;
  }
  // sort by (key0, key1, value): indexing.py:178-194 (sort by value, then stable by key1, then stable by key0)
  std::vector<int64_t> order((size_t)n);
  std::iota(order.begin(), order.end(), (int64_t)0);
  std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) {
    const int64_t* x = triples + 3 * a;
    const int64_t* y = triples + 3 * b;
    if (x[key_col0] != y[key_col0]) return x[key_col0] < y[key_col0];
    if (x[key_col1] != y[key_col1]) return x[key_col1] < y[key_col1];
    return x[value_col] < y[value_col];
  });
  // unique keys + start offset of each (np.unique(..., axis=0, return_index=True), indexing.py:39-42)
  int64_t nk = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t* t = triples + 3 * order[(size_t)i];
    if (i == 0 || t[key_col0] != keys_out[2 * (nk - 1)] || t[key_col1] != keys_out[2 * (nk - 1) + 1]) {
      keys_out[2 * nk] = t[key_col0];
      keys_out[2 * nk + 1] = t[key_col1];
      offsets_out[nk] = i;
      ++nk;
    }
    values_out[i] = t[value_col];          // duplicates are kept, as in the reference
  }
  offsets_out[nk] = n;
  *num_keys = nk;
  return 0;
}

int b200kge_kvsall_lookup(const int64_t* keys, const int64_t* offsets, const int64_t* values, int64_t num_keys,
                          const int64_t* query_keys, int64_t nq, int64_t col_shift, int64_t* offsets_out,
                          int64_t* cols_out) {
  if (!offsets_out || (nq > 0 && !query_keys) || (num_keys > 0 && (!keys || !offsets || !values)) || nq < 0 || num_keys < 0) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  // KvsAllIndex.get_all (indexing.py:113-166): absent keys contribute nothing
  int64_t total = 0;
  for (int64_t i = 0; i < nq; ++i) {
    offsets_out[i] = total;
    const int64_t k = find_key(keys, num_keys, query_keys[2 * i], query_keys[2 * i + 1]);
    if (k < 0) continue;
    const int64_t b = offsets[k], e = offsets[k + 1];
    if (cols_out)
      for (int64_t j = b; j < e; ++j) cols_out[total + (j - b)] = values[j] + col_shift;
    total += e - b;
  }
  offsets_out[nq] = total;
  return 0;
}

int b200kge_kvsall_gather(const int64_t* keys, const int64_t* offsets, const int64_t* values, int64_t num_keys,
                          const int64_t* examples, int64_t nb, int64_t* queries_out, int64_t* offsets_out,
                          int64_t* cols_out) {
  if (!offsets_out || (nb > 0 && (!examples || !keys || !offsets || !values || !queries_out)) || nb < 0) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  // the collate function of KvsAll training for one query type (train_KvsAll.py:116-203): example = key index
  int64_t total = 0;
  for (int64_t i = 0; i < nb; ++i) {
    const int64_t k = examples[i];
    if (k < 0 || k >= num_keys) { set_error("example index %lld out of range [0, %lld)", (long long)k, (long long)num_keys); return B200KGE_ERR_INVALID; }
    offsets_out[i] = total;
    queries_out[2 * i] = keys[2 * k];
    queries_out[2 * i + 1] = keys[2 * k + 1];
    const int64_t b = offsets[k], e = offsets[k + 1];
    if (cols_out)
      for (int64_t j = b; j < e; ++j) cols_out[total + (j - b)] = values[j];
    total += e - b;
  }
  offsets_out[nb] = total;
  return 0;
}

int b200kge_filter_index_build(const int64_t* keys, const int64_t* offsets, const int64_t* values, int64_t num_keys,
                               int64_t vocab, int64_t* keys_out, int64_t* offsets_out, int64_t* values_out,
                               int64_t* num_keys_out, int64_t* max_count) {
  if (num_keys < 0 || !offsets || !offsets_out || !num_keys_out || !max_count || (num_keys > 0 && !keys)) {
    set_error("null operand");
    return B200KGE_ERR_INVALID;
  }
  if (vocab <= 0) { set_error("vocabulary size must be positive"); return B200KGE_ERR_INVALID; }
  // every offset is checked before any value is read: nnz and the values' extent rest on them
  for (int64_t k = 0; k < num_keys; ++k)
    if (offsets[k + 1] < offsets[k]) { set_error("offsets must not decrease"); return B200KGE_ERR_INVALID; }
  const int64_t base = offsets[0], nnz = offsets[num_keys] - base;
  if (nnz > 0 && (!values || !keys_out || !values_out)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  // one (key0, key1, value) entry per listed value; sorting and dropping repeats gives sorted unique keys and sorted
  // distinct values per key whatever order or repeats the input had (a split may repeat a triple)
  struct Entry { int64_t a, b, v; };
  std::vector<Entry> ent;
  ent.reserve((size_t)nnz);
  for (int64_t k = 0; k < num_keys; ++k) {
    for (int64_t j = offsets[k]; j < offsets[k + 1]; ++j) {
      const int64_t v = values[j - base];
      if (v < 0 || v >= vocab) {
        set_error("value %lld of key (%lld, %lld) outside [0, %lld)", (long long)v, (long long)keys[2 * k],
                  (long long)keys[2 * k + 1], (long long)vocab);
        return B200KGE_ERR_INVALID;
      }
      ent.push_back({keys[2 * k], keys[2 * k + 1], v});
    }
  }
  auto lt = [](const Entry& x, const Entry& y) {
    return x.a != y.a ? x.a < y.a : x.b != y.b ? x.b < y.b : x.v < y.v;
  };
  std::sort(ent.begin(), ent.end(), lt);
  ent.erase(std::unique(ent.begin(), ent.end(),
                        [](const Entry& x, const Entry& y) { return x.a == y.a && x.b == y.b && x.v == y.v; }),
            ent.end());
  int64_t nk = 0, mx = 0;
  for (size_t i = 0; i < ent.size(); ++i) {
    if (i == 0 || ent[i].a != ent[i - 1].a || ent[i].b != ent[i - 1].b) {
      if (nk > 0) mx = std::max(mx, (int64_t)i - offsets_out[nk - 1]);
      keys_out[2 * nk] = ent[i].a;
      keys_out[2 * nk + 1] = ent[i].b;
      offsets_out[nk++] = (int64_t)i;
    }
    values_out[i] = ent[i].v;
  }
  if (nk > 0) mx = std::max(mx, (int64_t)ent.size() - offsets_out[nk - 1]);
  offsets_out[nk] = (int64_t)ent.size();
  *num_keys_out = nk;
  *max_count = mx;
  return 0;
}

int b200kge_frequency_cdf_build(const int64_t* counts, int64_t vocab, double smoothing, uint64_t* cdf_out) {
  if (vocab <= 0) { set_error("vocabulary size must be positive"); return B200KGE_ERR_INVALID; }
  if (!counts || !cdf_out) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (!std::isfinite(smoothing) || smoothing < 0) {
    set_error("smoothing must be finite and >= 0 (got %g)", smoothing);
    return B200KGE_ERR_INVALID;
  }
  for (int64_t x = 0; x < vocab; ++x)
    if (counts[x] < 0) { set_error("count %lld of id %lld is negative", (long long)counts[x], (long long)x); return B200KGE_ERR_INVALID; }
  // q_x(s) = c_x * 2^s + round(alpha * 2^s) = round((c_x + alpha) * 2^s) for s >= 0 (c_x * 2^s is an integer); ldexp
  // is exact and nearbyint rounds half to even, so every q_x is exact.  Q(s) = sum q_x does not decrease in s.
  if (!quantised_total(counts, vocab, smoothing, 0, nullptr)) {
    set_error("the smoothed counts sum to more than 2^62");
    return B200KGE_ERR_INVALID;
  }
  int lo = 0, hi = 2200;                  // fits at lo; beyond any alpha * 2^s a double can hold at hi
  while (hi - lo > 1) {
    const int mid = lo + (hi - lo) / 2;
    if (quantised_total(counts, vocab, smoothing, mid, nullptr)) lo = mid;
    else hi = mid;
  }
  quantised_total(counts, vocab, smoothing, lo, cdf_out);
  if (cdf_out[vocab] == 0) { set_error("every weight is zero (smoothing 0 and no id occurs)"); return B200KGE_ERR_INVALID; }
  return 0;
}

int b200kge_frequency_filter_build(const uint64_t* cdf, int64_t vocab, const int64_t* offsets, const int64_t* values,
                                   int64_t num_keys, uint64_t* below_out, int64_t* num_full, int64_t* first_full) {
  if (vocab <= 0) { set_error("vocabulary size must be positive"); return B200KGE_ERR_INVALID; }
  if (num_keys < 0 || !cdf || !offsets || !num_full || !first_full) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  if (cdf[0] != 0 || cdf[vocab] == 0) { set_error("cdf must start at 0 and end above 0"); return B200KGE_ERR_INVALID; }
  for (int64_t x = 0; x < vocab; ++x)
    if (cdf[x + 1] < cdf[x]) { set_error("cdf must not decrease"); return B200KGE_ERR_INVALID; }
  for (int64_t k = 0; k < num_keys; ++k)
    if (offsets[k + 1] < offsets[k]) { set_error("offsets must not decrease"); return B200KGE_ERR_INVALID; }
  const int64_t base = offsets[0];
  if (offsets[num_keys] > base && (!values || !below_out)) { set_error("null operand"); return B200KGE_ERR_INVALID; }
  const uint64_t Q = cdf[vocab];
  int64_t full = 0, first = -1;
  for (int64_t k = 0; k < num_keys; ++k) {
    uint64_t pos = 0;                     // mass of the key's positives below values[j]
    for (int64_t j = offsets[k]; j < offsets[k + 1]; ++j) {
      const int64_t v = values[j - base];
      if (v < 0 || v >= vocab || (j > offsets[k] && v <= values[j - 1 - base])) {
        set_error("values of key %lld must be ascending, distinct and in [0, %lld)", (long long)k, (long long)vocab);
        return B200KGE_ERR_INVALID;
      }
      below_out[j - base] = cdf[v] - pos;
      pos += cdf[v + 1] - cdf[v];
    }
    if (pos == Q) {
      if (first < 0) first = k;
      ++full;
    }
  }
  *num_full = full;
  *first_full = first;
  return 0;
}

}  // extern "C"
