// Slot table of the paired Clenshaw launch (cheby_pair_tiled, csrc/cheby_tiled.cu).  Host code:
// it runs once per matrix on a host copy of the CSR structure, and the tests run it without a GPU.
//
// Tile t is rows [t R, t R + R), t < T = n / R.  nbr[t] lists, in increasing order, the tiles that
// hold a column of t's rows, and t itself: the A tiles that B(t) reads.  (Columns past the last
// full tile belong to rows that the caller completes before the launch.)  A slot is
// (tile << 1) | which.  The forward table holds A(0), A(1), ... with B(t) inserted directly after
// A(min(max nbr[t] + lag, T - 1)); the reverse table holds A(T-1), A(T-2), ... with B(t) directly
// after A(max(min nbr[t] - lag, 0)).  Slots that are close in the table run at the same time on
// different CTAs, so with lag = 0 every B tile would start while the A tile before it is still
// running and wait for it; the lag (in A tiles, about two slots each) puts more than one wave of
// the grid between the two.  Either table is a topological order of "B(t) after A(s), s in
// nbr[t]", which is verified here before a table is handed out.
#include <algorithm>
#include <climits>
#include <vector>
#include "common.cuh"
#include "gspb200.h"

namespace gsp {

static bool slots_are_safe(int64_t T, const int32_t* nbr_ptr, const int32_t* nbr_idx,
                           const int32_t* slots) {
  std::vector<int64_t> pos_a(T, -1), pos_b(T, -1);
  for (int64_t i = 0; i < 2 * T; ++i) {
    const int64_t t = slots[i] >> 1;
    if (t < 0 || t >= T) return false;
    int64_t& p = (slots[i] & 1) ? pos_b[t] : pos_a[t];
    if (p >= 0) return false;                       // a tile twice in one role
    p = i;
  }
  for (int64_t t = 0; t < T; ++t) {
    if (pos_a[t] < 0 || pos_b[t] < 0) return false;
    for (int32_t e = nbr_ptr[t]; e < nbr_ptr[t + 1]; ++e)
      if (pos_a[nbr_idx[e]] > pos_b[t]) return false;
  }
  return true;
}

}  // namespace gsp

extern "C" int gsp_cheby_pair_plan_host(int64_t n, const int32_t* indptr_host,
                                        const int32_t* indices_host, int rows_per_tile, int lag,
                                        int64_t nbr_capacity, int32_t* nbr_ptr, int32_t* nbr_idx,
                                        int32_t* slots_fwd, int32_t* slots_rev,
                                        int64_t* nbr_count_out) {
  GSP_REQUIRE(n >= 0 && rows_per_tile > 0 && lag >= 0 && indptr_host && indices_host &&
                  nbr_count_out, "bad pair plan arguments");
  const int64_t R = rows_per_tile, T = n / R;
  GSP_REQUIRE(T >= 1 && T < (int64_t(1) << 30), "tile count out of range");
  std::vector<int32_t> stamp(T, -1), lo(T), hi(T), list;
  std::vector<int64_t> start(T + 1, 0);
  list.reserve(size_t(T) * 12);
  for (int64_t t = 0; t < T; ++t) {
    const size_t first = list.size();
    stamp[t] = int32_t(t);
    list.push_back(int32_t(t));
    for (int64_t j = indptr_host[t * R]; j < indptr_host[t * R + R]; ++j) {
      GSP_REQUIRE(indices_host[j] >= 0 && indices_host[j] < n, "column index out of range");
      const int64_t c = indices_host[j] / R;
      if (c < T && stamp[c] != t) {
        stamp[c] = int32_t(t);
        list.push_back(int32_t(c));
      }
    }
    std::sort(list.begin() + first, list.end());
    lo[t] = int32_t(std::max<int64_t>(int64_t(list[first]) - lag, 0));
    hi[t] = int32_t(std::min<int64_t>(int64_t(list.back()) + lag, T - 1));
    start[t + 1] = int64_t(list.size());
  }
  *nbr_count_out = int64_t(list.size());
  GSP_REQUIRE(list.size() < (size_t(1) << 31), "too many tile neighbours");
  if (int64_t(list.size()) > nbr_capacity) return GSP_OK;      // the caller retries with room
  GSP_REQUIRE(nbr_ptr && nbr_idx && slots_fwd && slots_rev, "bad pair plan arguments");
  for (int64_t t = 0; t <= T; ++t) nbr_ptr[t] = int32_t(start[t]);
  std::copy(list.begin(), list.end(), nbr_idx);
  // bucket the B tiles by the A tile they follow (counting sort keeps them in tile order)
  for (int dir = 0; dir < 2; ++dir) {
    const std::vector<int32_t>& key = dir == 0 ? hi : lo;
    int32_t* slots = dir == 0 ? slots_fwd : slots_rev;
    std::vector<int64_t> begin(T + 1, 0);
    for (int64_t t = 0; t < T; ++t) ++begin[key[t] + 1];
    for (int64_t t = 0; t < T; ++t) begin[t + 1] += begin[t];
    std::vector<int32_t> after(T);
    std::vector<int64_t> fill(begin.begin(), begin.end() - 1);
    for (int64_t t = 0; t < T; ++t) after[fill[key[t]]++] = int32_t(t);
    int64_t i = 0;
    for (int64_t rank = 0; rank < T; ++rank) {
      const int64_t at = dir == 0 ? rank : T - 1 - rank;
      slots[i++] = int32_t(at << 1);
      for (int64_t e = begin[at]; e < begin[at + 1]; ++e) slots[i++] = (after[e] << 1) | 1;
    }
    GSP_REQUIRE(i == 2 * T && gsp::slots_are_safe(T, nbr_ptr, nbr_idx, slots),
                "slot table is not a topological order");
  }
  return GSP_OK;
}

// Neighbour rings (gsp_cheby_ring_plan_host in the header).  A tile's own rows are always in its
// ring, so they form one stretch of it and the step reads its x_cur rows there too.
extern "C" int gsp_cheby_ring_plan_host(int64_t n, const int32_t* indptr_host,
                                        const int32_t* indices_host, int rows_per_tile,
                                        int64_t run_capacity, int32_t* tile_meta, int32_t* runs,
                                        uint16_t* local, int64_t* run_count_out,
                                        int32_t* ring_max_out) {
  GSP_REQUIRE(n >= 0 && rows_per_tile > 0 && indptr_host && indices_host && run_count_out &&
                  ring_max_out, "bad ring plan arguments");
  const int64_t R = rows_per_tile, T = n / R;
  GSP_REQUIRE(T >= 1 && T < (int64_t(1) << 30), "tile count out of range");
  std::vector<int32_t> ring;
  int64_t n_runs = 0, ring_max = 0;
  for (int pass = 0; pass < 2; ++pass) {
    // pass 0 counts; pass 1 writes, when everything fits
    if (pass == 1) {
      *run_count_out = n_runs;
      *ring_max_out = int32_t(std::min<int64_t>(ring_max, INT32_MAX));
      if (n_runs > run_capacity || ring_max > 65535) return GSP_OK;
      GSP_REQUIRE(tile_meta && runs && local, "bad ring plan arguments");
      const int64_t nnz = indptr_host[n];
      for (int64_t j = indptr_host[T * R]; j < nnz; ++j) local[j] = 0;
    }
    std::vector<int32_t> pos(pass == 1 ? n : 0);
    int64_t run = 0;
    for (int64_t t = 0; t < T; ++t) {
      ring.clear();
      for (int64_t i = t * R; i < t * R + R; ++i) ring.push_back(int32_t(i));
      for (int64_t j = indptr_host[t * R]; j < indptr_host[t * R + R]; ++j) {
        GSP_REQUIRE(indices_host[j] >= 0 && indices_host[j] < n, "column index out of range");
        ring.push_back(indices_host[j]);
      }
      std::sort(ring.begin(), ring.end());
      ring.erase(std::unique(ring.begin(), ring.end()), ring.end());
      const int64_t size = int64_t(ring.size());
      ring_max = std::max(ring_max, size);
      const int64_t first_run = run;
      int64_t self = 0;
      for (int64_t k = 0; k < size; ++k) {
        if (k == 0 || ring[k] != ring[k - 1] + 1) {
          if (pass == 1) {
            runs[2 * run] = ring[k];
            runs[2 * run + 1] = int32_t(k);
          }
          ++run;
        }
        if (ring[k] == t * R) self = k;
        if (pass == 1) pos[ring[k]] = int32_t(k);
      }
      if (pass == 0) continue;
      tile_meta[4 * t] = int32_t(first_run);
      tile_meta[4 * t + 1] = int32_t(run);
      tile_meta[4 * t + 2] = int32_t(size);
      tile_meta[4 * t + 3] = int32_t(self);
      for (int64_t j = indptr_host[t * R]; j < indptr_host[t * R + R]; ++j)
        local[j] = uint16_t(pos[indices_host[j]]);
    }
    n_runs = run;
    GSP_REQUIRE(n_runs < (int64_t(1) << 31), "too many ring runs");
  }
  return GSP_OK;
}
