// The vertex-partitioned cheby_op of ONE rank as a single C entry point.
//
// pygsp/filters/approximations.py:58-114 on rows [lo, hi) of a 1-D partitioned Laplacian
// (SURVEY.md 8e): K fused recurrence steps, each of which also carries this rank's part of
// the halo exchange -- boundary rows of T_k are stored straight into the neighbours' halo
// rows over NVLink peer memory from the step kernel's epilogue, flags order the steps.
// No collective library is involved in the per-step path; the communicator is only needed
// once, on the host side, to build the plan (who needs which rows, IPC handles).
//
// Sequence numbers (one uint64 per rank, advanced by M + 2 per call, identical on all ranks):
//   base+1      entry barrier: nobody writes into a rank that is still in its previous call
//   base+2      halo of T_0 (the input block) is in place
//   base+2+s    halo of the block written by step s is in place, s = 1 .. K-1
#include <vector>
#include <cstdio>
#include "step.cuh"

namespace gsp {

template <typename T> struct DistTraits;
template <> struct DistTraits<float> {
  static int push(const gsp_dist_plan* p, int64_t n_send, int b, uint64_t value, int64_t nsig,
                  void* st) {
    return gsp_halo_push_f32(n_send, p->src_row, p->dst_peer, p->dst_row,
                             static_cast<const float*>(p->buf[b]),
                             reinterpret_cast<float* const*>(p->peer_base[b]), nsig, p->peer_flags,
                             p->n_neighbors, value, p->push_counter, st);
  }
};
template <> struct DistTraits<double> {
  static int push(const gsp_dist_plan* p, int64_t n_send, int b, uint64_t value, int64_t nsig,
                  void* st) {
    return gsp_halo_push_f64(n_send, p->src_row, p->dst_peer, p->dst_row,
                             static_cast<const double*>(p->buf[b]),
                             reinterpret_cast<double* const*>(p->peer_base[b]), nsig, p->peer_flags,
                             p->n_neighbors, value, p->push_counter, st);
  }
};

// One step on the whole local block.  Fused form (the exchange fusable and the tiled kernel taking
// the step): wait, push and publish happen inside the step kernel; otherwise wait kernel -> step ->
// push kernel.  new_buf: the window block s.x_new points into (-1: the caller's r, not pushed).
template <typename T>
static int dist_step(const gsp_dist_plan* p, const gsp_tile_plan* tile, bool fusable,
                     const Step<T>& s, int new_buf, uint64_t wait_value, uint64_t publish_value,
                     bool publish, void* stream) {
  cudaStream_t st = as_stream(stream);
  const int64_t n = p->n_local;
  if (fusable && tiled_step_applies(s, 0, tile)) {
    gsp_halo_fusion h;
    memset(&h, 0, sizeof(h));
    h.n_push_rows = publish ? p->n_push_rows : 0;
    h.push_ptr = p->push_ptr;
    h.push_peer = p->push_peer;
    h.push_row = p->push_row;
    h.peer_base = new_buf >= 0 ? p->peer_base[new_buf] : nullptr;
    h.peer_flags = p->peer_flags;
    h.push_counter = p->fused_counter;
    h.wait_flags = p->flags;
    h.wait_ids = p->neighbor_ids;
    h.publish_value = publish_value;
    h.wait_value = wait_value;
    h.n_neighbors = p->n_neighbors;
    h.n_wait = p->n_neighbors;
    h.n_boundary_rows = p->n_boundary_rows;
    h.n_owned = n;
    h.publish = publish ? 1 : 0;
    return run_step<T>(s, 0, n, tile, &h, st);
  }
  int rc = gsp_halo_wait(p->flags, p->neighbor_ids, p->n_neighbors, wait_value, stream);
  if (rc != GSP_OK) return rc;
  // the halo is complete (the wait kernel ran): a step without the fused exchange
  rc = run_step<T>(s, 0, n, tile, nullptr, st);
  if (rc != GSP_OK) return rc;
  if (publish) return DistTraits<T>::push(p, p->n_send, new_buf, publish_value, s.nsig, stream);
  return GSP_OK;
}

// GSPB200_DIST_TRACE=1: per-step CUDA-event times of one call on stderr (diagnosis; synchronises)
struct StepTrace {
  bool on = false;
  cudaStream_t st = nullptr;
  std::vector<cudaEvent_t> ev;
  explicit StepTrace(cudaStream_t s) : st(s) {
    const char* v = getenv("GSPB200_DIST_TRACE");
    on = v && *v == '1';
  }
  void mark() {
    if (!on) return;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, st);
    ev.push_back(e);
  }
  ~StepTrace() {
    if (!on || ev.size() < 2) return;
    cudaEventSynchronize(ev.back());
    fprintf(stderr, "[gspb200 dist trace] ms between marks:");
    for (size_t i = 1; i < ev.size(); ++i) {
      float ms = 0;
      cudaEventElapsedTime(&ms, ev[i - 1], ev[i]);
      fprintf(stderr, " %.3f", ms);
    }
    fprintf(stderr, "\n");
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
  }
};

template <typename T>
int cheby_op_dist(const gsp_dist_plan* p, const gsp_tile_plan* tile, double lmax, const double* c,
                  int nscales, int m, const T* x, int64_t nsig64, T* r, int clenshaw,
                  uint64_t* seq, int phase_begin, int phase_end, void* stream) {
  GSP_REQUIRE(p && seq && r, "null argument");
  GSP_REQUIRE(m >= 2, "The coefficients have an invalid shape");        // approximations.py:83-84
  GSP_REQUIRE(nscales >= 1 && nscales <= 16, "1..16 filters per call");
  GSP_REQUIRE(lmax > 0 && lmax == lmax, "lmax must be positive");
  GSP_REQUIRE(nsig64 >= 1 && nsig64 <= (1 << 20), "nsig out of range");
  const int K = m - 1;
  // phases: 0 entry barrier, 1 input block and halo of T_0, 1 + s recurrence step s = 1 .. K
  GSP_REQUIRE(0 <= phase_begin && phase_begin <= phase_end && phase_end <= K + 2,
              "phase range out of bounds");
  const bool whole = phase_begin == 0 && phase_end == K + 2;
  auto in = [&](int phase) { return phase >= phase_begin && phase < phase_end; };
  const int nsig = int(nsig64);
  const int64_t n = p->n_local;
  cudaStream_t st = as_stream(stream);
  T* buf[3] = {static_cast<T*>(p->buf[0]), static_cast<T*>(p->buf[1]), static_cast<T*>(p->buf[2])};
  // a step fuses the exchange when this holds and the tiled kernel takes it (dist_step)
  const bool fusable =
      tile && tile->rows_per_tile > 0 && !p->separate_exchange && p->n_neighbors >= 1 &&
      p->n_neighbors <= 32 &&
      std::max(p->n_push_rows, p->n_boundary_rows) <= (n / tile->rows_per_tile) * tile->rows_per_tile;
  if (clenshaw && (nscales != 1 || K < 2 || !buf[2])) clenshaw = 0;
  const int64_t* perm = p->perm;      // local row i is row perm[i] of the caller's block
  // the forward form keeps its accumulators in call-local scratch when it permutes rows
  GSP_REQUIRE(whole || clenshaw || !perm, "a phased forward call takes no row permutation");
  const uint64_t base = *seq;
  if (phase_end == K + 2) *seq = base + uint64_t(m) + 2;

  StepTrace trace(st);
  trace.mark();
  int rc = GSP_OK;
  if (in(0)) {        // entry barrier
    rc = DistTraits<T>::push(p, 0, 0, base + 1, nsig, stream);
    if (rc != GSP_OK) return rc;
  }
  if (in(1)) {        // input block, halo of T_0
    rc = gsp_halo_wait(p->flags, p->neighbor_ids, p->n_neighbors, base + 1, stream);
    if (rc != GSP_OK) return rc;
    if (x && perm) {
      rc = move_rows<T>(false, n, perm, x, nsig, buf[0], st);
      if (rc != GSP_OK) return rc;
    } else if (x && x != buf[0]) {
      GSP_CUDA(cudaMemcpyAsync(buf[0], x, sizeof(T) * size_t(n) * nsig, cudaMemcpyDeviceToDevice, st));
    }
    rc = DistTraits<T>::push(p, p->n_send, 0, base + 2, nsig, stream);
    if (rc != GSP_OK) return rc;
    trace.mark();
  }

  // Step s runs in phase 1 + s; the blocks it reads and writes depend on s alone.
  double ck[16], c0[16];
  Step<T> s{p->nnz, p->indptr, p->indices, static_cast<const T*>(p->data)};
  s.r_rows = n;
  s.nsig = nsig;
  if (!clenshaw) {
    // forward recurrence, reference order (approximations.py:99-112).  With a row
    // permutation the accumulators live in local order in stream-ordered scratch and are
    // scattered to the caller's order at the end.
    Scratch<T> local(st);
    if (perm && n > 0) GSP_CUDA(local.alloc(size_t(nscales) * n * nsig));
    s.r = local.get() ? local.get() : r;
    int cur = 0, old = 1;
    for (int k = 1; k <= K; ++k) {
      if (in(1 + k)) {
        forward_coefs(s, k, m, nscales, lmax, c, ck, c0);
        s.x_cur = buf[cur];
        s.x_old = s.first ? nullptr : buf[old];
        s.x_new = buf[old];
        rc = dist_step<T>(p, tile, fusable, s, old, base + 1 + k, base + 2 + k, k < K, stream);
        if (rc != GSP_OK) return rc;
        trace.mark();
      }
      std::swap(cur, old);
    }
    if (local.get()) {
      for (int i = 0; i < nscales && rc == GSP_OK; ++i)
        rc = move_rows<T>(true, n, perm, local.get() + int64_t(i) * n * nsig, nsig,
                          r + int64_t(i) * n * nsig, st);
    }
    return rc;
  }
  // Clenshaw, single filter (see cheby_clenshaw in cheby.cu): buf[0] keeps x (the source),
  // b_{K-1} -> buf[1], b_{K-2} -> buf[2], b_{K-3} -> buf[1], ...; the last step writes r.
  if (in(2)) {
    clenshaw_coefs(s, K - 1, m, 1, lmax, c, ck);
    s.x_cur = buf[0];
    s.x_new = s.r = buf[1];
    rc = dist_step<T>(p, tile, fusable, s, 1, base + 2, base + 3, true, stream);
    if (rc != GSP_OK) return rc;
    trace.mark();
  }
  int cur = 1, old = -1, step = 1;
  for (int k = K - 2; k >= 0; --k) {
    ++step;
    const bool last = k == 0;
    const int dst = last ? -1 : (old >= 0 ? old : 2);
    if (in(1 + step)) {
      clenshaw_coefs(s, k, m, 1, lmax, c, ck);
      s.r = buf[0];
      s.x_cur = buf[cur];
      s.x_old = buf[old >= 0 ? old : cur];   // no b_{k+2} yet: any valid block, times gamma = 0
      s.x_new = last ? r : buf[dst];
      s.out_perm = last ? perm : nullptr;
      rc = dist_step<T>(p, tile, fusable, s, dst, base + 1 + step, base + 2 + step, !last, stream);
      if (rc != GSP_OK) return rc;
      trace.mark();
    }
    old = cur;
    cur = dst;
  }
  return GSP_OK;
}

}  // namespace gsp

extern "C" {
int gsp_cheby_op_dist_phases_f32(const gsp_dist_plan* plan_host, const gsp_tile_plan* tile_host,
                                 double lmax, const double* coeffs_host, int nscales, int m,
                                 const float* x, int64_t nsig, float* r, int clenshaw,
                                 uint64_t* seq_host, int phase_begin, int phase_end, void* stream) {
  return gsp::cheby_op_dist<float>(plan_host, tile_host, lmax, coeffs_host, nscales, m, x, nsig, r,
                                   clenshaw, seq_host, phase_begin, phase_end, stream);
}
int gsp_cheby_op_dist_phases_f64(const gsp_dist_plan* plan_host, const gsp_tile_plan* tile_host,
                                 double lmax, const double* coeffs_host, int nscales, int m,
                                 const double* x, int64_t nsig, double* r, int clenshaw,
                                 uint64_t* seq_host, int phase_begin, int phase_end, void* stream) {
  return gsp::cheby_op_dist<double>(plan_host, nullptr, lmax, coeffs_host, nscales, m, x, nsig, r,
                                    clenshaw, seq_host, phase_begin, phase_end, stream);
}
int gsp_cheby_op_dist_f32(const gsp_dist_plan* plan_host, const gsp_tile_plan* tile_host,
                          double lmax, const double* coeffs_host, int nscales, int m, const float* x,
                          int64_t nsig, float* r, int clenshaw, uint64_t* seq_host, void* stream) {
  return gsp_cheby_op_dist_phases_f32(plan_host, tile_host, lmax, coeffs_host, nscales, m, x, nsig,
                                      r, clenshaw, seq_host, 0, m + 1, stream);
}
int gsp_cheby_op_dist_f64(const gsp_dist_plan* plan_host, const gsp_tile_plan* tile_host,
                          double lmax, const double* coeffs_host, int nscales, int m, const double* x,
                          int64_t nsig, double* r, int clenshaw, uint64_t* seq_host, void* stream) {
  return gsp_cheby_op_dist_phases_f64(plan_host, tile_host, lmax, coeffs_host, nscales, m, x, nsig,
                                      r, clenshaw, seq_host, 0, m + 1, stream);
}
}
