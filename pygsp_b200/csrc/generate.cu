// On-device graph construction: the step *before* the filtering path (SURVEY.md 8f-4).
//
//   * Grid2d adjacency (pygsp/graphs/grid2d.py:40-89): 4-neighbour stencil, unit weights,
//     row-major vertex numbering, rows sorted -- count / scan / fill.
//   * k-nearest-neighbour search on a uniform cell grid (replaces scipy.spatial.KDTree
//     in pygsp/graphs/nngraphs/nngraph.py:213-216 and the per-vertex Python loop
//     :221-226): points are binned and sorted by cell (radix sort), every point scans
//     growing rings of cells, keeping its k best candidates sorted, until the k-th
//     distance is provably final; then the directed k-NN matrix with Gaussian weights
//     exp(-d^2/sigma) is emitted as CSR with sorted rows.  Symmetrisation
//     ((W + W^T)/2, nngraph.py:297) is done by the kernels of graph.cu.
// Distances are computed in double, like the reference.
#include <cub/cub.cuh>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {

constexpr int kGenThreads = 256;
constexpr int kMaxK = 32;

// --------------------------------------------------------------------- Grid2d
__global__ void grid2d_count_kernel(int64_t n1, int64_t n2, int32_t* indptr) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i == 0) indptr[0] = 0;
  if (i >= n1 * n2) return;
  const int64_t r = i / n2, c = i - r * n2;
  indptr[i + 1] = int(r > 0) + int(c > 0) + int(c < n2 - 1) + int(r < n1 - 1);
}

template <typename T>
__global__ void grid2d_fill_kernel(int64_t n1, int64_t n2, const int32_t* __restrict__ indptr,
                                   int32_t* indices, T* data) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n1 * n2) return;
  const int64_t r = i / n2, c = i - r * n2;
  int o = indptr[i];
  if (r > 0) { indices[o] = int32_t(i - n2); data[o++] = T(1); }
  if (c > 0) { indices[o] = int32_t(i - 1); data[o++] = T(1); }
  if (c < n2 - 1) { indices[o] = int32_t(i + 1); data[o++] = T(1); }
  if (r < n1 - 1) { indices[o] = int32_t(i + n2); data[o++] = T(1); }
}

// ------------------------------------------------------------------------ kNN
// Cells per axis are bounded by kMaxAxisCells, so home +- ring (ring <= the largest axis) stays
// in int32.
constexpr int kMaxAxisCells = 1 << 30;

struct GridSpec {
  double lo[3];
  double inv_h[3];
  double h[3];
  double slack[3];   // 2^-44 max(|lo|, |hi|): rounding margin of the stopping test
  int cells[3];
  int dim;
};

__device__ __forceinline__ int cell_coord(double x, const GridSpec& g, int d) {
  int c = int(floor((x - g.lo[d]) * g.inv_h[d]));
  return min(max(c, 0), g.cells[d] - 1);
}

__global__ void knn_cell_keys_kernel(int64_t n, const double* __restrict__ pts, GridSpec g,
                                     uint32_t* keys, int32_t* ids) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int cx = cell_coord(pts[i * g.dim + 0], g, 0);
  int cy = cell_coord(pts[i * g.dim + 1], g, 1);
  int cz = g.dim == 3 ? cell_coord(pts[i * g.dim + 2], g, 2) : 0;
  keys[i] = uint32_t((int64_t(cz) * g.cells[1] + cy) * g.cells[0] + cx);
  ids[i] = int32_t(i);
}

// cell_start[c] = first sorted position whose key >= c  (c = 0 .. ncells)
__global__ void knn_cell_start_kernel(int64_t n, int64_t ncells,
                                      const uint32_t* __restrict__ sorted_keys,
                                      int32_t* cell_start) {
  const int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c > ncells) return;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (int64_t(sorted_keys[mid]) < c) lo = mid + 1; else hi = mid;
  }
  cell_start[c] = int32_t(lo);
}

__global__ void knn_gather_points_kernel(int64_t n, int dim, const double* __restrict__ pts,
                                         const int32_t* __restrict__ sorted_ids, double* out) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t src = sorted_ids[i];
  for (int d = 0; d < dim; ++d) out[i * dim + d] = pts[src * dim + d];
}

// One thread per point (in cell order, so that a warp's points share cells).
__global__ void knn_query_kernel(int64_t n, int k, GridSpec g,
                                 const double* __restrict__ sp,          // sorted points
                                 const int32_t* __restrict__ sorted_ids,
                                 const int32_t* __restrict__ cell_start,
                                 int32_t* nn_idx, double* nn_dist) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n) return;
  double best_d[kMaxK];
  int32_t best_i[kMaxK];
  int found = 0;
  double p[3] = {0, 0, 0};
  int home[3] = {0, 0, 0};
  for (int d = 0; d < g.dim; ++d) {
    p[d] = sp[t * g.dim + d];
    home[d] = cell_coord(p[d], g, d);
  }
  const int self = sorted_ids[t];
  const int zdim = g.dim == 3 ? 1 : 0;
  int max_ring = max(g.cells[0], g.cells[1]);
  if (zdim) max_ring = max(max_ring, g.cells[2]);
  for (int ring = 0; ring <= max_ring; ++ring) {
    // the cells at Chebyshev distance `ring` from home, clipped to the grid
    const int x0 = home[0] - ring, x1 = home[0] + ring, y0 = home[1] - ring, y1 = home[1] + ring;
    const int z0 = zdim ? home[2] - ring : 0, z1 = zdim ? home[2] + ring : 0;
    for (int cz = max(z0, 0); cz <= min(z1, g.cells[2] - 1); ++cz) {
      for (int cy = max(y0, 0); cy <= min(y1, g.cells[1] - 1); ++cy) {
        // on a face of the ring's box every cell belongs to the ring, on an inner (z, y) line
        // only the two end cells x0 and x1
        const bool face = (zdim && (cz == z0 || cz == z1)) || cy == y0 || cy == y1;
        for (int cx = face ? max(x0, 0) : x0; cx <= min(x1, g.cells[0] - 1);
             cx = (face || cx == x1) ? cx + 1 : x1) {
          if (cx < 0) continue;
          const int64_t cell = (int64_t(cz) * g.cells[1] + cy) * g.cells[0] + cx;
          for (int q = cell_start[cell]; q < cell_start[cell + 1]; ++q) {
            const int cand = sorted_ids[q];
            if (cand == self) continue;
            // squares summed in dimension order by FMA: gsp_knn_brute's arithmetic, bit for bit
            double d2 = 0;
            for (int d = 0; d < g.dim; ++d) {
              const double diff = sp[int64_t(q) * g.dim + d] - p[d];
              d2 = fma(diff, diff, d2);
            }
            if (found == k && !(d2 < best_d[k - 1] || (d2 == best_d[k - 1] && cand < best_i[k - 1])))
              continue;
            // sorted insertion (distance, then index: deterministic on ties)
            int pos = found < k ? found : k - 1;
            while (pos > 0 && (best_d[pos - 1] > d2 || (best_d[pos - 1] == d2 && best_i[pos - 1] > cand))) {
              best_d[pos] = best_d[pos - 1];
              best_i[pos] = best_i[pos - 1];
              --pos;
            }
            best_d[pos] = d2;
            best_i[pos] = cand;
            if (found < k) ++found;
          }
        }
      }
    }
    if (found == k) {
      // Every unvisited point lies in a cell outside the box searched so far, so it is at least
      // `reach` away, less rounding: a point binned at or above cell c has
      // fl(fl(x - lo) * fl(1 / h)) >= c, so x >= lo + c h (1 - 3u) (and symmetrically below), and
      // the face lo + c h and the distance to it are rounded once each.  Both errors are below 2^-48 max(|lo|, |hi|), and
      // slack = 2^-44 max(|lo|, |hi|) leaves room for the rounding of d^2 too: the d^2 of every
      // unvisited point is strictly above reach^2, so a tie at the k-th distance is always seen.
      double reach = INFINITY;
      bool whole = true;
      for (int d = 0; d < g.dim; ++d) {
        const int lo_c = home[d] - ring, hi_c = home[d] + ring;
        if (lo_c > 0) {
          reach = fmin(reach, p[d] - fma(double(lo_c), g.h[d], g.lo[d]) - g.slack[d]);
          whole = false;
        }
        if (hi_c < g.cells[d] - 1) {
          reach = fmin(reach, fma(double(hi_c + 1), g.h[d], g.lo[d]) - p[d] - g.slack[d]);
          whole = false;
        }
      }
      if (whole || (reach > 0 && best_d[k - 1] < reach * reach)) break;
    }
  }
  for (int j = 0; j < k; ++j) {
    nn_idx[int64_t(self) * k + j] = j < found ? best_i[j] : -1;
    nn_dist[int64_t(self) * k + j] = j < found ? sqrt(best_d[j]) : 0.0;
  }
}

// directed k-NN matrix as CSR with sorted rows: W[i, nn] = exp(-d^2 / sigma)
template <typename T>
__global__ void knn_to_csr_kernel(int64_t n, int k, const int32_t* __restrict__ nn_idx,
                                  const double* __restrict__ nn_dist, double sigma,
                                  int32_t* indptr, int32_t* indices, T* data) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i == 0) indptr[0] = 0;
  if (i >= n) return;
  int32_t col[kMaxK];
  double w[kMaxK];
  for (int j = 0; j < k; ++j) {            // insertion sort by column
    const int32_t c = nn_idx[i * k + j];
    const double d = nn_dist[i * k + j];
    int pos = j;
    while (pos > 0 && col[pos - 1] > c) { col[pos] = col[pos - 1]; w[pos] = w[pos - 1]; --pos; }
    col[pos] = c;
    w[pos] = exp(-(d * d) / sigma);
  }
  indptr[i + 1] = int32_t((i + 1) * k);
  for (int j = 0; j < k; ++j) {
    indices[i * k + j] = col[j];
    data[i * k + j] = T(w[j]);
  }
}

static inline int blocks_for(int64_t n) { return (int)ceil_div(n > 0 ? n : 1, kGenThreads); }

}  // namespace gsp

extern "C" {

int gsp_grid2d_count(int64_t n1, int64_t n2, int32_t* indptr, int64_t* nnz, void* stream) {
  GSP_REQUIRE(n1 >= 1 && n2 >= 1 && n1 * n2 < (int64_t(1) << 31), "grid too large");
  cudaStream_t st = gsp::as_stream(stream);
  gsp::grid2d_count_kernel<<<gsp::blocks_for(n1 * n2), gsp::kGenThreads, 0, st>>>(n1, n2, indptr);
  GSP_LAUNCH_CHECK("grid2d_count");
  return gsp::scan_rows(indptr, n1 * n2, nnz, st);
}

int gsp_grid2d_fill_f32(int64_t n1, int64_t n2, const int32_t* indptr, int32_t* indices,
                        float* data, void* stream) {
  gsp::grid2d_fill_kernel<float><<<gsp::blocks_for(n1 * n2), gsp::kGenThreads, 0,
                                   gsp::as_stream(stream)>>>(n1, n2, indptr, indices, data);
  GSP_LAUNCH_CHECK("grid2d_fill");
  return GSP_OK;
}

int gsp_grid2d_fill_f64(int64_t n1, int64_t n2, const int32_t* indptr, int32_t* indices,
                        double* data, void* stream) {
  gsp::grid2d_fill_kernel<double><<<gsp::blocks_for(n1 * n2), gsp::kGenThreads, 0,
                                    gsp::as_stream(stream)>>>(n1, n2, indptr, indices, data);
  GSP_LAUNCH_CHECK("grid2d_fill");
  return GSP_OK;
}

int gsp_knn_grid(int64_t n, int dim, const double* points, int k, const double* lo_host,
                 const double* hi_host, const int32_t* cells_host, int32_t* nn_idx,
                 double* nn_dist, void* stream) {
  GSP_REQUIRE(dim == 2 || dim == 3, "dim must be 2 or 3");
  GSP_REQUIRE(k >= 1 && k <= gsp::kMaxK && k < n, "k must be in [1, 32] and < n");
  GSP_REQUIRE(n < (int64_t(1) << 31), "too many points");
  cudaStream_t st = gsp::as_stream(stream);
  gsp::GridSpec g;
  memset(&g, 0, sizeof(g));
  g.dim = dim;
  int64_t ncells = 1;
  for (int d = 0; d < 3; ++d) {
    g.cells[d] = d < dim ? cells_host[d] : 1;
    GSP_REQUIRE(g.cells[d] >= 1 && g.cells[d] <= gsp::kMaxAxisCells, "cells must be in [1, 2^30]");
    ncells *= g.cells[d];
    g.lo[d] = d < dim ? lo_host[d] : 0.0;
    const double hi = d < dim ? hi_host[d] : 0.0;
    const double span = hi - g.lo[d];
    GSP_REQUIRE(std::isfinite(span) && span >= 0, "the bounding box must be finite, lo <= hi");
    g.h[d] = span > 0 ? span / g.cells[d] : 1.0;
    g.inv_h[d] = 1.0 / g.h[d];
    g.slack[d] = ldexp(fmax(fabs(g.lo[d]), fabs(hi)), -44);
  }
  GSP_REQUIRE(ncells < (int64_t(1) << 31), "too many cells");
  gsp::Scratch<uint32_t> keys(st), keys_sorted(st);
  gsp::Scratch<int32_t> ids(st), ids_sorted(st), cell_start(st);
  gsp::Scratch<double> sorted_pts(st);
  GSP_CUDA(keys.alloc(n));
  GSP_CUDA(keys_sorted.alloc(n));
  GSP_CUDA(ids.alloc(n));
  GSP_CUDA(ids_sorted.alloc(n));
  GSP_CUDA(cell_start.alloc(ncells + 1));
  GSP_CUDA(sorted_pts.alloc(n * dim));
  const int nb = gsp::blocks_for(n);
  gsp::knn_cell_keys_kernel<<<nb, gsp::kGenThreads, 0, st>>>(n, points, g, keys.get(), ids.get());
  GSP_LAUNCH_CHECK("knn_cell_keys");
  int bits = 1;
  while ((int64_t(1) << bits) < ncells) ++bits;
  const int rc = gsp::cub_temp("cub::DeviceRadixSort::SortPairs", st, [&](void* tmp, size_t& b) {
    return cub::DeviceRadixSort::SortPairs(tmp, b, keys.get(), keys_sorted.get(), ids.get(),
                                           ids_sorted.get(), (int)n, 0, bits, st);
  });
  if (rc != GSP_OK) return rc;
  gsp::knn_cell_start_kernel<<<gsp::blocks_for(ncells + 1), gsp::kGenThreads, 0, st>>>(
      n, ncells, keys_sorted.get(), cell_start.get());
  GSP_LAUNCH_CHECK("knn_cell_start");
  gsp::knn_gather_points_kernel<<<nb, gsp::kGenThreads, 0, st>>>(n, dim, points, ids_sorted.get(),
                                                                sorted_pts.get());
  GSP_LAUNCH_CHECK("knn_gather_points");
  gsp::knn_query_kernel<<<nb, gsp::kGenThreads, 0, st>>>(n, k, g, sorted_pts.get(),
                                                        ids_sorted.get(), cell_start.get(), nn_idx,
                                                        nn_dist);
  GSP_LAUNCH_CHECK("knn_query");
  return GSP_OK;
}

int gsp_knn_to_csr_f32(int64_t n, int k, const int32_t* nn_idx, const double* nn_dist,
                       double sigma, int32_t* indptr, int32_t* indices, float* data,
                       void* stream) {
  GSP_REQUIRE(k >= 1 && k <= gsp::kMaxK && n * k < (int64_t(1) << 31), "bad k / nnz");
  gsp::knn_to_csr_kernel<float><<<gsp::blocks_for(n), gsp::kGenThreads, 0,
                                  gsp::as_stream(stream)>>>(n, k, nn_idx, nn_dist, sigma, indptr,
                                                            indices, data);
  GSP_LAUNCH_CHECK("knn_to_csr");
  return GSP_OK;
}

int gsp_knn_to_csr_f64(int64_t n, int k, const int32_t* nn_idx, const double* nn_dist,
                       double sigma, int32_t* indptr, int32_t* indices, double* data,
                       void* stream) {
  GSP_REQUIRE(k >= 1 && k <= gsp::kMaxK && n * k < (int64_t(1) << 31), "bad k / nnz");
  gsp::knn_to_csr_kernel<double><<<gsp::blocks_for(n), gsp::kGenThreads, 0,
                                   gsp::as_stream(stream)>>>(n, k, nn_idx, nn_dist, sigma,
                                                             indptr, indices, data);
  GSP_LAUNCH_CHECK("knn_to_csr");
  return GSP_OK;
}

}  // extern "C"
