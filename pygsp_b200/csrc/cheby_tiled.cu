// Tiled, warp-specialised Chebyshev step for sm_90a: the float32 fast path.
//
// Same arithmetic as cheby_step_rowgroup (csrc/cheby.cu) -- and therefore the same
// reference lines, pygsp/filters/approximations.py:99-112 -- but every operand
// that is read *contiguously* no longer passes through registers/L1:
//
//   * a persistent CTA owns row tiles t = blockIdx.x, blockIdx.x + gridDim.x, ...
//   * warp 0 is a producer: for each tile it issues 1-D TMA bulk copies
//     (cp.async.bulk ... mbarrier::complete_tx, L2 evict-first) of the tile's CSR slab
//     (indptr / indices / values) and of the tile's x_old and r rows into a
//     ring of `stages` shared-memory stages; the tile's first/last CSR offsets are
//     fetched one tile ahead so that their latency is off the critical path;
//   * the consumer warps wait on the stage's "full" mbarrier, read the CSR
//     entries from shared memory four at a time (LDS.128, no shuffles), gather x_cur
//     rows with coalesced 16-byte loads through L1/L2 (the only traffic left on that
//     path, so L1 holds nothing but x_cur), accumulate in registers in stored CSR
//     order, apply the three-term recurrence and the coefficient AXPYs and store
//     x_new / r with streaming 16-byte stores; then release the stage ("empty").
//
// With neighbour rings (single-source Clenshaw steps whose rings fit, RING instantiations) the
// producer warp also copies the tile's ring -- the x_cur rows its rows reference, and its own --
// into the stage, and the gather reads shared memory (stage_ring_tile, DESIGN.md section 4.1).
//
// Two optional roles of the same kernel:
//   * add_source (Clenshaw form): the r tiles are read-only source blocks,
//     x_new += sum_i ck_i s_i, nothing is written to r  (single-filter Clenshaw and
//     the fused synthesis of Filter.filter);
//   * halo fusion (vertex-partitioned path): wait for the neighbours' flags in the
//     prologue, store boundary rows of x_new into the neighbours' halo rows from
//     the epilogue (peer stores over NVLink), publish the step when the last
//     boundary tile is done  (gsp_halo_fusion in the header).
//
// Lane mapping: G = nsig/4 lanes own one row (a float4 packet each), 32/G rows
// per warp in flight.  A tile's slab must fit `slab_cap` entries: the caller
// obtains the bound from tile_nnz_max() once per matrix (see gsp_cheby_tile_plan).
#include "step.cuh"

namespace gsp {

constexpr int kTiledMaxScales = 16;

struct TileArgs {
  int64_t n_tiles;
  int64_t row_begin;   // first row of tile 0 (multiple of 4)
  int64_t r_rows;
  int64_t nnz;
  const int32_t* indptr;
  const int32_t* indices;
  const float* vals;
  const float* x_cur;
  const float* x_old;
  float* x_new;
  float* r;
  int rows_per_tile;   // R, multiple of 4
  int slab_cap;        // entries per stage for indices / values (multiple of 4)
  int stages;
  int consumer_warps;
  int nsig;
  int nscales;
  float alpha, beta, gamma;
  float half_c0[kTiledMaxScales];
  float ck[kTiledMaxScales];
  gsp_halo_fusion halo;   // all zero when the step does not exchange a halo
  int l2_hint;            // evict-first hint on the streamed TMA copies
  int keep_writes;        // plain instead of evict-first stores for x_new / r
  int reverse;            // walk the tiles from the last to the first (see cheby_op)
  int64_t n_front;        // tiles [0, n_front) always run first, in order (halo: boundary tiles)
  int add_source;         // Clenshaw form: x_new += sum_i ck[i] * (tile i of r), r is not written
  const int64_t* out_perm;  // x_new row of local row i is out_perm[i] (NULL: i); last step of a partitioned call
  int vec_direct;           // x_old / r rows are read straight from global memory (not staged by TMA)
  // Paired launch (cheby_pair_tiled): slot i runs tile slots[i] >> 1 as step A (bit 0 clear: the
  // blocks above) or as step B (bit 0 set: the blocks below, which differ from A's in the three
  // block pointers and in ck only).  B(t) starts once tile_done[s] >= done_target for every s in
  // nbr_idx[nbr_ptr[t] .. nbr_ptr[t + 1]).
  const int32_t* slots = nullptr;
  int64_t n_slots = 0;
  const int32_t* nbr_ptr = nullptr;
  const int32_t* nbr_idx = nullptr;
  unsigned* tile_done = nullptr;
  unsigned done_target = 0;
  const float* x_cur2 = nullptr;
  const float* x_old2 = nullptr;
  float* x_new2 = nullptr;
  float ck2 = 0.f;
  // Neighbour rings (gsp_ring_plan; ring_cap == 0: none).  The producer copies tile t's ring rows
  // of the gathered block into the stage, and the CSR slab carries ring positions (ring_local)
  // instead of column ids.  Only with row_begin == 0, a stage without vector tiles and no halo.
  const int4* ring_meta = nullptr;     // per tile: first run, end of runs, ring rows, position of row t R
  const int2* ring_runs = nullptr;     // per run: first row, ring position
  const uint16_t* ring_local = nullptr;
  int ring_cap = 0;                    // ring rows a stage holds
};

// ----------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_addr(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
// 1-D TMA bulk copy global -> shared, completion counted on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_addr(dst)),
      "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(smem_addr(bar))
      : "memory");
}

// same, with an L2 eviction-priority hint (streamed operands: read once per step)
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes,
                                              uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_addr(dst)),
      "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(smem_addr(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}

__device__ __forceinline__ float4 ldg_f4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}
__device__ __forceinline__ void stcs_f4(float* p, const float4& v) {
  __stcs(reinterpret_cast<float4*>(p), v);
}
// x_new / r: streaming (evict-first) stores, or plain ones when the next step walks the
// tiles in the opposite direction and re-reads the lines this step wrote last
__device__ __forceinline__ void store_f4(float* p, const float4& v, bool keep) {
  if (keep) *reinterpret_cast<float4*>(p) = v; else stcs_f4(p, v);
}

// shared-memory carve-up, identical on host and device
// Without a ring a stage is [vector tiles | column ids | values | indptr]; with one (no vector
// tiles then) it is [ring rows | values | ring positions | indptr].
struct TileLayout {
  int vec_bytes;      // x_old + r tiles of one stage, or the ring rows
  int slab_bytes;     // the values slab (4-byte column ids: as large, 2-byte ring positions: half)
  int idx_bytes;
  int ptr_bytes;      // indptr slab + trailing slot
  int stage_bytes;
  int bar_bytes;
  __host__ __device__ TileLayout(int R, int cap, int nsig, int nscales, bool first, int stages,
                                 int ring_cap = 0) {
    vec_bytes = ring_cap ? ring_cap * nsig * 4 : (first ? 0 : (1 + nscales) * R * nsig * 4);
    slab_bytes = (cap + 16) * 4;                // +16: aligned groups may run past the end
    idx_bytes = ring_cap ? slab_bytes / 2 : slab_bytes;
    ptr_bytes = (R + 4) * 4;
    stage_bytes = vec_bytes + slab_bytes + idx_bytes + ptr_bytes + 16;   // +16: slab offset, ring position of the tile
    bar_bytes = ((2 * stages * 8 + 15) / 16) * 16;
  }
  __host__ __device__ int total(int stages) const { return bar_bytes + stages * stage_bytes; }
};

// Order in which the persistent CTAs visit the tiles.  Tiles [0, n_front) come first, in
// order (vertex-partitioned path: the boundary tiles, whose rows the neighbours wait for);
// the others are walked forwards or backwards (`reverse`: the lines the previous step wrote
// last are still in L2 and are the first ones this step reads).
__device__ __forceinline__ int64_t tile_of_slot(const TileArgs& a, int64_t slot) {
  if (slot < a.n_front) return slot;
  return a.reverse ? a.n_tiles - 1 - (slot - a.n_front) : slot;
}

// Halo rows of x_cur are written by the neighbours (peer stores) while this kernel may
// already be running: a tile whose rows reference halo columns (the boundary tiles of a
// partitioned step, a few per launch) gathers through L2 (ld.global.cg), never through the
// non-coherent path.  Interior tiles only touch rows this GPU owns, which are read-only for the
// whole launch: ld.global.nc.
// Step B of a paired launch gathers a block that step A writes during the same launch (each row
// only after the acquire that proves it was written): a plain ld.global, cached in L1 like the
// non-coherent gather but never turned into one by the compiler.
__device__ __forceinline__ float4 ld_plain_f4(const float* p) {
  float4 v;
  asm volatile("ld.global.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
// kGatherRing: the rows come from the tile's neighbour ring in shared memory, `col` is a ring
// position.
constexpr int kGatherNc = 0, kGatherL2 = 1, kGatherPlain = 2, kGatherRing = 3;
template <int COH>
__device__ __forceinline__ float4 gather_f4(const float* __restrict__ xg, int col, int ns) {
  if (COH == kGatherRing) return *reinterpret_cast<const float4*>(xg + col * ns);
  const float* p = xg + int64_t(col) * ns;
  if (COH == kGatherL2) return __ldcg(reinterpret_cast<const float4*>(p));
  if (COH == kGatherPlain) return ld_plain_f4(p);
  return ldg_f4(p);
}

// four column ids (one LDS.128) or four 16-bit ring positions (one LDS.64) of an aligned group
__device__ __forceinline__ void load_idx4(const int32_t* p, int (&c)[4]) {
  const int4 v = *reinterpret_cast<const int4*>(p);
  c[0] = v.x; c[1] = v.y; c[2] = v.z; c[3] = v.w;
}
__device__ __forceinline__ void load_idx4(const uint16_t* p, int (&c)[4]) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  c[0] = int(v.x & 0xffffu); c[1] = int(v.x >> 16); c[2] = int(v.y & 0xffffu); c[3] = int(v.y >> 16);
}

// sum_j w_j x_cur[col_j, packets of this lane] over the stored entries [jb, je) of one row
// (slab-relative offsets).  The slab offset is a multiple of 4, so groups of four CSR entries
// are 16-byte aligned in shared memory: one LDS.128 brings four column indices, one four
// weights.  Slots outside [jb, je) (row head / tail) are predicated off, so the sum runs over
// the row's entries in stored order.  A lane owns P float4 packets of the row, 16 G bytes apart
// (P = 1: G lanes cover the row once; P = 2: G lanes cover it twice, so a row group is a quarter
// warp for 64 signals and one LDS.128 of CSR entries serves four rows instead of two -- the
// broadcast read costs one L1 wavefront per quarter warp whatever it delivers).  4 / P entries
// are in flight per lane at a time (the same 64 bytes either way).
// COH: the row may reference halo columns (boundary tiles of a partitioned step) -- the tile
// gathers through L2 then; interior tiles use the plain non-coherent gather only.
template <int G, int P, int COH, typename IDX>
__device__ __forceinline__ void row_gather_sum(const IDX* __restrict__ sm_col,
                                               const float* __restrict__ sm_val, int jb, int je,
                                               const float* __restrict__ xg, float4 (&acc)[P]) {
  constexpr int NS = 4 * G * P;
  constexpr int E = 4 / P;                         // entries requested back to back
  const unsigned span = unsigned(je - jb);
#pragma unroll
  for (int p = 0; p < P; ++p) acc[p] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int jj = jb & ~3; jj < je; jj += 4) {
    int cq[4];
    load_idx4(sm_col + jj, cq);
    const float4 w4 = *reinterpret_cast<const float4*>(sm_val + jj);
    const int base = jj - jb;
    const float wq[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
    for (int h = 0; h < P; ++h) {
      float4 xv[E][P];
      bool ok[E];
#pragma unroll
      for (int e = 0; e < E; ++e) {
        ok[e] = unsigned(base + h * E + e) < span;
#pragma unroll
        for (int p = 0; p < P; ++p)
          if (ok[e]) xv[e][p] = gather_f4<COH>(xg + p * 4 * G, cq[h * E + e], NS);
      }
#pragma unroll
      for (int e = 0; e < E; ++e) {
        if (ok[e]) {
          const float w = wq[h * E + e];
#pragma unroll
          for (int p = 0; p < P; ++p) {
            acc[p].x = fmaf(w, xv[e][p].x, acc[p].x);
            acc[p].y = fmaf(w, xv[e][p].y, acc[p].y);
            acc[p].z = fmaf(w, xv[e][p].z, acc[p].z);
            acc[p].w = fmaf(w, xv[e][p].w, acc[p].w);
          }
        }
      }
    }
  }
}

// What a consumer lane needs to process one staged tile.
struct TileCtx {
  const float* sm_vec;      // x_old tile, then one r / source tile per scale (empty in direct
                            // mode); with a ring: the ring rows
  const void* sm_col;       // CSR slab: column indices (int32), with a ring ring positions (uint16)
  const float* sm_val;      //           values
  const int32_t* sm_ptr;    // indptr[r0 .. r0 + R], slab offset at [R + 4], ring position of r0 at [R + 5]
  int64_t tile;
  int64_t r0;               // first row of the tile (block-local row index)
  int cw, sub, c0;          // consumer warp, row slot inside the warp, first column of the lane
  bool vd;                  // direct mode: x_old / r rows come straight from global memory
};

__device__ __forceinline__ void fma4(float4& d, float w, const float4& v) {
  d.x = fmaf(w, v.x, d.x);
  d.y = fmaf(w, v.y, d.y);
  d.z = fmaf(w, v.z, d.z);
  d.w = fmaf(w, v.w, d.w);
}

// The rows of one tile: gather + three-term recurrence + coefficient AXPYs + stores.
// COH: the tile's rows may reference halo columns (coherent gathers through L2).
// COH == kGatherRing: the x_cur rows (the gathered ones and the tile's own) come from the ring.
// PAIR (paired launch): 1 = step A, 2 = step B.  B takes its blocks and ck from the second operand
// set and reads the gathered block, which A writes in the same launch, with plain loads.  A reads
// the source rows through L2 without the evict-first mark, since B reads them again.
template <int G, bool FIRST, int NSC, int COH, int P, int PAIR = 0>
__device__ __forceinline__ void tile_rows(const TileArgs& a, const TileCtx t) {
  const float* x_cur_blk = PAIR == 2 ? a.x_cur2 : a.x_cur;
  const float* x_old_blk = PAIR == 2 ? a.x_old2 : a.x_old;
  float* x_new_blk = PAIR == 2 ? a.x_new2 : a.x_new;
  constexpr int RP = 32 / G;               // rows in flight per warp
  constexpr int NS = 4 * G * P;            // signal columns (compile-time: cheap addressing)
  constexpr int PS = 4 * G;                // column distance between a lane's packets
  const int R = a.rows_per_tile;
  const int NW = a.consumer_warps;
  const int c0 = t.c0;
  constexpr bool RING = COH == kGatherRing;
  // this lane's first column packet of x_cur, or of the ring
  const float* __restrict__ xg = (RING ? t.sm_vec : x_cur_blk) + c0;
  const int nscales = NSC >= 0 ? NSC : a.nscales;
  const float alpha = a.alpha, beta = a.beta, gamma = a.gamma;
  // (B's stores are evict-first: nothing reads them before the next launch, and L2 is what the
  //  pair lives on; config 2, H100: 12.25 -> 12.02 ms per call)
  const bool keep_writes = a.keep_writes != 0 && PAIR != 2;
  const bool VD = t.vd;
  const float* sm_vec = t.sm_vec;
  const int a0 = t.sm_ptr[R + 4];
  const int64_t r0 = t.r0;
  const float* __restrict__ xc_tile = xg + (RING ? int64_t(t.sm_ptr[R + 5]) : r0) * NS;
  float* __restrict__ xn_tile = x_new_blk + r0 * NS + c0;
  float* __restrict__ r_tile = a.r + r0 * NS + c0;
  const int64_t r_stride = a.r_rows * NS;

  for (int lr = t.cw * RP + t.sub; lr < R; lr += NW * RP) {
    const int off = lr * NS;
    const int jb = t.sm_ptr[lr] - a0;
    const int je = t.sm_ptr[lr + 1] - a0;
    float4 xc[P];
#pragma unroll
    for (int p = 0; p < P; ++p)
      xc[p] = COH == kGatherPlain ? ld_plain_f4(xc_tile + off + p * PS)
              : RING ? *reinterpret_cast<const float4*>(xc_tile + off + p * PS)
                     : ldg_f4(xc_tile + off + p * PS);
    // direct mode: this row's x_old and first r / source packets are requested now (streaming
    // loads, no L1 allocation) and consumed after the gather loop, which hides their latency
    float4 xo_d[P], r0_d[P];
#pragma unroll
    for (int p = 0; p < P; ++p) xo_d[p] = r0_d[p] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!FIRST && VD) {
#pragma unroll
      for (int p = 0; p < P; ++p) {
        xo_d[p] = __ldcs(reinterpret_cast<const float4*>(x_old_blk + (r0 + lr) * NS + c0 + p * PS));
        if (NSC != 0 && nscales > 0) {
          const float4* rp = reinterpret_cast<const float4*>(a.r + (r0 + lr) * NS + c0 + p * PS);
          r0_d[p] = PAIR == 1 ? __ldcg(rp) : __ldcs(rp);
        }
      }
    }
    float4 acc[P];
    if constexpr (RING)
      row_gather_sum<G, P, COH>(static_cast<const uint16_t*>(t.sm_col), t.sm_val, jb, je, xg, acc);
    else
      row_gather_sum<G, P, COH>(static_cast<const int32_t*>(t.sm_col), t.sm_val, jb, je, xg, acc);
    float4 xn[P];
#pragma unroll
    for (int p = 0; p < P; ++p) {
      xn[p].x = fmaf(alpha, acc[p].x, beta * xc[p].x);
      xn[p].y = fmaf(alpha, acc[p].y, beta * xc[p].y);
      xn[p].z = fmaf(alpha, acc[p].z, beta * xc[p].z);
      xn[p].w = fmaf(alpha, acc[p].w, beta * xc[p].w);
      if (!FIRST) {
        const float4 xo =
            VD ? xo_d[p] : *reinterpret_cast<const float4*>(sm_vec + off + c0 + p * PS);
        fma4(xn[p], gamma, xo);
      }
    }
    if (!FIRST && NSC != 0 && a.add_source) {
      // Clenshaw form: the r tiles are read-only source blocks, x_new += sum_i ck_i s_i
#pragma unroll
      for (int i = 0; i < (NSC >= 0 ? NSC : kTiledMaxScales); ++i) {
        if (NSC < 0 && i >= nscales) break;
        const float w = PAIR == 2 ? a.ck2 : a.ck[i];
#pragma unroll
        for (int p = 0; p < P; ++p) {
          const float4 sv =
              VD ? (i == 0 ? r0_d[p]
                           : __ldcs(reinterpret_cast<const float4*>(
                                 a.r + i * r_stride + (r0 + lr) * NS + c0 + p * PS)))
                 : *reinterpret_cast<const float4*>(sm_vec + (i + 1) * R * NS + off + c0 + p * PS);
          fma4(xn[p], w, sv);
        }
      }
    }
    if (a.out_perm) {    // the caller's row order: local row -> original row (uniform branch)
      float* dst = x_new_blk + __ldg(a.out_perm + r0 + lr) * NS + c0;
#pragma unroll
      for (int p = 0; p < P; ++p) store_f4(dst + p * PS, xn[p], keep_writes);
    } else {
#pragma unroll
      for (int p = 0; p < P; ++p) store_f4(xn_tile + off + p * PS, xn[p], keep_writes);
    }
#pragma unroll
    for (int i = 0; i < (NSC >= 0 ? NSC : kTiledMaxScales); ++i) {
      if (NSC < 0 && i >= nscales) break;
      if (!FIRST && a.add_source) break;
      const float ck = a.ck[i];
#pragma unroll
      for (int p = 0; p < P; ++p) {
        float4 rv;
        if (FIRST) {
          const float h0 = a.half_c0[i];
          rv.x = fmaf(ck, xn[p].x, h0 * xc[p].x);
          rv.y = fmaf(ck, xn[p].y, h0 * xc[p].y);
          rv.z = fmaf(ck, xn[p].z, h0 * xc[p].z);
          rv.w = fmaf(ck, xn[p].w, h0 * xc[p].w);
        } else {
          rv = VD ? (i == 0 ? r0_d[p]
                            : __ldcs(reinterpret_cast<const float4*>(
                                  a.r + i * r_stride + (r0 + lr) * NS + c0 + p * PS)))
                  : *reinterpret_cast<const float4*>(sm_vec + (i + 1) * R * NS + off + c0 + p * PS);
          fma4(rv, ck, xn[p]);
        }
        store_f4(r_tile + i * r_stride + off + p * PS, rv, keep_writes);
      }
    }
  }
}

// A boundary ("front") tile of a partitioned step -- a few tiles per launch.  It is a real
// function call on purpose: inlined, its extra state (flags, peer tables, a second copy of
// the gather loop) made ptxas spill registers in the interior tiles' loop as well
// (slower steps).  Does, for one consumer warp:
//   wait   : until the neighbours have published the halo of x_cur (they stored it straight
//            into this GPU's memory and released wait_value afterwards);
//   rows   : the tile's rows with coherent gathers;
//   push   : every lane re-reads the packets it has just stored (its own writes, program
//            order) and stores them into the halo rows of the neighbours that reference the
//            row -- peer stores over NVLink;
//   publish: every warp of every CTA checks in once per front tile; when the last one has,
//            (a) all boundary rows of x_new are stored in the neighbours and (b) nobody on this
//            GPU reads the halo of x_cur any more: the step is released to the neighbours,
//            which may then read their halo of x_new and overwrite our halo of x_cur's buffer.
template <int G, bool FIRST, int NSC>
__device__ __noinline__ void boundary_tile(const TileArgs& a, const TileCtx t, int lane) {
  constexpr int RP = 32 / G;
  constexpr int NS = 4 * G;
  const int R = a.rows_per_tile;
  const int NW = a.consumer_warps;
  if (t.tile < a.halo.n_wait_tiles && a.halo.n_wait > 0) {
    if (lane < a.halo.n_wait) {
      const unsigned long long* f =
          reinterpret_cast<const unsigned long long*>(a.halo.wait_flags) + a.halo.wait_ids[lane];
      unsigned long long seen;
      do {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(f) : "memory");
      } while (seen < a.halo.wait_value);
    }
    __syncwarp();
  }
  tile_rows<G, FIRST, NSC, kGatherL2, 1>(a, t);
  if (t.tile >= a.halo.n_push_tiles) return;
  if (!a.out_perm) {
    const float* xn_tile = a.x_new + t.r0 * NS + t.c0;
    for (int lr = t.cw * RP + t.sub; lr < R; lr += NW * RP) {
      const int64_t lrow = t.tile * R + lr;
      if (lrow >= a.halo.n_push_rows) continue;
      const int e0 = a.halo.push_ptr[lrow], e1 = a.halo.push_ptr[lrow + 1];
      if (e0 == e1) continue;
      const float4 xn = *reinterpret_cast<const float4*>(xn_tile + lr * NS);
      for (int e = e0; e < e1; ++e) {
        float* dst = reinterpret_cast<float* const*>(a.halo.peer_base)[a.halo.push_peer[e]] +
                     a.halo.push_row[e] * NS + t.c0;
        *reinterpret_cast<float4*>(dst) = xn;
      }
    }
  }
  __threadfence_system();
  __syncwarp();
  if (lane == 0) {
    const unsigned long long want =
        (unsigned long long)a.halo.n_push_tiles * (unsigned long long)NW;
    const unsigned long long prev =
        atomicAdd(reinterpret_cast<unsigned long long*>(a.halo.push_counter), 1ull);
    if (prev + 1 == want) {
      *reinterpret_cast<volatile unsigned long long*>(a.halo.push_counter) = 0ull;
      __threadfence_system();
      for (int q = 0; q < a.halo.n_neighbors; ++q)
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(
                         reinterpret_cast<unsigned long long* const*>(a.halo.peer_flags)[q]),
                     "l"((unsigned long long)a.halo.publish_value)
                     : "memory");
    }
  }
}

// Ring mode, the whole producer warp: stage tile `tile` (CSR entries [begin, end), ring `m`) in
// stage `st` -- indptr, values and ring positions by lane 0, then one bulk copy of the rows of
// `xg` per run of the ring, spread over the lanes.  One expect_tx covers the stage.  The slab
// starts at a multiple of 8 entries, so that the 2-byte positions are 16-byte aligned as well.
__device__ __forceinline__ void stage_ring_tile(const TileArgs& a, const TileLayout& lay,
                                                unsigned char* st, uint64_t* full, int64_t tile,
                                                int begin, int end, int4 m, const float* xg,
                                                bool evict, uint64_t pol, int lane) {
  const int R = a.rows_per_tile;
  const int nsig = a.nsig;
  float* sm_ring = reinterpret_cast<float*>(st);
  float* sm_val = reinterpret_cast<float*>(st + lay.vec_bytes);
  uint16_t* sm_loc = reinterpret_cast<uint16_t*>(st + lay.vec_bytes + lay.slab_bytes);
  int32_t* sm_ptr = reinterpret_cast<int32_t*>(st + lay.vec_bytes + lay.slab_bytes + lay.idx_bytes);
  const uint32_t row_bytes = uint32_t(nsig) * 4u;
  if (lane == 0) {
    const int64_t r0 = tile * R;
    const int a0 = begin & ~7;
    int a1 = (end + 7) & ~7;
    if (int64_t(a1) > a.nnz) a1 = end & ~7;     // never read past the arrays
    sm_ptr[R] = end;                            // the bulk copy brings indptr[r0 .. r0+R)
    sm_ptr[R + 4] = a0;
    sm_ptr[R + 5] = m.w;
    for (int k = (a1 > a0 ? a1 : a0); k < end; ++k) {   // <= 7 trailing entries, last tile only
      sm_val[k - a0] = __ldg(a.vals + k);
      sm_loc[k - a0] = __ldg(a.ring_local + k);
    }
    const uint32_t len = a1 > a0 ? uint32_t(a1 - a0) : 0u;
    mbar_expect_tx(full, uint32_t(R) * 4u + 6u * len + uint32_t(m.z) * row_bytes);
    bulk_g2s(sm_ptr, a.indptr + r0, uint32_t(R) * 4u, full);
    if (len && evict) {
      bulk_g2s_hint(sm_val, a.vals + a0, 4u * len, full, pol);
      bulk_g2s_hint(sm_loc, a.ring_local + a0, 2u * len, full, pol);
    } else if (len) {
      bulk_g2s(sm_val, a.vals + a0, 4u * len, full);
      bulk_g2s(sm_loc, a.ring_local + a0, 2u * len, full);
    }
  }
  __syncwarp();                                 // the expect_tx precedes every complete_tx
  for (int i = m.x + lane; i < m.y; i += 32) {
    const int2 run = __ldg(a.ring_runs + i);
    const int next = i + 1 < m.y ? __ldg(a.ring_runs + i + 1).y : m.z;
    bulk_g2s(sm_ring + size_t(run.y) * nsig, xg + int64_t(run.x) * nsig,
             uint32_t(next - run.y) * row_bytes, full);
  }
}

// One packet per lane: 1 + 16 warps per CTA, 2 CTAs per SM (<= 60 registers).  Two packets per
// lane keep twice the state per lane: 1 + 8 warps, 3 CTAs per SM (<= 75 registers).
// RING: the gather reads the tile's neighbour ring, staged by the whole producer warp (no halo,
// first step or direct vectors).
template <int G, bool FIRST, int NSC, bool HALO, int P, bool RING>
__global__ void __launch_bounds__(32 * (P == 2 ? 9 : 17), P == 2 ? 3 : 2)
cheby_step_tiled(const __grid_constant__ TileArgs a) {
  static_assert(!(RING && HALO), "the halo path keeps the gather from global memory");
  extern __shared__ __align__(128) unsigned char smem[];
  const int R = a.rows_per_tile;
  const int S = a.stages;
  const int NW = a.consumer_warps;
  const int nsig = a.nsig;
  const bool VD = !FIRST && a.vec_direct != 0;     // CTA-uniform
  const TileLayout lay(R, a.slab_cap, nsig, a.nscales, FIRST || VD, S, RING ? a.ring_cap : 0);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + S;
  unsigned char* stage0 = smem + lay.bar_bytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full + s, 1);
      mbar_init(empty + s, NW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ------------------------------------------------------------- producer
    // (nothing the producer stages depends on the halo: CSR slabs, x_old and r rows are local)
    // x_old / r / CSR are touched once per step: mark them evict-first so that the
    // L2 keeps the x_cur lines the gathers re-use (GSPB200_TILE_HINT=0 disables)
    const bool hint = a.l2_hint != 0;
    const uint64_t pol = l2_policy_evict_first();
    if (RING) {
      int it = 0;
      for (int64_t slot = blockIdx.x; slot < a.n_tiles; slot += gridDim.x, ++it) {
        const int64_t tile = tile_of_slot(a, slot);
        const int begin = __ldg(a.indptr + tile * R), end = __ldg(a.indptr + tile * R + R);
        const int4 m = __ldg(a.ring_meta + tile);
        const int s = it % S;
        mbar_wait(empty + s, (uint32_t(it / S) & 1u) ^ 1u);
        stage_ring_tile(a, lay, stage0 + size_t(s) * lay.stage_bytes, full + s, tile, begin, end,
                        m, a.x_cur, hint, pol, lane);
      }
      return;
    }
    if (lane != 0) return;
    int it = 0;
    // the tile's first / last CSR offsets are fetched one tile ahead, so that their
    // DRAM latency is not in series with the wait for a free slot
    int nbegin = 0, nend = 0;
    if (int64_t(blockIdx.x) < a.n_tiles) {
      const int64_t rn = a.row_begin + tile_of_slot(a, blockIdx.x) * R;
      nbegin = __ldg(a.indptr + rn);
      nend = __ldg(a.indptr + rn + R);
    }
    for (int64_t slot = blockIdx.x; slot < a.n_tiles; slot += gridDim.x, ++it) {
      const int64_t tile = tile_of_slot(a, slot);
      const int s = it % S;
      const uint32_t round = uint32_t(it / S);
      const int begin = nbegin, end = nend;
      if (slot + gridDim.x < a.n_tiles) {
        const int64_t rn = a.row_begin + tile_of_slot(a, slot + gridDim.x) * R;
        nbegin = __ldg(a.indptr + rn);
        nend = __ldg(a.indptr + rn + R);
      }
      mbar_wait(empty + s, (round & 1u) ^ 1u);      // slot free (passes at once in round 0)
      unsigned char* st = stage0 + size_t(s) * lay.stage_bytes;
      float* sm_vec = reinterpret_cast<float*>(st);
      int32_t* sm_col = reinterpret_cast<int32_t*>(st + lay.vec_bytes);
      float* sm_val = reinterpret_cast<float*>(st + lay.vec_bytes + lay.slab_bytes);
      int32_t* sm_ptr = reinterpret_cast<int32_t*>(st + lay.vec_bytes + 2 * lay.slab_bytes);
      int32_t* sm_meta = sm_ptr + (R + 4);

      const int64_t r0 = a.row_begin + tile * R;
      const int a0 = begin & ~3;                    // 16-byte aligned slab start
      int a1 = (end + 3) & ~3;
      if (int64_t(a1) > a.nnz) a1 = end & ~3;      // never read past the arrays
      sm_ptr[R] = end;                              // the bulk copy brings indptr[r0 .. r0+R)
      sm_meta[0] = a0;
      for (int k = (a1 > a0 ? a1 : a0); k < end; ++k) {   // <= 3 trailing entries, last tile only
        sm_col[k - a0] = __ldg(a.indices + k);
        sm_val[k - a0] = __ldg(a.vals + k);
      }
      const uint32_t slab = a1 > a0 ? uint32_t(a1 - a0) * 4u : 0u;
      const uint32_t tile_vec = uint32_t(R) * nsig * 4u;
      const bool stage_vec = !FIRST && !VD;
      const uint32_t bytes = uint32_t(R) * 4u + 2u * slab +
                             (stage_vec ? tile_vec * (1 + a.nscales) : 0u);
      mbar_expect_tx(full + s, bytes);
      bulk_g2s(sm_ptr, a.indptr + r0, uint32_t(R) * 4u, full + s);
      if (hint) {
        if (slab) {
          bulk_g2s_hint(sm_col, a.indices + a0, slab, full + s, pol);
          bulk_g2s_hint(sm_val, a.vals + a0, slab, full + s, pol);
        }
        if (stage_vec) {
          bulk_g2s_hint(sm_vec, a.x_old + r0 * nsig, tile_vec, full + s, pol);
          for (int i = 0; i < a.nscales; ++i)
            bulk_g2s_hint(sm_vec + size_t(i + 1) * R * nsig,
                          a.r + (int64_t(i) * a.r_rows + r0) * nsig, tile_vec, full + s, pol);
        }
      } else {
        if (slab) {
          bulk_g2s(sm_col, a.indices + a0, slab, full + s);
          bulk_g2s(sm_val, a.vals + a0, slab, full + s);
        }
        if (stage_vec) {
          bulk_g2s(sm_vec, a.x_old + r0 * nsig, tile_vec, full + s);
          for (int i = 0; i < a.nscales; ++i)
            bulk_g2s(sm_vec + size_t(i + 1) * R * nsig,
                     a.r + (int64_t(i) * a.r_rows + r0) * nsig, tile_vec, full + s);
        }
      }
    }
    return;
  }

  // ---------------------------------------------------------------- consumers
  const int cw = warp - 1;
  const int sub = lane / G;
  const int c0 = (lane % G) * 4;
  int it = 0;
  for (int64_t slot = blockIdx.x; slot < a.n_tiles; slot += gridDim.x, ++it) {
    const int64_t tile = tile_of_slot(a, slot);
    const int s = it % S;
    const uint32_t round = uint32_t(it / S);
    mbar_wait(full + s, round & 1u);
    unsigned char* st = stage0 + size_t(s) * lay.stage_bytes;
    // (the context is built per use and passed BY VALUE: a struct whose address escapes to the
    //  non-inlined boundary routine would live in local memory for the interior path too)
    // (ring: [ring | values | positions | indptr], else [vectors | columns | values | indptr])
    const unsigned char* sl0 = st + lay.vec_bytes;
    const unsigned char* sl1 = sl0 + lay.slab_bytes;
    const TileCtx t = {reinterpret_cast<const float*>(st), RING ? sl1 : sl0,
                       reinterpret_cast<const float*>(RING ? sl0 : sl1),
                       reinterpret_cast<const int32_t*>(sl1 + lay.idx_bytes),
                       tile, a.row_begin + tile * R, cw, sub, c0, VD};
    if (HALO && tile < a.n_front)          // warp-uniform; interior tiles never wait
      boundary_tile<G, FIRST, NSC>(a, t, lane);
    else
      tile_rows<G, FIRST, NSC, RING ? kGatherRing : kGatherNc, P>(a, t);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + s);
  }
}

// Two middle Clenshaw steps in one launch (float32, one source, direct vectors, one-stage ring).
// Step A forms b_k = a2 L P - 2 P - Q + c_k x into a third block W; step B forms
// b_{k-1} = a2 L W - 2 W - P + c_{k-1} x over Q.  The CTAs walk a slot table (built once per
// matrix, csrc/pair_plan.cu) round-robin: the A tiles in walk order, and B(t) a fixed lag after
// the last A tile among t and the tiles t's rows reference -- late enough that those A tiles are
// done when B(t) starts (slots that are neighbours in the table run at the same time on
// different CTAs), early enough that W, P and x are still in L2: five passes over a signal block
// per pair instead of eight.  No block is both gathered and written in the launch: P and x are
// read-only, W is written by A and read by B only, and the rows of Q that B(t) overwrites are
// read by A(t) alone.  Per row the instructions are those of the single step: the same bits.
//
// On the release side each warp's stores are ordered by __syncwarp before lane 0's red.release (a
// fence without L1 invalidation).  The acquire side has two forms.
//
// RING (the neighbour rings fit): A(t) stages the ring of P, B(t) the ring of W, and the producer
// warp waits for B(t)'s A tiles before it stages B(t), while the consumers still work on the slots
// before it: its lanes poll the flags with relaxed loads, then every lane issues
// fence.acq_rel.gpu -- with the relaxed reads of the flags and the releasing red of the A warps
// this is the fence-based release / acquire pattern that makes A's stores of W visible (PTX ISA,
// "Memory Consistency Model", sections on release / acquire patterns and causality order) -- and
// fence.proxy.async.global, which orders those generic-proxy stores before the async-proxy reads
// of the bulk copies that follow (same chapter, "Proxies").  The consumers see the staged rows
// through the stage's mbarrier.  Nothing the gathers read lives in L1, so the L1 invalidation that
// the acquire implies costs nothing.  No deadlock: the producer stages its CTA's slots in order,
// at most `stages` ahead of the consumers; an A slot waits for nothing, a B slot only for A slots
// lower in the table (checked when the table is built); so the lowest unfinished slot of the
// launch -- whose CTA has finished, and so has freed the stages of, every slot before it -- can
// always be staged and run, given that every CTA of the grid is resident (the launch requires it).
//
// Without a ring, the gathers of all resident CTAs live on L1, so the acquire is paid once per B
// tile and CTA and never inside a poll loop: consumer warp 0 polls with relaxed loads, fences once,
// and a named barrier hands the tile to the other consumer warps (one stage).
template <int G, int P, bool RING>
__global__ void __launch_bounds__(32 * (P == 2 ? 9 : 17), P == 2 ? 3 : 2)
cheby_pair_tiled(const __grid_constant__ TileArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int R = a.rows_per_tile;
  const int NW = a.consumer_warps;
  const int S = RING ? a.stages : 1;
  const TileLayout lay(R, a.slab_cap, a.nsig, a.nscales, true, S, RING ? a.ring_cap : 0);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + S;
  unsigned char* stage0 = smem + lay.bar_bytes;
  unsigned char* st = stage0;
  int32_t* sm_col = reinterpret_cast<int32_t*>(st);
  float* sm_val = reinterpret_cast<float*>(st + lay.slab_bytes);
  int32_t* sm_ptr = reinterpret_cast<int32_t*>(st + 2 * lay.slab_bytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full + s, 1);
      mbar_init(empty + s, NW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (RING && warp == 0) {
    const uint64_t pol = l2_policy_evict_first();
    uint32_t it = 0;
    for (int64_t slot = blockIdx.x; slot < a.n_slots; slot += gridDim.x, ++it) {
      const int code = __ldg(a.slots + slot);
      const int64_t tile = code >> 1;
      const int begin = __ldg(a.indptr + tile * R), end = __ldg(a.indptr + tile * R + R);
      const int4 m = __ldg(a.ring_meta + tile);
      if (code & 1) {
        // the wait of B(tile); bounded all the same: a wait of seconds can only be a broken table,
        // and a trapped launch is reported to the caller where a spinning one would hold the device
        const int e1 = __ldg(a.nbr_ptr + tile + 1);
        for (int e = __ldg(a.nbr_ptr + tile) + lane; e < e1; e += 32) {
          const unsigned* f = a.tile_done + __ldg(a.nbr_idx + e);
          unsigned seen, polls = 0;
          for (;;) {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(f) : "memory");
            if (seen >= a.done_target) break;
            if (++polls > (1u << 24)) __trap();
            __nanosleep(128);
          }
        }
        __syncwarp();
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
        asm volatile("fence.proxy.async.global;" ::: "memory");
      }
      const int s = int(it % uint32_t(S));
      mbar_wait(empty + s, ((it / uint32_t(S)) & 1u) ^ 1u);
      // A's slab stays in L2 for B(t): 12.16 -> 12.02 ms
      stage_ring_tile(a, lay, stage0 + size_t(s) * lay.stage_bytes, full + s, tile, begin, end, m,
                      (code & 1) ? a.x_cur2 : a.x_cur, a.l2_hint != 0 && (code & 1), pol, lane);
    }
    return;
  }
  if (RING) {
    const int cw = warp - 1;
    const int sub = lane / G;
    const int c0 = (lane % G) * 4;
    uint32_t it = 0;
    for (int64_t slot = blockIdx.x; slot < a.n_slots; slot += gridDim.x, ++it) {
      const int code = __ldg(a.slots + slot);
      const int64_t tile = code >> 1;
      const int s = int(it % uint32_t(S));
      mbar_wait(full + s, (it / uint32_t(S)) & 1u);
      const unsigned char* sg = stage0 + size_t(s) * lay.stage_bytes;
      const TileCtx t = {reinterpret_cast<const float*>(sg), sg + lay.vec_bytes + lay.slab_bytes,
                         reinterpret_cast<const float*>(sg + lay.vec_bytes),
                         reinterpret_cast<const int32_t*>(sg + lay.vec_bytes + lay.slab_bytes +
                                                          lay.idx_bytes),
                         tile, tile * R, cw, sub, c0, true};
      if (code & 1) {
        tile_rows<G, false, 1, kGatherRing, P, 2>(a, t);
      } else {
        tile_rows<G, false, 1, kGatherRing, P, 1>(a, t);
        __syncwarp();
        if (lane == 0)
          asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.tile_done + tile) : "memory");
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty + s);
    }
    return;
  }

  if (warp == 0) {
    // producer: the CSR slab of the slot's tile (the same slab for A(t) and B(t)); the slot table
    // and the tile's first / last CSR offsets are read one slot ahead
    if (lane != 0) return;
    const bool hint = a.l2_hint != 0;
    const uint64_t pol = l2_policy_evict_first();
    int64_t ntile = 0;
    int nbegin = 0, nend = 0, ncode = 0;
    if (int64_t(blockIdx.x) < a.n_slots) {
      ncode = __ldg(a.slots + blockIdx.x);
      ntile = ncode >> 1;
      nbegin = __ldg(a.indptr + a.row_begin + ntile * R);
      nend = __ldg(a.indptr + a.row_begin + ntile * R + R);
    }
    uint32_t it = 0;
    for (int64_t slot = blockIdx.x; slot < a.n_slots; slot += gridDim.x, ++it) {
      const int64_t tile = ntile;
      const int begin = nbegin, end = nend;
      const bool evict = hint && (ncode & 1);     // A's slab stays in L2 for B(t): 12.16 -> 12.02 ms
      if (slot + gridDim.x < a.n_slots) {
        ncode = __ldg(a.slots + slot + gridDim.x);
        ntile = ncode >> 1;
        nbegin = __ldg(a.indptr + a.row_begin + ntile * R);
        nend = __ldg(a.indptr + a.row_begin + ntile * R + R);
      }
      mbar_wait(empty, (it & 1u) ^ 1u);
      const int64_t r0 = a.row_begin + tile * R;
      const int a0 = begin & ~3;
      int a1 = (end + 3) & ~3;
      if (int64_t(a1) > a.nnz) a1 = end & ~3;
      sm_ptr[R] = end;
      sm_ptr[R + 4] = a0;
      for (int k = (a1 > a0 ? a1 : a0); k < end; ++k) {
        sm_col[k - a0] = __ldg(a.indices + k);
        sm_val[k - a0] = __ldg(a.vals + k);
      }
      const uint32_t slab = a1 > a0 ? uint32_t(a1 - a0) * 4u : 0u;
      mbar_expect_tx(full, uint32_t(R) * 4u + 2u * slab);
      bulk_g2s(sm_ptr, a.indptr + r0, uint32_t(R) * 4u, full);
      if (slab && evict) {
        bulk_g2s_hint(sm_col, a.indices + a0, slab, full, pol);
        bulk_g2s_hint(sm_val, a.vals + a0, slab, full, pol);
      } else if (slab) {
        bulk_g2s(sm_col, a.indices + a0, slab, full);
        bulk_g2s(sm_val, a.vals + a0, slab, full);
      }
    }
    return;
  }

  const int cw = warp - 1;
  const int sub = lane / G;
  const int c0 = (lane % G) * 4;
  uint32_t it = 0;
  for (int64_t slot = blockIdx.x; slot < a.n_slots; slot += gridDim.x, ++it) {
    const int code = __ldg(a.slots + slot);
    const int64_t tile = code >> 1;
    mbar_wait(full, it & 1u);
    const TileCtx t = {nullptr, sm_col, sm_val, sm_ptr, tile, a.row_begin + tile * R, cw, sub, c0, true};
    if (code & 1) {
      // Wait until every A tile that B(tile) reads is stored.  This cannot deadlock: all CTAs of
      // the grid are resident (the launch requires it), each walks its slots in increasing order,
      // a B slot waits only for A tiles in lower slots (checked when the table is built), and an
      // A slot waits for nothing; so the lowest unfinished slot of the launch can always finish.
      // The poll is bounded all the same: a wait of seconds can only be a broken table, and a
      // trapped launch is reported to the caller where a spinning one would hold the device.
      if (cw == 0) {
        const int e1 = __ldg(a.nbr_ptr + tile + 1);
        for (int e = __ldg(a.nbr_ptr + tile) + lane; e < e1; e += 32) {
          const unsigned* f = a.tile_done + __ldg(a.nbr_idx + e);
          unsigned seen, polls = 0;
          for (;;) {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(f) : "memory");
            if (seen >= a.done_target) break;
            if (++polls > (1u << 24)) __trap();
            __nanosleep(128);
          }
        }
        __syncwarp();
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
      }
      asm volatile("bar.sync 1, %0;" ::"r"(NW * 32) : "memory");
      tile_rows<G, false, 1, kGatherPlain, P, 2>(a, t);
    } else {
      tile_rows<G, false, 1, kGatherNc, P, 1>(a, t);
      // publish: the warp's stores, then its arrival (the tile is done at NW arrivals)
      __syncwarp();
      if (lane == 0)
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(a.tile_done + tile) : "memory");
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty);
  }
}

// max over every window of `rows_per_tile` rows that starts at a multiple of 4 of
// the window's 16-byte-aligned CSR slab length: a bound valid for any tiling of
// any row range [rb, re) with rb % 4 == 0
__global__ void tile_nnz_max_kernel(int64_t n, int rows_per_tile,
                                    const int32_t* __restrict__ indptr, int* out) {
  int best = 0;
  const int64_t windows = (n - rows_per_tile) / 4 + 1;
  for (int64_t w = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; w < windows;
       w += int64_t(gridDim.x) * blockDim.x) {
    const int begin = indptr[4 * w] & ~3;
    const int end = (indptr[4 * w + rows_per_tile] + 3) & ~3;
    best = max(best, end - begin);
  }
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, best);
}

static int env_int(const char* name, int fallback) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : fallback;
}

// Decide the tiling for (matrix, nsig, nscales).  Synchronises `st` once.
int tile_plan(int64_t n, const int32_t* indptr, int64_t nsig, int nscales, gsp_tile_plan* plan,
              cudaStream_t st) {
  memset(plan, 0, sizeof(*plan));
  const char* force = getenv("GSPB200_KERNEL");
  if (force && strcmp(force, "rowgroup") == 0) return GSP_OK;
  if (!(nsig == 8 || nsig == 16 || nsig == 32 || nsig == 64 || nsig == 128)) return GSP_OK;
  if (nscales < 0 || nscales > kTiledMaxScales) return GSP_OK;
  // vector tiles per stage: x_old + one r tile per scale; keep a stage near 40 KB
  int R = env_int("GSPB200_TILE_R", nscales <= 1 ? 64 : (nscales <= 2 ? 32 : 16));
  if (nsig == 128) R = std::max(8, R / 2);
  R = std::max(8, (R / 8) * 8);
  const int warps_default = 16;
  // narrow blocks: a warp carries 32 / (nsig/4) rows, a tile should feed every warp
  if (nsig <= 16 && !getenv("GSPB200_TILE_R")) R = std::max(R, warps_default * (128 / (int)nsig));
  const int64_t n_tiles = n / R;
  if (n_tiles < 1) return GSP_OK;
  Scratch<int> dmax(st);
  GSP_CUDA(dmax.alloc(1));
  GSP_CUDA(cudaMemsetAsync(dmax.get(), 0, sizeof(int), st));
  const int blocks = (int)std::min<int64_t>(ceil_div(n / 4 + 1, 256), 2048);
  tile_nnz_max_kernel<<<blocks, 256, 0, st>>>(n, R, indptr, dmax.get());
  GSP_LAUNCH_CHECK("tile_nnz_max");
  int hmax = 0;
  GSP_CUDA(cudaMemcpyAsync(&hmax, dmax.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  GSP_CUDA(cudaStreamSynchronize(st));
  const int cap = ((hmax + 8 + 31) / 32) * 32;
  int stages = env_int("GSPB200_TILE_S", nscales <= 1 ? 2 : 3);
  const int warps = std::min(16, std::max(1, env_int("GSPB200_TILE_NW", 16)));
  // keep a CTA's ring within ~100 KB so that L1 keeps room for the x_cur gather
  const int budget = env_int("GSPB200_TILE_SMEM", 100 * 1024);
  const bool vd = env_int("GSPB200_TILE_VDIR", 0) != 0;     // vectors not staged: small stages
  TileLayout lay(R, cap, (int)nsig, nscales, vd, stages);
  while (stages > 2 && lay.total(stages) > budget) { --stages; lay = TileLayout(R, cap, (int)nsig, nscales, vd, stages); }
  if (lay.total(stages) > 200 * 1024) return GSP_OK;        // heavy rows: row-group kernel
  plan->rows_per_tile = R;
  plan->slab_capacity = cap;
  plan->stages = stages;
  plan->consumer_warps = warps;
  plan->gather_unroll = env_int("GSPB200_TILE_U", 4);
  plan->blocks_per_sm = env_int("GSPB200_TILE_BPS", 0);
  return GSP_OK;
}

// Stages of a step with neighbour rings of up to ring_max rows: as many as the shared-memory
// budget of a CTA holds, at most GSPB200_RING_S (default kRingStages); 0 when not even one fits.
// The budget lets two CTAs share an SM (2 x (113 + 1) KB of 228 KB).  Measured on an H100 SXM
// (700 W), config 2 of bench.py (1e6-vertex Morton k-NN, 64 signals, order 30, R = 64, largest
// ring 178 rows, a stage of about 54 KB): one stage and three CTAs per SM 10.12 ms per call, two
// stages and two CTAs per SM 9.68 ms; R = 32 12.15 ms, R = 128 10.87 ms (DESIGN.md section 4.1).
constexpr int kRingStages = 2;
constexpr int kRingBudget = 113 * 1024;
static int ring_stages(const gsp_tile_plan& plan, int nsig, int ring_max) {
  if (plan.rows_per_tile <= 0 || ring_max <= 0 || env_int("GSPB200_TILE_RING", 1) == 0) return 0;
  const int budget = env_int("GSPB200_RING_SMEM", kRingBudget);
  for (int s = std::max(1, env_int("GSPB200_RING_S", kRingStages)); s >= 1; --s)
    if (TileLayout(plan.rows_per_tile, plan.slab_capacity, nsig, 0, true, s, ring_max).total(s) <=
        budget)
      return s;
  return 0;
}

template <int G, int NSC, bool HALO, int P, bool RING = false>
static int launch_tiled_k(bool first, const TileArgs& a, int blocks_per_sm, cudaStream_t st) {
  const TileLayout lay(a.rows_per_tile, a.slab_cap, a.nsig, a.nscales, first || a.vec_direct,
                       a.stages, a.ring_cap);
  const int smem = lay.total(a.stages);
  const int threads = 32 * (1 + a.consumer_warps);
  GSP_REQUIRE(threads <= 32 * (P == 2 ? 9 : 17), "too many consumer warps for this mapping");
  auto kern = first ? cheby_step_tiled<G, true, NSC, HALO, P, RING>
                    : cheby_step_tiled<G, false, NSC, HALO, P, RING>;
  GSP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 0;
  GSP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
  if (per_sm < 1) return fail(GSP_ERR_UNSUPPORTED, "tiled kernel does not fit (%s)", "smem");
  if (blocks_per_sm > 0) per_sm = std::min(per_sm, blocks_per_sm);
  const int64_t grid = std::min<int64_t>(a.n_tiles, int64_t(sm_count()) * per_sm);
  kern<<<(unsigned)grid, threads, smem, st>>>(a);
  GSP_LAUNCH_CHECK("cheby_step_tiled");
  return GSP_OK;
}

template <int G, bool HALO, int P>
static int launch_tiled_gh(bool first, const TileArgs& a, int bps, cudaStream_t st) {
  if constexpr (!HALO) {
    // rings: the single-source Clenshaw steps (the first one has no source block)
    if (a.ring_cap && a.nscales == 0) return launch_tiled_k<G, 0, false, P, true>(first, a, bps, st);
    if (a.ring_cap && a.nscales == 1) return launch_tiled_k<G, 1, false, P, true>(first, a, bps, st);
  }
  switch (a.nscales) {          // common bank widths get the scale loop unrolled
    case 0: return launch_tiled_k<G, 0, HALO, P>(first, a, bps, st);
    case 1: return launch_tiled_k<G, 1, HALO, P>(first, a, bps, st);
    case 2: return launch_tiled_k<G, 2, HALO, P>(first, a, bps, st);
    default: return launch_tiled_k<G, -1, HALO, P>(first, a, bps, st);
  }
}

// G lanes x P packets x 4 columns = nsig.  The boundary tiles of a partitioned step (halo) always
// take the one-packet mapping; `two` selects the two-packet mapping for the others.
template <int G>
static int launch_tiled_g(bool first, const TileArgs& a, bool halo, bool two, int bps,
                          cudaStream_t st) {
  if (halo) return launch_tiled_gh<G, true, 1>(first, a, bps, st);
  if (two && G >= 8) return launch_tiled_gh<(G >= 8 ? G / 2 : G), false, (G >= 8 ? 2 : 1)>(first, a, bps, st);
  return launch_tiled_gh<G, false, 1>(first, a, bps, st);
}

template <int G, int P>
static int launch_pair_k(const TileArgs& a, int blocks_per_sm, cudaStream_t st) {
  const TileLayout lay(a.rows_per_tile, a.slab_cap, a.nsig, a.nscales, true, a.stages, a.ring_cap);
  const int smem = lay.total(a.stages);
  const int threads = 32 * (1 + a.consumer_warps);
  GSP_REQUIRE(threads <= 32 * (P == 2 ? 9 : 17), "too many consumer warps for this mapping");
  auto kern = a.ring_cap ? cheby_pair_tiled<G, P, true> : cheby_pair_tiled<G, P, false>;
  GSP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 0;
  GSP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
  // B tiles wait for A tiles of other CTAs: every CTA of the grid must be resident
  GSP_REQUIRE(per_sm >= 1, "paired tiled kernel does not fit");
  if (blocks_per_sm > 0) per_sm = std::min(per_sm, blocks_per_sm);
  const int64_t grid = std::min<int64_t>(a.n_slots, int64_t(sm_count()) * per_sm);
  kern<<<(unsigned)grid, threads, smem, st>>>(a);
  GSP_LAUNCH_CHECK("cheby_pair_tiled");
  return GSP_OK;
}

// the lane mappings of launch_tiled_g without a halo
template <int G>
static int launch_pair_g(const TileArgs& a, bool two, int bps, cudaStream_t st) {
  if (two && G >= 8) return launch_pair_k<(G >= 8 ? G / 2 : G), (G >= 8 ? 2 : 1)>(a, bps, st);
  return launch_pair_k<G, 1>(a, bps, st);
}

int cheby_step_tiled_f32(const Step<float>& s, int64_t rb, int64_t re, const gsp_tile_plan& plan,
                         const gsp_halo_fusion* halo, int64_t* rows_done, cudaStream_t st,
                         const PairLaunch* pair) {
  const bool first = s.first;
  const int nsig = s.nsig, nscales = s.nscales;
  TileArgs a;
  a.out_perm = s.out_perm;
  a.vec_direct = (!first && env_int("GSPB200_TILE_VDIR", s.add_source ? 1 : 0)) ? 1 : 0;
  a.keep_writes = env_int("GSPB200_TILE_REV", 1);
  a.reverse = (s.reverse && a.keep_writes) ? 1 : 0;
  a.add_source = s.add_source ? 1 : 0;
  a.l2_hint = env_int("GSPB200_TILE_HINT", 1);
  a.n_front = 0;
  GSP_REQUIRE(!s.add_source || (nscales >= 1 && !first), "add_source needs source blocks");
  memset(&a.halo, 0, sizeof(a.halo));
  const int64_t full_tiles = (re - rb) / plan.rows_per_tile;
  gsp_halo_fusion probe;                       // GSPB200_FORCE_HALO=1: run the halo-capable
  if (!halo && !pair && rb == 0 && env_int("GSPB200_FORCE_HALO", 0)) {   // variant with no neighbours
    memset(&probe, 0, sizeof(probe));          // (single-GPU A/B of the two instantiations)
    probe.n_owned = 0x7fffffff;
    halo = &probe;
  }
  if (halo) {
    a.halo = *halo;
    const int R = plan.rows_per_tile;
    GSP_REQUIRE(rb == 0, "fused halo push needs the whole row block in one launch");
    GSP_REQUIRE(halo->n_wait <= 32, "at most 32 neighbours");
    GSP_REQUIRE(halo->n_push_rows >= 0 && halo->n_boundary_rows >= 0, "negative row counts");
    // tiles whose rows read halo columns wait for the neighbours' flags; the step is
    // published once those AND the tiles that push rows are done (both sets are "front")
    a.halo.n_wait_tiles = ceil_div(halo->n_boundary_rows, R);
    a.halo.n_push_tiles =
        halo->publish ? ceil_div(std::max(halo->n_push_rows, halo->n_boundary_rows), R) : 0;
    a.n_front = std::max(a.halo.n_wait_tiles, a.halo.n_push_tiles);
    GSP_REQUIRE(a.n_front <= full_tiles, "boundary rows must lie inside the full tiles");
  }
  a.row_begin = rb;
  a.n_tiles = full_tiles;
  *rows_done = a.n_tiles * plan.rows_per_tile;
  if (a.n_tiles == 0) return GSP_OK;
  a.r_rows = s.r_rows;
  a.nnz = s.nnz;
  a.indptr = s.indptr; a.indices = s.indices; a.vals = s.vals;
  a.x_cur = s.x_cur; a.x_old = s.x_old; a.x_new = s.x_new; a.r = s.r;
  a.rows_per_tile = plan.rows_per_tile;
  a.slab_cap = plan.slab_capacity;
  // A stage that carries no vector tiles (the first step, or x_old / r read directly) holds only
  // the tile's CSR slab, and the ring then has one stage: the shared memory of three CTAs stays
  // within the 32 KB carveout, which leaves the most L1 to the x_cur gather.  That is worth more
  // than the producer running a tile ahead; the SM's other CTAs cover one CTA's wait for its TMA.
  // H100, 1e6-vertex k-NN, Clenshaw form: 14.8 -> 12.7 ms per call (DESIGN.md section 4.1).
  a.stages = (first || a.vec_direct) ? 1 : plan.stages;
  // Neighbour rings: the gather reads shared memory only, so L1 no longer needs the room the
  // one-stage argument above keeps for it (DESIGN.md section 4.1).
  if (s.ring && !halo && rb == 0 && (first || a.vec_direct) && nscales <= 1 &&
      s.ring->rows_per_tile == plan.rows_per_tile) {
    const int rs = ring_stages(plan, nsig, s.ring->ring_max);
    if (rs > 0) {
      a.ring_meta = reinterpret_cast<const int4*>(s.ring->tile_meta);
      a.ring_runs = reinterpret_cast<const int2*>(s.ring->runs);
      a.ring_local = s.ring->local;
      a.ring_cap = s.ring->ring_max;
      a.stages = rs;
    }
  }
  a.consumer_warps = plan.consumer_warps;
  a.nsig = nsig;
  a.nscales = nscales;
  a.alpha = float(s.alpha); a.beta = float(s.beta); a.gamma = float(s.gamma);
  for (int i = 0; i < kTiledMaxScales; ++i) {
    a.ck[i] = i < nscales ? float(s.ck[i]) : 0.f;
    a.half_c0[i] = (first && i < nscales) ? float(0.5 * s.c0[i]) : 0.f;
  }
  const bool h = halo != nullptr;
  // two packets per lane (32 / 64 / 128 signals): a CSR read in shared memory serves twice
  // as many rows; GSPB200_TILE_P2=0 / 1 forces one / two packets per lane.
  // Measured on an H100 SXM (400 W limit), 1e6-vertex graphs, interleaved A/B, one -> two packets:
  // Clenshaw form (direct vectors), order 30: 64 signals 18.4 -> 15.7 ms per call, 128 signals
  // 38.0 -> 31.6 ms, 32 signals 10.2 -> 8.9 ms; forward form (TMA-staged vectors): one filter at
  // 64 signals 23.5 -> 19.2 ms, two filters 29.2 / 30.8 -> 27.6 / 27.3 ms, a 6-filter MexicanHat
  // bank at order 50 on a grid 89.8 / 97.1 -> 84.0 / 84.1 ms.  So two packets are the default.
  const bool two = !h && nsig >= 32 && env_int("GSPB200_TILE_P2", 1) != 0;
  if (two) a.consumer_warps = std::min(a.consumer_warps, 8);
  if (pair) {
    const Step<float>& b = *pair->second;
    GSP_REQUIRE(!h && !first && s.add_source && nscales == 1 && a.vec_direct && !s.out_perm,
                "a paired launch takes two middle Clenshaw steps of one source");
    GSP_REQUIRE(float(b.alpha) == a.alpha && float(b.beta) == a.beta && float(b.gamma) == a.gamma,
                "paired steps share alpha, beta and gamma");
    GSP_REQUIRE(a.n_tiles < (int64_t(1) << 30), "too many tiles for the slot table");
    a.slots = pair->slots;
    a.n_slots = 2 * a.n_tiles;
    a.nbr_ptr = pair->nbr_ptr;
    a.nbr_idx = pair->nbr_idx;
    a.tile_done = pair->tile_done;
    a.done_target = pair->launch_index * unsigned(a.consumer_warps);
    a.x_cur2 = b.x_cur; a.x_old2 = b.x_old; a.x_new2 = b.x_new;
    a.ck2 = float(b.ck[0]);
    switch (nsig) {
      case 8: return launch_pair_g<2>(a, false, plan.blocks_per_sm, st);
      case 16: return launch_pair_g<4>(a, false, plan.blocks_per_sm, st);
      case 32: return launch_pair_g<8>(a, two, plan.blocks_per_sm, st);
      case 64: return launch_pair_g<16>(a, two, plan.blocks_per_sm, st);
      case 128: return launch_pair_g<32>(a, two, plan.blocks_per_sm, st);
    }
  }
  switch (nsig) {
    case 8: return launch_tiled_g<2>(first, a, h, false, plan.blocks_per_sm, st);
    case 16: return launch_tiled_g<4>(first, a, h, false, plan.blocks_per_sm, st);
    case 32: return launch_tiled_g<8>(first, a, h, two, plan.blocks_per_sm, st);
    case 64: return launch_tiled_g<16>(first, a, h, two, plan.blocks_per_sm, st);
    case 128: return launch_tiled_g<32>(first, a, h, two, plan.blocks_per_sm, st);
  }
  return fail(GSP_ERR_UNSUPPORTED, "tiled kernel: nsig must be 8, 16, 32, 64 or 128 (%s)", "nsig");
}

}  // namespace gsp

extern "C" int gsp_cheby_tile_plan(int64_t n, const int32_t* indptr, int64_t nsig, int nscales,
                                   gsp_tile_plan* plan_host_out, void* stream) {
  GSP_REQUIRE(plan_host_out != nullptr, "plan must not be NULL");
  return gsp::tile_plan(n, indptr, nsig, nscales, plan_host_out, gsp::as_stream(stream));
}

extern "C" int gsp_cheby_ring_fits(int ring_max, int64_t nsig, const gsp_tile_plan* plan_host) {
  if (!plan_host || nsig < 1 || nsig > 128) return 0;
  return gsp::ring_stages(*plan_host, int(nsig), ring_max) > 0;
}
