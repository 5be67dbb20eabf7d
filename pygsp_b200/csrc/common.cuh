// Shared helpers for libgspb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <stdio.h>
#include <string.h>

#define GSP_OK 0
#define GSP_ERR_ARG (-1)
#define GSP_ERR_CUDA (-2)
#define GSP_ERR_UNSUPPORTED (-3)

namespace gsp {

// thread-local message returned by gsp_last_error()
char* error_buffer();

inline int fail(int code, const char* fmt, const char* a = "", const char* b = "") {
  snprintf(error_buffer(), 512, fmt, a, b);
  return code;
}

// kernels launched by this library since load (bench.py's gpu_launches)
void note_launch(int n);

inline int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return GSP_OK;
  return fail(GSP_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

#define GSP_CUDA(call)                                        \
  do {                                                        \
    int _rc = gsp::check_cuda((call), #call);                 \
    if (_rc != GSP_OK) return _rc;                            \
  } while (0)

#define GSP_LAUNCH_CHECK(name)                                \
  do {                                                        \
    gsp::note_launch(1);                                      \
    int _rc = gsp::check_cuda(cudaGetLastError(), name);      \
    if (_rc != GSP_OK) return _rc;                            \
  } while (0)

#define GSP_REQUIRE(cond, msg)                                \
  do {                                                        \
    if (!(cond)) return gsp::fail(GSP_ERR_ARG, "%s (%s)", msg, #cond); \
  } while (0)

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Stream-ordered device scratch of one C entry point: allocated on `st` by alloc(), freed on
// `st` when the owner goes out of scope, so every return path releases it.  An owner that is
// never allocated holds nullptr and frees nothing.
template <typename T>
class Scratch {
 public:
  explicit Scratch(cudaStream_t st) : st_(st) {}
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  // The status is ignored: a pointer from cudaMallocAsync freed on its own stream can only fail
  // to free if the context is already broken, and every later call reports that anyway.
  ~Scratch() {
    if (p_) (void)cudaFreeAsync(p_, st_);
  }
  // count elements of T; call once per owner
  cudaError_t alloc(size_t count) {
    void* p = nullptr;
    const cudaError_t e = cudaMallocAsync(&p, count * sizeof(T), st_);
    if (e == cudaSuccess) p_ = static_cast<T*>(p);
    return e;
  }
  T* get() const { return p_; }

 private:
  T* p_ = nullptr;
  cudaStream_t st_;
};

// CUB's two-phase protocol: run(nullptr, bytes) sizes the temporary storage, run(tmp, bytes)
// does the work; `run` is a callable (void* tmp, size_t& bytes) -> cudaError_t.
template <typename F>
int cub_temp(const char* what, cudaStream_t st, F&& run) {
  size_t bytes = 0;
  int rc = check_cuda(run(nullptr, bytes), what);
  if (rc != GSP_OK) return rc;
  Scratch<char> tmp(st);
  GSP_CUDA(tmp.alloc(std::max<size_t>(bytes, 16)));
  return check_cuda(run(tmp.get(), bytes), what);
}

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// number of SMs of the current device (cached per device)
int sm_count();

// indptr[1..n] (row sizes on entry) := their inclusive scan, indptr[0] = 0.  When nnz (device)
// is not null it first receives the int64 sum of the row sizes, which stays exact where the int32
// scan wraps -- csrc/graph.cu
int scan_rows(int32_t* indptr, int64_t n, int64_t* nnz, cudaStream_t st);

// dst[i,:] = src[idx[i],:] (scatter: dst[idx[i],:] = src[i,:]) -- csrc/graph.cu
template <typename T>
int move_rows(bool scatter, int64_t rows, const int64_t* idx, const T* src, int64_t width, T* dst,
              cudaStream_t st);

// counter-based generator (splitmix64): uniform in [-1, 1), a function of (seed, index) only,
// so that seeded start vectors / blocks are reproducible (csrc/lanczos.cu, csrc/block.cu)
__device__ __forceinline__ double hash_uniform(uint64_t seed, uint64_t i) {
  uint64_t z = seed + 0x9E3779B97F4A7C15ull * (i + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return double(z >> 11) * (1.0 / 9007199254740992.0) * 2.0 - 1.0;
}

// ----- vector types: 16-byte packets of T --------------------------------
template <typename T, int VEC> struct Pack;
template <> struct Pack<float, 4> { typedef float4 type; };
template <> struct Pack<float, 2> { typedef float2 type; };
template <> struct Pack<float, 1> { typedef float type; };
template <> struct Pack<double, 2> { typedef double2 type; };
template <> struct Pack<double, 1> { typedef double type; };

template <typename T, int VEC>
struct Vec {
  T v[VEC];
};

template <typename T, int VEC>
__device__ __forceinline__ Vec<T, VEC> load_vec(const T* p) {
  typedef typename Pack<T, VEC>::type P;
  union { P p; Vec<T, VEC> v; } u;
  u.p = *reinterpret_cast<const P*>(p);
  return u.v;
}

// read-only (non-coherent) path: data that no thread of this launch writes
template <typename T, int VEC>
__device__ __forceinline__ Vec<T, VEC> load_vec_ro(const T* p) {
  typedef typename Pack<T, VEC>::type P;
  union { P p; Vec<T, VEC> v; } u;
  u.p = __ldg(reinterpret_cast<const P*>(p));
  return u.v;
}

// streaming load: touched once per launch, do not keep in L1
template <typename T, int VEC>
__device__ __forceinline__ Vec<T, VEC> load_vec_stream(const T* p) {
  typedef typename Pack<T, VEC>::type P;
  union { P p; Vec<T, VEC> v; } u;
  u.p = __ldcs(reinterpret_cast<const P*>(p));
  return u.v;
}

template <typename T, int VEC>
__device__ __forceinline__ void store_vec_stream(T* p, const Vec<T, VEC>& v) {
  typedef typename Pack<T, VEC>::type P;
  union { P p; Vec<T, VEC> v; } u;
  u.v = v;
  __stcs(reinterpret_cast<P*>(p), u.p);
}

}  // namespace gsp
