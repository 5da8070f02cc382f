// dalm_b200 — shared device/host helpers for the sm_90a kernels.
// Everything in csrc/ is compiled with: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

struct CUtensorMap_st;          // CUtensorMap (cuda.h)

namespace dalm {

// ---------------------------------------------------------------------------------------------
// error plumbing for the C ABI: every entry point returns 0 on success, non-zero otherwise and
// leaves a message retrievable through dalm_b200_last_error().
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int  check_launch(const char* what);          // cudaPeekAtLastError → error code + message
void count_launch(int n = 1);                 // bumps the global launch counter (bench.py reads it)

#define DALM_REQUIRE(cond, ...)                                   \
  do {                                                            \
    if (!(cond)) { ::dalm::set_error(__VA_ARGS__); return 1; }    \
  } while (0)

#define DALM_CUDA(expr)                                                                   \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::dalm::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                        __LINE__);                                                        \
      return 2;                                                                           \
    }                                                                                     \
  } while (0)

// true when p (which may be null) is a multiple of `bytes`: vector loads / stores of that width are legal at p
__host__ __device__ inline bool aligned(const void* p, unsigned bytes) { return (reinterpret_cast<uintptr_t>(p) % bytes) == 0; }

// SM count and L2 size of the device the library first runs on (read once; persistent grids and L2 heuristics use them)
int num_sms();
long long l2_bytes();

// cached TMA descriptor of a row-major [rows, cols] bf16 (or fp32) matrix with row stride ld; box = {128 bytes, box_rows},
// 128B swizzle (defined in gemm_wgmma.cu)
int get_tmap(const void* ptr, long long rows, long long cols, long long ld, int box_rows, ::CUtensorMap_st* out, int f32 = 0);

// ---------------------------------------------------------------------------------------------
// warp / block reductions (shuffle based, no atomics)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum; `red` must hold >= 32 floats of shared memory. All threads get the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();                       // protect `red` against the previous use
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : 0.f;
  r = warp_sum(r);
  return r;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : -INFINITY;
  r = warp_max(r);
  return r;
}

// ---------------------------------------------------------------------------------------------
// vector helpers
// ---------------------------------------------------------------------------------------------
struct __align__(16) bf16x8 { __nv_bfloat162 v[4]; };

__device__ __forceinline__ void unpack8(const bf16x8& p, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x; f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf16x8 pack8(const float* f) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}

__device__ __forceinline__ float gelu_erf(float x) {           // HF "gelu": x * 0.5 * (1 + erf(x/sqrt2))
  return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}


// ---------------------------------------------------------------------------------------------
// dropout: counter-based Philox4x32-10 (same generator family as torch/curand), keyed by (seed), counter =
// (element index / 4, stream). Nothing is stored: backward kernels regenerate the keep-mask from the same
// (seed, stream, index). `stream` identifies the call site (layer, tensor, call); `*offset` (device memory, may be
// null) is added to it so that a CUDA-graph replay of the step draws fresh masks (the graph bumps the counter).
// ---------------------------------------------------------------------------------------------
struct DropCfg {
  float p;                              // requested drop probability; 0 => disabled
  float inv_keep;                       // 1 / (1 - p_eff), p_eff = thresh / 65536 (the probability actually realised)
  unsigned int thresh;                  // keep iff rand16 >= thresh
  unsigned long long seed, stream;
  const unsigned long long* offset;     // device counter or nullptr
};
inline DropCfg make_drop(float p, unsigned long long seed, unsigned long long stream, const void* offset) {
  DropCfg d;
  d.p = p;
  double t = (double)p * 65536.0 + 0.5;
  d.thresh = p > 0.f ? (t >= 65535.0 ? 65535u : (unsigned int)t) : 0u;
  d.inv_keep = p > 0.f ? (float)(1.0 / (1.0 - (double)d.thresh / 65536.0)) : 1.f;
  d.seed = seed; d.stream = stream; d.offset = (const unsigned long long*)offset;
  return d;
}
// Philox4x32 with 7 rounds (the Random123 "crush-resistant" minimum; 10 is the library default's safety margin)
__device__ __forceinline__ uint4 philox4x32_7(uint2 key, uint4 c) {
#pragma unroll
  for (int r = 0; r < 7; ++r) {
    const unsigned int hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const unsigned int hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ key.x, lo1, hi0 ^ c.w ^ key.y, lo0);
    key.x += 0x9E3779B9u; key.y += 0xBB67AE85u;
  }
  return c;
}
__device__ __forceinline__ unsigned long long drop_stream(const DropCfg& d) {
  return d.stream + (d.offset ? (*d.offset) * 0x9E3779B97F4A7C15ull : 0ull);
}
// One Philox call serves EIGHT consecutive elements (16 random bits each): word j holds the bits of elements 2j (low half)
// and 2j + 1 (high half) of [8*idx8, 8*idx8 + 8).
__device__ __forceinline__ uint4 drop_bits8(const DropCfg& d, unsigned long long stream, unsigned long long idx8) {
  return philox4x32_7(make_uint2((unsigned int)d.seed, (unsigned int)(d.seed >> 32)),
                      make_uint4((unsigned int)idx8, (unsigned int)(idx8 >> 32), (unsigned int)stream, (unsigned int)(stream >> 32)));
}
// scale[j] = 0 or 1/(1-p_eff) for elements [8*idx8, 8*idx8 + 8) of the tensor the mask applies to.
__device__ __forceinline__ void drop_scale8(const DropCfg& d, unsigned long long stream, unsigned long long idx8, float* scale) {
  const uint4 r = drop_bits8(d, stream, idx8);
  const unsigned int w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    scale[2 * j]     = (w[j] & 0xFFFFu) >= d.thresh ? d.inv_keep : 0.f;
    scale[2 * j + 1] = (w[j] >> 16)     >= d.thresh ? d.inv_keep : 0.f;
  }
}
// scalar access (recomputes the group of 8): tests / cold paths
__device__ __forceinline__ float drop_scale1(const DropCfg& d, unsigned long long stream, unsigned long long idx) {
  float sc[8];
  drop_scale8(d, stream, idx >> 3, sc);
  float v = sc[0];
#pragma unroll
  for (int j = 1; j < 8; ++j) if ((idx & 7) == (unsigned long long)j) v = sc[j];
  return v;
}

}  // namespace dalm
