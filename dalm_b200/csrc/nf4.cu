// dalm_b200 — NF4 (bitsandbytes 4-bit NormalFloat) quantise -> dequantise round trip of a weight tensor, in place.
//
// `use_bnb` in the reference (dalm/models/rag_e2e_base_model.py:136-142, retriever_only_base_model.py:85-91) loads the
// nn.Linear weights through BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type="nf4",
// bnb_4bit_compute_dtype=bfloat16): weights are cast to fp16, split into blocks of 64 consecutive elements, each block
// stores absmax (fp32) and sixteen-level codes of x / absmax; every forward dequantises code * absmax back to fp16 and runs
// the matmul in bf16. The values the GEMM sees are therefore a pure function of the checkpoint — this kernel computes them
// once at load time, and the product keeps them resident as bf16 (an H100 has the HBM for 7B; the reference quantises to fit 7B
// models on smaller parts). Same numerics as bnb's forward, none of its per-step dequantisation.
#include "common.cuh"
#include <cuda_fp16.h>

namespace dalm {

__constant__ float kNF4Code[16] = {-1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f,
                                   -0.28444138169288635f, -0.18477343022823334f, -0.09105003625154495f, 0.0f,
                                   0.07958029955625534f, 0.16093020141124725f, 0.24611230194568634f, 0.33791524171829224f,
                                   0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f, 1.0f};

// nearest NF4 level; decision boundaries are the midpoints between adjacent levels, a value exactly on a boundary goes down
// (bitsandbytes' dQuantizeNF4 decision tree tests `x > boundary`)
__device__ __forceinline__ int nf4_index(float x) {
  int idx = 0;
#pragma unroll
  for (int i = 0; i < 15; ++i) idx += (x > 0.5f * (kNF4Code[i] + kNF4Code[i + 1])) ? 1 : 0;
  return idx;
}

// one warp per block of 64 elements (2 per lane)
__global__ void nf4_roundtrip_kernel(float* __restrict__ w, long long n, unsigned char* __restrict__ codes, float* __restrict__ absmax) {
  const long long blk = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long base = blk * 64;
  if (base >= n) return;
  float v[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const long long i = base + lane + 32 * j;
    v[j] = i < n ? __half2float(__float2half_rn(w[i])) : 0.f;          // the checkpoint is cast to fp16 before quantisation
  }
  float m = fmaxf(fabsf(v[0]), fabsf(v[1]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const float inv = 1.0f / m;                                           // bnb multiplies by the reciprocal
  if (lane == 0 && absmax) absmax[blk] = m;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const long long i = base + lane + 32 * j;
    if (i >= n) continue;
    const int q = m > 0.f ? nf4_index(v[j] * inv) : 7;                  // an all-zero block: level 0.0
    if (codes) codes[i] = (unsigned char)q;
    w[i] = __half2float(__float2half_rn(kNF4Code[q] * m));              // dequantised to fp16, as the forward sees it
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// 4-bit STORAGE (DALM_B200_NF4_STORAGE=1): what bitsandbytes keeps resident - two codes per byte (first element in the high
// nibble, as bnb's kQuantizeBlockwise packs them) + one fp32 absmax per 64-element block = 0.5625 B per parameter instead of
// the 2 B (4 B with the resident transpose) of the dequantised-resident default. A weight is expanded to bf16 right before
// the GEMM that needs it (bnb does the same in its forward: dequantize_4bit -> matmul), into a scratch shared by all layers.
// ---------------------------------------------------------------------------------------------------------------------
// one warp per 64-element block; lane l owns elements 2l, 2l+1 -> one packed byte
__global__ void nf4_quantize_kernel(const float* __restrict__ w, long long n, unsigned char* __restrict__ packed, float* __restrict__ absmax) {
  const long long blk = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long base = blk * 64;
  if (base >= n) return;
  float v[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const long long i = base + 2 * lane + j;
    v[j] = i < n ? __half2float(__float2half_rn(w[i])) : 0.f;          // the checkpoint is cast to fp16 before quantisation
  }
  float m = fmaxf(fabsf(v[0]), fabsf(v[1]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const float inv = 1.0f / m;
  if (lane == 0) absmax[blk] = m;
  const int q0 = m > 0.f ? nf4_index(v[0] * inv) : 7, q1 = m > 0.f ? nf4_index(v[1] * inv) : 7;
  const long long i0 = base + 2 * lane;
  if (i0 < n) packed[i0 >> 1] = (unsigned char)((q0 << 4) | (i0 + 1 < n ? q1 : 7));
}

// bf16 out[r, c] = bf16(fp16(code * absmax))  (the value the dequantised-resident mode keeps). grid (ceil((cols/16 + 1)/256), rows):
// a thread expands 16 codes (8 bytes in, 32 bytes out); the sixteen levels sit in shared memory (divergent indices into
// __constant__ memory serialise); the last thread of a row copies the row's
// `tail_cols` extra columns (the LoRA block of a K-augmented weight) from `tail`
__global__ void __launch_bounds__(256) nf4_dequant_bf16_kernel(const unsigned char* __restrict__ packed, const float* __restrict__ absmax,
                                                               long long rows, int cols, __nv_bfloat16* __restrict__ out, long long ldo,
                                                               const __nv_bfloat16* __restrict__ tail, long long ldt, int tail_cols) {
  __shared__ float lut[16];
  if (threadIdx.x < 16) lut[threadIdx.x] = kNF4Code[threadIdx.x];
  __syncthreads();
  const int groups = cols >> 4;                                         // 16-code groups per row
  const long long r = blockIdx.y;
  const int gi = blockIdx.x * blockDim.x + threadIdx.x;
  if (gi > groups) return;
  if (gi == groups) {                                                   // this row's tail
    for (int c = 0; c < tail_cols; ++c) out[r * ldo + cols + c] = tail[r * ldt + c];
    return;
  }
  const long long e0 = r * cols + (long long)gi * 16;                   // first element (flattened row-major weight)
  const uint2 raw = __ldg(reinterpret_cast<const uint2*>(packed + (e0 >> 1)));
  const float m = __ldg(absmax + (e0 >> 6));
  const unsigned char* b = reinterpret_cast<const unsigned char*>(&raw);
  float f[16];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    f[2 * i]     = __half2float(__float2half_rn(lut[b[i] >> 4] * m));
    f[2 * i + 1] = __half2float(__float2half_rn(lut[b[i] & 15] * m));
  }
  __nv_bfloat16* o = out + r * ldo + (long long)gi * 16;
  *reinterpret_cast<bf16x8*>(o) = pack8(f);
  *reinterpret_cast<bf16x8*>(o + 8) = pack8(f + 8);
}

}  // namespace dalm

using namespace dalm;

// w: fp32 [n] (row-major weight, flattened) -> packed codes uint8 [ceil(n/2)] + absmax fp32 [ceil(n/64)]
extern "C" int dalm_b200_nf4_quantize(const float* w, long long n, void* packed, float* absmax, void* stream) {
  DALM_REQUIRE(n > 0 && w && packed && absmax, "nf4_quantize: empty tensor / null output");
  const long long threads = ((n + 63) / 64) * 32;
  nf4_quantize_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, n, (unsigned char*)packed, absmax);
  count_launch();
  return check_launch("nf4_quantize_kernel");
}

// packed / absmax of a [rows, cols] weight (cols % 64 == 0: blocks never straddle rows) -> bf16 out[rows, ldo] columns [0, cols);
// tail (bf16 [rows, ldt], may be NULL) is copied into columns [cols, cols + tail_cols)
extern "C" int dalm_b200_nf4_dequant_bf16(const void* packed, const float* absmax, long long rows, int cols, void* out, long long ldo,
                                          const void* tail, long long ldt, int tail_cols, void* stream) {
  DALM_REQUIRE(rows > 0 && cols > 0 && (cols % 64) == 0, "nf4_dequant: cols=%d must be a positive multiple of 64", cols);
  DALM_REQUIRE(ldo >= cols + tail_cols && (ldo % 8) == 0 && ((uintptr_t)out & 15) == 0 && ((uintptr_t)packed & 7) == 0,
               "nf4_dequant: output stride / alignment");
  DALM_REQUIRE(tail_cols == 0 || (tail != nullptr && ldt >= tail_cols), "nf4_dequant: tail");
  DALM_REQUIRE(rows <= 65535, "nf4_dequant: %lld rows exceed the grid's y extent of 65535", rows);
  const dim3 grid((unsigned)(((cols >> 4) + 1 + 255) / 256), (unsigned)rows);
  nf4_dequant_bf16_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      (const unsigned char*)packed, absmax, rows, cols, (__nv_bfloat16*)out, ldo, (const __nv_bfloat16*)tail, ldt, tail_cols);
  count_launch();
  return check_launch("nf4_dequant_bf16_kernel");
}

// w: fp32 [n] (a row-major weight, flattened) overwritten with its NF4 round trip. codes (uint8 [n]) and absmax
// (fp32 [ceil(n/64)]) are optional outputs for inspection / tests.
extern "C" int dalm_b200_nf4_roundtrip(float* w, long long n, void* codes, float* absmax, void* stream) {
  DALM_REQUIRE(n > 0, "nf4_roundtrip: empty tensor");
  const long long blocks64 = (n + 63) / 64;
  const long long threads = blocks64 * 32;
  nf4_roundtrip_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, n, (unsigned char*)codes, absmax);
  count_launch();
  return check_launch("nf4_roundtrip_kernel");
}
