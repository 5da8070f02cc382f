// dalm_b200 — LoRA adapter kernels that are contractions over the TOKEN dimension or have a skinny output:
//
//   lora_wgrad_mma_kernel : out[r,k] += scale * sum_m G[m,r] * X[m,k]           (dA = g^T x,  dB^T = u^T dY)
//   skinny_gemm_kernel    : out[m,r]  = sum_k X[m,k] * W[r,k],  r <= 16          (u = x A^T,   g = dY (sB))
//
// Both are HBM-bound (X is read exactly once: 38 MB per call at cfg-3) with a trivial amount of math, so they use
// warp-level mma.sync (m16n8k16, the 16-row tile IS the LoRA rank) fed by cp.async double buffering instead of the
// wgmma path: there is no reuse to stage, only bytes to stream.
// Replaces the two skinny GEMMs per adapted Linear that peft's LoRA layer adds per pass (reference
// dalm/models/rag_e2e_base_model.py:61-80,144-160) and their autograd backward.
#include "common.cuh"

namespace dalm {

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const int sz = valid ? 16 : 0;                              // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm4(uint32_t* r, const void* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm4t(uint32_t* r, const void* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void mma_bf16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// in-place dropout of a [rows x 128-col] bf16 smem tile (row stride lds) whose element (r, c) is x[m0 + r, k0 + c] of a
// logical [M, K] tensor: the SAME (seed, stream, m*K + k) indexing in the forward skinny GEMM, the wgrad and lora_dx
template <int NT>
__device__ __forceinline__ void drop_tile(__nv_bfloat16* tile, int lds, int rows, int m0, int k0, int M, int K,
                                          const DropCfg& d, unsigned long long dstream) {
  for (int i = threadIdx.x; i < rows * 16; i += NT) {
    const int r = i >> 4, p = i & 15;
    const int m = m0 + r, k = k0 + p * 8;
    if (m < M && k < K) {
      const unsigned long long idx = (unsigned long long)m * K + k;          // multiple of 8 (K % 8 == 0)
      float sc[8], f[8];
      drop_scale8(d, dstream, idx >> 3, sc);
      bf16x8* ptr = reinterpret_cast<bf16x8*>(tile + r * lds + p * 8);
      unpack8(*ptr, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] *= sc[j];
      *ptr = pack8(f);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// wgrad: grid (ceil(K/128), ceil(M/TOK)); 4 warps, warp w owns columns [w*32, w*32+32) of the CTA's 128-column slab.
// G has R (8 or 16) valid columns; rows 0-7 of the result go to out0, rows 8-15 to out1 (two adapters that share X).
// ------------------------------------------------------------------------------------------------------------
constexpr int WG_TOK = 512, WG_CH = 64, WG_XS = 128 + 8, WG_GS = 16 + 8;

__global__ void __launch_bounds__(128) lora_wgrad_mma_kernel(const __nv_bfloat16* __restrict__ X, long long ldx,
                                                             const __nv_bfloat16* __restrict__ G, long long ldg, int R,
                                                             float* __restrict__ out0, float* __restrict__ out1,
                                                             long long so_r, long long so_k, int M, int K, float scale,
                                                             DropCfg dropx) {
  __shared__ __align__(16) __nv_bfloat16 Xs[2][WG_CH][WG_XS];
  __shared__ __align__(16) __nv_bfloat16 Gs[2][WG_CH][WG_GS];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int col0 = blockIdx.x * 128;
  const int m_begin = blockIdx.y * WG_TOK, m_end = min(M, m_begin + WG_TOK);
  const int nchunks = (m_end - m_begin + WG_CH - 1) / WG_CH;

  // zero the G columns that are never loaded (R == 8 -> columns 8..15)
  for (int i = tid; i < 2 * WG_CH * WG_GS; i += 128) (&Gs[0][0][0])[i] = __float2bfloat16(0.f);
  __syncthreads();

  auto load_chunk = [&](int c, int buf) {
    const int m0 = m_begin + c * WG_CH;
    for (int i = tid; i < WG_CH * 16; i += 128) {               // X: 64 rows x 16 sixteen-byte pieces
      const int r = i >> 4, p = i & 15;
      const int m = m0 + r, col = col0 + p * 8;
      const bool ok = (m < m_end) && (col < K);
      cp_async16(&Xs[buf][r][p * 8], X + (size_t)(ok ? m : 0) * ldx + (ok ? col : 0), ok);
    }
    for (int i = tid; i < WG_CH * (R / 8); i += 128) {          // G: 64 rows x (1 or 2) pieces
      const int r = i / (R / 8), p = i - r * (R / 8);
      const int m = m0 + r;
      const bool ok = m < m_end;
      cp_async16(&Gs[buf][r][p * 8], G + (size_t)(ok ? m : 0) * ldg + p * 8, ok);
    }
    cp_async_commit();
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;

  if (nchunks > 0) load_chunk(0, 0);
  for (int c = 0; c < nchunks; ++c) {
    const int buf = c & 1;
    if (c + 1 < nchunks) { load_chunk(c + 1, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    if (dropx.p > 0.f) {                                         // X is the LoRA branch input: dA = g^T dropout(x)
      drop_tile<128>(&Xs[buf][0][0], WG_XS, WG_CH, m_begin + c * WG_CH, col0, m_end, K, dropx, drop_stream(dropx));
      __syncthreads();
    }
#pragma unroll
    for (int ks = 0; ks < WG_CH / 16; ++ks) {
      const int tok0 = ks * 16;
      uint32_t a[4];
      // A = G^T (16 x 16 tokens): transposed 8x8 blocks of Gs[tok][r]
      ldsm4t(a, &Gs[buf][tok0 + (lane & 7) + ((lane >> 4) << 3)][((lane >> 3) & 1) * 8]);
#pragma unroll
      for (int np = 0; np < 2; ++np) {                           // two pairs of n-tiles = this warp's 32 columns
        uint32_t b[4];
        ldsm4t(b, &Xs[buf][tok0 + (lane & 7) + (((lane >> 3) & 1) << 3)][warp * 32 + np * 16 + ((lane >> 4) << 3)]);
        mma_bf16(acc[2 * np], a, b[0], b[1]);
        mma_bf16(acc[2 * np + 1], a, b[2], b[3]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = g + ((e >> 1) << 3);                         // c0,c1: row g ; c2,c3: row g+8
      const int col = col0 + warp * 32 + nt * 8 + t * 2 + (e & 1);
      if (col < K && r < R) {
        float* o = (r < 8) ? out0 : out1;
        atomicAdd(o + (long long)(r & 7) * so_r + (long long)col * so_k, acc[nt][e] * scale);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// skinny GEMM: out[m, 0..R) = X[m,:] . W[0..R,:]^T   (R in {8,16,24,32} rows of W, zero-padded in smem).
// grid = ceil(M/32) CTAs of 256 threads. The 8 warps split the CTA's work 2 (row halves of 16) x 4 (quarters of each
// 128-wide K chunk), so every SM holds enough warps to keep HBM busy; the 4 partial sums per row half are combined through
// shared memory at the end. X is streamed once with cp.async double buffering. Output is written bf16 with row stride ldo
// (the tail columns of an augmented activation buffer).
// ------------------------------------------------------------------------------------------------------------
constexpr int SK_ROWS = 32, SK_KC = 128, SK_LD = SK_KC + 8;

__global__ void __launch_bounds__(256) skinny_gemm_kernel(const __nv_bfloat16* __restrict__ X, long long ldx,
                                                          const __nv_bfloat16* __restrict__ W, long long ldw, int R,
                                                          __nv_bfloat16* __restrict__ out, long long ldo, int M, int K,
                                                          DropCfg dropx) {
  __shared__ __align__(16) __nv_bfloat16 Xs[2][SK_ROWS][SK_LD];
  __shared__ __align__(16) __nv_bfloat16 Ws[2][32][SK_LD];
  __shared__ float red[3][2][4][4][32];                          // partial sums of k-quarters 1..3: [kq-1][rg][nt][e][lane]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int rg = warp & 1, kq = warp >> 1;                       // row half, K quarter
  const int m0 = blockIdx.x * SK_ROWS;
  const int nchunks = (K + SK_KC - 1) / SK_KC;
  for (int i = tid; i < 2 * 32 * SK_LD; i += 256) (&Ws[0][0][0])[i] = __float2bfloat16(0.f);
  __syncthreads();

  auto load_chunk = [&](int c, int buf) {
    const int k0 = c * SK_KC;
    for (int i = tid; i < SK_ROWS * 16; i += 256) {
      const int r = i >> 4, p = i & 15;
      const int m = m0 + r, k = k0 + p * 8;
      const bool ok = (m < M) && (k < K);
      cp_async16(&Xs[buf][r][p * 8], X + (size_t)(ok ? m : 0) * ldx + (ok ? k : 0), ok);
    }
    for (int i = tid; i < R * 16; i += 256) {
      const int r = i >> 4, p = i & 15;
      const int k = k0 + p * 8;
      const bool ok = k < K;
      cp_async16(&Ws[buf][r][p * 8], W + (size_t)r * ldw + (ok ? k : 0), ok);
    }
    cp_async_commit();
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
  const int npairs = (R + 15) / 16;                              // pairs of 8-row n-tiles of W
  load_chunk(0, 0);
  for (int c = 0; c < nchunks; ++c) {
    const int buf = c & 1;
    if (c + 1 < nchunks) { load_chunk(c + 1, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    if (dropx.p > 0.f) {                                         // u = dropout(x) A^T (peft LoRA input dropout)
      drop_tile<256>(&Xs[buf][0][0], SK_LD, SK_ROWS, m0, c * SK_KC, M, K, dropx, drop_stream(dropx));
      __syncthreads();
    }
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      const int ks = kq * 2 + kk;                                // this warp's two 16-wide k-steps of the chunk
      uint32_t a[4], b[4];
      ldsm4(a, &Xs[buf][rg * 16 + (lane & 15)][ks * 16 + ((lane >> 4) << 3)]);             // A: rows x k, K-contiguous
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        if (np < npairs) {
          ldsm4(b, &Ws[buf][np * 16 + (lane & 7) + ((lane >> 4) << 3)][ks * 16 + (((lane >> 3) & 1) << 3)]);   // B stored [n][k]
          mma_bf16(acc[2 * np], a, b[0], b[1]);
          mma_bf16(acc[2 * np + 1], a, b[2], b[3]);
        }
      }
    }
    __syncthreads();
  }
  if (kq > 0) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) red[kq - 1][rg][nt][e][lane] = acc[nt][e];
  }
  __syncthreads();
  if (kq == 0) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      if (nt * 8 >= R) break;
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[nt][e] += red[0][rg][nt][e][lane] + red[1][rg][nt][e][lane] + red[2][rg][nt][e][lane];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + rg * 16 + g + h * 8;
        if (m < M) {
          __nv_bfloat162 v = __floats2bfloat162_rn(acc[nt][2 * h], acc[nt][2 * h + 1]);
          *reinterpret_cast<__nv_bfloat162*>(out + (size_t)m * ldo + nt * 8 + t * 2) = v;
        }
      }
    }
  }
}

}  // namespace dalm

using namespace dalm;

// out0[r*so_r + k*so_k] += scale * sum_m G[m,r] X[m,k] for r<8 ; rows 8..R-1 go to out1 (R == 16). G: bf16 [M, >=R].
extern "C" int dalm_b200_lora_wgrad(const void* X, long long ldx, const void* G, long long ldg, float* out0,
                                    float* out1, long long so_r, long long so_k, int M, int K, int R, float scale,
                                    float drop_p, unsigned long long drop_seed, unsigned long long drop_stream_id,
                                    const void* drop_offset, void* stream) {
  DALM_REQUIRE(R == 8 || R == 16, "lora_wgrad: rank rows %d unsupported (8 or 16)", R);
  DALM_REQUIRE(R == 8 || out1 != nullptr, "lora_wgrad: R=16 needs a second output");
  DALM_REQUIRE((ldx % 8) == 0 && (ldg % 8) == 0 && (K % 8) == 0, "lora_wgrad: K and strides must be multiples of 8");
  DALM_REQUIRE(((uintptr_t)X & 15) == 0 && ((uintptr_t)G & 15) == 0, "lora_wgrad: X and G must be 16-byte aligned");
  DALM_REQUIRE(M > 0 && K > 0, "lora_wgrad: empty problem");
  dim3 grid((K + 127) / 128, (M + WG_TOK - 1) / WG_TOK);
  lora_wgrad_mma_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)X, ldx, (const __nv_bfloat16*)G, ldg, R,
                                                               out0, out1, so_r, so_k, M, K, scale,
                                                               make_drop(drop_p, drop_seed, drop_stream_id, drop_offset));
  count_launch();
  return check_launch("lora_wgrad_mma_kernel");
}

// out[M, R] (bf16, row stride ldo) = X[M,K] . W[R,K]^T
extern "C" int dalm_b200_skinny_gemm(const void* X, long long ldx, const void* W, long long ldw, void* out, long long ldo,
                                     int M, int K, int R, float drop_p, unsigned long long drop_seed,
                                     unsigned long long drop_stream_id, const void* drop_offset, void* stream) {
  DALM_REQUIRE(R == 8 || R == 16 || R == 24 || R == 32, "skinny_gemm: R=%d unsupported (8/16/24/32)", R);
  DALM_REQUIRE((ldx % 8) == 0 && (ldw % 8) == 0 && (K % 8) == 0 && (ldo % 2) == 0, "skinny_gemm: alignment");
  DALM_REQUIRE(((uintptr_t)X & 15) == 0 && ((uintptr_t)W & 15) == 0 && ((uintptr_t)out & 3) == 0, "skinny_gemm: pointer alignment");
  DALM_REQUIRE(M > 0 && K > 0, "skinny_gemm: empty problem");
  skinny_gemm_kernel<<<(M + SK_ROWS - 1) / SK_ROWS, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)X, ldx, (const __nv_bfloat16*)W,
                                                                                  ldw, R, (__nv_bfloat16*)out, ldo, M, K,
                                                                                  make_drop(drop_p, drop_seed, drop_stream_id, drop_offset));
  count_launch();
  return check_launch("skinny_gemm_kernel");
}
