// dalm_b200 — parameter-gradient kernels of FULL fine-tuning (reference default `use_peft=None`: every parameter of the
// HF model the wrapper holds is trainable, dalm/models/rag_e2e_base_model.py:45-59 + train_rage2e.py:336). The dense
// weight gradients dW = dY^T X are wgmma GEMMs (gemm_wgmma.cu, layout 2); what is left is HBM-bound row/column work:
//   col_reduce      bias gradients (column sums of dY) and LayerNorm / RMSNorm gain+bias gradients (sum_m dy, sum_m dy*zhat)
//   embed_scatter   word / position embedding gradients (scatter-add of the embedding-LayerNorm input gradient)
//   masked_add      g = (a_f32 + b_bf16) * dropout_mask  (gradient through the embedding dropout)
//   adam_shadow     Adam over the flat fp32 master buffer + refresh of the bf16 shadow the GEMMs read
#include "common.cuh"

namespace dalm {

// out_sum[h] (+)= sum_m dy[m,h] ;  out_prod[h] (+)= sum_m dy[m,h] * zhat[m,h],  zhat = (z - mean[m]) * rstd[m]  (mean may be null)
// dy = dy_a (fp32, optional) + dy_b (bf16, optional). Each thread owns 4 consecutive columns (16-byte fp32 / 8-byte bf16
// loads: a warp reads 512 contiguous bytes of a row), 8 row lanes per CTA walk the CTA's row range, shared-memory tree
// over the row lanes, one fp32 atomicAdd per column per CTA.
constexpr int kCrCols = 128, kCrLanes = 8;
__global__ void __launch_bounds__(256) col_reduce_kernel(const float* __restrict__ dy_a, const __nv_bfloat16* __restrict__ dy_b,
                                                         long long ldb, const float* __restrict__ z,
                                                         const float* __restrict__ mean, const float* __restrict__ rstd,
                                                         float* __restrict__ out_sum, float* __restrict__ out_prod, int M, int H,
                                                         int rows_per_cta) {
  __shared__ float4 red_s[kCrLanes][32], red_p[kCrLanes][32];
  const int cq = threadIdx.x & 31, lane = threadIdx.x >> 5;
  const int col = blockIdx.x * kCrCols + cq * 4;
  const int r0 = blockIdx.y * rows_per_cta, r1 = min(M, r0 + rows_per_cta);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f), p = s;
  if (col < H) {
    for (int r = r0 + lane; r < r1; r += kCrLanes) {
      float4 d = dy_a ? *reinterpret_cast<const float4*>(dy_a + (size_t)r * H + col) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (dy_b) {
        const uint2 raw = *reinterpret_cast<const uint2*>(dy_b + (size_t)r * ldb + col);
        const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
        const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
        d.x += lo.x; d.y += lo.y; d.z += hi.x; d.w += hi.y;
      }
      s.x += d.x; s.y += d.y; s.z += d.z; s.w += d.w;
      if (out_prod) {
        const float4 zz = *reinterpret_cast<const float4*>(z + (size_t)r * H + col);
        const float mu = mean ? mean[r] : 0.f, rs = rstd[r];
        p.x += d.x * (zz.x - mu) * rs; p.y += d.y * (zz.y - mu) * rs; p.z += d.z * (zz.z - mu) * rs; p.w += d.w * (zz.w - mu) * rs;
      }
    }
  }
  red_s[lane][cq] = s; red_p[lane][cq] = p;
  __syncthreads();
  if (lane == 0 && col < H) {
#pragma unroll
    for (int l = 1; l < kCrLanes; ++l) {
      const float4 a = red_s[l][cq], b = red_p[l][cq];
      s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
      p.x += b.x; p.y += b.y; p.z += b.z; p.w += b.w;
    }
    if (out_sum)  { atomicAdd(out_sum + col, s.x);  atomicAdd(out_sum + col + 1, s.y);  atomicAdd(out_sum + col + 2, s.z);  atomicAdd(out_sum + col + 3, s.w); }
    if (out_prod) { atomicAdd(out_prod + col, p.x); atomicAdd(out_prod + col + 1, p.y); atomicAdd(out_prod + col + 2, p.z); atomicAdd(out_prod + col + 3, p.w); }
  }
}

// dword[ids[m], :] += d[m, :] ;  dpos[pos_ids ? pos_ids[m] : m % L, :] += d[m, :]  (dpos optional). With pad >= 0, tokens whose
// id is pad add nothing to dword and positions equal to pad add nothing to dpos (nn.Embedding padding_idx). One CTA per token
// row, float4 reads, fp32 atomics.
__global__ void __launch_bounds__(256) embed_scatter_kernel(const float* __restrict__ d, const long long* __restrict__ ids,
                                                            const long long* __restrict__ pos_ids, float* __restrict__ dword,
                                                            float* __restrict__ dpos, int M, int H, int L, int V, long long pad) {
  const int m = blockIdx.x;
  const long long raw = ids[m];
  const long long id = (raw < 0 || raw >= V) ? 0 : raw;               // the forward gathers read row 0 for any out-of-range id
  const float* src = d + (size_t)m * H;
  float* w = (pad >= 0 && raw == pad) ? nullptr : dword + (size_t)id * H;
  float* pp = nullptr;
  if (dpos) {
    const long long p = pos_ids ? pos_ids[m] : m % L;
    if (pad < 0 || p != pad) pp = dpos + (size_t)p * H;
  }
  if (!w && !pp) return;
  for (int i = threadIdx.x * 4; i < H; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(src + i);
    if (w) { atomicAdd(w + i, v.x); atomicAdd(w + i + 1, v.y); atomicAdd(w + i + 2, v.z); atomicAdd(w + i + 3, v.w); }
    if (pp) { atomicAdd(pp + i, v.x); atomicAdd(pp + i + 1, v.y); atomicAdd(pp + i + 2, v.z); atomicAdd(pp + i + 3, v.w); }
  }
}

// out[m,h] = (a[m,h] + b[m,h]) * dropout_scale(m*H + h)     a fp32 (optional), b bf16 (optional), out fp32 (may alias a)
__global__ void masked_add_kernel(const float* a, const __nv_bfloat16* __restrict__ b, long long ldb, float* out, int M, int H,
                                  DropCfg drop) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;    // one thread per 8 columns (one Philox call)
  const int per_row = H / 8;
  if (g >= (long long)M * per_row) return;
  const int m = (int)(g / per_row), c = (int)(g % per_row) * 8;
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = 0.f;
  if (a) {
    const float4 x0 = *reinterpret_cast<const float4*>(a + (size_t)m * H + c), x1 = *reinterpret_cast<const float4*>(a + (size_t)m * H + c + 4);
    v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
  }
  if (b) {
    float t[8];
    unpack8(*reinterpret_cast<const bf16x8*>(b + (size_t)m * ldb + c), t);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] += t[i];
  }
  if (drop.p > 0.f) {
    float sc[8];
    drop_scale8(drop, drop_stream(drop), ((unsigned long long)m * H + c) >> 3, sc);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] *= sc[i];
  }
  *reinterpret_cast<float4*>(out + (size_t)m * H + c) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(out + (size_t)m * H + c + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// torch.optim.Adam (no weight decay / amsgrad) on 4 parameters per thread + bf16 shadow refresh. 30 B of HBM traffic per
// parameter (p,g,m,v read; p,m,v + shadow written): the optimizer of a 7B full fine-tune is a ~200 GB pass.
__global__ void __launch_bounds__(256) adam_shadow_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                          float* __restrict__ v, __nv_bfloat16* __restrict__ shadow, long long n4,
                                                          float lr_bc1, float beta1, float beta2, float eps, float bc2_sqrt,
                                                          float grad_scale) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 P = reinterpret_cast<float4*>(p)[i], Mv = reinterpret_cast<float4*>(m)[i], Vv = reinterpret_cast<float4*>(v)[i];
  const float4 G = reinterpret_cast<const float4*>(g)[i];
  float* pp = &P.x; float* mm = &Mv.x; float* vv = &Vv.x; const float* gg = &G.x;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float gi = gg[j] * grad_scale;
    mm[j] = beta1 * mm[j] + (1.f - beta1) * gi;
    vv[j] = beta2 * vv[j] + (1.f - beta2) * gi * gi;
    pp[j] -= lr_bc1 * (mm[j] / (sqrtf(vv[j]) / bc2_sqrt + eps));
  }
  reinterpret_cast<float4*>(p)[i] = P; reinterpret_cast<float4*>(m)[i] = Mv; reinterpret_cast<float4*>(v)[i] = Vv;
  if (shadow) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(P.x, P.y), hi = __floats2bfloat162_rn(P.z, P.w);
    uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
    reinterpret_cast<uint2*>(shadow)[i] = pk;
  }
}

}  // namespace dalm

using namespace dalm;
#define ST(s) ((cudaStream_t)(s))

// out_sum / out_prod are ACCUMULATED into (zero them for a fresh gradient). mean may be NULL (RMSNorm); z / rstd are only
// read when out_prod is given. Shapes: dy_f32 [M,H] dense, dy_bf16 [M,H] row stride lddy.
extern "C" int dalm_b200_col_reduce(const float* dy_f32, const void* dy_bf16, long long lddy, const float* z, const float* mean,
                                    const float* rstd, float* out_sum, float* out_prod, int M, int H, void* stream) {
  DALM_REQUIRE(M > 0 && H > 0 && (H % 4) == 0, "col_reduce: bad shape M=%d H=%d (H must be a multiple of 4)", M, H);
  DALM_REQUIRE(dy_f32 || dy_bf16, "col_reduce: no gradient input");
  DALM_REQUIRE(!dy_bf16 || (lddy % 4) == 0, "col_reduce: lddy=%lld must be a multiple of 4", lddy);
  DALM_REQUIRE(out_sum || out_prod, "col_reduce: no output");
  DALM_REQUIRE(!out_prod || (z && rstd), "col_reduce: out_prod needs z and rstd");
  DALM_REQUIRE(aligned(dy_f32, 16) && aligned(z, 16) && aligned(dy_bf16, 8), "col_reduce: fp32 rows must be 16-byte, bf16 rows 8-byte aligned");
  const int colblocks = (H + kCrCols - 1) / kCrCols;
  int splits = (4 * num_sms() + colblocks - 1) / colblocks;
  const int max_splits = (M + 63) / 64;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  const int rows_per_cta = (M + splits - 1) / splits;
  dim3 grid(colblocks, (M + rows_per_cta - 1) / rows_per_cta);
  col_reduce_kernel<<<grid, 256, 0, ST(stream)>>>(dy_f32, (const __nv_bfloat16*)dy_bf16, lddy, z, mean, rstd, out_sum, out_prod, M, H,
                                                  rows_per_cta);
  count_launch();
  return check_launch("col_reduce_kernel");
}

extern "C" int dalm_b200_embed_scatter_add(const float* d, const int64_t* ids, const int64_t* pos_ids, float* dword, float* dpos,
                                           int M, int H, int L, int V, int pad_id, void* stream) {
  DALM_REQUIRE(M > 0 && (H % 4) == 0 && L > 0 && V > 0 && pad_id >= -1, "embed_scatter_add: bad shape M=%d H=%d L=%d V=%d pad_id=%d",
               M, H, L, V, pad_id);
  DALM_REQUIRE(aligned(d, 16), "embed_scatter_add: d must be 16-byte aligned");
  embed_scatter_kernel<<<M, 256, 0, ST(stream)>>>(d, (const long long*)ids, (const long long*)pos_ids, dword, dpos, M, H, L, V,
                                                  pad_id);
  count_launch();
  return check_launch("embed_scatter_kernel");
}

extern "C" int dalm_b200_masked_add(const float* a, const void* b, long long ldb, float* out, int M, int H, float p,
                                    unsigned long long seed, unsigned long long stream_id, const void* offset, void* stream) {
  DALM_REQUIRE(M > 0 && (H % 8) == 0, "masked_add: H=%d must be a multiple of 8", H);
  DALM_REQUIRE(a || b, "masked_add: no input");
  DALM_REQUIRE(!b || (ldb % 8) == 0, "masked_add: ldb must be a multiple of 8");
  DALM_REQUIRE(p >= 0.f && p < 1.f, "masked_add: p must be in [0,1)");
  DALM_REQUIRE(aligned(a, 16) && aligned(out, 16) && aligned(b, 16), "masked_add: operands must be 16-byte aligned");
  const long long n = (long long)M * (H / 8);
  masked_add_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(a, (const __nv_bfloat16*)b, ldb, out, M, H,
                                                                         make_drop(p, seed, stream_id, offset));
  count_launch();
  return check_launch("masked_add_kernel");
}

// n must be a multiple of 4 and the buffers 16-byte aligned (the flat parameter banks are padded accordingly)
extern "C" int dalm_b200_adam_step_shadow(float* p, const float* g, float* m, float* v, void* shadow_bf16, long long n, float lr,
                                          float beta1, float beta2, float eps, int step, float grad_scale, void* stream) {
  DALM_REQUIRE(n >= 0 && step >= 1 && (n % 4) == 0, "adam_shadow: n=%lld must be a non-negative multiple of 4, step >= 1", n);
  if (n == 0) return 0;
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2s = sqrtf(1.f - powf(beta2, (float)step));
  const long long n4 = n / 4;
  adam_shadow_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, ST(stream)>>>(p, g, m, v, (__nv_bfloat16*)shadow_bf16, n4, lr / bc1, beta1,
                                                                           beta2, eps, bc2s, grad_scale);
  count_launch();
  return check_launch("adam_shadow_kernel");
}
