// dalm_b200 — HBM-bound row-wise kernels of the encoder/decoder blocks (everything that is not a tensor-core tile):
// LayerNorm / RMSNorm forward+backward, embedding gathers, RoPE, SwiGLU, GeGLU, GELU, masked mean-pool + L2 normalise,
// LoRA weight-gradients, fused Adam. All use 16-byte vector accesses, warp-shuffle reductions and one CTA per row
// (rows = tokens; 3204..26700 per launch => several waves over 132 SMs).
//
// Reference semantics: HF BertModel / LlamaForCausalLM blocks reached via dalm/models/rag_e2e_base_model.py:93,105;
// mean_pooling + F.normalize: rag_e2e_base_model.py:96-97,108-111; torch.optim.Adam: train_rage2e.py:336.
#include "common.cuh"

namespace dalm {

// ------------------------------------------------------------------------------------------------------------
// LayerNorm forward: z fp32 [M,H] -> y = (z-mean)*rstd*gamma+beta, written as fp32 (residual path) and bf16 (GEMM input)
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) layernorm_fwd_kernel(const float* __restrict__ z, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float* __restrict__ y32,
                                                            __nv_bfloat16* __restrict__ y16, long long ld16,
                                                            float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                            int H, float eps, DropCfg drop) {
  extern __shared__ float row[];
  __shared__ float red[32];
  const size_t r = blockIdx.x;
  const float* zr = z + r * H;
  // the vector paths need 16-byte aligned fp32 operands and a y16 aligned to its access width (a view may start mid-row)
  const bool v32 = aligned(z, 16) && aligned(gamma, 16) && aligned(beta, 16) && aligned(y32, 16);
  float s = 0.f;
  if ((H & 3) == 0 && aligned(z, 16)) {
    const float4* z4 = reinterpret_cast<const float4*>(zr);
    float4* row4 = reinterpret_cast<float4*>(row);
    for (int i = threadIdx.x; i < H / 4; i += blockDim.x) { const float4 v = z4[i]; row4[i] = v; s += (v.x + v.y) + (v.z + v.w); }
  } else {
    for (int i = threadIdx.x; i < H; i += blockDim.x) { const float v = zr[i]; row[i] = v; s += v; }
  }
  const float mean = block_sum(s, red) / H;
  float q = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) { const float d = row[i] - mean; q += d * d; }
  const float var = block_sum(q, red) / H;
  const float rstd = rsqrtf(var + eps);
  if (threadIdx.x == 0) { mean_out[r] = mean; rstd_out[r] = rstd; }
  if (drop.p > 0.f && (H & 7) == 0 && v32) {                   // embeddings dropout: one Philox call per 8 outputs
    const unsigned long long dstream = drop_stream(drop);
    const bool y16_v8 = (ld16 & 7) == 0 && aligned(y16, 16);
    for (int i8 = threadIdx.x; i8 < H / 8; i8 += blockDim.x) {
      float sc[8];
      drop_scale8(drop, dstream, ((unsigned long long)r * H >> 3) + i8, sc);
      const int i0 = i8 * 8;
      float v[8];
      const float4 g0 = *reinterpret_cast<const float4*>(gamma + i0), g1 = *reinterpret_cast<const float4*>(gamma + i0 + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(beta + i0), b1 = *reinterpret_cast<const float4*>(beta + i0 + 4);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = ((row[i0 + j] - mean) * rstd * gg[j] + bb[j]) * sc[j];
      if (y32) {
        *reinterpret_cast<float4*>(y32 + r * H + i0) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(y32 + r * H + i0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
      }
      if (y16_v8) *reinterpret_cast<bf16x8*>(y16 + r * ld16 + i0) = pack8(v);
      else {
#pragma unroll
        for (int j = 0; j < 8; ++j) y16[r * ld16 + i0 + j] = __float2bfloat16_rn(v[j]);
      }
    }
    return;
  }
  if (drop.p == 0.f && (H & 3) == 0 && v32 && (ld16 & 3) == 0 && aligned(y16, 8)) {   // vectorised plain path: 4 outputs per thread
    const float4* row4 = reinterpret_cast<const float4*>(row);
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
    for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
      const float4 x = row4[i], g = g4[i], b = b4[i];
      const float4 v = make_float4((x.x - mean) * rstd * g.x + b.x, (x.y - mean) * rstd * g.y + b.y,
                                   (x.z - mean) * rstd * g.z + b.z, (x.w - mean) * rstd * g.w + b.w);
      if (y32) reinterpret_cast<float4*>(y32 + r * H)[i] = v;
      __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
      uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(y16 + r * ld16 + i * 4) = pk;
    }
    return;
  }
  const unsigned long long dstream = drop.p > 0.f ? drop_stream(drop) : 0ull;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    float v = (row[i] - mean) * rstd * gamma[i] + beta[i];
    if (drop.p > 0.f) v *= drop_scale1(drop, dstream, (unsigned long long)r * H + i);
    if (y32) y32[r * H + i] = v;
    y16[r * ld16 + i] = __float2bfloat16_rn(v);
  }
}

// LayerNorm backward (input gradient only; gamma/beta frozen in PEFT mode, see layernorm_bwd_params_kernel):
//   dz = rstd * (g - mean(g) - zhat * mean(g*zhat)),  g = dy*gamma ; dy = dy_a (fp32, residual stream) + dy_b (bf16, GEMM dgrad)
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const float* __restrict__ z, const float* __restrict__ gamma,
                                                            const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                                                            const float* __restrict__ dy_a, const __nv_bfloat16* __restrict__ dy_b,
                                                            long long ldb, float* dz32,
                                                            __nv_bfloat16* __restrict__ dz16, long long ld16, int H,
                                                            DropCfg drop16, const float* dres) {
  // dres (optional, may alias dz32): gradient arriving through a residual connection AROUND the norm (pre-LN blocks:
  // Falcon's x_out = x + attn(LN(x)) + mlp(LN(x))), added to both outputs; each element is read and written by one thread
  extern __shared__ float sm[];
  float* gbuf = sm;          // g = dy*gamma
  float* zh = sm + H;        // zhat
  __shared__ float red[32];
  const size_t r = blockIdx.x;
  const float mean = mean_in[r], rstd = rstd_in[r];
  float s1 = 0.f, s2 = 0.f;
  const bool v32 = aligned(dz32, 16) && aligned(dres, 16);         // vector stores of the fp32 output
  if ((H & 3) == 0 && (ldb & 3) == 0 && aligned(z, 16) && aligned(gamma, 16) && aligned(dy_a, 16) && aligned(dy_b, 8)) {
    const float4* z4 = reinterpret_cast<const float4*>(z + r * H);
    const float4* a4 = dy_a ? reinterpret_cast<const float4*>(dy_a + r * H) : nullptr;
    const uint2* b2 = dy_b ? reinterpret_cast<const uint2*>(dy_b + r * ldb) : nullptr;
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
      float4 dy = a4 ? a4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      if (b2) {
        const uint2 raw = b2[i];
        const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
        const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
        dy.x += lo.x; dy.y += lo.y; dy.z += hi.x; dy.w += hi.y;
      }
      const float4 gg = g4[i], zz4 = z4[i];
      const float4 g = make_float4(dy.x * gg.x, dy.y * gg.y, dy.z * gg.z, dy.w * gg.w);
      const float4 zz = make_float4((zz4.x - mean) * rstd, (zz4.y - mean) * rstd, (zz4.z - mean) * rstd, (zz4.w - mean) * rstd);
      reinterpret_cast<float4*>(gbuf)[i] = g;
      reinterpret_cast<float4*>(zh)[i] = zz;
      s1 += (g.x + g.y) + (g.z + g.w);
      s2 += (g.x * zz.x + g.y * zz.y) + (g.z * zz.z + g.w * zz.w);
    }
  } else {
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
      float dy = 0.f;
      if (dy_a) dy += dy_a[r * H + i];
      if (dy_b) dy += __bfloat162float(dy_b[r * ldb + i]);
      const float g = dy * gamma[i];
      const float zz = (z[r * H + i] - mean) * rstd;
      gbuf[i] = g; zh[i] = zz;
      s1 += g; s2 += g * zz;
    }
  }
  s1 = block_sum(s1, red) / H;
  s2 = block_sum(s2, red) / H;
  // z = dropout(dense_out) + residual: the residual branch takes dz as is (dz32), the dense branch takes mask*dz/(1-p)
  if (drop16.p > 0.f && (H & 7) == 0 && v32) {
    const unsigned long long dstream = drop_stream(drop16);
    const bool dz16_v8 = (ld16 & 7) == 0 && aligned(dz16, 16);
    for (int i8 = threadIdx.x; i8 < H / 8; i8 += blockDim.x) {
      float sc[8];
      drop_scale8(drop16, dstream, ((unsigned long long)r * H >> 3) + i8, sc);
      const int i0 = i8 * 8;
      float d[8], dm[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) { d[j] = rstd * (gbuf[i0 + j] - s1 - zh[i0 + j] * s2); dm[j] = d[j] * sc[j]; }
      if (dz32) {
        *reinterpret_cast<float4*>(dz32 + r * H + i0) = make_float4(d[0], d[1], d[2], d[3]);
        *reinterpret_cast<float4*>(dz32 + r * H + i0 + 4) = make_float4(d[4], d[5], d[6], d[7]);
      }
      if (dz16) {
        if (dz16_v8) *reinterpret_cast<bf16x8*>(dz16 + r * ld16 + i0) = pack8(dm);
        else {
#pragma unroll
          for (int j = 0; j < 8; ++j) dz16[r * ld16 + i0 + j] = __float2bfloat16_rn(dm[j]);
        }
      }
    }
    return;
  }
  if (drop16.p == 0.f && (H & 3) == 0 && v32 && (ld16 & 3) == 0 && aligned(dz16, 8)) {
    for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
      const float4 g = reinterpret_cast<const float4*>(gbuf)[i], zz = reinterpret_cast<const float4*>(zh)[i];
      float4 d = make_float4(rstd * (g.x - s1 - zz.x * s2), rstd * (g.y - s1 - zz.y * s2), rstd * (g.z - s1 - zz.z * s2),
                             rstd * (g.w - s1 - zz.w * s2));
      if (dres) {
        const float4 t = reinterpret_cast<const float4*>(dres + r * H)[i];
        d.x += t.x; d.y += t.y; d.z += t.z; d.w += t.w;
      }
      if (dz32) reinterpret_cast<float4*>(dz32 + r * H)[i] = d;
      if (dz16) {
        __nv_bfloat162 lo = __floats2bfloat162_rn(d.x, d.y), hi = __floats2bfloat162_rn(d.z, d.w);
        uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(dz16 + r * ld16 + i * 4) = pk;
      }
    }
    return;
  }
  const unsigned long long dstream = drop16.p > 0.f ? drop_stream(drop16) : 0ull;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const float d = rstd * (gbuf[i] - s1 - zh[i] * s2) + (dres ? dres[r * H + i] : 0.f);
    if (dz32) dz32[r * H + i] = d;
    if (dz16) {
      const float m = drop16.p > 0.f ? drop_scale1(drop16, dstream, (unsigned long long)r * H + i) : 1.f;
      dz16[r * ld16 + i] = __float2bfloat16_rn(d * m);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// RMSNorm forward: x fp32 [M,H] -> h bf16 = x * rsqrt(mean(x^2)+eps) * g
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rmsnorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                          __nv_bfloat16* __restrict__ h, long long ldh,
                                                          float* __restrict__ rstd_out, int H, float eps) {
  extern __shared__ float row[];
  __shared__ float red[32];
  const size_t r = blockIdx.x;
  const float4* x4 = reinterpret_cast<const float4*>(x + r * H);
  float4* row4 = reinterpret_cast<float4*>(row);
  float q = 0.f;
  for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
    const float4 v = x4[i]; row4[i] = v;
    q += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  const float rstd = rsqrtf(block_sum(q, red) / H + eps);
  if (threadIdx.x == 0) rstd_out[r] = rstd;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
    const float4 v = row4[i], w = g4[i];
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x * rstd * w.x, v.y * rstd * w.y);
    __nv_bfloat162 b = __floats2bfloat162_rn(v.z * rstd * w.z, v.w * rstd * w.w);
    uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&a); pk.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(h + r * ldh + i * 4) = pk;
  }
}

// RMSNorm backward, fused with the residual-gradient stream:
//   dx = rstd * (gd - xhat * mean(gd * xhat)), gd = dh * g;   dres_out = dres_in + dx  (fp32) and its bf16 copy
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                          const float* __restrict__ rstd_in,
                                                          const __nv_bfloat16* __restrict__ dh, long long lddh,
                                                          const float* __restrict__ dres_in, float* __restrict__ dres_out,
                                                          __nv_bfloat16* __restrict__ dres16, long long ld16, int H) {
  // 4 elements per thread per iteration (float4 / 8-byte bf16x4); the row's g*dh and xhat stay in shared memory
  extern __shared__ float sm[];
  float4* gd4 = reinterpret_cast<float4*>(sm);
  float4* xh4 = reinterpret_cast<float4*>(sm + H);
  __shared__ float red[32];
  const size_t r = blockIdx.x;
  const float rstd = rstd_in[r];
  const float4* x4 = reinterpret_cast<const float4*>(x + r * H);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const uint2* dh2 = reinterpret_cast<const uint2*>(dh + r * lddh);
  float s = 0.f;
  for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
    const uint2 raw = dh2[i];
    const float2 d01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
    const float2 d23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
    const float4 gg = g4[i], xx = x4[i];
    const float4 a = make_float4(d01.x * gg.x, d01.y * gg.y, d23.x * gg.z, d23.y * gg.w);
    const float4 b = make_float4(xx.x * rstd, xx.y * rstd, xx.z * rstd, xx.w * rstd);
    gd4[i] = a; xh4[i] = b;
    s += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
  }
  s = block_sum(s, red) / H;
  const float4* din4 = dres_in ? reinterpret_cast<const float4*>(dres_in + r * H) : nullptr;
  float4* dout4 = reinterpret_cast<float4*>(dres_out + r * H);
  uint2* d16 = dres16 ? reinterpret_cast<uint2*>(dres16 + r * ld16) : nullptr;
  for (int i = threadIdx.x; i < H / 4; i += blockDim.x) {
    const float4 a = gd4[i], b = xh4[i];
    float4 d = make_float4(rstd * (a.x - b.x * s), rstd * (a.y - b.y * s), rstd * (a.z - b.z * s), rstd * (a.w - b.w * s));
    if (din4) { const float4 t = din4[i]; d.x += t.x; d.y += t.y; d.z += t.z; d.w += t.w; }
    dout4[i] = d;
    if (d16) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(d.x, d.y), hi = __floats2bfloat162_rn(d.z, d.w);
      uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
      d16[i] = pk;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// OLMo 2 / OLMo 3 post-sublayer RMSNorm with the residual add (transformers Olmo2DecoderLayer: x + post_norm(sublayer(x))):
//   forward:  out (fp32) = resid + bf16(w * (y * rstd)),  rstd = rsqrt(mean(y^2) + eps),  y = the bf16 o_proj / down output;
//             out16 (optional) = bf16(out), the next GEMM's operand
//   backward: d = dres_in (+ dh, the bf16 gradient of the sublayer below that joins the residual stream here) -> dres_out = d
//             (the residual gradient passes on unchanged) and dy (bf16) = rstd (w d - y_hat mean(w d y_hat)), y_hat = y rstd
// One CTA per row; each thread holds up to kPostNormUnits 8-column units of the row in registers (H <= 8192, H % 8 == 0).
// ------------------------------------------------------------------------------------------------------------
constexpr int kPostNormUnits = 4;

__device__ __forceinline__ void ld_bf16x8(const __nv_bfloat16* p, float* v) {
  const uint4 raw = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[e]));
    v[2 * e] = f.x; v[2 * e + 1] = f.y;
  }
}
__device__ __forceinline__ void st_bf16x8(__nv_bfloat16* p, const float* v) {
  uint32_t w[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    __nv_bfloat162 t = __floats2bfloat162_rn(v[2 * e], v[2 * e + 1]);
    w[e] = *reinterpret_cast<uint32_t*>(&t);
  }
  *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ void ld_f32x8(const float* p, float* v) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void st_f32x8(float* p, const float* v) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

__global__ void __launch_bounds__(256) postnorm_fwd_kernel(const __nv_bfloat16* __restrict__ y, long long ldy,
                                                           const float* __restrict__ w, const float* __restrict__ resid,
                                                           float* __restrict__ out, __nv_bfloat16* __restrict__ out16, long long ld16,
                                                           float* __restrict__ rstd_out, int H, float eps) {
  __shared__ float red[32];
  const size_t r = blockIdx.x;
  const int units = H / 8;
  float v[kPostNormUnits][8];
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < kPostNormUnits; ++k) {
    const int i = threadIdx.x + k * 256;
    if (i < units) {
      ld_bf16x8(y + r * ldy + i * 8, v[k]);
#pragma unroll
      for (int e = 0; e < 8; ++e) q = fmaf(v[k][e], v[k][e], q);
    }
  }
  const float rstd = rsqrtf(block_sum(q, red) / H + eps);
  if (threadIdx.x == 0) rstd_out[r] = rstd;
#pragma unroll
  for (int k = 0; k < kPostNormUnits; ++k) {
    const int i = threadIdx.x + k * 256;
    if (i < units) {
      float ww[8], x[8];
      ld_f32x8(w + i * 8, ww);
      ld_f32x8(resid + r * H + i * 8, x);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] += __bfloat162float(__float2bfloat16_rn(ww[e] * (v[k][e] * rstd)));
      st_f32x8(out + r * H + i * 8, x);
      if (out16 != nullptr) st_bf16x8(out16 + r * ld16 + i * 8, x);
    }
  }
}

__global__ void __launch_bounds__(256) postnorm_bwd_kernel(const __nv_bfloat16* __restrict__ y, long long ldy,
                                                           const float* __restrict__ w, const float* __restrict__ rstd_in,
                                                           const float* __restrict__ dres_in, const __nv_bfloat16* __restrict__ dh,
                                                           long long lddh, float* __restrict__ dres_out,
                                                           __nv_bfloat16* __restrict__ dy, long long lddy, int H) {
  __shared__ float red[32];
  const size_t r = blockIdx.x;
  const int units = H / 8;
  const float rstd = rstd_in[r];
  float wd[kPostNormUnits][8], yh[kPostNormUnits][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kPostNormUnits; ++k) {
    const int i = threadIdx.x + k * 256;
    if (i < units) {
      float d[8], ww[8];
      ld_f32x8(dres_in + r * H + i * 8, d);
      if (dh != nullptr) {
        float t[8];
        ld_bf16x8(dh + r * lddh + i * 8, t);
#pragma unroll
        for (int e = 0; e < 8; ++e) d[e] += t[e];
      }
      st_f32x8(dres_out + r * H + i * 8, d);
      ld_f32x8(w + i * 8, ww);
      ld_bf16x8(y + r * ldy + i * 8, yh[k]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        wd[k][e] = ww[e] * d[e];
        yh[k][e] *= rstd;
        s = fmaf(wd[k][e], yh[k][e], s);
      }
    }
  }
  const float m = block_sum(s, red) / H;
#pragma unroll
  for (int k = 0; k < kPostNormUnits; ++k) {
    const int i = threadIdx.x + k * 256;
    if (i < units) {
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = rstd * fmaf(-yh[k][e], m, wd[k][e]);
      st_bf16x8(dy + r * lddy + i * 8, o);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// embeddings
// ------------------------------------------------------------------------------------------------------------
// BERT: z = word[id] + pos[l] + type[0]  (fp32 sum, LayerNorm follows as a separate launch)
__global__ void bert_embed_kernel(const int64_t* __restrict__ ids, const __nv_bfloat16* __restrict__ word,
                                  const __nv_bfloat16* __restrict__ pos, const __nv_bfloat16* __restrict__ type0,
                                  float* __restrict__ z, int L, int H, int V) {
  const size_t r = blockIdx.x;
  const int l = (int)(r % L);
  int64_t id = ids[r];
  if (id < 0 || id >= V) id = 0;
  for (int i = threadIdx.x; i < H; i += blockDim.x)
    z[r * H + i] = __bfloat162float(word[(size_t)id * H + i]) + __bfloat162float(pos[(size_t)l * H + i]) +
                   __bfloat162float(type0[i]);
}
// RoBERTa / XLM-RoBERTa: the position comes from the ids (HF create_position_ids_from_input_ids), not the column:
// pos = pad + (id != pad) * (number of non-pad ids in columns 0..l of the row), clamped into [0, P) as a guard. One CTA per
// (row, chunk of 32 columns), so the grid scales with B*L: the CTA counts the row's non-pad ids before its chunk, one warp
// ballot ranks the chunk, then z = word[id] + pos[position] + type[0] in bert_embed's order of additions. Position ids of the
// chunk go to pos_ids (may be NULL) for the backward's scatter.
constexpr int kReChunk = 32;
__global__ void __launch_bounds__(256) roberta_embed_kernel(const int64_t* __restrict__ ids, const __nv_bfloat16* __restrict__ word,
                                                            const __nv_bfloat16* __restrict__ pos,
                                                            const __nv_bfloat16* __restrict__ type0, long long pad,
                                                            float* __restrict__ z, int64_t* __restrict__ pos_ids, int L, int H,
                                                            int V, int P) {
  __shared__ int red[32];
  __shared__ long long s_pos[kReChunk];
  const int c0 = blockIdx.x * kReChunk;
  const int64_t* row = ids + (size_t)blockIdx.y * L;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int cnt = 0;
  for (int l = threadIdx.x; l < c0; l += blockDim.x) cnt += row[l] != pad;
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if (lane == 0) red[warp] = cnt;
  __syncthreads();
  if (warp == 0) {
    const int before = __reduce_add_sync(0xffffffffu, lane < (int)(blockDim.x >> 5) ? red[lane] : 0);
    const int l = c0 + lane;
    const bool tok = l < L && row[l] != pad;
    const unsigned bal = __ballot_sync(0xffffffffu, tok);
    long long p = tok ? pad + before + __popc(bal & (0xffffffffu >> (31 - lane))) : pad;
    p = p < 0 ? 0 : (p >= P ? P - 1 : p);
    s_pos[lane] = p;
    if (pos_ids && l < L) pos_ids[(size_t)blockIdx.y * L + l] = p;
  }
  __syncthreads();
  const int n = min(kReChunk, L - c0), H4 = H >> 2;
  for (int e = threadIdx.x; e < n * H4; e += blockDim.x) {           // 4 columns per thread: 8-byte bf16 reads, float4 store
    const int t = e / H4, c = (e - t * H4) * 4;
    int64_t id = row[c0 + t];
    if (id < 0 || id >= V) id = 0;
    const uint2 w = *reinterpret_cast<const uint2*>(word + (size_t)id * H + c);
    const uint2 q = *reinterpret_cast<const uint2*>(pos + (size_t)s_pos[t] * H + c);
    const uint2 y = *reinterpret_cast<const uint2*>(type0 + c);
    const float2 w0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w.x)), w1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w.y));
    const float2 q0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&q.x)), q1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&q.y));
    const float2 y0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&y.x)), y1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&y.y));
    *reinterpret_cast<float4*>(z + ((size_t)blockIdx.y * L + c0 + t) * H + c) =
        make_float4(w0.x + q0.x + y0.x, w0.y + q0.y + y0.y, w1.x + q1.x + y1.x, w1.y + q1.y + y1.y);
  }
}
// decoder: x[r,:] = table[id,:] (bf16 -> fp32 residual stream)
__global__ void embed_gather_kernel(const int64_t* __restrict__ ids, const __nv_bfloat16* __restrict__ table,
                                    float* __restrict__ x, int H, int V) {
  const size_t r = blockIdx.x;
  int64_t id = ids[r];
  if (id < 0 || id >= V) id = 0;
  for (int i = threadIdx.x; i < H; i += blockDim.x) x[r * H + i] = __bfloat162float(table[(size_t)id * H + i]);
}

// ------------------------------------------------------------------------------------------------------------
// RoPE (HF rotate_half convention), in place on `nheads` heads of width D starting at column col0 of a token-major
// bf16 buffer. position = row % L. sign = +1 forward, -1 backward (inverse rotation = transpose of the forward map).
// ------------------------------------------------------------------------------------------------------------
__global__ void rope_kernel(__nv_bfloat16* __restrict__ buf, long long ld, int col0, int nheads, int D,
                            const float* __restrict__ cos_t, const float* __restrict__ sin_t, int L, float sign) {
  // one CTA per token row; each thread rotates 8 (j, j+D/2) pairs with 16-byte accesses
  const size_t r = blockIdx.x;
  const int l = (int)(r % L), half = D / 2, chunks = half / 8;
  __nv_bfloat16* base = buf + r * ld + col0;
  for (int i = threadIdx.x; i < nheads * chunks; i += blockDim.x) {
    const int hd = i / chunks, j = (i - hd * chunks) * 8;
    __nv_bfloat16* p = base + hd * D + j;
    float x1[8], x2[8], o1[8], o2[8];
    unpack8(*reinterpret_cast<const bf16x8*>(p), x1);
    unpack8(*reinterpret_cast<const bf16x8*>(p + half), x2);
    const float4 c0 = *reinterpret_cast<const float4*>(cos_t + (size_t)l * half + j);
    const float4 c1 = *reinterpret_cast<const float4*>(cos_t + (size_t)l * half + j + 4);
    const float4 s0 = *reinterpret_cast<const float4*>(sin_t + (size_t)l * half + j);
    const float4 s1 = *reinterpret_cast<const float4*>(sin_t + (size_t)l * half + j + 4);
    const float c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float s = sn[k] * sign;
      o1[k] = x1[k] * c[k] - x2[k] * s;
      o2[k] = x2[k] * c[k] + x1[k] * s;
    }
    *reinterpret_cast<bf16x8*>(p) = pack8(o1);
    *reinterpret_cast<bf16x8*>(p + half) = pack8(o2);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Gated MLP activations on a [first | second] buffer (bf16 [M,2F]): act = A(first) * second.
//   SwiGLU (Llama): gu = [gate | up], A = silu.   GeGLU (ModernBERT): [input | gate] = Wi(x).chunk(2), A = gelu_erf.
// ------------------------------------------------------------------------------------------------------------
// gate / up column of feature i inside a [M, 2F] gate|up buffer: il == 0: [gate 0..F | up 0..F] (HF order); il > 0: blocks of il
// features interleaved [gate blk | up blk | gate blk+1 | ...] - the layout that puts a feature's gate AND up accumulator in the
// same 128 x 256 GEMM tile (gemm_wgmma.cu: SwiGLU epilogue)
__device__ __forceinline__ int gate_col(int i, int F, int il, int& up_off) {
  if (il == 0) { up_off = F; return i; }
  up_off = il;
  return (i / il) * 2 * il + (i % il);
}
// A(x), and the backward of act = A(g) * u given d = d act: dg = d * u * A'(g), du = d * A(g)
struct SiluAct {
  static __device__ __forceinline__ float fwd(float x) { return x / (1.f + __expf(-x)); }
  static __device__ __forceinline__ void bwd(float g, float u, float d, float& dg, float& du) {
    const float sg = 1.f / (1.f + __expf(-g));
    const float silu = g * sg;
    dg = d * u * sg * (1.f + g * (1.f - sg));
    du = d * silu;
  }
};
struct GeluAct {
  static __device__ __forceinline__ float fwd(float x) { return gelu_erf(x); }
  static __device__ __forceinline__ void bwd(float g, float u, float d, float& dg, float& du) {
    dg = d * u * gelu_erf_grad(g);
    du = d * gelu_erf(g);
  }
};
template <class Act>
__global__ void glu_fwd_kernel(const __nv_bfloat16* __restrict__ gu, long long ldgu, __nv_bfloat16* __restrict__ act,
                               long long lda, int F, int il) {
  const size_t r = blockIdx.y;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= F) return;
  float g[8], u[8], o[8];
  int uo;
  const int gc = gate_col(i, F, il, uo);
  unpack8(*reinterpret_cast<const bf16x8*>(gu + r * ldgu + gc), g);
  unpack8(*reinterpret_cast<const bf16x8*>(gu + r * ldgu + gc + uo), u);
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = Act::fwd(g[k]) * u[k];
  *reinterpret_cast<bf16x8*>(act + r * lda + i) = pack8(o);
}
// in place: gu <- [d first | d second]
template <class Act>
__global__ void glu_bwd_kernel(__nv_bfloat16* __restrict__ gu, long long ldgu, const __nv_bfloat16* __restrict__ dact,
                               long long ldd, int F, int il) {
  const size_t r = blockIdx.y;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= F) return;
  float g[8], u[8], d[8], dg[8], du[8];
  int uo;
  const int gc = gate_col(i, F, il, uo);
  unpack8(*reinterpret_cast<const bf16x8*>(gu + r * ldgu + gc), g);
  unpack8(*reinterpret_cast<const bf16x8*>(gu + r * ldgu + gc + uo), u);
  unpack8(*reinterpret_cast<const bf16x8*>(dact + r * ldd + i), d);
#pragma unroll
  for (int k = 0; k < 8; ++k) Act::bwd(g[k], u[k], d[k], dg[k], du[k]);
  *reinterpret_cast<bf16x8*>(gu + r * ldgu + gc) = pack8(dg);
  *reinterpret_cast<bf16x8*>(gu + r * ldgu + gc + uo) = pack8(du);
}

// GELU(erf) forward on a pre-activation buffer, and backward in place on the incoming gradient
// GELU forward / backward: each thread walks GELU_ROWS rows of one 8-column group with all of its 16-byte loads issued before
// the first use (one row per thread leaves most of the HBM bandwidth unused)
constexpr int GELU_ROWS = 4;
__global__ void gelu_fwd_kernel(const __nv_bfloat16* __restrict__ pre, long long ldp, __nv_bfloat16* __restrict__ act,
                                long long lda, int M, int F) {
  const size_t r0 = (size_t)blockIdx.y * GELU_ROWS;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= F) return;
  bf16x8 raw[GELU_ROWS];
#pragma unroll
  for (int u = 0; u < GELU_ROWS; ++u)
    if (r0 + u < (size_t)M) raw[u] = *reinterpret_cast<const bf16x8*>(pre + (r0 + u) * ldp + i);
#pragma unroll
  for (int u = 0; u < GELU_ROWS; ++u) {
    if (r0 + u >= (size_t)M) break;
    float x[8];
    unpack8(raw[u], x);
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = gelu_erf(x[k]);
    *reinterpret_cast<bf16x8*>(act + (r0 + u) * lda + i) = pack8(x);
  }
}
__global__ void gelu_bwd_kernel(const __nv_bfloat16* __restrict__ pre, long long ldp, __nv_bfloat16* __restrict__ dact,
                                long long ldd, int M, int F) {
  const size_t r0 = (size_t)blockIdx.y * GELU_ROWS;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= F) return;
  bf16x8 rx[GELU_ROWS], rd[GELU_ROWS];
#pragma unroll
  for (int u = 0; u < GELU_ROWS; ++u)
    if (r0 + u < (size_t)M) {
      rx[u] = *reinterpret_cast<const bf16x8*>(pre + (r0 + u) * ldp + i);
      rd[u] = *reinterpret_cast<const bf16x8*>(dact + (r0 + u) * ldd + i);
    }
#pragma unroll
  for (int u = 0; u < GELU_ROWS; ++u) {
    if (r0 + u >= (size_t)M) break;
    float x[8], d[8];
    unpack8(rx[u], x);
    unpack8(rd[u], d);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] *= gelu_erf_grad(x[k]);
    *reinterpret_cast<bf16x8*>(dact + (r0 + u) * ldd + i) = pack8(d);
  }
}

// ------------------------------------------------------------------------------------------------------------
// LayerNorm, one WARP per row (H = 256 NV8, NV8 <= 8: bge-large's 1024). The CTA-per-row kernels above give a 1024-wide row to
// 256 threads - one float4 each - and spend their time in two block-wide reductions, far from the HBM bandwidth. Here a lane keeps its 8 NV8 elements in registers
// (8 consecutive floats per 256-wide chunk: one Philox group per chunk when dropout is on), statistics by warp shuffles, no
// shared memory, 8 rows per CTA.
// ------------------------------------------------------------------------------------------------------------
template <int NV8>
__global__ void __launch_bounds__(256) layernorm_fwd_warp_kernel(const float* __restrict__ z, const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, float* __restrict__ y32,
                                                                 __nv_bfloat16* __restrict__ y16, long long ld16,
                                                                 float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                                 int M, float eps, DropCfg drop) {
  constexpr int H = NV8 * 256;
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= M) return;
  float v[NV8][8];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < NV8; ++c) {
    const float4* p = reinterpret_cast<const float4*>(z + r * H + c * 256 + lane * 8);
    const float4 a = p[0], b = p[1];
    v[c][0] = a.x; v[c][1] = a.y; v[c][2] = a.z; v[c][3] = a.w; v[c][4] = b.x; v[c][5] = b.y; v[c][6] = b.z; v[c][7] = b.w;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += v[c][j];
  }
  const float mean = warp_sum(s) / H;
  float q = 0.f;
#pragma unroll
  for (int c = 0; c < NV8; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float d = v[c][j] - mean; q += d * d; }
  const float rstd = rsqrtf(warp_sum(q) / H + eps);
  if (lane == 0) { mean_out[r] = mean; rstd_out[r] = rstd; }
  const unsigned long long dstream = drop.p > 0.f ? drop_stream(drop) : 0ull;
#pragma unroll
  for (int c = 0; c < NV8; ++c) {
    const int i0 = c * 256 + lane * 8;
    const float4 g0 = *reinterpret_cast<const float4*>(gamma + i0), g1 = *reinterpret_cast<const float4*>(gamma + i0 + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(beta + i0), b1 = *reinterpret_cast<const float4*>(beta + i0 + 4);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rstd * gg[j] + bb[j];
    if (drop.p > 0.f) {
      float sc[8];
      drop_scale8(drop, dstream, (((unsigned long long)r * H) >> 3) + (unsigned long long)(i0 >> 3), sc);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] *= sc[j];
    }
    if (y32) {
      *reinterpret_cast<float4*>(y32 + r * H + i0) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(y32 + r * H + i0 + 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
    *reinterpret_cast<bf16x8*>(y16 + r * ld16 + i0) = pack8(o);
  }
}

template <int NV8>
__global__ void __launch_bounds__(256) layernorm_bwd_warp_kernel(const float* __restrict__ z, const float* __restrict__ gamma,
                                                                 const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                                                                 const float* __restrict__ dy_a, const __nv_bfloat16* __restrict__ dy_b,
                                                                 long long ldb, float* dz32, __nv_bfloat16* __restrict__ dz16,
                                                                 long long ld16, int M, DropCfg drop16, const float* dres) {
  constexpr int H = NV8 * 256;
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= M) return;
  const float mean = mean_in[r], rstd = rstd_in[r];
  float g[NV8][8], zh[NV8][8];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int c = 0; c < NV8; ++c) {
    const int i0 = c * 256 + lane * 8;
    float dy[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (dy_a) {
      const float4 a = *reinterpret_cast<const float4*>(dy_a + r * H + i0), b = *reinterpret_cast<const float4*>(dy_a + r * H + i0 + 4);
      dy[0] = a.x; dy[1] = a.y; dy[2] = a.z; dy[3] = a.w; dy[4] = b.x; dy[5] = b.y; dy[6] = b.z; dy[7] = b.w;
    }
    if (dy_b) {
      float t[8];
      unpack8(*reinterpret_cast<const bf16x8*>(dy_b + r * ldb + i0), t);
#pragma unroll
      for (int j = 0; j < 8; ++j) dy[j] += t[j];
    }
    const float4 z0 = *reinterpret_cast<const float4*>(z + r * H + i0), z1 = *reinterpret_cast<const float4*>(z + r * H + i0 + 4);
    const float4 g0 = *reinterpret_cast<const float4*>(gamma + i0), g1 = *reinterpret_cast<const float4*>(gamma + i0 + 4);
    const float zz[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      g[c][j] = dy[j] * gg[j];
      zh[c][j] = (zz[j] - mean) * rstd;
      s1 += g[c][j];
      s2 += g[c][j] * zh[c][j];
    }
  }
  s1 = warp_sum(s1) / H;
  s2 = warp_sum(s2) / H;
  const unsigned long long dstream = drop16.p > 0.f ? drop_stream(drop16) : 0ull;
#pragma unroll
  for (int c = 0; c < NV8; ++c) {
    const int i0 = c * 256 + lane * 8;
    float d[8], dm[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = rstd * (g[c][j] - s1 - zh[c][j] * s2);
    if (dres) {                                                // residual around the norm (pre-LN blocks): added to both outputs
      const float4 a = *reinterpret_cast<const float4*>(dres + r * H + i0), b = *reinterpret_cast<const float4*>(dres + r * H + i0 + 4);
      d[0] += a.x; d[1] += a.y; d[2] += a.z; d[3] += a.w; d[4] += b.x; d[5] += b.y; d[6] += b.z; d[7] += b.w;
    }
    if (drop16.p > 0.f) {                                      // z = dropout(dense_out) + residual: the dense branch gets mask*dz/(1-p)
      float sc[8];
      drop_scale8(drop16, dstream, (((unsigned long long)r * H) >> 3) + (unsigned long long)(i0 >> 3), sc);
#pragma unroll
      for (int j = 0; j < 8; ++j) dm[j] = d[j] * sc[j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) dm[j] = d[j];
    }
    if (dz32) {
      *reinterpret_cast<float4*>(dz32 + r * H + i0) = make_float4(d[0], d[1], d[2], d[3]);
      *reinterpret_cast<float4*>(dz32 + r * H + i0 + 4) = make_float4(d[4], d[5], d[6], d[7]);
    }
    if (dz16) *reinterpret_cast<bf16x8*>(dz16 + r * ld16 + i0) = pack8(dm);
  }
}

template <int NV8>
static int launch_ln_fwd_warp(const float* z, const float* gamma, const float* beta, float* y32, __nv_bfloat16* y16, long long ld16,
                              float* mean, float* rstd, int M, float eps, const DropCfg& d, cudaStream_t st) {
  layernorm_fwd_warp_kernel<NV8><<<(M + 7) / 8, 256, 0, st>>>(z, gamma, beta, y32, y16, ld16, mean, rstd, M, eps, d);
  count_launch();
  return check_launch("layernorm_fwd_warp_kernel");
}
template <int NV8>
static int launch_ln_bwd_warp(const float* z, const float* gamma, const float* mean, const float* rstd, const float* dy_a,
                              const __nv_bfloat16* dy_b, long long ldb, float* dz32, __nv_bfloat16* dz16, long long ld16, int M,
                              const DropCfg& d, const float* dres, cudaStream_t st) {
  layernorm_bwd_warp_kernel<NV8><<<(M + 7) / 8, 256, 0, st>>>(z, gamma, mean, rstd, dy_a, dy_b, ldb, dz32, dz16, ld16, M, d, dres);
  count_launch();
  return check_launch("layernorm_bwd_warp_kernel");
}
// the warp-per-row kernels serve H in {256, 512, 1024, 2048} with 16-byte aligned rows
static bool ln_warp_ok(int H, long long ld16, const void* a, const void* b, const void* c, long long ldb) {
  auto al = [](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return (H == 256 || H == 512 || H == 1024 || H == 2048) && (ld16 % 8) == 0 && (ldb % 8) == 0 && al(a) && al(b) && al(c);
}

// ------------------------------------------------------------------------------------------------------------
// masked mean-pool + L2 normalise (forward) and its backward. hidden fp32 [B,L,H]; mask int64 [B,L].
//   pooled = sum_l h*m / clamp(sum_l m, 1e-9);  emb = pooled / max(||pooled||, 1e-12)   (if normalize)
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pool_norm_fwd_kernel(const float* __restrict__ hidden, const int64_t* __restrict__ mask,
                                                            float* __restrict__ pooled, float* __restrict__ emb,
                                                            float* __restrict__ norm_out, int L, int H, int normalize) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  float cnt = 0.f;
  for (int l = 0; l < L; ++l) cnt += (float)mask[(size_t)b * L + l];
  const float inv = 1.f / fmaxf(cnt, 1e-9f);
  float sq = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    float acc = 0.f;
    for (int l = 0; l < L; ++l) {
      const float m = (float)mask[(size_t)b * L + l];
      if (m != 0.f) acc += hidden[((size_t)b * L + l) * H + i] * m;
    }
    acc *= inv;
    pooled[(size_t)b * H + i] = acc;
    sq += acc * acc;
  }
  const float nrm = sqrtf(block_sum(sq, red));
  if (threadIdx.x == 0) norm_out[b] = nrm;
  const float s = normalize ? 1.f / fmaxf(nrm, 1e-12f) : 1.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) emb[(size_t)b * H + i] = pooled[(size_t)b * H + i] * s;
}
// The same forward for H % 128 == 0, spread over the machine: the one-CTA-per-sample kernel above walks the L rows serially
// (B CTAs: a small fraction of the machine). Here CTA (chunk, b) owns 128 columns of sample b: each of its 8 warps
// streams the rows l = warp, warp + 8, ... (one coalesced 512-byte float4 row piece per warp-load, masked rows skipped), the
// warps' partial sums meet in shared memory. B x H/128 CTAs (144 at cfg-3, 1200 at cfg-2). A second tiny launch normalises.
__global__ void __launch_bounds__(256) pool_sum_kernel(const float* __restrict__ hidden, const int64_t* __restrict__ mask,
                                                       float* __restrict__ pooled, int L, int H) {
  __shared__ float4 part[8][32];
  __shared__ float s_cnt;
  const int b = blockIdx.y, c0 = blockIdx.x * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float cnt = 0.f;
  for (int l = warp; l < L; l += 8) {
    const float m = (float)mask[(size_t)b * L + l];
    if (m != 0.f) {
      const float4 v = *reinterpret_cast<const float4*>(hidden + ((size_t)b * L + l) * H + c0 + lane * 4);
      acc.x += v.x * m; acc.y += v.y * m; acc.z += v.z * m; acc.w += v.w * m;
    }
  }
  if (warp == 0) {                                               // token count of the sample (one warp)
    for (int l = lane; l < L; l += 32) cnt += (float)mask[(size_t)b * L + l];
    cnt = warp_sum(cnt);
    if (lane == 0) s_cnt = cnt;
  }
  part[warp][lane] = acc;
  __syncthreads();
  if (warp == 0) {
    float4 t = part[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) { const float4 u = part[w][lane]; t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w; }
    const float inv = 1.f / fmaxf(s_cnt, 1e-9f);
    t.x *= inv; t.y *= inv; t.z *= inv; t.w *= inv;
    *reinterpret_cast<float4*>(pooled + (size_t)b * H + c0 + lane * 4) = t;
  }
}
__global__ void __launch_bounds__(256) pool_finish_kernel(const float* __restrict__ pooled, float* __restrict__ emb,
                                                          float* __restrict__ norm_out, int H, int normalize) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  float sq = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) { const float v = pooled[(size_t)b * H + i]; sq += v * v; }
  const float nrm = sqrtf(block_sum(sq, red));
  if (threadIdx.x == 0) norm_out[b] = nrm;
  const float s = normalize ? 1.f / fmaxf(nrm, 1e-12f) : 1.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) emb[(size_t)b * H + i] = pooled[(size_t)b * H + i] * s;
}
// d_hidden[b,l,:] = m[b,l]/cnt * d_pooled;  d_pooled = (d_emb - emb*(emb.d_emb)) / max(norm,eps)  (if normalize)
__global__ void __launch_bounds__(256) pool_norm_bwd_kernel(const float* __restrict__ emb, const float* __restrict__ norm_in,
                                                            const float* __restrict__ d_emb, const int64_t* __restrict__ mask,
                                                            float* __restrict__ d_hidden, int L, int H, int normalize) {
  extern __shared__ float dp[];     // [H] d_pooled
  __shared__ float red[32];
  const int b = blockIdx.x;
  float cnt = 0.f;
  for (int l = 0; l < L; ++l) cnt += (float)mask[(size_t)b * L + l];
  const float inv = 1.f / fmaxf(cnt, 1e-9f);
  float dot = 0.f;
  if (normalize) {
    for (int i = threadIdx.x; i < H; i += blockDim.x) dot += emb[(size_t)b * H + i] * d_emb[(size_t)b * H + i];
    dot = block_sum(dot, red);
  }
  const float nrm = norm_in[b];
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    float d = d_emb[(size_t)b * H + i];
    if (normalize) {
      if (nrm > 1e-12f) d = (d - emb[(size_t)b * H + i] * dot) / nrm;
      else d = d / 1e-12f;
    }
    dp[i] = d * inv;
  }
  __syncthreads();
  for (int l = 0; l < L; ++l) {
    const float m = (float)mask[(size_t)b * L + l];
    for (int i = threadIdx.x; i < H; i += blockDim.x) d_hidden[((size_t)b * L + l) * H + i] = m * dp[i];
  }
}

// ------------------------------------------------------------------------------------------------------------
// fused Adam over a flat fp32 buffer (torch.optim.Adam semantics, no weight decay, no amsgrad), optional bf16 shadow copy
// ------------------------------------------------------------------------------------------------------------
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            long long n, float lr, float beta1, float beta2, float eps, float bc1, float bc2_sqrt,
                            float grad_scale) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i] * grad_scale;
  const float mi = beta1 * m[i] + (1.f - beta1) * gi;
  const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
  m[i] = mi; v[i] = vi;
  const float denom = sqrtf(vi) / bc2_sqrt + eps;
  p[i] -= (lr / bc1) * (mi / denom);
}

// dropout plumbing: the per-replay counter bump, and the keep-mask itself (for tests: lets a torch reference apply the
// identical mask)
__global__ void bump_counter_kernel(unsigned long long* c) { if (threadIdx.x == 0 && blockIdx.x == 0) c[0] += 1ull; }
__global__ void dropout_scale_kernel(float* __restrict__ out, long long n, DropCfg drop) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = drop.p > 0.f ? drop_scale1(drop, drop_stream(drop), (unsigned long long)i) : 1.f;
}

// LoRA input-dropout backward: dh[m,k] += mask(m,k)/(1-p) * sum_r G[m,r] * A[r,k]   (G bf16 [M,R], A bf16 [R,K] = A_stack)
// The un-dropped case folds this term into the dgrad GEMM (K-augmentation); with dropout the mask makes it elementwise.
// HBM-bound (dh read + written once). Each thread owns 8 fixed columns: its slice of A (R x 8) stays in registers
// (packed bf16), the CTA's rows stream through with one 16-byte load/store of dh per row.
template <int R>
__global__ void __launch_bounds__(256) lora_dx_kernel(__nv_bfloat16* __restrict__ dh, long long lddh,
                                                      const __nv_bfloat16* __restrict__ G, long long ldg,
                                                      const __nv_bfloat16* __restrict__ A, long long lda, int M, int K,
                                                      DropCfg drop) {
  constexpr int ROWS = 16;
  __shared__ __align__(16) float Gs[ROWS][R];
  const int m0 = blockIdx.y * ROWS;
  for (int i = threadIdx.x; i < ROWS * R; i += blockDim.x) {
    const int mm = i / R, r = i - mm * R;
    Gs[mm][r] = (m0 + mm < M) ? __bfloat162float(G[(size_t)(m0 + mm) * ldg + r]) : 0.f;
  }
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  bf16x8 areg[R];
  if (c < K) {
#pragma unroll
    for (int r = 0; r < R; ++r) areg[r] = *reinterpret_cast<const bf16x8*>(A + (size_t)r * lda + c);
  }
  __syncthreads();
  if (c >= K) return;
  const unsigned long long dstream = drop_stream(drop);
  const int nrows = min(ROWS, M - m0);
  // four rows per step with their loads issued together: the read-modify-write of dh otherwise serialises one 16-byte
  // load per thread per iteration
  for (int mm = 0; mm < nrows; mm += 4) {
    bf16x8 raw[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (mm + u < nrows) raw[u] = *reinterpret_cast<const bf16x8*>(dh + (size_t)(m0 + mm + u) * lddh + c);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (mm + u >= nrows) break;
      const int m = m0 + mm + u;
      float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float gv = Gs[mm + u][r];
        float av[8];
        unpack8(areg[r], av);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(gv, av[j], acc[j]);
      }
      float sc[8], cur[8];
      drop_scale8(drop, dstream, ((unsigned long long)m * K + c) >> 3, sc);
      unpack8(raw[u], cur);
#pragma unroll
      for (int j = 0; j < 8; ++j) cur[j] = fmaf(sc[j], acc[j], cur[j]);
      *reinterpret_cast<bf16x8*>(dh + (size_t)m * lddh + c) = pack8(cur);
    }
  }
}

// out_bf16[r*ldo + c] = scale * in_f32[r*si_r + c*si_c]   (LoRA factor packing into the augmented weights)
__global__ void pack_scaled_bf16_kernel(const float* __restrict__ in, long long si_r, long long si_c,
                                        __nv_bfloat16* __restrict__ out, long long ldo, int rows, int cols, float scale) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * cols) return;
  const int r = (int)(i / cols), c = (int)(i - (long long)r * cols);
  out[(size_t)r * ldo + c] = __float2bfloat16_rn(in[r * si_r + c * si_c] * scale);
}

// table-driven variant: one launch refreshes every LoRA block of a model (blockIdx.y = table entry)
struct PackEntry { const float* in; long long si_r, si_c; __nv_bfloat16* out; long long ldo; int rows, cols; float scale; };
__global__ void pack_table_kernel(const PackEntry* __restrict__ table) {
  const PackEntry e = table[blockIdx.y];
  const long long n = (long long)e.rows * e.cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / e.cols), c = (int)(i - (long long)r * e.cols);
    e.out[(size_t)r * e.ldo + c] = __float2bfloat16_rn(e.in[r * e.si_r + c * e.si_c] * e.scale);
  }
}

// out_bf16 [rows, ldo] <- fp32 [rows, cols]  (plain cast, vectorised)
__global__ void cast_f32_bf16_kernel(const float* __restrict__ in, long long ldi, __nv_bfloat16* __restrict__ out,
                                     long long ldo, int rows, int cols) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (c >= cols) return;
  for (size_t r = blockIdx.y; r < (size_t)rows; r += gridDim.y) {     // gridDim.y is capped at 65535: rows stride over it
    const float4 v = *reinterpret_cast<const float4*>(in + r * ldi + c);
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&a); pk.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(out + r * ldo + c) = pk;
  }
}

}  // namespace dalm

using namespace dalm;
#define ST(s) ((cudaStream_t)(s))

// The CTA-per-row norms stage rows in dynamic shared memory up to 48 KB. The default per-kernel limit leaves out the
// kernel's static shared memory (`red`), so each of them opts in to the full size once.
static int allow_ln_bwd_smem() {
  static bool attr = false;
  if (!attr) { DALM_CUDA(cudaFuncSetAttribute(layernorm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024)); attr = true; }
  return 0;
}

extern "C" int dalm_b200_layernorm_fwd(const float* z, const float* gamma, const float* beta, float* y32, void* y16,
                                       long long ld16, float* mean, float* rstd, int M, int H, float eps, float drop_p,
                                       unsigned long long drop_seed, unsigned long long drop_stream_id,
                                       const void* drop_offset, void* stream) {
  DALM_REQUIRE(M > 0 && H > 0 && H * 4 <= 64 * 1024, "layernorm_fwd: bad shape M=%d H=%d", M, H);
  DALM_REQUIRE(drop_p >= 0.f && drop_p < 1.f, "layernorm_fwd: dropout p must be in [0,1)");
  if (y16 != nullptr && ln_warp_ok(H, ld16, z, y32, y16, 0)) {
    const DropCfg d = make_drop(drop_p, drop_seed, drop_stream_id, drop_offset);
    auto* y = (__nv_bfloat16*)y16;
    switch (H / 256) {
      case 1: return launch_ln_fwd_warp<1>(z, gamma, beta, y32, y, ld16, mean, rstd, M, eps, d, ST(stream));
      case 2: return launch_ln_fwd_warp<2>(z, gamma, beta, y32, y, ld16, mean, rstd, M, eps, d, ST(stream));
      case 4: return launch_ln_fwd_warp<4>(z, gamma, beta, y32, y, ld16, mean, rstd, M, eps, d, ST(stream));
      default: return launch_ln_fwd_warp<8>(z, gamma, beta, y32, y, ld16, mean, rstd, M, eps, d, ST(stream));
    }
  }
  // the row is staged in H * 4 bytes of dynamic shared memory: above 48 KB (less the static `red`) only with the opt-in
  static bool attr = false;
  if (!attr) { DALM_CUDA(cudaFuncSetAttribute(layernorm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); attr = true; }
  layernorm_fwd_kernel<<<M, 256, H * sizeof(float), ST(stream)>>>(z, gamma, beta, y32, (__nv_bfloat16*)y16, ld16, mean, rstd, H, eps,
                                                                  make_drop(drop_p, drop_seed, drop_stream_id, drop_offset));
  count_launch();
  return check_launch("layernorm_fwd_kernel");
}
extern "C" int dalm_b200_layernorm_bwd(const float* z, const float* gamma, const float* mean, const float* rstd,
                                       const float* dy_f32, const void* dy_bf16, long long ldb, float* dz32, void* dz16,
                                       long long ld16, int M, int H, float drop_p, unsigned long long drop_seed,
                                       unsigned long long drop_stream_id, const void* drop_offset, void* stream) {
  DALM_REQUIRE(M > 0 && H > 0 && H * 8 <= 48 * 1024, "layernorm_bwd: bad shape M=%d H=%d", M, H);
  DALM_REQUIRE(dy_f32 || dy_bf16, "layernorm_bwd: no incoming gradient");
  if (ln_warp_ok(H, dz16 ? ld16 : 0, z, dy_f32, dz32, dy_bf16 ? ldb : 0) && ((uintptr_t)dy_bf16 & 15) == 0 && ((uintptr_t)dz16 & 15) == 0) {
    const DropCfg d = make_drop(drop_p, drop_seed, drop_stream_id, drop_offset);
    auto* b = (const __nv_bfloat16*)dy_bf16; auto* o = (__nv_bfloat16*)dz16;
    switch (H / 256) {
      case 1: return launch_ln_bwd_warp<1>(z, gamma, mean, rstd, dy_f32, b, ldb, dz32, o, ld16, M, d, nullptr, ST(stream));
      case 2: return launch_ln_bwd_warp<2>(z, gamma, mean, rstd, dy_f32, b, ldb, dz32, o, ld16, M, d, nullptr, ST(stream));
      case 4: return launch_ln_bwd_warp<4>(z, gamma, mean, rstd, dy_f32, b, ldb, dz32, o, ld16, M, d, nullptr, ST(stream));
      default: return launch_ln_bwd_warp<8>(z, gamma, mean, rstd, dy_f32, b, ldb, dz32, o, ld16, M, d, nullptr, ST(stream));
    }
  }
  if (int e = allow_ln_bwd_smem()) return e;
  layernorm_bwd_kernel<<<M, 256, 2 * H * sizeof(float), ST(stream)>>>(z, gamma, mean, rstd, dy_f32, (const __nv_bfloat16*)dy_bf16, ldb,
                                                                     dz32, (__nv_bfloat16*)dz16, ld16, H,
                                                                     make_drop(drop_p, drop_seed, drop_stream_id, drop_offset), nullptr);
  count_launch();
  return check_launch("layernorm_bwd_kernel");
}
// pre-LN variant: dz = LayerNorm-backward(dy) + dres  (dres fp32 [M,H], may alias dz32)
extern "C" int dalm_b200_layernorm_bwd_res(const float* z, const float* gamma, const float* mean, const float* rstd,
                                           const float* dy_f32, const void* dy_bf16, long long ldb, const float* dres,
                                           float* dz32, void* dz16, long long ld16, int M, int H, void* stream) {
  DALM_REQUIRE(M > 0 && H > 0 && H * 8 <= 48 * 1024, "layernorm_bwd_res: bad shape M=%d H=%d", M, H);
  DALM_REQUIRE(dy_f32 || dy_bf16, "layernorm_bwd_res: no incoming gradient");
  if (ln_warp_ok(H, dz16 ? ld16 : 0, z, dy_f32, dz32, dy_bf16 ? ldb : 0) && ((uintptr_t)dy_bf16 & 15) == 0 && ((uintptr_t)dz16 & 15) == 0 &&
      ((uintptr_t)dres & 15) == 0) {
    const DropCfg d = make_drop(0.f, 0, 0, nullptr);
    auto* b = (const __nv_bfloat16*)dy_bf16; auto* o = (__nv_bfloat16*)dz16;
    switch (H / 256) {
      case 1: return launch_ln_bwd_warp<1>(z, gamma, mean, rstd, dy_f32, b, ldb, dz32, o, ld16, M, d, dres, ST(stream));
      case 2: return launch_ln_bwd_warp<2>(z, gamma, mean, rstd, dy_f32, b, ldb, dz32, o, ld16, M, d, dres, ST(stream));
      case 4: return launch_ln_bwd_warp<4>(z, gamma, mean, rstd, dy_f32, b, ldb, dz32, o, ld16, M, d, dres, ST(stream));
      default: return launch_ln_bwd_warp<8>(z, gamma, mean, rstd, dy_f32, b, ldb, dz32, o, ld16, M, d, dres, ST(stream));
    }
  }
  if (int e = allow_ln_bwd_smem()) return e;
  layernorm_bwd_kernel<<<M, 256, 2 * H * sizeof(float), ST(stream)>>>(z, gamma, mean, rstd, dy_f32, (const __nv_bfloat16*)dy_bf16, ldb,
                                                                     dz32, (__nv_bfloat16*)dz16, ld16, H, make_drop(0.f, 0, 0, nullptr), dres);
  count_launch();
  return check_launch("layernorm_bwd_kernel");
}
extern "C" int dalm_b200_rmsnorm_fwd(const float* x, const float* g, void* h, long long ldh, float* rstd, int M, int H,
                                     float eps, void* stream) {
  DALM_REQUIRE(M > 0 && H > 0 && (H % 4) == 0 && H * 4 <= 48 * 1024 && (ldh % 4) == 0, "rmsnorm_fwd: bad shape M=%d H=%d", M, H);
  DALM_REQUIRE(aligned(x, 16) && aligned(g, 16) && aligned(h, 8), "rmsnorm_fwd: x / g must be 16-byte and h 8-byte aligned");
  static bool attr = false;
  if (!attr) { DALM_CUDA(cudaFuncSetAttribute(rmsnorm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024)); attr = true; }
  rmsnorm_fwd_kernel<<<M, 256, H * sizeof(float), ST(stream)>>>(x, g, (__nv_bfloat16*)h, ldh, rstd, H, eps);
  count_launch();
  return check_launch("rmsnorm_fwd_kernel");
}
extern "C" int dalm_b200_rmsnorm_bwd(const float* x, const float* g, const float* rstd, const void* dh, long long lddh,
                                     const float* dres_in, float* dres_out, void* dres16, long long ld16, int M, int H,
                                     void* stream) {
  DALM_REQUIRE(M > 0 && H > 0 && (H % 4) == 0 && H * 8 <= 96 * 1024 && (lddh % 4) == 0 && (ld16 % 4) == 0,
               "rmsnorm_bwd: bad shape M=%d H=%d", M, H);
  DALM_REQUIRE(aligned(x, 16) && aligned(g, 16) && aligned(dres_in, 16) && aligned(dres_out, 16) && aligned(dh, 8) && aligned(dres16, 8),
               "rmsnorm_bwd: fp32 operands must be 16-byte and bf16 ones 8-byte aligned");
  static bool attr = false;
  if (!attr) { DALM_CUDA(cudaFuncSetAttribute(rmsnorm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024)); attr = true; }
  rmsnorm_bwd_kernel<<<M, 256, 2 * H * sizeof(float), ST(stream)>>>(x, g, rstd, (const __nv_bfloat16*)dh, lddh, dres_in, dres_out,
                                                                   (__nv_bfloat16*)dres16, ld16, H);
  count_launch();
  return check_launch("rmsnorm_bwd_kernel");
}
extern "C" int dalm_b200_postnorm_fwd(const void* y, long long ldy, const float* w, const float* resid, float* out, void* out16,
                                      long long ld16, float* rstd, int M, int H, float eps, void* stream) {
  DALM_REQUIRE(M > 0 && H > 0 && (H % 8) == 0 && H <= 8 * kPostNormUnits * 256, "postnorm_fwd: bad shape M=%d H=%d (H %% 8 == 0, <= %d)",
               M, H, 8 * kPostNormUnits * 256);
  DALM_REQUIRE(y && w && resid && out && rstd && (ldy % 8) == 0 && (out16 == nullptr || (ld16 % 8) == 0), "postnorm_fwd: operands / strides");
  DALM_REQUIRE(aligned(y, 16) && aligned(w, 16) && aligned(resid, 16) && aligned(out, 16) && aligned(out16, 16),
               "postnorm_fwd: operands must be 16-byte aligned");
  postnorm_fwd_kernel<<<M, 256, 0, ST(stream)>>>((const __nv_bfloat16*)y, ldy, w, resid, out, (__nv_bfloat16*)out16, ld16, rstd, H, eps);
  count_launch();
  return check_launch("postnorm_fwd_kernel");
}
extern "C" int dalm_b200_postnorm_bwd(const void* y, long long ldy, const float* w, const float* rstd, const float* dres_in,
                                      const void* dh, long long lddh, float* dres_out, void* dy, long long lddy, int M, int H,
                                      void* stream) {
  DALM_REQUIRE(M > 0 && H > 0 && (H % 8) == 0 && H <= 8 * kPostNormUnits * 256, "postnorm_bwd: bad shape M=%d H=%d", M, H);
  DALM_REQUIRE(y && w && rstd && dres_in && dres_out && dy && (ldy % 8) == 0 && (lddy % 8) == 0 && (dh == nullptr || (lddh % 8) == 0),
               "postnorm_bwd: operands / strides");
  DALM_REQUIRE(aligned(y, 16) && aligned(w, 16) && aligned(dres_in, 16) && aligned(dres_out, 16) && aligned(dh, 16) && aligned(dy, 16),
               "postnorm_bwd: operands must be 16-byte aligned");
  postnorm_bwd_kernel<<<M, 256, 0, ST(stream)>>>((const __nv_bfloat16*)y, ldy, w, rstd, dres_in, (const __nv_bfloat16*)dh, lddh, dres_out,
                                                 (__nv_bfloat16*)dy, lddy, H);
  count_launch();
  return check_launch("postnorm_bwd_kernel");
}
extern "C" int dalm_b200_bert_embed(const int64_t* ids, const void* word, const void* pos, const void* type0, float* z,
                                    int M, int L, int H, int V, void* stream) {
  bert_embed_kernel<<<M, 256, 0, ST(stream)>>>(ids, (const __nv_bfloat16*)word, (const __nv_bfloat16*)pos,
                                               (const __nv_bfloat16*)type0, z, L, H, V);
  count_launch();
  return check_launch("bert_embed_kernel");
}
extern "C" int dalm_b200_roberta_embed(const int64_t* ids, const void* word, const void* pos, const void* type0, int pad_id,
                                       float* z, int64_t* pos_ids_out, int B, int L, int H, int V, int P, void* stream) {
  DALM_REQUIRE(B > 0 && B <= 65535 && L > 0 && V > 0 && P > 0 && H > 0 && (H % 4) == 0 && pad_id >= 0,
               "roberta_embed: bad shape B=%d L=%d H=%d V=%d P=%d pad_id=%d (B at most 65535: a grid extent)", B, L, H, V, P, pad_id);
  DALM_REQUIRE(aligned(word, 8) && aligned(pos, 8) && aligned(type0, 8) && aligned(z, 16),
               "roberta_embed: tables must be 8-byte and z 16-byte aligned");
  roberta_embed_kernel<<<dim3((L + kReChunk - 1) / kReChunk, B), 256, 0, ST(stream)>>>(
      ids, (const __nv_bfloat16*)word, (const __nv_bfloat16*)pos, (const __nv_bfloat16*)type0, pad_id, z, pos_ids_out, L, H, V, P);
  count_launch();
  return check_launch("roberta_embed_kernel");
}
extern "C" int dalm_b200_embed_gather(const int64_t* ids, const void* table, float* x, int M, int H, int V, void* stream) {
  embed_gather_kernel<<<M, 256, 0, ST(stream)>>>(ids, (const __nv_bfloat16*)table, x, H, V);
  count_launch();
  return check_launch("embed_gather_kernel");
}
extern "C" int dalm_b200_rope(void* buf, long long ld, int col0, int nheads, int D, const float* cos_t, const float* sin_t,
                              int M, int L, int backward, void* stream) {
  DALM_REQUIRE((D % 16) == 0 && (ld % 8) == 0 && (col0 % 8) == 0, "rope: head_dim must be a multiple of 16 and rows 16-byte aligned");
  rope_kernel<<<M, 256, 0, ST(stream)>>>((__nv_bfloat16*)buf, ld, col0, nheads, D, cos_t, sin_t, L, backward ? -1.f : 1.f);
  count_launch();
  return check_launch("rope_kernel");
}
// rows go to grid.y, which holds at most 65535: longer batches (bs 8 x 8192 tokens) are launched in chunks of rows, each
// chunk a view that starts at its first row (a batch of <= 65535 rows stays one launch)
constexpr int GLU_ROWS = 65535;
template <class Act>
static int launch_glu_fwd(const void* gu, long long ldgu, void* act, long long lda, int M, int F, int il, const char* name,
                          cudaStream_t st) {
  for (long long r0 = 0; r0 < M; r0 += GLU_ROWS) {
    dim3 grid((F / 8 + 255) / 256, (unsigned)min((long long)GLU_ROWS, M - r0));
    glu_fwd_kernel<Act><<<grid, 256, 0, st>>>((const __nv_bfloat16*)gu + r0 * ldgu, ldgu, (__nv_bfloat16*)act + r0 * lda, lda, F, il);
    count_launch();
    if (int e = check_launch(name)) return e;
  }
  return 0;
}
template <class Act>
static int launch_glu_bwd(void* gu, long long ldgu, const void* dact, long long ldd, int M, int F, int il, const char* name,
                          cudaStream_t st) {
  for (long long r0 = 0; r0 < M; r0 += GLU_ROWS) {
    dim3 grid((F / 8 + 255) / 256, (unsigned)min((long long)GLU_ROWS, M - r0));
    glu_bwd_kernel<Act><<<grid, 256, 0, st>>>((__nv_bfloat16*)gu + r0 * ldgu, ldgu, (const __nv_bfloat16*)dact + r0 * ldd, ldd, F, il);
    count_launch();
    if (int e = check_launch(name)) return e;
  }
  return 0;
}
extern "C" int dalm_b200_swiglu_fwd(const void* gu, long long ldgu, void* act, long long lda, int M, int F, int interleave, void* stream) {
  DALM_REQUIRE((F % 8) == 0 && (ldgu % 8) == 0 && (lda % 8) == 0, "swiglu: F and strides must be multiples of 8");
  DALM_REQUIRE(interleave == 0 || ((interleave % 8) == 0 && (F % interleave) == 0), "swiglu: interleave block must divide F and be a multiple of 8");
  return launch_glu_fwd<SiluAct>(gu, ldgu, act, lda, M, F, interleave, "swiglu_fwd_kernel", ST(stream));
}
extern "C" int dalm_b200_swiglu_bwd(void* gu, long long ldgu, const void* dact, long long ldd, int M, int F, int interleave, void* stream) {
  DALM_REQUIRE((F % 8) == 0 && (ldgu % 8) == 0 && (ldd % 8) == 0, "swiglu: F and strides must be multiples of 8");
  DALM_REQUIRE(interleave == 0 || ((interleave % 8) == 0 && (F % interleave) == 0), "swiglu: interleave block must divide F and be a multiple of 8");
  return launch_glu_bwd<SiluAct>(gu, ldgu, dact, ldd, M, F, interleave, "swiglu_bwd_kernel", ST(stream));
}
extern "C" int dalm_b200_geglu_fwd(const void* x, long long ldx, void* act, long long lda, int M, int F, void* stream) {
  DALM_REQUIRE((F % 8) == 0 && (ldx % 8) == 0 && (lda % 8) == 0, "geglu: F and strides must be multiples of 8");
  return launch_glu_fwd<GeluAct>(x, ldx, act, lda, M, F, 0, "geglu_fwd_kernel", ST(stream));
}
extern "C" int dalm_b200_geglu_bwd(void* x, long long ldx, const void* dact, long long ldd, int M, int F, void* stream) {
  DALM_REQUIRE((F % 8) == 0 && (ldx % 8) == 0 && (ldd % 8) == 0, "geglu: F and strides must be multiples of 8");
  return launch_glu_bwd<GeluAct>(x, ldx, dact, ldd, M, F, 0, "geglu_bwd_kernel", ST(stream));
}
// a CTA row of the GELU grid covers GELU_ROWS rows and grid.y holds at most 65535: longer batches go in chunks of
// GELU_CHUNK rows (a whole number of CTA rows, so every chunk but the last is full and a batch of <= GELU_CHUNK rows is one launch)
constexpr long long GELU_CHUNK = 65535LL * GELU_ROWS;
extern "C" int dalm_b200_gelu_fwd(const void* pre, long long ldp, void* act, long long lda, int M, int F, void* stream) {
  DALM_REQUIRE((F % 8) == 0 && (ldp % 8) == 0 && (lda % 8) == 0, "gelu: F and strides must be multiples of 8");
  for (long long r0 = 0; r0 < M; r0 += GELU_CHUNK) {
    const int m = (int)min(GELU_CHUNK, M - r0);
    dim3 grid((F / 8 + 255) / 256, (m + GELU_ROWS - 1) / GELU_ROWS);
    gelu_fwd_kernel<<<grid, 256, 0, ST(stream)>>>((const __nv_bfloat16*)pre + r0 * ldp, ldp, (__nv_bfloat16*)act + r0 * lda, lda, m, F);
    count_launch();
    if (int e = check_launch("gelu_fwd_kernel")) return e;
  }
  return 0;
}
extern "C" int dalm_b200_gelu_bwd(const void* pre, long long ldp, void* dact, long long ldd, int M, int F, void* stream) {
  DALM_REQUIRE((F % 8) == 0 && (ldp % 8) == 0 && (ldd % 8) == 0, "gelu: F and strides must be multiples of 8");
  for (long long r0 = 0; r0 < M; r0 += GELU_CHUNK) {
    const int m = (int)min(GELU_CHUNK, M - r0);
    dim3 grid((F / 8 + 255) / 256, (m + GELU_ROWS - 1) / GELU_ROWS);
    gelu_bwd_kernel<<<grid, 256, 0, ST(stream)>>>((const __nv_bfloat16*)pre + r0 * ldp, ldp, (__nv_bfloat16*)dact + r0 * ldd, ldd, m, F);
    count_launch();
    if (int e = check_launch("gelu_bwd_kernel")) return e;
  }
  return 0;
}
extern "C" int dalm_b200_pool_norm_fwd(const float* hidden, const int64_t* mask, float* pooled, float* emb, float* norm,
                                       int B, int L, int H, int normalize, void* stream) {
  DALM_REQUIRE(B > 0 && B <= 65535 && L > 0 && H > 0, "pool_norm_fwd: bad shape B=%d L=%d H=%d (at most 65535 samples: B is a grid "
               "extent)", B, L, H);
  if ((H % 128) == 0 && (reinterpret_cast<uintptr_t>(hidden) & 15) == 0) {
    pool_sum_kernel<<<dim3(H / 128, B), 256, 0, ST(stream)>>>(hidden, mask, pooled, L, H);
    if (int e = check_launch("pool_sum_kernel")) return e;
    pool_finish_kernel<<<B, 256, 0, ST(stream)>>>(pooled, emb, norm, H, normalize);
    count_launch(2);
    return check_launch("pool_finish_kernel");
  }
  pool_norm_fwd_kernel<<<B, 256, 0, ST(stream)>>>(hidden, mask, pooled, emb, norm, L, H, normalize);
  count_launch();
  return check_launch("pool_norm_fwd_kernel");
}
extern "C" int dalm_b200_pool_norm_bwd(const float* emb, const float* norm, const float* d_emb, const int64_t* mask,
                                       float* d_hidden, int B, int L, int H, int normalize, void* stream) {
  DALM_REQUIRE(H * 4 <= 48 * 1024, "pool_norm_bwd: H too large");
  // d_pooled takes H * 4 bytes of dynamic shared memory next to the kernel's static `red`: at H = 12288 the sum passes the
  // 48 KB a launch gets without opting in
  static bool attr_set = false;
  if (!attr_set) {
    DALM_CUDA(cudaFuncSetAttribute(pool_norm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024));
    attr_set = true;
  }
  pool_norm_bwd_kernel<<<B, 256, H * sizeof(float), ST(stream)>>>(emb, norm, d_emb, mask, d_hidden, L, H, normalize);
  count_launch();
  return check_launch("pool_norm_bwd_kernel");
}
extern "C" int dalm_b200_adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1,
                                   float beta2, float eps, int step, float grad_scale, void* stream) {
  DALM_REQUIRE(n >= 0 && step >= 1, "adam: bad n/step");
  if (n == 0) return 0;
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2s = sqrtf(1.f - powf(beta2, (float)step));
  adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(p, g, m, v, n, lr, beta1, beta2, eps, bc1, bc2s, grad_scale);
  count_launch();
  return check_launch("adam_kernel");
}
extern "C" int dalm_b200_pack_scaled_bf16(const float* in, long long si_r, long long si_c, void* out, long long ldo,
                                          int rows, int cols, float scale, void* stream) {
  const long long n = (long long)rows * cols;
  if (n == 0) return 0;
  pack_scaled_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(in, si_r, si_c, (__nv_bfloat16*)out, ldo, rows, cols, scale);
  count_launch();
  return check_launch("pack_scaled_bf16_kernel");
}
extern "C" int dalm_b200_bump_counter(void* counter, void* stream) {
  bump_counter_kernel<<<1, 32, 0, ST(stream)>>>((unsigned long long*)counter);
  count_launch();
  return check_launch("bump_counter_kernel");
}
// out[i] = 0 or 1/(1-p): the scale dropout applies to element i of a tensor under (seed, stream, *offset)
extern "C" int dalm_b200_dropout_scale(float* out, long long n, float p, unsigned long long seed, unsigned long long stream_id,
                                       const void* offset, void* stream) {
  DALM_REQUIRE(p >= 0.f && p < 1.f, "dropout_scale: p must be in [0,1)");
  if (n <= 0) return 0;
  dropout_scale_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ST(stream)>>>(out, n, make_drop(p, seed, stream_id, offset));
  count_launch();
  return check_launch("dropout_scale_kernel");
}
extern "C" int dalm_b200_lora_dx(void* dh, long long lddh, const void* G, long long ldg, const void* A, long long lda, int M,
                                 int K, int R, float p, unsigned long long seed, unsigned long long stream_id,
                                 const void* offset, void* stream) {
  DALM_REQUIRE((R == 8 || R == 16 || R == 24) && (K % 8) == 0 && (lddh % 8) == 0 && (lda % 8) == 0, "lora_dx: bad shape R=%d K=%d", R, K);
  DALM_REQUIRE(p >= 0.f && p < 1.f, "lora_dx: p must be in [0,1)");
  DALM_REQUIRE(M >= 0 && M <= 65535 * 16, "lora_dx: M=%d rows past the grid's 65535 blocks of 16", M);
  // one thread per 8 columns: a CTA no wider than the row (bge-large, K = 1024: 128 threads - a 256-thread CTA keeps half of its
  // warps resident but idle)
  const int cols8 = K / 8;
  const int threads = cols8 >= 256 ? 256 : ((cols8 + 31) / 32) * 32;
  dim3 grid((cols8 + threads - 1) / threads, (M + 15) / 16);
  const DropCfg dc = make_drop(p, seed, stream_id, offset);
  auto* dhp = (__nv_bfloat16*)dh; auto* gp = (const __nv_bfloat16*)G; auto* ap = (const __nv_bfloat16*)A;
  if (R == 8)       lora_dx_kernel<8><<<grid, threads, 0, ST(stream)>>>(dhp, lddh, gp, ldg, ap, lda, M, K, dc);
  else if (R == 16) lora_dx_kernel<16><<<grid, threads, 0, ST(stream)>>>(dhp, lddh, gp, ldg, ap, lda, M, K, dc);
  else              lora_dx_kernel<24><<<grid, threads, 0, ST(stream)>>>(dhp, lddh, gp, ldg, ap, lda, M, K, dc);
  count_launch();
  return check_launch("lora_dx_kernel");
}
// table: device array of n_entries records {const float* in; int64 si_r, si_c; bf16* out; int64 ldo; int32 rows, cols; float scale}
// (48 bytes each, natural alignment) — see dalm_b200/engine/lora.py:pack_table
extern "C" int dalm_b200_pack_table(const void* table, int n_entries, void* stream) {
  static_assert(sizeof(PackEntry) == 56, "PackEntry layout");
  if (n_entries <= 0) return 0;
  dim3 grid(32, n_entries);
  pack_table_kernel<<<grid, 256, 0, ST(stream)>>>((const PackEntry*)table);
  count_launch();
  return check_launch("pack_table_kernel");
}
extern "C" int dalm_b200_cast_f32_bf16(const float* in, long long ldi, void* out, long long ldo, int rows, int cols, void* stream) {
  DALM_REQUIRE((cols % 4) == 0 && (ldi % 4) == 0 && (ldo % 4) == 0, "cast: cols/strides must be multiples of 4");
  DALM_REQUIRE(aligned(in, 16) && aligned(out, 8), "cast: in must be 16-byte and out 8-byte aligned");
  if (rows <= 0 || cols <= 0) return 0;
  dim3 grid((cols / 4 + 255) / 256, rows < 65535 ? rows : 65535);
  cast_f32_bf16_kernel<<<grid, 256, 0, ST(stream)>>>(in, ldi, (__nv_bfloat16*)out, ldo, rows, cols);
  count_launch();
  return check_launch("cast_f32_bf16_kernel");
}
