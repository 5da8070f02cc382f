// dalm_b200 — Qwen3's per-head q/k RMSNorm with the rotary embedding, for the paths the QKV GEMM epilogue does not serve, and
// its backward (transformers models/qwen3/modeling_qwen3.py, Qwen3Attention.forward):
//
//     q = rotate_half_rope(q_norm(q_proj(h).view(..., nh, 128)))     k likewise with k_norm; v untouched
//     RMSNorm(x) = x * rsqrt(mean(x^2) + eps) * w                     w: [128], one per projection, shared by its heads
//
//   qk_norm_rope_kernel     : in place on the q|k heads of a token-major bf16 buffer (decode step, the prefill of `generate` with
//                             explicit positions, and training shapes whose q|k width is not a whole number of 256-wide tiles);
//                             optionally emits the pre-norm values and the rstd the backward needs
//   qk_norm_rope_bwd_kernel : in place on d(q|k): un-rotate, then the RMSNorm backward from the saved pre-norm values and rstd;
//                             optionally accumulates d(q_norm.weight) / d(k_norm.weight)
//
// One warp per (row, head): lane l owns the rotate_half pairs (2l, 64+2l) and (2l+1, 64+2l+1), so the rotation is lane-local
// and the head's sums are one butterfly reduction. No allocation and no host synchronisation: safe inside a captured graph.
#include "common.cuh"

namespace dalm {

constexpr int kNormRopeWarps = 8;

__device__ __forceinline__ void ld_pair(const __nv_bfloat16* p, float& a, float& b) {
  const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
  a = t.x; b = t.y;
}
__device__ __forceinline__ void st_pair(__nv_bfloat16* p, float a, float b) {
  *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(a, b);
}

// x[0..1] = columns 2l, 2l+1 (first half), x[2..3] = columns 64+2l, 64+2l+1 (second half)
__global__ void __launch_bounds__(kNormRopeWarps * 32)
qk_norm_rope_kernel(__nv_bfloat16* __restrict__ buf, long long ld, int nheads, int nq_heads, const float* __restrict__ q_norm,
                    const float* __restrict__ k_norm, float eps, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                    int T, int L, const int64_t* __restrict__ pos, int M, __nv_bfloat16* __restrict__ pre, long long ld_pre,
                    float* __restrict__ rstd_out, long long ld_rstd) {
  const int lane = threadIdx.x & 31;
  const long long items = (long long)M * nheads;
  const long long item = (long long)blockIdx.x * kNormRopeWarps + (threadIdx.x >> 5);
  if (item >= items) return;
  const int r = (int)(item / nheads), hd = (int)(item - (long long)r * nheads);
  int p;
  if (pos != nullptr) {
    const long long t = pos[r];
    p = (int)(t < 0 ? 0 : (t >= T ? T - 1 : t));
  } else {
    p = r % L;
  }
  __nv_bfloat16* x = buf + (size_t)r * ld + hd * 128;
  const int j = 2 * lane;
  float v[4];
  ld_pair(x + j, v[0], v[1]);
  ld_pair(x + 64 + j, v[2], v[3]);
  if (pre != nullptr) {
    __nv_bfloat16* q = pre + (size_t)r * ld_pre + hd * 128;
    st_pair(q + j, v[0], v[1]);
    st_pair(q + 64 + j, v[2], v[3]);
  }
  const float ss = warp_sum(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
  const float rstd = rsqrtf(ss * (1.f / 128.f) + eps);
  if (rstd_out != nullptr && lane == 0) rstd_out[(size_t)r * ld_rstd + hd] = rstd;
  const float* w = hd < nq_heads ? q_norm : k_norm;
  const float2 w1 = *reinterpret_cast<const float2*>(w + j), w2 = *reinterpret_cast<const float2*>(w + 64 + j);
  const float n0 = v[0] * rstd * w1.x, n1 = v[1] * rstd * w1.y, n2 = v[2] * rstd * w2.x, n3 = v[3] * rstd * w2.y;
  const float2 c = *reinterpret_cast<const float2*>(cos_t + (size_t)p * 64 + j);
  const float2 s = *reinterpret_cast<const float2*>(sin_t + (size_t)p * 64 + j);
  st_pair(x + j, fmaf(n0, c.x, -n2 * s.x), fmaf(n1, c.y, -n3 * s.y));
  st_pair(x + 64 + j, fmaf(n2, c.x, n0 * s.x), fmaf(n3, c.y, n1 * s.y));
}

// d(q|k) in place: g = un-rotated gradient of the normalised head y = x_hat * w (x_hat = pre * rstd);
//   dx = rstd * (w g - x_hat * mean(w g x_hat)),   d w += g x_hat   (summed over rows and over the heads that share w)
// A persistent grid: each warp walks (row, head) items, keeps its weight-gradient partials in registers, and the block adds
// them with one atomic per column at the end.
__global__ void __launch_bounds__(kNormRopeWarps * 32)
qk_norm_rope_bwd_kernel(__nv_bfloat16* __restrict__ dbuf, long long ld, int nheads, int nq_heads, const float* __restrict__ q_norm,
                        const float* __restrict__ k_norm, const float* __restrict__ cos_t, const float* __restrict__ sin_t, int L,
                        const __nv_bfloat16* __restrict__ pre, long long ld_pre, const float* __restrict__ rstd_in, long long ld_rstd,
                        int M, float* __restrict__ dw_q, float* __restrict__ dw_k) {
  __shared__ float red[kNormRopeWarps][2][128];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = 2 * lane;
  const bool want_dw = dw_q != nullptr;
  float dq[4] = {0.f, 0.f, 0.f, 0.f}, dk[4] = {0.f, 0.f, 0.f, 0.f};
  const long long items = (long long)M * nheads;
  for (long long item = (long long)blockIdx.x * kNormRopeWarps + warp; item < items; item += (long long)gridDim.x * kNormRopeWarps) {
    const int r = (int)(item / nheads), hd = (int)(item - (long long)r * nheads);
    const int p = r % L;
    __nv_bfloat16* d = dbuf + (size_t)r * ld + hd * 128;
    float dy[4], x[4];
    ld_pair(d + j, dy[0], dy[1]);
    ld_pair(d + 64 + j, dy[2], dy[3]);
    const __nv_bfloat16* xp = pre + (size_t)r * ld_pre + hd * 128;
    ld_pair(xp + j, x[0], x[1]);
    ld_pair(xp + 64 + j, x[2], x[3]);
    const float rstd = rstd_in[(size_t)r * ld_rstd + hd];
    const float2 c = *reinterpret_cast<const float2*>(cos_t + (size_t)p * 64 + j);
    const float2 s = *reinterpret_cast<const float2*>(sin_t + (size_t)p * 64 + j);
    // inverse rotation (the transpose of the forward map)
    float g[4];
    g[0] = fmaf(dy[0], c.x, dy[2] * s.x); g[1] = fmaf(dy[1], c.y, dy[3] * s.y);
    g[2] = fmaf(dy[2], c.x, -dy[0] * s.x); g[3] = fmaf(dy[3], c.y, -dy[1] * s.y);
    const float* wp = hd < nq_heads ? q_norm : k_norm;
    const float2 w1 = *reinterpret_cast<const float2*>(wp + j), w2 = *reinterpret_cast<const float2*>(wp + 64 + j);
    const float w[4] = {w1.x, w1.y, w2.x, w2.y};
    float xh[4], wg[4], dot = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      xh[i] = x[i] * rstd;
      wg[i] = w[i] * g[i];
      dot = fmaf(wg[i], xh[i], dot);
    }
    const float m = warp_sum(dot) * (1.f / 128.f);
    st_pair(d + j, rstd * fmaf(-xh[0], m, wg[0]), rstd * fmaf(-xh[1], m, wg[1]));
    st_pair(d + 64 + j, rstd * fmaf(-xh[2], m, wg[2]), rstd * fmaf(-xh[3], m, wg[3]));
    if (want_dw) {
      float* acc = hd < nq_heads ? dq : dk;
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = fmaf(g[i], xh[i], acc[i]);
    }
  }
  if (!want_dw) return;
  red[warp][0][j] = dq[0]; red[warp][0][j + 1] = dq[1]; red[warp][0][64 + j] = dq[2]; red[warp][0][64 + j + 1] = dq[3];
  red[warp][1][j] = dk[0]; red[warp][1][j + 1] = dk[1]; red[warp][1][64 + j] = dk[2]; red[warp][1][64 + j + 1] = dk[3];
  __syncthreads();
  const int t = threadIdx.x;                                    // 256 threads = 2 x 128 weight columns
  float sum = 0.f;
#pragma unroll
  for (int w = 0; w < kNormRopeWarps; ++w) sum += red[w][t >> 7][t & 127];
  atomicAdd((t >> 7) ? dw_k + (t & 127) : dw_q + (t & 127), sum);
}

// ---- OLMo 2 / OLMo 3 / OLMoE: q/k RMSNorm over the whole projection width (transformers Olmo2Attention / OlmoeAttention) ----
//
//     q = rotate_half_rope(q_norm(q_proj(h)))     q_norm: RMSNorm over all Nq = nq_heads * hd columns, weight [Nq]
//     k = rotate_half_rope(k_norm(k_proj(h)))     k_norm: over all Nkv columns, weight [Nkv]
//
// One CTA per row. A "unit" is four consecutive columns of a head's first half and the four columns hd/2 further on, so the
// rotation stays thread-local; a row's units live in registers between the sum-of-squares pass and the normalising pass.
// Rounding of the normalised value follows transformers: Olmo2RMSNorm returns bf16(w * (x rstd)) (round_first = 0),
// OlmoeRMSNorm w * bf16(x rstd) rounded again (round_first = 1); RoPE then runs in fp32 on that bf16 value.
constexpr int kFullNormThreads = 256, kFullNormUnits = 5;        // up to 5 * 8 * 256 = 10 240 q|k columns (OLMo-2-13B)

struct Unit8 { float v[8]; };

__device__ __forceinline__ void ld_unit(const __nv_bfloat16* p, int half, Unit8& u) {
  const uint2 a = *reinterpret_cast<const uint2*>(p), b = *reinterpret_cast<const uint2*>(p + half);
  const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&a.x));
  const float2 a1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&a.y));
  const float2 b0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&b.x));
  const float2 b1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&b.y));
  u.v[0] = a0.x; u.v[1] = a0.y; u.v[2] = a1.x; u.v[3] = a1.y; u.v[4] = b0.x; u.v[5] = b0.y; u.v[6] = b1.x; u.v[7] = b1.y;
}
__device__ __forceinline__ void st_unit(__nv_bfloat16* p, int half, const float* v) {
  __nv_bfloat162 t[4] = {__floats2bfloat162_rn(v[0], v[1]), __floats2bfloat162_rn(v[2], v[3]),
                         __floats2bfloat162_rn(v[4], v[5]), __floats2bfloat162_rn(v[6], v[7])};
  uint2 a, b;
  a.x = *reinterpret_cast<uint32_t*>(&t[0]); a.y = *reinterpret_cast<uint32_t*>(&t[1]);
  b.x = *reinterpret_cast<uint32_t*>(&t[2]); b.y = *reinterpret_cast<uint32_t*>(&t[3]);
  *reinterpret_cast<uint2*>(p) = a;
  *reinterpret_cast<uint2*>(p + half) = b;
}
// unit i of a row -> its first column and its frequency index j (columns c .. c+3 and c+half .. c+half+3)
__device__ __forceinline__ int unit_col(int i, int hd, int& j) {
  const int per_head = hd >> 3, h = i / per_head;
  j = (i - h * per_head) * 4;
  return h * hd + j;
}
__device__ __forceinline__ float2 block_sum2(float a, float b, float (*red)[32]) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  a = warp_sum(a); b = warp_sum(b);
  if (lane == 0) { red[0][w] = a; red[1][w] = b; }
  __syncthreads();
  a = lane < nw ? red[0][lane] : 0.f; b = lane < nw ? red[1][lane] : 0.f;
  return make_float2(warp_sum(a), warp_sum(b));
}

__global__ void __launch_bounds__(kFullNormThreads)
qk_fullnorm_rope_kernel(__nv_bfloat16* __restrict__ buf, long long ld, int nq_heads, int nheads, int hd,
                        const float* __restrict__ q_norm, const float* __restrict__ k_norm, float eps, int round_first,
                        const float* __restrict__ cos_t, const float* __restrict__ sin_t, int T, int L,
                        const int64_t* __restrict__ pos, __nv_bfloat16* __restrict__ pre, long long ld_pre,
                        float* __restrict__ rstd_out, long long ld_rstd) {
  __shared__ float red[2][32];
  const size_t r = blockIdx.x;
  const int half = hd >> 1, units = nheads * hd / 8, units_q = nq_heads * hd / 8;
  const int Nq = nq_heads * hd, Nk = (nheads - nq_heads) * hd;
  __nv_bfloat16* x = buf + r * ld;
  Unit8 u[kFullNormUnits];
  float sq = 0.f, sk = 0.f;
#pragma unroll
  for (int k = 0; k < kFullNormUnits; ++k) {
    const int i = threadIdx.x + k * kFullNormThreads;
    if (i < units) {
      int j;
      const int c = unit_col(i, hd, j);
      ld_unit(x + c, half, u[k]);
      if (pre != nullptr) st_unit(pre + r * ld_pre + c, half, u[k].v);
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) s = fmaf(u[k].v[e], u[k].v[e], s);
      if (i < units_q) sq += s; else sk += s;
    }
  }
  const float2 ss = block_sum2(sq, sk, red);
  const float rq = rsqrtf(ss.x / (float)Nq + eps), rk = Nk > 0 ? rsqrtf(ss.y / (float)Nk + eps) : 0.f;
  if (rstd_out != nullptr && threadIdx.x == 0) { rstd_out[r * ld_rstd] = rq; rstd_out[r * ld_rstd + 1] = rk; }
  int p;
  if (pos != nullptr) {
    const long long t = pos[r];
    p = (int)(t < 0 ? 0 : (t >= T ? T - 1 : t));
  } else {
    p = (int)(r % L);
  }
#pragma unroll
  for (int k = 0; k < kFullNormUnits; ++k) {
    const int i = threadIdx.x + k * kFullNormThreads;
    if (i < units) {
      int j;
      const int c = unit_col(i, hd, j);
      const bool isq = i < units_q;
      const float rs = isq ? rq : rk;
      const float* w = isq ? q_norm + c : k_norm + (c - Nq);
      const float4 w1 = *reinterpret_cast<const float4*>(w), w2 = *reinterpret_cast<const float4*>(w + half);
      const float ww[8] = {w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w};
      float n[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float xh = u[k].v[e] * rs;
        n[e] = __bfloat162float(__float2bfloat16_rn(ww[e] * (round_first ? __bfloat162float(__float2bfloat16_rn(xh)) : xh)));
      }
      const float4 c4 = *reinterpret_cast<const float4*>(cos_t + (size_t)p * half + j);
      const float4 s4 = *reinterpret_cast<const float4*>(sin_t + (size_t)p * half + j);
      const float cc[4] = {c4.x, c4.y, c4.z, c4.w}, sn[4] = {s4.x, s4.y, s4.z, s4.w};
      float o[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        o[e] = fmaf(n[e], cc[e], -n[e + 4] * sn[e]);
        o[e + 4] = fmaf(n[e + 4], cc[e], n[e] * sn[e]);
      }
      st_unit(x + c, half, o);
    }
  }
}

// d(q|k) in place: g = un-rotated gradient of y = w x_hat (x_hat = pre rstd, one rstd per row for q and one for k);
//   dx = rstd (w g - x_hat mean(w g x_hat)), the mean over the q (or k) width
__global__ void __launch_bounds__(kFullNormThreads)
qk_fullnorm_rope_bwd_kernel(__nv_bfloat16* __restrict__ dbuf, long long ld, int nq_heads, int nheads, int hd,
                            const float* __restrict__ q_norm, const float* __restrict__ k_norm, const float* __restrict__ cos_t,
                            const float* __restrict__ sin_t, int L, const __nv_bfloat16* __restrict__ pre, long long ld_pre,
                            const float* __restrict__ rstd_in, long long ld_rstd) {
  __shared__ float red[2][32];
  const size_t r = blockIdx.x;
  const int half = hd >> 1, units = nheads * hd / 8, units_q = nq_heads * hd / 8;
  const int Nq = nq_heads * hd, Nk = (nheads - nq_heads) * hd;
  const int p = (int)(r % L);
  const float rq = rstd_in[r * ld_rstd], rk = rstd_in[r * ld_rstd + 1];
  __nv_bfloat16* d = dbuf + r * ld;
  Unit8 wg[kFullNormUnits], xh[kFullNormUnits];
  float dq = 0.f, dk = 0.f;
#pragma unroll
  for (int k = 0; k < kFullNormUnits; ++k) {
    const int i = threadIdx.x + k * kFullNormThreads;
    if (i < units) {
      int j;
      const int c = unit_col(i, hd, j);
      const bool isq = i < units_q;
      const float rs = isq ? rq : rk;
      Unit8 dy;
      ld_unit(d + c, half, dy);
      ld_unit(pre + r * ld_pre + c, half, xh[k]);
      const float4 c4 = *reinterpret_cast<const float4*>(cos_t + (size_t)p * half + j);
      const float4 s4 = *reinterpret_cast<const float4*>(sin_t + (size_t)p * half + j);
      const float cc[4] = {c4.x, c4.y, c4.z, c4.w}, sn[4] = {s4.x, s4.y, s4.z, s4.w};
      const float* w = isq ? q_norm + c : k_norm + (c - Nq);
      const float4 w1 = *reinterpret_cast<const float4*>(w), w2 = *reinterpret_cast<const float4*>(w + half);
      const float ww[8] = {w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w};
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {                              // inverse rotation (the transpose of the forward map)
        wg[k].v[e] = ww[e] * fmaf(dy.v[e], cc[e], dy.v[e + 4] * sn[e]);
        wg[k].v[e + 4] = ww[e + 4] * fmaf(dy.v[e + 4], cc[e], -dy.v[e] * sn[e]);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        xh[k].v[e] *= rs;
        s = fmaf(wg[k].v[e], xh[k].v[e], s);
      }
      if (isq) dq += s; else dk += s;
    }
  }
  const float2 dots = block_sum2(dq, dk, red);
  const float mq = dots.x / (float)Nq, mk = Nk > 0 ? dots.y / (float)Nk : 0.f;
#pragma unroll
  for (int k = 0; k < kFullNormUnits; ++k) {
    const int i = threadIdx.x + k * kFullNormThreads;
    if (i < units) {
      int j;
      const int c = unit_col(i, hd, j);
      const bool isq = i < units_q;
      const float rs = isq ? rq : rk, m = isq ? mq : mk;
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = rs * fmaf(-xh[k].v[e], m, wg[k].v[e]);
      st_unit(d + c, half, o);
    }
  }
}

// Deterministic RMSNorm weight gradient over bf16 normalised inputs: dw[c] += sum_r g[r,c] x[r,c] rstd[r, c >= ncols0], where
// g = dy (fp32 or bf16), un-rotated within heads of width hd when cos_t is given (the q|k norm under RoPE); without RoPE hd = 8
// only groups the columns. Rows split into fixed slices: each CTA writes its slice's partial column sums, and
// norm_wgrad_finish adds the slices in order. No atomics: the same bits on every run.
constexpr int kWgUnits = 64, kWgLanes = 4;

__device__ __forceinline__ void ld_unit(const float* p, int half, Unit8& u) {
  const float4 a0 = *reinterpret_cast<const float4*>(p), b0 = *reinterpret_cast<const float4*>(p + half);
  u.v[0] = a0.x; u.v[1] = a0.y; u.v[2] = a0.z; u.v[3] = a0.w; u.v[4] = b0.x; u.v[5] = b0.y; u.v[6] = b0.z; u.v[7] = b0.w;
}

template <typename TD>
__global__ void __launch_bounds__(kWgUnits * kWgLanes)
norm_wgrad_partial_kernel(const TD* __restrict__ dy, long long ld_dy, const __nv_bfloat16* __restrict__ x, long long ld_x,
                          const float* __restrict__ rstd, long long ld_rstd, int ncols0, int ncols, int hd,
                          const float* __restrict__ cos_t, const float* __restrict__ sin_t, int L, int M, int rows_per_split,
                          float* __restrict__ part) {
  __shared__ float red[kWgLanes][kWgUnits][9];
  const int ul = threadIdx.x % kWgUnits, lane = threadIdx.x / kWgUnits;
  const int i = blockIdx.x * kWgUnits + ul, half = hd >> 1;
  const int r0 = blockIdx.y * rows_per_split, r1 = min(M, r0 + rows_per_split);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int j = 0, c = 0;
  const bool live = i < ncols / 8;
  if (live) c = unit_col(i, hd, j);
  if (live) {
    const int seg = c >= ncols0 ? 1 : 0;
    for (int r = r0 + lane; r < r1; r += kWgLanes) {
      Unit8 g, xv;
      ld_unit(dy + (size_t)r * ld_dy + c, half, g);
      ld_unit(x + (size_t)r * ld_x + c, half, xv);
      if (cos_t != nullptr) {
        const int p = r % L;
        const float4 c4 = *reinterpret_cast<const float4*>(cos_t + (size_t)p * half + j);
        const float4 s4 = *reinterpret_cast<const float4*>(sin_t + (size_t)p * half + j);
        const float cc[4] = {c4.x, c4.y, c4.z, c4.w}, sn[4] = {s4.x, s4.y, s4.z, s4.w};
        float t[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          t[e] = fmaf(g.v[e], cc[e], g.v[e + 4] * sn[e]);
          t[e + 4] = fmaf(g.v[e + 4], cc[e], -g.v[e] * sn[e]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) g.v[e] = t[e];
      }
      const float rs = rstd[(size_t)r * ld_rstd + seg];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = fmaf(g.v[e], xv.v[e] * rs, acc[e]);
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[lane][ul][e] = acc[e];
  __syncthreads();
  if (lane == 0 && live) {
#pragma unroll
    for (int l = 1; l < kWgLanes; ++l)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += red[l][ul][e];
    float* o = part + (size_t)blockIdx.y * ncols + c;
    *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(o + half) = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
}

__global__ void norm_wgrad_finish_kernel(const float* __restrict__ part, int splits, int ncols0, int ncols, float* __restrict__ dw0,
                                         float* __restrict__ dw1) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncols) return;
  float s = 0.f;
  for (int k = 0; k < splits; ++k) s += part[(size_t)k * ncols + c];
  if (c < ncols0) dw0[c] += s; else dw1[c - ncols0] += s;
}

}  // namespace dalm

using namespace dalm;

extern "C" int dalm_b200_qk_norm_rope(void* buf, long long ld, int nheads, int nq_heads, const float* q_norm, const float* k_norm,
                                      float eps, const float* cos_t, const float* sin_t, int T, int L, const int64_t* pos, int M,
                                      void* pre, long long ld_pre, float* rstd, long long ld_rstd, void* stream) {
  DALM_REQUIRE(M > 0 && nheads > 0 && nq_heads >= 0 && nq_heads <= nheads, "qk_norm_rope: bad shape M=%d heads=%d q heads=%d", M, nheads, nq_heads);
  DALM_REQUIRE(buf != nullptr && ld >= 128LL * nheads && (ld % 2) == 0 && ((uintptr_t)buf & 3) == 0, "qk_norm_rope: buffer / ld=%lld", ld);
  DALM_REQUIRE(q_norm != nullptr && k_norm != nullptr && ((uintptr_t)q_norm & 7) == 0 && ((uintptr_t)k_norm & 7) == 0, "qk_norm_rope: norm weights");
  DALM_REQUIRE(cos_t != nullptr && sin_t != nullptr && ((uintptr_t)cos_t & 7) == 0 && ((uintptr_t)sin_t & 7) == 0 && T > 0, "qk_norm_rope: cos / sin tables");
  DALM_REQUIRE(pos != nullptr || (L > 0 && L <= T), "qk_norm_rope: row positions need 0 < L=%d <= T=%d", L, T);
  DALM_REQUIRE(pre == nullptr || (ld_pre >= 128LL * nheads && (ld_pre % 2) == 0 && ((uintptr_t)pre & 3) == 0), "qk_norm_rope: pre / ld_pre");
  DALM_REQUIRE(rstd == nullptr || ld_rstd >= nheads, "qk_norm_rope: ld_rstd=%lld < %d heads", ld_rstd, nheads);
  DALM_REQUIRE(eps >= 0.f, "qk_norm_rope: eps must be >= 0");
  const long long items = (long long)M * nheads;
  const int grid = (int)((items + kNormRopeWarps - 1) / kNormRopeWarps);
  qk_norm_rope_kernel<<<grid, kNormRopeWarps * 32, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16*)buf, ld, nheads, nq_heads, q_norm, k_norm, eps, cos_t, sin_t, T, L, pos, M, (__nv_bfloat16*)pre, ld_pre, rstd, ld_rstd);
  count_launch();
  return check_launch("qk_norm_rope_kernel");
}

extern "C" int dalm_b200_qk_norm_rope_bwd(void* dbuf, long long ld, int nheads, int nq_heads, const float* q_norm, const float* k_norm,
                                          const float* cos_t, const float* sin_t, int L, const void* pre, long long ld_pre,
                                          const float* rstd, long long ld_rstd, int M, float* dw_q, float* dw_k, void* stream) {
  DALM_REQUIRE(M > 0 && nheads > 0 && nq_heads >= 0 && nq_heads <= nheads && L > 0, "qk_norm_rope_bwd: bad shape M=%d heads=%d L=%d", M, nheads, L);
  DALM_REQUIRE(dbuf != nullptr && ld >= 128LL * nheads && (ld % 2) == 0 && ((uintptr_t)dbuf & 3) == 0, "qk_norm_rope_bwd: buffer / ld=%lld", ld);
  DALM_REQUIRE(q_norm != nullptr && k_norm != nullptr && ((uintptr_t)q_norm & 7) == 0 && ((uintptr_t)k_norm & 7) == 0, "qk_norm_rope_bwd: norm weights");
  DALM_REQUIRE(cos_t != nullptr && sin_t != nullptr && ((uintptr_t)cos_t & 7) == 0 && ((uintptr_t)sin_t & 7) == 0, "qk_norm_rope_bwd: cos / sin tables");
  DALM_REQUIRE(pre != nullptr && ld_pre >= 128LL * nheads && (ld_pre % 2) == 0 && ((uintptr_t)pre & 3) == 0, "qk_norm_rope_bwd: pre / ld_pre");
  DALM_REQUIRE(rstd != nullptr && ld_rstd >= nheads, "qk_norm_rope_bwd: rstd / ld_rstd=%lld", ld_rstd);
  DALM_REQUIRE((dw_q == nullptr) == (dw_k == nullptr), "qk_norm_rope_bwd: dw_q and dw_k go together");
  const long long items = (long long)M * nheads;
  long long want = (items + kNormRopeWarps - 1) / kNormRopeWarps;
  const long long cap = (long long)num_sms() * 8;               // enough blocks to fill the GPU; each adds its dw once
  const int grid = (int)(want < cap ? want : cap);
  qk_norm_rope_bwd_kernel<<<grid, kNormRopeWarps * 32, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16*)dbuf, ld, nheads, nq_heads, q_norm, k_norm, cos_t, sin_t, L, (const __nv_bfloat16*)pre, ld_pre, rstd, ld_rstd, M,
      dw_q, dw_k);
  count_launch();
  return check_launch("qk_norm_rope_bwd_kernel");
}

static bool fullnorm_shape_ok(int nq_heads, int nheads, int hd) {
  return nq_heads > 0 && nheads > nq_heads && (hd == 64 || hd == 128) &&
         (long long)nheads * hd <= 8LL * kFullNormUnits * kFullNormThreads;
}

extern "C" int dalm_b200_qk_fullnorm_rope(void* buf, long long ld, int nq_heads, int nheads, int hd, const float* q_norm,
                                          const float* k_norm, float eps, int round_first, const float* cos_t, const float* sin_t,
                                          int T, int L, const int64_t* pos, int M, void* pre, long long ld_pre, float* rstd,
                                          long long ld_rstd, void* stream) {
  DALM_REQUIRE(M > 0 && M <= 0x7fffffff && fullnorm_shape_ok(nq_heads, nheads, hd),
               "qk_fullnorm_rope: bad shape M=%d heads=%d q heads=%d head_dim=%d (head_dim 64 / 128, at most %d q|k columns)",
               M, nheads, nq_heads, hd, 8 * kFullNormUnits * kFullNormThreads);
  DALM_REQUIRE(buf != nullptr && ld >= (long long)hd * nheads && (ld % 4) == 0 && aligned(buf, 8), "qk_fullnorm_rope: buffer / ld=%lld", ld);
  DALM_REQUIRE(aligned(q_norm, 16) && aligned(k_norm, 16) && q_norm && k_norm, "qk_fullnorm_rope: norm weights must be 16-byte aligned");
  DALM_REQUIRE(cos_t && sin_t && aligned(cos_t, 16) && aligned(sin_t, 16) && T > 0, "qk_fullnorm_rope: cos / sin tables");
  DALM_REQUIRE(pos != nullptr || (L > 0 && L <= T), "qk_fullnorm_rope: row positions need 0 < L=%d <= T=%d", L, T);
  DALM_REQUIRE(pre == nullptr || (ld_pre >= (long long)hd * nheads && (ld_pre % 4) == 0 && aligned(pre, 8)), "qk_fullnorm_rope: pre / ld_pre");
  DALM_REQUIRE(rstd == nullptr || ld_rstd >= 2, "qk_fullnorm_rope: ld_rstd=%lld < 2", ld_rstd);
  DALM_REQUIRE(eps >= 0.f, "qk_fullnorm_rope: eps must be >= 0");
  qk_fullnorm_rope_kernel<<<M, kFullNormThreads, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16*)buf, ld, nq_heads, nheads, hd, q_norm, k_norm, eps, round_first, cos_t, sin_t, T, L, pos, (__nv_bfloat16*)pre,
      ld_pre, rstd, ld_rstd);
  count_launch();
  return check_launch("qk_fullnorm_rope_kernel");
}

extern "C" int dalm_b200_qk_fullnorm_rope_bwd(void* dbuf, long long ld, int nq_heads, int nheads, int hd, const float* q_norm,
                                              const float* k_norm, const float* cos_t, const float* sin_t, int L, const void* pre,
                                              long long ld_pre, const float* rstd, long long ld_rstd, int M, void* stream) {
  DALM_REQUIRE(M > 0 && L > 0 && fullnorm_shape_ok(nq_heads, nheads, hd), "qk_fullnorm_rope_bwd: bad shape M=%d heads=%d q heads=%d head_dim=%d L=%d",
               M, nheads, nq_heads, hd, L);
  DALM_REQUIRE(dbuf != nullptr && ld >= (long long)hd * nheads && (ld % 4) == 0 && aligned(dbuf, 8), "qk_fullnorm_rope_bwd: buffer / ld=%lld", ld);
  DALM_REQUIRE(aligned(q_norm, 16) && aligned(k_norm, 16) && q_norm && k_norm, "qk_fullnorm_rope_bwd: norm weights must be 16-byte aligned");
  DALM_REQUIRE(cos_t && sin_t && aligned(cos_t, 16) && aligned(sin_t, 16), "qk_fullnorm_rope_bwd: cos / sin tables");
  DALM_REQUIRE(pre != nullptr && ld_pre >= (long long)hd * nheads && (ld_pre % 4) == 0 && aligned(pre, 8), "qk_fullnorm_rope_bwd: pre / ld_pre");
  DALM_REQUIRE(rstd != nullptr && ld_rstd >= 2, "qk_fullnorm_rope_bwd: rstd / ld_rstd=%lld", ld_rstd);
  qk_fullnorm_rope_bwd_kernel<<<M, kFullNormThreads, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16*)dbuf, ld, nq_heads, nheads, hd, q_norm, k_norm, cos_t, sin_t, L, (const __nv_bfloat16*)pre, ld_pre, rstd, ld_rstd);
  count_launch();
  return check_launch("qk_fullnorm_rope_bwd_kernel");
}

extern "C" int dalm_b200_norm_wgrad(const void* dy, int dy_f32, long long ld_dy, const void* x, long long ld_x, const float* rstd,
                                    long long ld_rstd, int ncols0, int ncols, int hd, const float* cos_t, const float* sin_t, int L,
                                    int M, float* part, int splits, float* dw0, float* dw1, void* stream) {
  DALM_REQUIRE(M > 0 && ncols > 0 && (hd == 8 || hd == 64 || hd == 128) && (ncols % hd) == 0 && ncols0 > 0 && ncols0 <= ncols &&
               (ncols0 % hd) == 0 && splits >= 1 && splits <= 65535,
               "norm_wgrad: bad shape M=%d ncols=%d ncols0=%d hd=%d splits=%d", M, ncols, ncols0, hd, splits);
  DALM_REQUIRE(dy && x && rstd && part && dw0 && (dw1 || ncols0 == ncols), "norm_wgrad: missing operand");
  DALM_REQUIRE(ld_rstd >= (ncols0 < ncols ? 2 : 1), "norm_wgrad: ld_rstd=%lld", ld_rstd);
  DALM_REQUIRE((ld_dy % 4) == 0 && (ld_x % 4) == 0 && aligned(dy, 16) && aligned(x, 8) && aligned(part, 16),
               "norm_wgrad: rows must be 4-element strided and aligned");
  DALM_REQUIRE(cos_t == nullptr || (sin_t && L > 0 && hd >= 64 && aligned(cos_t, 16) && aligned(sin_t, 16)), "norm_wgrad: cos / sin tables");
  const int rows = (M + splits - 1) / splits;
  const dim3 grid((ncols / 8 + kWgUnits - 1) / kWgUnits, (M + rows - 1) / rows);
  if (dy_f32)
    norm_wgrad_partial_kernel<float><<<grid, kWgUnits * kWgLanes, 0, (cudaStream_t)stream>>>(
        (const float*)dy, ld_dy, (const __nv_bfloat16*)x, ld_x, rstd, ld_rstd, ncols0, ncols, hd, cos_t, sin_t, L, M, rows, part);
  else
    norm_wgrad_partial_kernel<__nv_bfloat16><<<grid, kWgUnits * kWgLanes, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)dy, ld_dy, (const __nv_bfloat16*)x, ld_x, rstd, ld_rstd, ncols0, ncols, hd, cos_t, sin_t, L, M, rows, part);
  count_launch();
  if (int e = check_launch("norm_wgrad_partial_kernel")) return e;
  norm_wgrad_finish_kernel<<<(ncols + 255) / 256, 256, 0, (cudaStream_t)stream>>>(part, (int)grid.y, ncols0, ncols, dw0, dw1);
  count_launch();
  return check_launch("norm_wgrad_finish_kernel");
}
