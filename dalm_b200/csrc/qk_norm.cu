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
