// dalm_b200 — routing kernels of a top-k mixture-of-experts MLP (Qwen3-MoE's Qwen3MoeSparseMoeBlock).
//
// The experts run on the grouped wgmma GEMM (dalm_b200_gemm_bf16_grouped), which wants each expert's rows contiguous and
// padded to its 128-row M tile. These kernels build that layout and undo it:
//
//   router        fp32 logits [M, E] -> softmax -> top-k ids (descending) and weights, renormalised when norm_topk
//   permute       per-expert counts, padded segment offsets, the M-tile -> expert table, the live tile count, and the
//                 (token, slot) pair <-> row maps. Within a segment rows follow the pair order: by token, then by slot
//   gather        rows[r] = x[token of row r] (0 on padding rows)
//   combine       out[t] = resid[t] + sum_s w[t, s] y[row(t, s)]                   (w == NULL: weights of 1)
//   down_bwd      dw[t, s] = <da[row], act[row]>, d_act[row] = w[t, s] da[row]     (da = W_down^T dy of the row)
//   router_bwd    d logits from d weights: renormalisation, top-k and softmax backward
//
// Every sum runs in a fixed order and nothing uses floating-point atomics, so routing, outputs and gradients are the same
// bits from run to run. No kernel needs a host synchronisation: the live tile count stays in device memory.
#include "common.cuh"

namespace dalm {

constexpr int kMoeMaxExperts = 256;      // the router holds a token's logits in registers, 8 per lane
constexpr int kMoeMaxTopK = 16;
constexpr int kMoeChunk = 1024;          // (token, slot) pairs ranked per CTA of the permutation

// --------------------------------------------------------------------------------------------------------------
// router: one warp per token. Expert j = lane + 32 i lives in v[i] of its lane.
// --------------------------------------------------------------------------------------------------------------
struct RouterRow {
  float v[kMoeMaxExperts / 32];          // logits, then probabilities
  int sel[kMoeMaxTopK];                  // selected experts, descending
};

// softmax in fp32 (max-subtracted, expf, one butterfly sum) and top-k by logit, ties to the lower index
__device__ __forceinline__ void router_row(const float* __restrict__ lg, int E, int k, RouterRow& r) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) {
    const int j = lane + 32 * i;
    r.v[i] = j < E ? lg[j] : -INFINITY;
    mx = fmaxf(mx, r.v[i]);
  }
  mx = warp_max(mx);
  unsigned taken = 0u;                   // bit i: v[i] already selected
  for (int s = 0; s < k; ++s) {
    float bv = -INFINITY; int bj = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < kMoeMaxExperts / 32; ++i) {
      const int j = lane + 32 * i;
      if (j < E && !(taken >> i & 1u) && (r.v[i] > bv || (r.v[i] == bv && j < bj))) { bv = r.v[i]; bj = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (ov > bv || (ov == bv && oj < bj)) { bv = ov; bj = oj; }
    }
    r.sel[s] = bj;
    if ((bj & 31) == lane) taken |= 1u << (bj >> 5);
  }
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) {
    r.v[i] = lane + 32 * i < E ? expf(r.v[i] - mx) : 0.f;
    sum += r.v[i];
  }
  sum = warp_sum(sum);
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) r.v[i] /= sum;
}

// probability of expert j (held by lane j % 32), broadcast to the warp
__device__ __forceinline__ float router_prob(const RouterRow& r, int j) {
  float x = 0.f;
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) if (i == (j >> 5)) x = r.v[i];
  return __shfl_sync(0xffffffffu, x, j & 31);
}

__global__ void __launch_bounds__(256) moe_router_kernel(const float* __restrict__ logits, long long ld, int M, int E, int k,
                                                         int norm_topk, int* __restrict__ ids, float* __restrict__ w) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= M) return;
  RouterRow r;
  router_row(logits + (size_t)t * ld, E, k, r);
  float p[kMoeMaxTopK], s = 0.f;
  for (int q = 0; q < k; ++q) { p[q] = router_prob(r, r.sel[q]); s += p[q]; }
  if (lane < k) {
    float pq = 0.f;
    for (int q = 0; q < k; ++q) if (q == lane) pq = p[q];
    ids[(size_t)t * k + lane] = r.sel[lane];
    w[(size_t)t * k + lane] = norm_topk ? pq / s : pq;
  }
}

// w_s = p_s (/ S, S = sum of the k selected p): g_s = dL/dp_{e_s} = dw_s (or (dw_s - sum_r dw_r w_r) / S), and
// dlogit_j = p_j (g_j - sum_s p_{e_s} g_s) with g_j = 0 off the selection
__global__ void __launch_bounds__(256) moe_router_bwd_kernel(const float* __restrict__ logits, long long ld, const int* __restrict__ ids,
                                                             const float* __restrict__ w, const float* __restrict__ dw, int M, int E,
                                                             int k, int norm_topk, __nv_bfloat16* __restrict__ dlogits, long long ldd) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= M) return;
  RouterRow r;
  router_row(logits + (size_t)t * ld, E, 0, r);   // probabilities only; the selection is the forward's
  const int* id = ids + (size_t)t * k;
  float S = 0.f, dot = 0.f;
  for (int q = 0; q < k; ++q) {
    S += router_prob(r, id[q]);
    dot += dw[(size_t)t * k + q] * w[(size_t)t * k + q];
  }
  float g[kMoeMaxTopK], pg = 0.f;
  for (int q = 0; q < k; ++q) {
    const float d = dw[(size_t)t * k + q];
    g[q] = norm_topk ? (d - dot) / S : d;
    pg += router_prob(r, id[q]) * g[q];
  }
#pragma unroll
  for (int i = 0; i < kMoeMaxExperts / 32; ++i) {
    const int j = lane + 32 * i;
    if (j >= E) break;
    float gj = 0.f;
    for (int q = 0; q < k; ++q) if (id[q] == j) gj = g[q];
    dlogits[(size_t)t * ldd + j] = __float2bfloat16_rn(r.v[i] * (gj - pg));
  }
}

// --------------------------------------------------------------------------------------------------------------
// permutation: count per chunk of 1024 pairs, one CTA scans, then every chunk ranks its pairs in pair order.
// Integer shared-memory atomics only count; the rank of a pair comes from warp match masks and a scan over warps.
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMoeChunk) moe_count_kernel(const int* __restrict__ ids, int P, int E, int* __restrict__ chunk_counts) {
  __shared__ int cnt[kMoeMaxExperts];
  for (int e = threadIdx.x; e < E; e += blockDim.x) cnt[e] = 0;
  __syncthreads();
  const int p = blockIdx.x * kMoeChunk + threadIdx.x;
  if (p < P) {
    const int e = ids[p];
    if (e >= 0 && e < E) atomicAdd(&cnt[e], 1);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) chunk_counts[(size_t)blockIdx.x * E + e] = cnt[e];
}

// chunk_counts -> each chunk's first rank per expert; seg_off[E + 1] padded offsets; counts[E]; tile_expert[n_tiles]; live;
// row_pair = -1 on every padding row of a segment
__global__ void __launch_bounds__(256) moe_scan_kernel(int* __restrict__ chunk_counts, int n_chunks, int E, int n_tiles,
                                                       int* __restrict__ counts, int* __restrict__ seg_off, int* __restrict__ tile_expert,
                                                       int* __restrict__ live, int* __restrict__ row_pair) {
  __shared__ int off[kMoeMaxExperts + 1];
  __shared__ int tot[kMoeMaxExperts];
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    int base = 0;
    for (int c = 0; c < n_chunks; ++c) {
      const int v = chunk_counts[(size_t)c * E + e];
      chunk_counts[(size_t)c * E + e] = base;
      base += v;
    }
    tot[e] = base;
    counts[e] = base;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int o = 0;
    for (int e = 0; e < E; ++e) { off[e] = o; o += (tot[e] + 127) & ~127; }
    off[E] = o;
    *live = o / 128;
  }
  __syncthreads();
  for (int e = threadIdx.x; e <= E; e += blockDim.x) seg_off[e] = off[e];
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    for (int r = off[e] + tot[e]; r < off[e + 1]; ++r) row_pair[r] = -1;
    for (int m = off[e] / 128; m < off[e + 1] / 128; ++m) tile_expert[m] = e;
  }
  for (int m = off[E] / 128 + threadIdx.x; m < n_tiles; m += blockDim.x) tile_expert[m] = -1;
}

__global__ void __launch_bounds__(kMoeChunk) moe_scatter_kernel(const int* __restrict__ ids, int P, int E, const int* __restrict__ chunk_base,
                                                                const int* __restrict__ seg_off, int* __restrict__ pair_row,
                                                                int* __restrict__ row_pair) {
  __shared__ int wc[kMoeChunk / 32][kMoeMaxExperts];  // per warp: its pairs per expert, then its first rank
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < (kMoeChunk / 32) * kMoeMaxExperts; i += blockDim.x) (&wc[0][0])[i] = 0;
  __syncthreads();
  const int p = blockIdx.x * kMoeChunk + threadIdx.x;
  int e = p < P ? ids[p] : -1;
  if (e >= E) e = -1;
  const unsigned same = __match_any_sync(0xffffffffu, e);
  const int rank = __popc(same & ((1u << lane) - 1u));
  if (e >= 0 && rank == 0) wc[warp][e] = __popc(same);
  __syncthreads();
  for (int x = threadIdx.x; x < E; x += blockDim.x) {
    int run = chunk_base[(size_t)blockIdx.x * E + x];
    for (int w = 0; w < kMoeChunk / 32; ++w) { const int c = wc[w][x]; wc[w][x] = run; run += c; }
  }
  __syncthreads();
  if (p < P) {
    if (e < 0) { pair_row[p] = -1; return; }
    const int row = seg_off[e] + wc[warp][e] + rank;
    pair_row[p] = row;
    row_pair[row] = p;
  }
}

// --------------------------------------------------------------------------------------------------------------
// row movement: 16-byte pieces, one CTA of 128 threads per row
// --------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load8(const void* base, int f32, size_t off, float* f) {
  if (f32) {
    const float4 a = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + off);
    const float4 b = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + off + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  } else {
    unpack8(*reinterpret_cast<const bf16x8*>(reinterpret_cast<const __nv_bfloat16*>(base) + off), f);
  }
}
__device__ __forceinline__ void store8(void* base, int f32, size_t off, const float* f) {
  if (f32) {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + off) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + off + 4) = make_float4(f[4], f[5], f[6], f[7]);
  } else {
    *reinterpret_cast<bf16x8*>(reinterpret_cast<__nv_bfloat16*>(base) + off) = pack8(f);
  }
}

__global__ void __launch_bounds__(128) moe_gather_kernel(const void* __restrict__ x, long long ldx, int x_f32, int H,
                                                         const int* __restrict__ row_pair, int k, const int* __restrict__ live,
                                                         __nv_bfloat16* __restrict__ out, long long ldo) {
  const int r = blockIdx.x;
  if (r >= __ldg(live) * 128) return;
  const int p = row_pair[r];
  for (int c = threadIdx.x * 8; c < H; c += 128 * 8) {
    float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (p >= 0) load8(x, x_f32, (size_t)(p / k) * ldx + c, f);
    store8(out, 0, (size_t)r * ldo + c, f);
  }
}

__global__ void __launch_bounds__(128) moe_combine_kernel(const __nv_bfloat16* __restrict__ y, long long ldy, const int* __restrict__ pair_row,
                                                          const float* __restrict__ w, int k, int H, const void* resid, long long ldr,
                                                          void* out, long long ldo, int f32) {
  const int t = blockIdx.x;
  for (int c = threadIdx.x * 8; c < H; c += 128 * 8) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < k; ++s) {
      const int r = pair_row[(size_t)t * k + s];
      if (r < 0) continue;
      const float ws = w ? w[(size_t)t * k + s] : 1.f;
      float f[8];
      unpack8(*reinterpret_cast<const bf16x8*>(y + (size_t)r * ldy + c), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(ws, f[i], acc[i]);
    }
    if (resid) {
      float f[8];
      load8(resid, f32, (size_t)t * ldr + c, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = f[i] + acc[i];
    }
    store8(out, f32, (size_t)t * ldo + c, acc);
  }
}

// one warp per (token, slot) pair
__global__ void __launch_bounds__(256) moe_down_bwd_kernel(const __nv_bfloat16* __restrict__ da, long long ldda,
                                                           const __nv_bfloat16* act, long long ldact,   // may be d_act
                                                           const int* __restrict__ pair_row, const float* __restrict__ w, int P, int I,
                                                           float* __restrict__ dw, __nv_bfloat16* d_act, long long ldd) {
  const int p = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= P) return;
  const int r = pair_row[p];
  if (r < 0) { if (lane == 0) dw[p] = 0.f; return; }
  const float ws = w[p];
  float dot = 0.f;
  for (int c = lane * 8; c < I; c += 32 * 8) {
    float a[8], g[8];
    unpack8(*reinterpret_cast<const bf16x8*>(da + (size_t)r * ldda + c), g);
    unpack8(*reinterpret_cast<const bf16x8*>(act + (size_t)r * ldact + c), a);
#pragma unroll
    for (int i = 0; i < 8; ++i) { dot = fmaf(g[i], a[i], dot); g[i] *= ws; }
    *reinterpret_cast<bf16x8*>(d_act + (size_t)r * ldd + c) = pack8(g);
  }
  dot = warp_sum(dot);
  if (lane == 0) dw[p] = dot;
}

static inline cudaStream_t ST(void* s) { return (cudaStream_t)s; }

}  // namespace dalm

using namespace dalm;

extern "C" int dalm_b200_moe_router(const float* logits, long long ld, int M, int E, int k, int norm_topk, int* ids, float* w,
                                    void* stream) {
  DALM_REQUIRE(M > 0 && E > 0 && E <= kMoeMaxExperts && ld >= E, "moe_router: E=%d must be in [1, %d] (ld %lld)", E, kMoeMaxExperts, ld);
  DALM_REQUIRE(k > 0 && k <= kMoeMaxTopK && k <= E, "moe_router: top-k=%d must be in [1, min(E, %d)]", k, kMoeMaxTopK);
  moe_router_kernel<<<(M + 7) / 8, 256, 0, ST(stream)>>>(logits, ld, M, E, k, norm_topk, ids, w);
  count_launch();
  return check_launch("moe_router_kernel");
}

extern "C" int dalm_b200_moe_router_bwd(const float* logits, long long ld, const int* ids, const float* w, const float* dw, int M,
                                        int E, int k, int norm_topk, void* dlogits, long long ldd, void* stream) {
  DALM_REQUIRE(M > 0 && E > 0 && E <= kMoeMaxExperts && ld >= E && ldd >= E, "moe_router_bwd: E=%d must be in [1, %d]", E, kMoeMaxExperts);
  DALM_REQUIRE(k > 0 && k <= kMoeMaxTopK && k <= E, "moe_router_bwd: top-k=%d must be in [1, min(E, %d)]", k, kMoeMaxTopK);
  moe_router_bwd_kernel<<<(M + 7) / 8, 256, 0, ST(stream)>>>(logits, ld, ids, w, dw, M, E, k, norm_topk,
                                                              reinterpret_cast<__nv_bfloat16*>(dlogits), ldd);
  count_launch();
  return check_launch("moe_router_bwd_kernel");
}

// int32 workspace: chunk_counts [ceil(P / 1024) * E]; outputs counts [E], seg_off [E + 1], tile_expert [n_tiles], live [1],
// pair_row [P], row_pair [128 n_tiles]. n_tiles * 128 must cover P + 127 E (every segment padded).
extern "C" int dalm_b200_moe_permute(const int* ids, int P, int E, int n_tiles, int* chunk_counts, int* counts, int* seg_off,
                                     int* tile_expert, int* live, int* pair_row, int* row_pair, void* stream) {
  DALM_REQUIRE(P > 0 && E > 0 && E <= kMoeMaxExperts, "moe_permute: P=%d pairs, E=%d experts (at most %d)", P, E, kMoeMaxExperts);
  DALM_REQUIRE((long long)n_tiles * 128 >= (long long)P + 127LL * E, "moe_permute: %d M tiles cannot hold %d pairs padded over %d experts",
               n_tiles, P, E);
  const int chunks = (P + kMoeChunk - 1) / kMoeChunk;
  moe_count_kernel<<<chunks, kMoeChunk, 0, ST(stream)>>>(ids, P, E, chunk_counts);
  moe_scan_kernel<<<1, 256, 0, ST(stream)>>>(chunk_counts, chunks, E, n_tiles, counts, seg_off, tile_expert, live, row_pair);
  moe_scatter_kernel<<<chunks, kMoeChunk, 0, ST(stream)>>>(ids, P, E, chunk_counts, seg_off, pair_row, row_pair);
  count_launch(3);
  return check_launch("moe_permute kernels");
}

extern "C" int dalm_b200_moe_gather(const void* x, long long ldx, int x_f32, int H, const int* row_pair, int k, const int* live,
                                    int n_rows, void* out, long long ldo, void* stream) {
  DALM_REQUIRE(H > 0 && (H % 8) == 0 && k > 0 && n_rows > 0, "moe_gather: H=%d must be a positive multiple of 8", H);
  DALM_REQUIRE(ldx >= H && ldo >= H && (ldx % 8) == 0 && (ldo % 8) == 0 && aligned(x, 16) && aligned(out, 16),
               "moe_gather: leading dimensions / 16-byte alignment");
  moe_gather_kernel<<<n_rows, 128, 0, ST(stream)>>>(x, ldx, x_f32, H, row_pair, k, live, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  count_launch();
  return check_launch("moe_gather_kernel");
}

extern "C" int dalm_b200_moe_combine(const void* y, long long ldy, const int* pair_row, const float* w, int M, int k, int H,
                                     const void* resid, long long ldr, void* out, long long ldo, int f32, void* stream) {
  DALM_REQUIRE(M > 0 && k > 0 && H > 0 && (H % 8) == 0, "moe_combine: H=%d must be a positive multiple of 8", H);
  DALM_REQUIRE(ldy >= H && ldo >= H && (ldy % 8) == 0 && (ldo % 8) == 0 && aligned(y, 16) && aligned(out, 16) &&
               (resid == nullptr || (ldr >= H && (ldr % 8) == 0 && aligned(resid, 16))),
               "moe_combine: leading dimensions / 16-byte alignment");
  moe_combine_kernel<<<M, 128, 0, ST(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(y), ldy, pair_row, w, k, H, resid, ldr, out, ldo, f32);
  count_launch();
  return check_launch("moe_combine_kernel");
}

extern "C" int dalm_b200_moe_down_bwd(const void* da, long long ldda, const void* act, long long ldact, const int* pair_row,
                                      const float* w, int P, int I, float* dw, void* d_act, long long ldd, void* stream) {
  DALM_REQUIRE(P > 0 && I > 0 && (I % 8) == 0, "moe_down_bwd: I=%d must be a positive multiple of 8", I);
  DALM_REQUIRE(ldda >= I && ldact >= I && ldd >= I && (ldda % 8) == 0 && (ldact % 8) == 0 && (ldd % 8) == 0 &&
               aligned(da, 16) && aligned(act, 16) && aligned(d_act, 16), "moe_down_bwd: leading dimensions / 16-byte alignment");
  moe_down_bwd_kernel<<<(P + 7) / 8, 256, 0, ST(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(da), ldda,
                                                           reinterpret_cast<const __nv_bfloat16*>(act), ldact, pair_row, w, P, I, dw,
                                                           reinterpret_cast<__nv_bfloat16*>(d_act), ldd);
  count_launch();
  return check_launch("moe_down_bwd_kernel");
}
