// dalm_b200 — exact maximum-inner-product top-k over a resident passage-embedding matrix.
//
// Replaces the approximate hnswlib index of the reference's evaluation path (dalm/eval/utils.py:18-66: space "ip",
// M=100, ef_construction=200, ef=100; `knn_query` returns labels sorted by distance = 1 - <q,p>) with an exact sweep:
// for 200k x 1024 fp32 passages one query batch reads 819 MB — about 0.25 ms at the H100's 3.35 TB/s — so there is no reason to
// approximate on an H100. HBM-bound: algorithmic bytes = N*D*4 (the passage matrix, read once per query tile of <= 8).
//
// Stage 1 (topk_scan_kernel): the grid walks the passage rows; each warp takes two rows at a time (lanes read consecutive
//   float4: 512 contiguous bytes per request), accumulates the dot products with the <= 8 queries of the tile held in
//   shared memory (fp32 FMA), butterfly-reduces them, and keeps the warp's best K (<= 32) per query as a sorted list
//   distributed over the lanes (lane j = j-th best); insertion is a ballot + shuffle. Warp lists are merged per CTA
//   and written as [cta][query][K] candidates.
// Stage 2 (topk_merge_kernel): one warp per query merges all CTA candidate lists with the same insertion network.
// Order: higher score first; equal scores -> lower passage index first (deterministic, independent of the grid).
#include "common.cuh"

namespace dalm {

constexpr int kTopkMaxK = 32;
constexpr int kTopkQT = 8;           // queries per tile (one pass over the passages serves 8 queries)

struct Cand { float s; int i; };

__device__ __forceinline__ bool better(float s, int i, float s2, int i2) { return s > s2 || (s == s2 && i < i2); }

// lane j holds the j-th best (s,i) of a list of length K (lanes >= K hold -inf). Inserts (ns,ni) if it belongs; returns
// whether it did (merging SORTED lists can stop at the first candidate that does not).
__device__ __forceinline__ bool warp_insert(float& s, int& i, float ns, int ni, int K, int lane) {
  const unsigned m = __ballot_sync(0xffffffffu, lane < K && better(ns, ni, s, i));
  if (m == 0u) return false;                                   // uniform: every lane sees the same ballot
  const int pos = __ffs(m) - 1;
  const float us = __shfl_up_sync(0xffffffffu, s, 1);
  const int ui = __shfl_up_sync(0xffffffffu, i, 1);
  if (lane > pos) { s = us; i = ui; }
  else if (lane == pos) { s = ns; i = ni; }
  return true;
}

// fold one sorted candidate list (lane j holds its j-th entry, -inf padded) into the running list
__device__ __forceinline__ void warp_merge_list(float& s, int& i, float ls, int li, int K, int lane) {
  for (int j = 0; j < K; ++j) {
    const float cs = __shfl_sync(0xffffffffu, ls, j);
    const int ci = __shfl_sync(0xffffffffu, li, j);
    if (cs == -INFINITY || !warp_insert(s, i, cs, ci, K, lane)) break;      // sorted: nothing later can qualify either
  }
}

// Two passage rows x 8 queries of per-lane partial dot products -> full sums -> top-K lists, with ~5x fewer instructions
// than 16 butterfly reductions + 16 ballots (the first version issued 1240 warp instructions per 8 KB of passages: the sweep
// was issue/latency bound at a third of HBM speed). Recursive halving: at each of 4 steps a lane keeps half of its values
// and hands the other half to its partner (16 -> 8 -> 4 -> 2 -> 1), so lane L ends up with the complete sum of value
// (row = L >> 4, query = (L >> 1) & 7) after 16 shuffles; each lane compares its one value with that query's current K-th
// best score (kept per lane in `mythr`), and only the rare survivors go through the insertion network.
template <int QT>
__device__ __forceinline__ void reduce_and_insert(const float2 (&acc2)[2][QT], float (&bs)[QT], int (&bi)[QT], float& mythr,
                                                  int row0, int nvalid, int K, int lane) {
  static_assert(QT == 8, "the halving network is written for 2 rows x 8 queries");
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
  float w[8], x[4], y[2];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float v0 = acc2[0][j].x + acc2[0][j].y, v1 = acc2[1][j].x + acc2[1][j].y;
    w[j] = (b4 ? v1 : v0) + __shfl_xor_sync(0xffffffffu, b4 ? v0 : v1, 16);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) x[j] = (b3 ? w[j + 4] : w[j]) + __shfl_xor_sync(0xffffffffu, b3 ? w[j] : w[j + 4], 8);
#pragma unroll
  for (int j = 0; j < 2; ++j) y[j] = (b2 ? x[j + 2] : x[j]) + __shfl_xor_sync(0xffffffffu, b2 ? x[j] : x[j + 2], 4);
  float z = (b1 ? y[1] : y[0]) + __shfl_xor_sync(0xffffffffu, b1 ? y[0] : y[1], 2);
  z += __shfl_xor_sync(0xffffffffu, z, 1);
  const int myq = (lane >> 1) & 7, myr = lane >> 4;
  unsigned m = __ballot_sync(0xffffffffu, z > mythr && !(lane & 1) && myr < nvalid);
  while (m) {                                                    // rare once the lists have warmed up
    const int l = __ffs(m) - 1;
    m &= m - 1;
    const float val = __shfl_sync(0xffffffffu, z, l);
    const int q = (l >> 1) & 7, row = row0 + (l >> 4);
#pragma unroll
    for (int qq = 0; qq < QT; ++qq) {
      if (qq == q) {                                             // warp-uniform
        if (warp_insert(bs[qq], bi[qq], val, row, K, lane)) {
          const float kth = __shfl_sync(0xffffffffu, bs[qq], K - 1);
          if (myq == qq) mythr = kth;
        }
      }
    }
  }
}

__device__ __forceinline__ float2 fma2(const float4& p, const float4& x, float2 acc) {
  acc.x = fmaf(p.x, x.x, acc.x);                               // two independent fp32 FMA chains per pair of lanes
  acc.y = fmaf(p.y, x.y, acc.y);
  acc.x = fmaf(p.z, x.z, acc.x);
  acc.y = fmaf(p.w, x.w, acc.y);
  return acc;
}

template <int QT>
__global__ void __launch_bounds__(256, 2) topk_scan_kernel(const float* __restrict__ Q, const float* __restrict__ P, long long ldp,
                                                        int nq, int N, int D, int K, float* __restrict__ cand_s,
                                                        int* __restrict__ cand_i) {
  extern __shared__ float smem[];                               // [QT][D] queries, then merge scratch
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int q0 = blockIdx.y * QT;
  const int nqt = min(QT, nq - q0);
  for (int t = threadIdx.x; t < QT * D; t += blockDim.x) {
    const int q = t / D, d = t - q * D;
    smem[t] = q < nqt ? Q[(size_t)(q0 + q) * D + d] : 0.f;
  }
  __syncthreads();
  float bs[QT]; int bi[QT];
#pragma unroll
  for (int q = 0; q < QT; ++q) { bs[q] = -INFINITY; bi[q] = 0x7fffffff; }
  float mythr = -INFINITY;
  const int D4 = D >> 2;
  const float4* q4 = reinterpret_cast<const float4*>(smem);
  // two passage rows per warp iteration: every shared-memory query read feeds two rows (the query tile would otherwise be
  // re-read 8x per HBM byte and cap the sweep at ~half of HBM speed)
  for (int row = (blockIdx.x * nwarps + warp) * 2; row < N; row += gridDim.x * nwarps * 2) {
    const bool two = row + 1 < N;
    const float4* pa = reinterpret_cast<const float4*>(P + (size_t)row * ldp);
    const float4* pb = reinterpret_cast<const float4*>(P + (size_t)(two ? row + 1 : row) * ldp);
    float2 acc[2][QT];
#pragma unroll
    for (int q = 0; q < QT; ++q) { acc[0][q] = make_float2(0.f, 0.f); acc[1][q] = make_float2(0.f, 0.f); }
    int c = lane;
    for (; c + 96 < D4; c += 128) {                              // 8 independent 16-byte loads in flight per lane
      float4 a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { a[u] = __ldg(pa + c + 32 * u); b[u] = __ldg(pb + c + 32 * u); }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
#pragma unroll
        for (int q = 0; q < QT; ++q) {
          const float4 x = q4[q * D4 + c + 32 * u];
          acc[0][q] = fma2(a[u], x, acc[0][q]);
          acc[1][q] = fma2(b[u], x, acc[1][q]);
        }
      }
    }
    for (; c < D4; c += 32) {
      const float4 a = __ldg(pa + c), b = __ldg(pb + c);
#pragma unroll
      for (int q = 0; q < QT; ++q) {
        const float4 x = q4[q * D4 + c];
        acc[0][q] = fma2(a, x, acc[0][q]);
        acc[1][q] = fma2(b, x, acc[1][q]);
      }
    }
    reduce_and_insert<QT>(acc, bs, bi, mythr, row, two ? 2 : 1, K, lane);
  }
  // CTA merge: warps publish their lists; one warp per query folds them (sorted lists: stop at the first miss)
  __syncthreads();
  float* ms = smem;                                             // reuse: [nwarps][QT][32] scores + indices
  int* mi = reinterpret_cast<int*>(smem + nwarps * QT * 32);
#pragma unroll
  for (int q = 0; q < QT; ++q) { ms[(warp * QT + q) * 32 + lane] = bs[q]; mi[(warp * QT + q) * 32 + lane] = bi[q]; }
  __syncthreads();
  if (warp < nqt) {                                             // one warp per query of the tile folds the 8 warp lists
    const int q = warp;
    float s = ms[(0 * QT + q) * 32 + lane]; int i = mi[(0 * QT + q) * 32 + lane];
    for (int w = 1; w < nwarps; ++w) warp_merge_list(s, i, ms[(w * QT + q) * 32 + lane], mi[(w * QT + q) * 32 + lane], K, lane);
    if (lane < K) {
      const size_t o = ((size_t)blockIdx.x * nq + (q0 + q)) * K + lane;
      cand_s[o] = s; cand_i[o] = i;
    }
  }
}

// Pipelined variant (D <= kTopkPipeMaxD): every warp owns a 2-slot shared-memory ring of R = 2 passage rows; lanes stream
// the NEXT 2 rows in with 16-byte cp.async while the warp computes on the current 2 from shared memory (no CTA-wide
// barrier: a warp only waits for its own copies). ncu of the register-load version above showed 16 warps/SM stalled on
// their own global loads: the loads of a warp were only in
// flight while it was not computing. Here 8 warps x 8 KB stay in flight per SM for the whole sweep (160 KB of shared
// memory at D = 1024: one CTA per SM).
constexpr int kTopkPipeMaxD = 1024;
constexpr int kTopkR = 2;
constexpr int kTopkPipeWarps = 8;   // 8 warps x 2 slots x 2 rows x 4 KB + the 32 KB query tile = 160 KB at D = 1024
__device__ __forceinline__ void cp_async16_topk(void* smem, const void* gmem) {
  const uint32_t sa = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem) : "memory");
}
template <int QT>
__global__ void __launch_bounds__(kTopkPipeWarps * 32, 1) topk_scan_pipe_kernel(const float* __restrict__ Q, const float* __restrict__ P, long long ldp,
                                                                int nq, int N, int D, int K, float* __restrict__ cand_s,
                                                                int* __restrict__ cand_i) {
  extern __shared__ float smem[];                               // [QT][D] queries | per warp: [2 slots][R rows][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int q0 = blockIdx.y * QT;
  const int nqt = min(QT, nq - q0);
  for (int t = threadIdx.x; t < QT * D; t += blockDim.x) {
    const int q = t / D, d = t - q * D;
    smem[t] = q < nqt ? Q[(size_t)(q0 + q) * D + d] : 0.f;
  }
  __syncthreads();
  const int D4 = D >> 2;
  const float4* q4 = reinterpret_cast<const float4*>(smem);
  float4* ring = reinterpret_cast<float4*>(smem + QT * D) + (size_t)warp * 2 * kTopkR * D4;
  float bs[QT]; int bi[QT];
#pragma unroll
  for (int q = 0; q < QT; ++q) { bs[q] = -INFINITY; bi[q] = 0x7fffffff; }
  float mythr = -INFINITY;
  static_assert(kTopkR == 2, "reduce_and_insert handles two rows per step");
  const int step = gridDim.x * nwarps * kTopkR;
  auto issue = [&](int row0, int slot) {
    if (row0 < N) {
#pragma unroll
      for (int r = 0; r < kTopkR; ++r) {
        const int row = min(row0 + r, N - 1);                   // tail: re-read the last row, ignored below
        const float4* src = reinterpret_cast<const float4*>(P + (size_t)row * ldp);
        float4* dst = ring + (size_t)(slot * kTopkR + r) * D4;
        for (int c = lane; c < D4; c += 32) cp_async16_topk(dst + c, src + c);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  int row0 = (blockIdx.x * nwarps + warp) * kTopkR, slot = 0;
  issue(row0, 0);
  for (; row0 < N; row0 += step, slot ^= 1) {
    issue(row0 + step, slot ^ 1);                               // prefetch the next group into the other slot
    asm volatile("cp.async.wait_group 1;" ::: "memory");        // this slot's copies (this lane's) have landed
    __syncwarp();                                               // ... and every other lane's
    const float4* base = ring + (size_t)slot * kTopkR * D4;
    float2 acc[kTopkR][QT];
#pragma unroll
    for (int r = 0; r < kTopkR; ++r)
#pragma unroll
      for (int q = 0; q < QT; ++q) acc[r][q] = make_float2(0.f, 0.f);
#pragma unroll 2
    for (int c = lane; c < D4; c += 32) {
      const float4 pa = base[c], pb = base[D4 + c];
#pragma unroll
      for (int q = 0; q < QT; ++q) {
        const float4 x = q4[q * D4 + c];
        acc[0][q] = fma2(pa, x, acc[0][q]);
        acc[1][q] = fma2(pb, x, acc[1][q]);
      }
    }
    reduce_and_insert<QT>(acc, bs, bi, mythr, row0, min(kTopkR, N - row0), K, lane);
    __syncwarp();                                               // all lanes are done reading this slot before it is refilled
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  float* ms = smem;                                             // reuse the query tile: [nwarps][QT][32] scores + indices
  int* mi = reinterpret_cast<int*>(smem + nwarps * QT * 32);
#pragma unroll
  for (int q = 0; q < QT; ++q) { ms[(warp * QT + q) * 32 + lane] = bs[q]; mi[(warp * QT + q) * 32 + lane] = bi[q]; }
  __syncthreads();
  for (int q = warp; q < nqt; q += nwarps) {
    float s = ms[(0 * QT + q) * 32 + lane]; int i = mi[(0 * QT + q) * 32 + lane];
    for (int w = 1; w < nwarps; ++w) warp_merge_list(s, i, ms[(w * QT + q) * 32 + lane], mi[(w * QT + q) * 32 + lane], K, lane);
    if (lane < K) {
      const size_t o = ((size_t)blockIdx.x * nq + (q0 + q)) * K + lane;
      cand_s[o] = s; cand_i[o] = i;
    }
  }
}

// one CTA (8 warps) per query: each warp folds every 8th per-CTA candidate list (one coalesced load per list: lane j reads
// entry j), warp 0 folds the 8 partial results
__global__ void __launch_bounds__(256) topk_merge_kernel(const float* __restrict__ cand_s, const int* __restrict__ cand_i, int ncta,
                                                         int nq, int K, float* __restrict__ out_s, int* __restrict__ out_i) {
  __shared__ float ps[8][32];
  __shared__ int pi[8][32];
  const int q = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float s = -INFINITY; int i = 0x7fffffff;
  for (int c = warp; c < ncta; c += 8) {
    const size_t o = ((size_t)c * nq + q) * K + lane;
    const float ls = lane < K ? cand_s[o] : -INFINITY;
    const int li = lane < K ? cand_i[o] : 0x7fffffff;
    warp_merge_list(s, i, ls, li, K, lane);
  }
  ps[warp][lane] = s; pi[warp][lane] = i;
  __syncthreads();
  if (warp == 0) {
    for (int w = 1; w < 8; ++w) warp_merge_list(s, i, ps[w][lane], pi[w][lane], K, lane);
    if (lane < K) {
      out_s[(size_t)q * K + lane] = s;
      out_i[(size_t)q * K + lane] = (s == -INFINITY) ? -1 : i;    // fewer than K passages: -1 padding
    }
  }
}

}  // namespace dalm

using namespace dalm;

// Queries go in chunks of kTopkChunk (2048 query tiles), so that the query tiles' grid.y stays far below its 65535 limit and the
// candidate workspace ([CTA][query][K] of one chunk, reused by the next) stays bounded for any nq: at most 1.1 GB at K = 32 on
// 132 SMs. Each query's result depends on its own row only, so the chunking changes no output bit.
constexpr int kTopkChunk = 16384;
// workspace the caller must provide: dalm_b200_topk_ip_workspace(nq, K) bytes
static int topk_grid_x() { return 2 * num_sms(); }
extern "C" long long dalm_b200_topk_ip_workspace(int nq, int K) {
  return (long long)topk_grid_x() * (nq < kTopkChunk ? nq : kTopkChunk) * K * (long long)(sizeof(float) + sizeof(int));
}

// out_scores [nq,K] fp32 (inner products, descending), out_idx [nq,K] int32 (passage rows; -1 past the end when N < K).
// Q [nq,D] fp32 dense; P [N,D] fp32 with row stride ldp (elements). D % 4 == 0, 1 <= K <= 32.
extern "C" int dalm_b200_topk_ip(const float* Q, const float* P, long long ldp, int nq, int N, int D, int K, float* out_scores,
                                 int* out_idx, void* workspace, void* stream) {
  DALM_REQUIRE(nq > 0 && N > 0 && D > 0 && (D % 4) == 0, "topk_ip: bad shape nq=%d N=%d D=%d (D must be a multiple of 4)", nq, N, D);
  DALM_REQUIRE(K >= 1 && K <= kTopkMaxK, "topk_ip: K=%d must be in [1,%d]", K, kTopkMaxK);
  DALM_REQUIRE((ldp % 4) == 0 && ldp >= D, "topk_ip: ldp=%lld must be a multiple of 4 and >= D", ldp);
  DALM_REQUIRE((reinterpret_cast<uintptr_t>(P) & 15) == 0 && (reinterpret_cast<uintptr_t>(Q) & 15) == 0, "topk_ip: operands must be 16-byte aligned");
  DALM_REQUIRE(workspace != nullptr, "topk_ip: workspace is NULL (size it with dalm_b200_topk_ip_workspace)");
  const int nwarps = 8;
  const int nq_max = nq < kTopkChunk ? nq : kTopkChunk;
  float* cs = reinterpret_cast<float*>(workspace);
  int* ci = reinterpret_cast<int*>(cs + (size_t)topk_grid_x() * nq_max * K);
  static bool attr_set = false;
  if (!attr_set) {
    DALM_CUDA(cudaFuncSetAttribute(topk_scan_kernel<kTopkQT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    DALM_CUDA(cudaFuncSetAttribute(topk_scan_pipe_kernel<kTopkQT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
    attr_set = true;
  }
  int gx;
  size_t smem;
  const size_t smem_m = (size_t)nwarps * kTopkQT * 32 * (sizeof(float) + sizeof(int));
  const size_t smem_pipe = (size_t)(kTopkQT + kTopkPipeWarps * 2 * kTopkR) * D * sizeof(float);
  const bool pipe = D <= kTopkPipeMaxD && smem_pipe >= smem_m;
  if (pipe) {
    // pipelined sweep: one CTA per SM (its rings take most of the shared memory), 2 rows per warp step
    gx = smem_pipe * 2 <= 200 * 1024 ? 2 * num_sms() : num_sms();   // small D: two CTAs per SM keep enough bytes in flight
    const int max_gx = (N + kTopkR * kTopkPipeWarps - 1) / (kTopkR * kTopkPipeWarps);
    if (gx > max_gx) gx = max_gx;
    smem = smem_pipe;
  } else {
    gx = topk_grid_x();
    const int max_gx = (N + 2 * nwarps - 1) / (2 * nwarps);
    if (gx > max_gx) gx = max_gx;
    const size_t smem_q = (size_t)kTopkQT * D * sizeof(float);
    smem = smem_q > smem_m ? smem_q : smem_m;
    DALM_REQUIRE(smem <= 200 * 1024, "topk_ip: D=%d too large for the query tile in shared memory", D);
  }
  for (int q0 = 0; q0 < nq; q0 += kTopkChunk) {
    const int n = nq - q0 < kTopkChunk ? nq - q0 : kTopkChunk;
    const float* Qc = Q + (size_t)q0 * D;
    dim3 grid(gx, (n + kTopkQT - 1) / kTopkQT);
    if (pipe) {
      topk_scan_pipe_kernel<kTopkQT><<<grid, kTopkPipeWarps * 32, smem, (cudaStream_t)stream>>>(Qc, P, ldp, n, N, D, K, cs, ci);
      count_launch();
      if (int e = check_launch("topk_scan_pipe_kernel")) return e;
    } else {
      topk_scan_kernel<kTopkQT><<<grid, nwarps * 32, smem, (cudaStream_t)stream>>>(Qc, P, ldp, n, N, D, K, cs, ci);
      count_launch();
      if (int e = check_launch("topk_scan_kernel")) return e;
    }
    topk_merge_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(cs, ci, gx, n, K, out_scores + (size_t)q0 * K, out_idx + (size_t)q0 * K);
    count_launch();
    if (int e = check_launch("topk_merge_kernel")) return e;
  }
  return 0;
}
