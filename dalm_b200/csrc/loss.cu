// dalm_b200 — loss kernels of the RAG-e2e / retriever-only training step.
//
//  * inbatch_loss_kernel : fused  S = scale * Q P^T  -> two-way contrastive cross-entropy (rows and columns)
//                          -> doc log-prob diag(log_softmax(S,1)) -> marginalisation coupling term
//                          -> dS -> dQ, dP, all in ONE cooperative launch.
//                          Replaces get_cosine_sim + 2x get_nt_xent_loss + the doc_logprobs part of
//                          compute_marginalized_loss_from_logits (reference dalm/training/utils/train_utils.py:76-88,124)
//                          and their autograd backward.
//  * marginal_counts_kernel : c_b = sum_t m[b,t+1] * [t >= qlen_b - 1],  N = sum m[:,1:]
//                          (the slicing of marginalize_log_probs, train_utils.py:96-110, reduced to counts)
//  * ce_rows_kernel      : per (b,t) row: log_softmax over the vocabulary, gather at ids[b,t+1], masked token-mean
//                          weights, and dlogits = m/N (softmax - onehot) in the same pass
//                          (train_utils.py:113-138 + autograd).
//  * finalize_loss_kernel: deterministic reduction of the per-token log-probs into Lm and the total loss.
#include "common.cuh"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace dalm {

// ------------------------------------------------------------------------------------------------------------
// marginal counts
// ------------------------------------------------------------------------------------------------------------
// grid = 1 block; B*L is tiny (4608 at cfg-3, 36864 at cfg-5).
__global__ void marginal_counts_kernel(const int64_t* __restrict__ mask, const int64_t* __restrict__ qlen, int B, int L,
                                       float* __restrict__ cvec, float* __restrict__ nsum) {
  __shared__ float red[32];
  float n_total = 0.f;
  for (int b = 0; b < B; ++b) {
    const int64_t q = qlen[b];
    // python slice semantics of logprobs[q-1:] on a length L-1 sequence (train_utils.py:101-104):
    // start = q-1; negative start wraps (q<=0 never occurs: BOS => q>=1); start > L-1 => empty.
    int64_t start = q - 1;
    if (start < 0) { start += (L - 1); if (start < 0) start = 0; }
    float c = 0.f, n = 0.f;
    for (int t = threadIdx.x; t < L - 1; t += blockDim.x) {
      const float m = (float)mask[(size_t)b * L + t + 1];
      n += m;
      if (t >= start) c += m;
    }
    c = block_sum(c, red);
    n = block_sum(n, red);
    if (threadIdx.x == 0) cvec[b] = c;
    n_total += n;
  }
  if (threadIdx.x == 0) nsum[0] = n_total;
}

// ------------------------------------------------------------------------------------------------------------
// fused in-batch similarity + contrastive CE + marginalisation coupling, forward and backward
// ------------------------------------------------------------------------------------------------------------
struct InbatchParams {
  const float* Q;        // [B,D] fp32 query embeddings (L2-normalised upstream)
  const float* P;        // [B,D] fp32 passage embeddings
  int B, D;
  float scale;           // logit_scale
  const float* cvec;     // [B] or nullptr (retriever-only: no marginal term)
  const float* nsum;     // [1] or nullptr
  float* S;              // [B,B] out
  float* dlp;            // [B]   out: log_softmax(S, dim=1).diag()
  float* losses;         // [4]   out: {Lc, doc_term, Lc+doc_term, N}
  float* dQ;             // [B,D] out (may be nullptr -> forward only)
  float* dP;             // [B,D] out
  float gout;            // upstream gradient of the scalar loss (1.0 in the trainers)
};

// dynamic smem layout: qrow[D] | rowlse[B] | collse[B] | wrow[B] | wcol[B] | red[32]
__global__ void __launch_bounds__(256) inbatch_loss_kernel(InbatchParams p) {
  extern __shared__ float smem[];
  const int B = p.B, D = p.D;
  float* qrow   = smem;
  float* rowlse = qrow + D;
  float* collse = rowlse + B;
  float* wrow   = collse + B;
  float* wcol   = wrow + B;
  float* red    = wcol + B;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nwarp = blockDim.x >> 5;
  cg::grid_group grid = cg::this_grid();

  // ---- phase 1: S[i,:] for the rows this CTA owns (one warp per (i,j) dot product, float4 coalesced) ----
  // float4 loads of P need D % 4 == 0 and a 16-byte aligned P (a contiguous view may start anywhere); Q is staged through
  // shared memory with scalar loads. Uniform over the grid.
  const bool vec_p = (D & 3) == 0 && (reinterpret_cast<uintptr_t>(p.P) & 15) == 0;
  for (int i = blockIdx.x; i < B; i += gridDim.x) {
    __syncthreads();
    for (int d = tid; d < D; d += blockDim.x) qrow[d] = p.Q[(size_t)i * D + d];
    __syncthreads();
    for (int j = wid; j < B; j += nwarp) {
      const float* prow = p.P + (size_t)j * D;
      float acc = 0.f;
      if (vec_p) {
        const float4* p4 = reinterpret_cast<const float4*>(prow);
        const float4* q4 = reinterpret_cast<const float4*>(qrow);
        for (int d = lane; d < (D >> 2); d += 32) {
          const float4 a = q4[d], b = __ldg(p4 + d);
          acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
          acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
        }
      } else {
        for (int d = lane; d < D; d += 32) acc = fmaf(qrow[d], __ldg(prow + d), acc);
      }
      acc = warp_sum(acc);
      if (lane == 0) p.S[(size_t)i * B + j] = acc * p.scale;
    }
  }
  __threadfence();
  grid.sync();

  // ---- phase 2: every CTA recomputes all row / column log-sum-exps (B^2 exps, S is L2 resident) ----
  for (int r = wid; r < B; r += nwarp) {                       // rows: coalesced along j
    const float* srow = p.S + (size_t)r * B;
    float mx = -INFINITY;
    for (int j = lane; j < B; j += 32) mx = fmaxf(mx, srow[j]);
    mx = warp_max(mx);
    float s = 0.f;
    for (int j = lane; j < B; j += 32) s += __expf(srow[j] - mx);
    s = warp_sum(s);
    if (lane == 0) rowlse[r] = mx + __logf(s);
  }
  for (int c = tid; c < B; c += blockDim.x) {                  // columns: thread per column, coalesced along c
    float mx = -INFINITY;
    for (int r = 0; r < B; ++r) mx = fmaxf(mx, p.S[(size_t)r * B + c]);
    float s = 0.f;
    for (int r = 0; r < B; ++r) s += __expf(p.S[(size_t)r * B + c] - mx);
    collse[c] = mx + __logf(s);
  }
  __syncthreads();

  const bool has_marg = (p.cvec != nullptr);
  const float N = has_marg ? p.nsum[0] : 1.f;
  const float invN = has_marg ? 1.f / N : 0.f;
  const float inv2B = 0.5f / (float)B;

  // ---- losses + doc log-probs: CTA 0 only, fixed summation order (deterministic) ----
  if (blockIdx.x == 0) {
    float lc = 0.f, doc = 0.f;
    for (int i = tid; i < B; i += blockDim.x) {
      const float sii = p.S[(size_t)i * B + i];
      const float d = sii - rowlse[i];
      p.dlp[i] = d;
      lc += -(d + (sii - collse[i]));
      if (has_marg) doc += -p.cvec[i] * d;
    }
    lc = block_sum(lc, red) * inv2B;
    doc = block_sum(doc, red) * invN;
    if (tid == 0) {
      p.losses[0] = lc;
      p.losses[1] = has_marg ? doc : 0.f;
      p.losses[2] = lc + (has_marg ? doc : 0.f);
      p.losses[3] = has_marg ? N : 0.f;
    }
  }
  if (p.dQ == nullptr) return;

  // ---- phase 3: dS row i and dS column i, then dQ[i,:] = scale * dS[i,:] P, dP[i,:] = scale * dS[:,i]^T Q ----
  for (int i = blockIdx.x; i < B; i += gridDim.x) {
    __syncthreads();
    for (int j = tid; j < B; j += blockDim.x) {
      const float kd = (i == j) ? 1.f : 0.f;
      {  // dS[i,j]
        const float s = p.S[(size_t)i * B + j];
        const float pr = __expf(s - rowlse[i]), pc = __expf(s - collse[j]);
        float g = inv2B * ((pr - kd) + (pc - kd));
        if (has_marg) g += p.cvec[i] * invN * (pr - kd);
        wrow[j] = g * p.gout * p.scale;
      }
      {  // dS[j,i]
        const float s = p.S[(size_t)j * B + i];
        const float pr = __expf(s - rowlse[j]), pc = __expf(s - collse[i]);
        float g = inv2B * ((pr - kd) + (pc - kd));
        if (has_marg) g += p.cvec[j] * invN * (pr - kd);
        wcol[j] = g * p.gout * p.scale;
      }
    }
    __syncthreads();
    for (int d = tid; d < D; d += blockDim.x) {
      float aq = 0.f, ap = 0.f;
#pragma unroll 4
      for (int j = 0; j < B; ++j) {
        aq = fmaf(wrow[j], __ldg(p.P + (size_t)j * D + d), aq);
        ap = fmaf(wcol[j], __ldg(p.Q + (size_t)j * D + d), ap);
      }
      p.dQ[(size_t)i * D + d] = aq;
      p.dP[(size_t)i * D + d] = ap;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// cross-entropy over the vocabulary with marginalisation weights; forward + backward in one pass
// ------------------------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

struct CeParams {
  const void* logits;      // [B*L, ldl] (T)
  void* dlogits;           // [B*L, ldl] (T) out, may alias logits; nullptr -> forward only
  const int64_t* ids;      // [B,L]
  const int64_t* mask;     // [B,L]
  const float* nsum;       // [1]  N = sum(mask[:,1:])
  float* tok_lp;           // [B,L] out: log p(ids[b,t+1] | ...) at (b,t), 0 where t = L-1
  int B, L, V;
  int64_t ldl;             // row stride in elements
  float gout;
  int cache_in_smem;       // 1: row staged in shared memory (V * sizeof(T) bytes)
  int row0;                // first (b*L + t) row of this launch: `logits` / `dlogits` point at that row (row-chunked lm_head + CE)
};

// one CTA per (b,t) row. bf16 rows are staged in shared memory (64 KB at V=32000) so HBM sees each logit once on
// the read side and once on the write side.
template <typename T>
__global__ void __launch_bounds__(512) ce_rows_kernel(CeParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float red[32];
  T* row_s = reinterpret_cast<T*>(smem_raw);
  const int row = p.row0 + blockIdx.x;        // = b*L + t
  const int b = row / p.L, t = row - b * p.L;
  const T* x = reinterpret_cast<const T*>(p.logits) + (size_t)blockIdx.x * p.ldl;
  T* dx = p.dlogits ? reinterpret_cast<T*>(p.dlogits) + (size_t)blockIdx.x * p.ldl : nullptr;
  const int V = p.V, tid = threadIdx.x, nt = blockDim.x;
  // 16-byte loads / stores need whole vectors per row and 16-byte aligned rows: ldl, V and both base pointers (a view such
  // as logits[..., 1:] keeps a padded ldl but starts mid-vector). Uniform over the grid.
  constexpr int VEC = 16 / sizeof(T);
  const bool vec_ok = (p.ldl % VEC) == 0 && (V % VEC) == 0 &&
                      ((reinterpret_cast<uintptr_t>(p.logits) | reinterpret_cast<uintptr_t>(p.dlogits)) & 15) == 0;

  float w = 0.f;
  int64_t label = -1;
  if (t < p.L - 1) {
    w = (float)p.mask[(size_t)b * p.L + t + 1];
    label = p.ids[(size_t)b * p.L + t + 1];
  }
  // masked rows (and the last position) contribute neither loss nor gradient: skip the read entirely.
  // NOTE: the reference still evaluates lp there but multiplies by mask 0 (train_utils.py:135).
  if (w == 0.f) {
    if (tid == 0) p.tok_lp[row] = 0.f;
    if (dx) {
      if (vec_ok) {
        uint4 z = make_uint4(0, 0, 0, 0);
        uint4* d4 = reinterpret_cast<uint4*>(dx);
        for (int i = tid; i < V / VEC; i += nt) d4[i] = z;
      } else {
        for (int i = tid; i < V; i += nt) dx[i] = from_f<T>(0.f);
      }
    }
    return;
  }

  const bool cache = p.cache_in_smem != 0;

  // ---- pass 1: stream the row (HBM -> smem), running max ----
  float mx = -INFINITY;
  if (vec_ok) {
    const uint4* x4 = reinterpret_cast<const uint4*>(x);
    uint4* s4 = reinterpret_cast<uint4*>(row_s);
    for (int i = tid; i < V / VEC; i += nt) {
      const uint4 v = __ldg(x4 + i);
      if (cache) s4[i] = v;
      const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int k = 0; k < VEC; ++k) mx = fmaxf(mx, to_f<T>(e[k]));
    }
  } else {
    for (int i = tid; i < V; i += nt) {
      const T v = x[i];
      if (cache) row_s[i] = v;
      mx = fmaxf(mx, to_f<T>(v));
    }
  }
  mx = block_max(mx, red);
  const T* src = cache ? row_s : x;

  // ---- pass 2 (on-chip when cached): sum of exponentials ----
  float s = 0.f;
  if (vec_ok) {
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    for (int i = tid; i < V / VEC; i += nt) {
      const uint4 v = s4[i];
      const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int k = 0; k < VEC; ++k) s += __expf(to_f<T>(e[k]) - mx);
    }
  } else {
    for (int i = tid; i < V; i += nt) s += __expf(to_f<T>(src[i]) - mx);
  }
  s = block_sum(s, red);
  const float lse = mx + __logf(s);
  const bool label_ok = (label >= 0 && label < V);
  const float xl = label_ok ? to_f<T>(src[label]) : 0.f;
  if (tid == 0) p.tok_lp[row] = xl - lse;
  if (!dx) return;

  // ---- pass 3: dlogits = gout * w/N * (softmax - onehot) ----
  const float coef = p.gout * w / p.nsum[0];
  __syncthreads();       // everyone has read src[label] before an in-place overwrite of x (non-cached aliasing case)
  if (vec_ok) {
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(dx);
    for (int i = tid; i < V / VEC; i += nt) {
      const uint4 v = s4[i];
      const T* e = reinterpret_cast<const T*>(&v);
      uint4 o;
      T* oe = reinterpret_cast<T*>(&o);
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        const int col = i * VEC + k;
        float g = __expf(to_f<T>(e[k]) - lse);
        if (col == (int)label) g -= 1.f;
        oe[k] = from_f<T>(g * coef);
      }
      d4[i] = o;
    }
  } else {
    for (int i = tid; i < V; i += nt) {
      float g = __expf(to_f<T>(src[i]) - lse);
      if (i == (int)label) g -= 1.f;
      dx[i] = from_f<T>(g * coef);
    }
  }
}

// Lm_tok = -sum(mask[:,1:] * tok_lp[:, :-1]) / N ; total = Lc + doc + Lm_tok.   single block, fixed order.
__global__ void finalize_loss_kernel(const float* __restrict__ tok_lp, const int64_t* __restrict__ mask, int B, int L,
                                     const float* __restrict__ nsum, const float* __restrict__ inbatch_losses,
                                     float* __restrict__ out /* [4]: Lc, Lm, total, N */) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int i = threadIdx.x; i < B * L; i += blockDim.x) {
    const int t = i % L;
    if (t < L - 1) acc += (float)mask[i + 1] * tok_lp[i];
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) {
    const float N = nsum[0];
    const float lm_tok = -acc / N;
    const float lc = inbatch_losses ? inbatch_losses[0] : 0.f;
    const float doc = inbatch_losses ? inbatch_losses[1] : 0.f;
    out[0] = lc;
    out[1] = lm_tok + doc;
    out[2] = lc + lm_tok + doc;
    out[3] = N;
  }
}

}  // namespace dalm

// ============================================================================================================
// C ABI
// ============================================================================================================
using namespace dalm;

extern "C" int dalm_b200_marginal_counts(const int64_t* gen_mask, const int64_t* qlen, int B, int L, float* cvec,
                                         float* nsum, void* stream) {
  DALM_REQUIRE(B > 0 && L > 1, "marginal_counts: need B>0, L>1 (got B=%d L=%d)", B, L);
  marginal_counts_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(gen_mask, qlen, B, L, cvec, nsum);
  count_launch();
  return check_launch("marginal_counts_kernel");
}

extern "C" int dalm_b200_inbatch_loss_fwd_bwd(const float* Q, const float* P, int B, int D, float logit_scale,
                                              const float* cvec, const float* nsum, float* S, float* dlp,
                                              float* losses, float* dQ, float* dP, float grad_out, void* stream) {
  DALM_REQUIRE(B > 0 && D > 0, "inbatch_loss: empty batch (B=%d D=%d)", B, D);
  DALM_REQUIRE((cvec == nullptr) == (nsum == nullptr), "inbatch_loss: cvec and nsum must both be given or both null");
  DALM_REQUIRE((dQ == nullptr) == (dP == nullptr), "inbatch_loss: dQ and dP must both be given or both null");
  InbatchParams p{Q, P, B, D, logit_scale, cvec, nsum, S, dlp, losses, dQ, dP, grad_out};
  const size_t smem = (size_t)(D + 4 * B + 32) * sizeof(float);
  DALM_REQUIRE(smem <= 200 * 1024, "inbatch_loss: B=%d D=%d needs %zu B of shared memory", B, D, smem);
  static bool attr_set = false;
  if (!attr_set) {
    DALM_CUDA(cudaFuncSetAttribute(inbatch_loss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  const int grid = B < num_sms() ? B : num_sms();     // co-resident by construction (<= 1 CTA per SM)
  void* args[] = {&p};
  DALM_CUDA(cudaLaunchCooperativeKernel((void*)inbatch_loss_kernel, dim3(grid), dim3(256), args, smem,
                                        (cudaStream_t)stream));
  count_launch();
  return check_launch("inbatch_loss_kernel");
}

// rows [row0, row0 + nrows) of the flattened [B*L] token rows; `logits` / `dlogits` point at row `row0` (their own buffer may
// hold just that chunk). tok_lp stays the whole [B,L] table (written at the global row index).
extern "C" int dalm_b200_ce_marginal_rows(const void* logits, void* dlogits, int dtype /*0=bf16,1=f32*/,
                                          const int64_t* ids, const int64_t* mask, const float* nsum,
                                          float* tok_lp, int B, int L, int V, int64_t ld, float grad_out,
                                          int row0, int nrows, void* stream) {
  DALM_REQUIRE(B > 0 && L > 1 && V > 0, "ce_marginal: bad shape B=%d L=%d V=%d", B, L, V);
  DALM_REQUIRE(dtype == 0 || dtype == 1, "ce_marginal: dtype must be 0 (bf16) or 1 (f32)");
  DALM_REQUIRE(ld >= V, "ce_marginal: ld < V");
  DALM_REQUIRE(row0 >= 0 && nrows > 0 && (long long)row0 + nrows <= (long long)B * L,
               "ce_marginal: rows [%d, %d + %d) outside the %d x %d token rows", row0, row0, nrows, B, L);
  CeParams p{logits, dlogits, ids, mask, nsum, tok_lp, B, L, V, ld, grad_out, 1, row0};
  const size_t esz = dtype == 0 ? 2 : 4;
  size_t smem = (size_t)V * esz;
  smem = (smem + 15) & ~size_t(15);
  if (smem > 200 * 1024) { p.cache_in_smem = 0; smem = 0; }
  static bool attr_set[2] = {false, false};
  if (!attr_set[dtype]) {
    if (dtype == 0)
      DALM_CUDA(cudaFuncSetAttribute(ce_rows_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    else
      DALM_CUDA(cudaFuncSetAttribute(ce_rows_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set[dtype] = true;
  }
  if (dtype == 0) ce_rows_kernel<__nv_bfloat16><<<nrows, 512, smem, (cudaStream_t)stream>>>(p);
  else            ce_rows_kernel<float><<<nrows, 512, smem, (cudaStream_t)stream>>>(p);
  count_launch();
  return check_launch("ce_rows_kernel");
}

extern "C" int dalm_b200_ce_marginal_fwd_bwd(const void* logits, void* dlogits, int dtype /*0=bf16,1=f32*/,
                                             const int64_t* ids, const int64_t* mask, const float* nsum,
                                             float* tok_lp, int B, int L, int V, int64_t ld, float grad_out,
                                             void* stream) {
  DALM_REQUIRE(B > 0 && L > 1, "ce_marginal: bad shape B=%d L=%d V=%d", B, L, V);
  return dalm_b200_ce_marginal_rows(logits, dlogits, dtype, ids, mask, nsum, tok_lp, B, L, V, ld, grad_out, 0, B * L, stream);
}

extern "C" int dalm_b200_finalize_loss(const float* tok_lp, const int64_t* mask, int B, int L, const float* nsum,
                                       const float* inbatch_losses, float* out4, void* stream) {
  finalize_loss_kernel<<<1, 512, 0, (cudaStream_t)stream>>>(tok_lp, mask, B, L, nsum, inbatch_losses, out4);
  count_launch();
  return check_launch("finalize_loss_kernel");
}

// ------------------------------------------------------------------------------------------------------------
// small fp32 matmul for the stand-alone (non-fused) API functions: get_cosine_sim forward/backward on [B,D] x [B,D]
// (reference train_utils.py:76-77). C[M,N] = alpha * opA(A)[M,K] * opB(B)[K,N]; row-major; 16x16 smem tiles.
// ------------------------------------------------------------------------------------------------------------
namespace dalm {
__global__ void small_matmul_f32_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C,
                                        int M, int N, int K, int transA, int transB, float alpha) {
  __shared__ float sa[16][17], sb[16][17];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int row = blockIdx.y * 16 + ty, col = blockIdx.x * 16 + tx;
  float acc = 0.f;
  for (int k0 = 0; k0 < K; k0 += 16) {
    const int ka = k0 + tx, kb = k0 + ty;
    sa[ty][tx] = (row < M && ka < K) ? (transA ? A[(size_t)ka * M + row] : A[(size_t)row * K + ka]) : 0.f;
    sb[ty][tx] = (kb < K && col < N) ? (transB ? B[(size_t)col * K + kb] : B[(size_t)kb * N + col]) : 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc = fmaf(sa[ty][k], sb[k][tx], acc);
    __syncthreads();
  }
  if (row < M && col < N) C[(size_t)row * N + col] = acc * alpha;
}
}  // namespace dalm

extern "C" int dalm_b200_small_matmul_f32(const float* A, const float* B, float* C, int M, int N, int K, int transA,
                                          int transB, float alpha, void* stream) {
  DALM_REQUIRE(M > 0 && N > 0 && K > 0, "small_matmul: empty problem");
  dim3 grid((N + 15) / 16, (M + 15) / 16), block(16, 16);
  dalm::small_matmul_f32_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(A, B, C, M, N, K, transA, transB, alpha);
  dalm::count_launch();
  return dalm::check_launch("small_matmul_f32_kernel");
}
