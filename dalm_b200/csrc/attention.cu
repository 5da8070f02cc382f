// dalm_b200 — fused multi-head attention, forward and backward, for the encoder (bidirectional + key-padding mask,
// head_dim 32/64) and the decoder (causal + key-padding mask, head_dim 64/128, MHA / GQA / MQA).
//
// Replaces the attention inside HF BertModel / LlamaForCausalLM / FalconForCausalLM that the reference reaches through
// dalm/models/rag_e2e_base_model.py:93,105 and its autograd backward. Flash-style: scores never touch HBM; the forward
// stores only the per-row log-sum-exp, the backward recomputes P tile by tile.
//
// Two implementations of the same tiles:
//   * warp-level mma.sync (HMMA) kernels with ldmatrix-fed fragments: head_dim 32 (bge-small, cfg-1), and the independent
//     cross-check of the wgmma kernels (dalm_b200_attention_fwd / _bwd);
//   * Hopper wgmma kernels (dalm_b200_attention_tc_fwd / _bwd, head_dim 64 / 128: the training path of bge-large, Llama
//     and Falcon): operands staged by TMA into 128B-swizzled shared-memory tiles through mbarriers, every contraction one
//     warpgroup MMA, P / dS fed to the second contraction from registers. Same masks, softmax and dropout indexing.
//
//   forward : grid (ceil(L/64), Hq, B), 4 warps, each warp owns 16 query rows, KV streamed in 64-key tiles
//   dKdV    : grid (ceil(L/64), Hkv, B), each warp owns 16 keys, loops over the q heads of its group and 32-query tiles
//   dQ      : grid (ceil(L/64), Hq, B), each warp owns 16 queries, loops over 64-key tiles
#include "common.cuh"
#include "ptx.cuh"

namespace dalm {

struct AttnParams {
  const __nv_bfloat16* q; const __nv_bfloat16* k; const __nv_bfloat16* v;   // token-major: row = b*L + l
  long long ldq, ldk, ldv;          // row strides (elements); head h lives at column h*D (k/v: (h/group)*D)
  const int64_t* mask;              // [B,L] key-padding mask (1 keep / 0 drop) or nullptr
  __nv_bfloat16* o; long long ldo;  // [B*L, Hq*D]
  float* lse;                       // [B,Hq,L]
  // backward only
  const __nv_bfloat16* d_o; long long lddo;
  float* delta;                     // [B,Hq,L] rowsum(dO * O)
  __nv_bfloat16* dq; __nv_bfloat16* dk; __nv_bfloat16* dv;
  long long lddq, lddk, lddv;
  int B, L, Hq, Hkv;
  float scale;                      // 1/sqrt(D)
  int causal;
  DropCfg drop;                     // attention-probability dropout (BERT attention_probs_dropout_prob); p = 0 => off.
                                    // element index of P[b,h,i,j] = ((b*Hq + h)*L + i)*Lp + j, Lp = L rounded up to 8
                                    // (rows start on a Philox group of 8, so one call covers an 8-key MMA n-tile)
  int window;                       // sliding window (WIN instances only): query i sees key j iff i - window < j <= i
                                    // (causal) or |i - j| < window (bidirectional); the host clamps it to L, so tile
                                    // bounds computed from it cannot overflow
};

// ---------------------------------------------------------------- fragment helpers
__device__ __forceinline__ void ldsm_x4(uint32_t* r, const void* smem_ptr) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(smem_ptr));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t* r, const void* smem_ptr) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(smem_ptr));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
// D(16x8, f32) += A(16x16, bf16 row) * B(16x8, bf16 col)
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

// cooperative copy of a [ROWS x D] bf16 tile (global row stride ld) into padded smem (row stride D+8); rows >= nvalid
// are zero-filled. 16-byte vector accesses (D % 8 == 0, ld % 8 == 0, 16B-aligned base).
template <int ROWS, int D, int NT>
__device__ __forceinline__ void load_tile(__nv_bfloat16* s, const __nv_bfloat16* g, long long ld, int nvalid) {
  constexpr int CH = D / 8;
  for (int i = threadIdx.x; i < ROWS * CH; i += NT) {
    const int r = i / CH, c = i - r * CH;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < nvalid) v = __ldg(reinterpret_cast<const uint4*>(g + (size_t)r * ld + c * 8));
    *reinterpret_cast<uint4*>(s + r * (D + 8) + c * 8) = v;
  }
}

// A-operand fragments (16 rows x 16 cols at [row0, col0]) from a padded smem tile
template <int D>
__device__ __forceinline__ void load_a_frag(uint32_t* a, const __nv_bfloat16* s, int row0, int col0, int lane) {
  ldsm_x4(a, s + (row0 + (lane & 15)) * (D + 8) + col0 + ((lane >> 4) << 3));
}
// B-operand fragments for TWO adjacent n-tiles (16 "n" rows at n0) x one k-step (16 cols at k0), tile stored [n][k]:
//   b[0],b[1] -> n-tile n0 ; b[2],b[3] -> n-tile n0+8
template <int D>
__device__ __forceinline__ void load_b_frag_nk(uint32_t* b, const __nv_bfloat16* s, int n0, int k0, int lane) {
  ldsm_x4(b, s + (n0 + (lane & 7) + ((lane >> 4) << 3)) * (D + 8) + k0 + (((lane >> 3) & 1) << 3));
}
// B-operand fragments for TWO adjacent n-tiles (16 cols at n0) x one k-step (16 "k" rows at k0), tile stored [k][n]:
//   b[0],b[1] -> n-tile n0 ; b[2],b[3] -> n-tile n0+8
template <int D>
__device__ __forceinline__ void load_b_frag_kn(uint32_t* b, const __nv_bfloat16* s, int k0, int n0, int lane) {
  ldsm_x4_t(b, s + (k0 + (lane & 7) + (((lane >> 3) & 1) << 3)) * (D + 8) + n0 + ((lane >> 4) << 3));
}

// first key of the KV loop of the query tile at q0: 0 without a window, else the tile holding key q0 - window + 1 (the
// first key any of its queries sees, causal or not). Mirrored, it is also the first query tile a bidirectional window lets
// see the key tile at kv0. The loops end at the last key (query) the tile's last query (key) sees: q0 + BQ - 1 + window - 1
// without causal. Every range holds the tile's own diagonal, so it is never empty. A skipped tile would be fully masked for every query of the tile (corr = 1, p = 0
// in the online softmax), so starting later changes no bit of the result.
template <bool WIN, int BKV> __device__ __forceinline__ int win_begin(int q0, int window) {
  return WIN ? (max(0, q0 - window + 1) / BKV) * BKV : 0;
}
// ============================================================================================================
// forward
// ============================================================================================================
template <int D, bool DROP, bool WIN>
__global__ void __launch_bounds__(128) attn_fwd_kernel(AttnParams p) {
  constexpr int BQ = 64, BKV = 64, LDS = D + 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sK = sQ + BQ * LDS;
  __nv_bfloat16* sV = sK + BKV * LDS;
  float* sMask = reinterpret_cast<float*>(sV + BKV * LDS);      // [BKV] additive 0 / -inf

  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (p.Hq / p.Hkv);
  const int L = p.L, q0 = qb * BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t tok0 = (size_t)b * L;

  load_tile<BQ, D, 128>(sQ, p.q + (tok0 + q0) * p.ldq + (size_t)h * D, p.ldq, min(BQ, L - q0));

  float o_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float sl2 = p.scale * 1.4426950408889634f;               // scores are exponentiated in base 2
  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;       // the two query rows this thread holds

  const int kv_end = p.causal ? min(L, q0 + BQ) : WIN ? min(L, q0 + BQ - 1 + p.window) : L;
  for (int kv0 = win_begin<WIN, BKV>(q0, p.window); kv0 < kv_end; kv0 += BKV) {
    __syncthreads();                                            // previous tile fully consumed
    const int nvalid = min(BKV, L - kv0);
    load_tile<BKV, D, 128>(sK, p.k + (tok0 + kv0) * p.ldk + (size_t)hk * D, p.ldk, nvalid);
    load_tile<BKV, D, 128>(sV, p.v + (tok0 + kv0) * p.ldv + (size_t)hk * D, p.ldv, nvalid);
    if (threadIdx.x < BKV) {
      const int key = kv0 + threadIdx.x;
      bool keep = key < L;
      if (keep && p.mask) keep = p.mask[tok0 + key] != 0;
      sMask[threadIdx.x] = keep ? 0.f : -INFINITY;
    }
    __syncthreads();

    // ---- S = Q K^T (16 x 64 per warp) ----
    float s[BKV / 8][4];
#pragma unroll
    for (int i = 0; i < BKV / 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      uint32_t a[4];
      load_a_frag<D>(a, sQ, warp * 16, kk * 16, lane);
#pragma unroll
      for (int nt = 0; nt < BKV / 16; ++nt) {
        uint32_t bf[4];
        load_b_frag_nk<D>(bf, sK, nt * 16, kk * 16, lane);
        mma16816(s[2 * nt], a, bf[0], bf[1]);
        mma16816(s[2 * nt + 1], a, bf[2], bf[3]);
      }
    }
    // ---- mask + online softmax (base-2) ----
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kc = nt * 8 + t * 2 + (e & 1);
        const int qr = (e < 2) ? row_a : row_b;
        float val = s[nt][e] * sl2 + sMask[kc];
        if (p.causal && (kv0 + kc) > qr) val = -INFINITY;
        if (WIN && (kv0 + kc) <= qr - p.window) val = -INFINITY;
        if (WIN && (kv0 + kc) >= qr + p.window) val = -INFINITY;
        s[nt][e] = val;
        mx[e >> 1] = fmaxf(mx[e >> 1], val);
      }
    }
    float corr[2], mnew[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      mnew[r] = fmaxf(m_run[r], mx[r]);
      const float msafe = (mnew[r] == -INFINITY) ? 0.f : mnew[r];
      corr[r] = exp2f(m_run[r] - msafe);                        // m_run = -inf -> 0
      m_run[r] = mnew[r];
      mnew[r] = msafe;
    }
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f(s[nt][e] - mnew[e >> 1]);
        s[nt][e] = pv;
        rs[e >> 1] += pv;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
      rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
      l_run[r] = l_run[r] * corr[r] + rs[r];
    }
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      o_acc[i][0] *= corr[0]; o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1]; o_acc[i][3] *= corr[1];
    }
    if (DROP) {
      // dropout acts on the normalised probabilities; the row sum above used the un-dropped values.
      // one Philox call per (row, 8-key n-tile); this thread uses components t*2, t*2+1
      const unsigned long long dstream = drop_stream(p.drop);
      const unsigned long long rbase = ((unsigned long long)b * p.Hq + h) * L;
      const int lp8 = (L + 7) >> 3;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int qr = r == 0 ? row_a : row_b;
          float sc[8];
          drop_scale8(p.drop, dstream, (rbase + qr) * lp8 + ((kv0 >> 3) + nt), sc);
          float s0 = sc[0], s1 = sc[1];
#pragma unroll
          for (int j = 1; j < 4; ++j) if (t == j) { s0 = sc[2 * j]; s1 = sc[2 * j + 1]; }
          s[nt][2 * r] *= s0; s[nt][2 * r + 1] *= s1;
        }
      }
    }
    // ---- O += P V ----
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
      a[1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
      a[2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int nt = 0; nt < D / 16; ++nt) {
        uint32_t bf[4];
        load_b_frag_kn<D>(bf, sV, kk * 16, nt * 16, lane);
        mma16816(o_acc[2 * nt], a, bf[0], bf[1]);
        mma16816(o_acc[2 * nt + 1], a, bf[2], bf[3]);
      }
    }
  }

  // ---- normalise, write O and LSE (natural log of sum exp(scale * s)) ----
  const float inv_l[2] = {l_run[0] > 0.f ? 1.f / l_run[0] : 0.f, l_run[1] > 0.f ? 1.f / l_run[1] : 0.f};
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r == 0 ? row_a : row_b;
    if (row < L) {
      __nv_bfloat16* orow = p.o + (tok0 + row) * p.ldo + (size_t)h * D;
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt) {
        const uint32_t pk = pack_bf16(o_acc[nt][2 * r] * inv_l[r], o_acc[nt][2 * r + 1] * inv_l[r]);
        *reinterpret_cast<uint32_t*>(orow + nt * 8 + t * 2) = pk;
      }
      if (t == 0) {
        // fully masked row: +inf makes the backward's exp(s - lse) vanish
        const float lse = l_run[r] > 0.f ? (m_run[r] + log2f(l_run[r])) * 0.6931471805599453f : INFINITY;
        p.lse[((size_t)b * p.Hq + h) * L + row] = lse;
      }
    }
  }
}

// ============================================================================================================
// backward pre-pass: delta[b,h,i] = sum_d dO[i,d] * O[i,d]
// ============================================================================================================
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ o, long long ldo, const __nv_bfloat16* __restrict__ d_o,
                                  long long lddo, float* __restrict__ delta, int B, int L, int Hq, int D) {
  // one warp per (token, head)
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int total = B * L * Hq;
  if (gw >= total) return;
  const int tok = gw / Hq, h = gw - tok * Hq;
  const __nv_bfloat16* a = o + (size_t)tok * ldo + (size_t)h * D;
  const __nv_bfloat16* c = d_o + (size_t)tok * lddo + (size_t)h * D;
  float acc = 0.f;
  for (int d = lane * 2; d < D; d += 64) {
    const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(a + d));
    const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(c + d));
    acc += x.x * y.x + x.y * y.y;
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    const int b = tok / L, l = tok - b * L;
    delta[((size_t)b * Hq + h) * L + l] = acc;
  }
}

// ============================================================================================================
// backward: dK, dV.  Each warp owns 16 keys; queries streamed in 32-row tiles.
// ============================================================================================================
template <int D, bool DROP, bool WIN>
__global__ void __launch_bounds__(128) attn_bwd_dkv_kernel(AttnParams p) {
  constexpr int BKV = 64, BQ = 32, LDS = D + 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __nv_bfloat16* sK  = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sV  = sK + BKV * LDS;
  __nv_bfloat16* sQ  = sV + BKV * LDS;
  __nv_bfloat16* sdO = sQ + BQ * LDS;
  float* sLse   = reinterpret_cast<float*>(sdO + BQ * LDS);     // [BQ]
  float* sDelta = sLse + BQ;                                    // [BQ]
  float* sMask  = sDelta + BQ;                                  // [BKV]

  const int kb = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int group = p.Hq / p.Hkv;
  const int L = p.L, kv0 = kb * BKV;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t tok0 = (size_t)b * L;
  const float sl2 = p.scale * 1.4426950408889634f;

  const int nvalid_kv = min(BKV, L - kv0);
  load_tile<BKV, D, 128>(sK, p.k + (tok0 + kv0) * p.ldk + (size_t)hk * D, p.ldk, nvalid_kv);
  load_tile<BKV, D, 128>(sV, p.v + (tok0 + kv0) * p.ldv + (size_t)hk * D, p.ldv, nvalid_kv);
  if (threadIdx.x < BKV) {
    const int key = kv0 + threadIdx.x;
    bool keep = key < L;
    if (keep && p.mask) keep = p.mask[tok0 + key] != 0;
    sMask[threadIdx.x] = keep ? 0.f : -INFINITY;
  }

  float dk_acc[D / 8][4], dv_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) {
    dk_acc[i][0] = dk_acc[i][1] = dk_acc[i][2] = dk_acc[i][3] = 0.f;
    dv_acc[i][0] = dv_acc[i][1] = dv_acc[i][2] = dv_acc[i][3] = 0.f;
  }
  const int key_a = kv0 + warp * 16 + g, key_b = key_a + 8;     // the two keys (rows of S^T) this thread holds
  const int q_begin = p.causal ? (kv0 / BQ) * BQ : win_begin<WIN, BQ>(kv0, p.window);  // queries before it see none of it
  const int q_end = WIN ? min(L, kv0 + BKV - 1 + p.window) : L;  // nor do queries past its last key's window

  for (int hq = hk * group; hq < (hk + 1) * group; ++hq) {
    for (int q0 = q_begin; q0 < q_end; q0 += BQ) {
      __syncthreads();
      const int nq = min(BQ, L - q0);
      load_tile<BQ, D, 128>(sQ, p.q + (tok0 + q0) * p.ldq + (size_t)hq * D, p.ldq, nq);
      load_tile<BQ, D, 128>(sdO, p.d_o + (tok0 + q0) * p.lddo + (size_t)hq * D, p.lddo, nq);
      if (threadIdx.x < BQ) {
        const int qi = q0 + threadIdx.x;
        const size_t idx = ((size_t)b * p.Hq + hq) * L + qi;
        sLse[threadIdx.x]   = qi < L ? p.lse[idx] * 1.4426950408889634f : INFINITY;   // base-2 units
        sDelta[threadIdx.x] = qi < L ? p.delta[idx] : 0.f;
      }
      __syncthreads();

      // ---- S^T = K Q^T : 16 keys x 32 queries per warp ----
      float st[BQ / 8][4];
#pragma unroll
      for (int i = 0; i < BQ / 8; ++i) { st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        uint32_t a[4];
        load_a_frag<D>(a, sK, warp * 16, kk * 16, lane);
#pragma unroll
        for (int nt = 0; nt < BQ / 16; ++nt) {
          uint32_t bf[4];
          load_b_frag_nk<D>(bf, sQ, nt * 16, kk * 16, lane);
          mma16816(st[2 * nt], a, bf[0], bf[1]);
          mma16816(st[2 * nt + 1], a, bf[2], bf[3]);
        }
      }
      // ---- P^T = exp2(S^T * sl2 - lse2[q]) with masks ----
      const float mk_a = sMask[warp * 16 + g], mk_b = sMask[warp * 16 + g + 8];
#pragma unroll
      for (int nt = 0; nt < BQ / 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = nt * 8 + t * 2 + (e & 1);
          const int key = (e < 2) ? key_a : key_b;
          float val = st[nt][e] * sl2 + ((e < 2) ? mk_a : mk_b);
          if (p.causal && key > (q0 + qc)) val = -INFINITY;
          if (WIN && key <= (q0 + qc) - p.window) val = -INFINITY;
          if (WIN && key >= (q0 + qc) + p.window) val = -INFINITY;
          st[nt][e] = exp2f(val - sLse[qc]);                     // -inf - x -> 0 ; x - (+inf) -> 0
        }
      }
      // dropout scale of each (key, query) element this thread holds (1 when dropout is off)
      float ms[DROP ? BQ / 8 : 1][4];
      if (DROP) {
        const unsigned long long dstream = drop_stream(p.drop);
        const unsigned long long rbase = ((unsigned long long)b * p.Hq + hq) * L;
        const int lp8 = (L + 7) >> 3;
        const int kg = (kv0 >> 3) + warp * 2;                    // Philox group of key_a (key_b is the next group), component g
#pragma unroll
        for (int nt = 0; nt < BQ / 8; ++nt) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int qi = q0 + nt * 8 + t * 2 + c;
            float sa[8], sb[8];
            drop_scale8(p.drop, dstream, (rbase + qi) * lp8 + kg, sa);
            drop_scale8(p.drop, dstream, (rbase + qi) * lp8 + kg + 1, sb);
            float va = sa[0], vb = sb[0];
#pragma unroll
            for (int j = 1; j < 8; ++j) if (g == j) { va = sa[j]; vb = sb[j]; }
            ms[nt][c] = va; ms[nt][2 + c] = vb;                  // e = c: key_a ; e = 2 + c: key_b
          }
        }
      }
      // ---- dV += P_drop^T dO ----
      uint32_t pa[BQ / 16][4];
#pragma unroll
      for (int kk = 0; kk < BQ / 16; ++kk) {
        if (DROP) {
          pa[kk][0] = pack_bf16(st[2 * kk][0] * ms[2 * kk][0], st[2 * kk][1] * ms[2 * kk][1]);
          pa[kk][1] = pack_bf16(st[2 * kk][2] * ms[2 * kk][2], st[2 * kk][3] * ms[2 * kk][3]);
          pa[kk][2] = pack_bf16(st[2 * kk + 1][0] * ms[2 * kk + 1][0], st[2 * kk + 1][1] * ms[2 * kk + 1][1]);
          pa[kk][3] = pack_bf16(st[2 * kk + 1][2] * ms[2 * kk + 1][2], st[2 * kk + 1][3] * ms[2 * kk + 1][3]);
        } else {
          pa[kk][0] = pack_bf16(st[2 * kk][0], st[2 * kk][1]);
          pa[kk][1] = pack_bf16(st[2 * kk][2], st[2 * kk][3]);
          pa[kk][2] = pack_bf16(st[2 * kk + 1][0], st[2 * kk + 1][1]);
          pa[kk][3] = pack_bf16(st[2 * kk + 1][2], st[2 * kk + 1][3]);
        }
      }
#pragma unroll
      for (int kk = 0; kk < BQ / 16; ++kk) {
#pragma unroll
        for (int nt = 0; nt < D / 16; ++nt) {
          uint32_t bf[4];
          load_b_frag_kn<D>(bf, sdO, kk * 16, nt * 16, lane);
          mma16816(dv_acc[2 * nt], pa[kk], bf[0], bf[1]);
          mma16816(dv_acc[2 * nt + 1], pa[kk], bf[2], bf[3]);
        }
      }
      // ---- dP^T = V dO^T : 16 keys x 32 queries ----
      float dpt[BQ / 8][4];
#pragma unroll
      for (int i = 0; i < BQ / 8; ++i) { dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        uint32_t a[4];
        load_a_frag<D>(a, sV, warp * 16, kk * 16, lane);
#pragma unroll
        for (int nt = 0; nt < BQ / 16; ++nt) {
          uint32_t bf[4];
          load_b_frag_nk<D>(bf, sdO, nt * 16, kk * 16, lane);
          mma16816(dpt[2 * nt], a, bf[0], bf[1]);
          mma16816(dpt[2 * nt + 1], a, bf[2], bf[3]);
        }
      }
      // ---- dS^T = P^T * (dP^T - delta[q]) * scale ;  dK += dS^T Q ----
      uint32_t da[BQ / 16][4];
#pragma unroll
      for (int kk = 0; kk < BQ / 16; ++kk) {
        float ds[2][4];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int nt = 2 * kk + half;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int qc = nt * 8 + t * 2 + (e & 1);
            const float dpv = DROP ? dpt[nt][e] * ms[nt][e] : dpt[nt][e];
            ds[half][e] = st[nt][e] * (dpv - sDelta[qc]) * p.scale;
          }
        }
        da[kk][0] = pack_bf16(ds[0][0], ds[0][1]);
        da[kk][1] = pack_bf16(ds[0][2], ds[0][3]);
        da[kk][2] = pack_bf16(ds[1][0], ds[1][1]);
        da[kk][3] = pack_bf16(ds[1][2], ds[1][3]);
      }
#pragma unroll
      for (int kk = 0; kk < BQ / 16; ++kk) {
#pragma unroll
        for (int nt = 0; nt < D / 16; ++nt) {
          uint32_t bf[4];
          load_b_frag_kn<D>(bf, sQ, kk * 16, nt * 16, lane);
          mma16816(dk_acc[2 * nt], da[kk], bf[0], bf[1]);
          mma16816(dk_acc[2 * nt + 1], da[kk], bf[2], bf[3]);
        }
      }
    }
  }
  // ---- write dK, dV ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = r == 0 ? key_a : key_b;
    if (key < L) {
      __nv_bfloat16* dkrow = p.dk + (tok0 + key) * p.lddk + (size_t)hk * D;
      __nv_bfloat16* dvrow = p.dv + (tok0 + key) * p.lddv + (size_t)hk * D;
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt) {
        *reinterpret_cast<uint32_t*>(dkrow + nt * 8 + t * 2) = pack_bf16(dk_acc[nt][2 * r], dk_acc[nt][2 * r + 1]);
        *reinterpret_cast<uint32_t*>(dvrow + nt * 8 + t * 2) = pack_bf16(dv_acc[nt][2 * r], dv_acc[nt][2 * r + 1]);
      }
    }
  }
}

// ============================================================================================================
// backward: dQ.  Each warp owns 16 queries; keys streamed in 64-row tiles.
// ============================================================================================================
template <int D, bool DROP, bool WIN>
__global__ void __launch_bounds__(128) attn_bwd_dq_kernel(AttnParams p) {
  constexpr int BQ = 64, BKV = 64, LDS = D + 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __nv_bfloat16* sQ  = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sdO = sQ + BQ * LDS;
  __nv_bfloat16* sK  = sdO + BQ * LDS;
  __nv_bfloat16* sV  = sK + BKV * LDS;
  float* sMask = reinterpret_cast<float*>(sV + BKV * LDS);      // [BKV]

  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (p.Hq / p.Hkv);
  const int L = p.L, q0 = qb * BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t tok0 = (size_t)b * L;
  const float sl2 = p.scale * 1.4426950408889634f;

  const int nq = min(BQ, L - q0);
  load_tile<BQ, D, 128>(sQ, p.q + (tok0 + q0) * p.ldq + (size_t)h * D, p.ldq, nq);
  load_tile<BQ, D, 128>(sdO, p.d_o + (tok0 + q0) * p.lddo + (size_t)h * D, p.lddo, nq);

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  float lse2[2], dl[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r == 0 ? row_a : row_b;
    const size_t idx = ((size_t)b * p.Hq + h) * L + row;
    lse2[r] = row < L ? p.lse[idx] * 1.4426950408889634f : INFINITY;
    dl[r]   = row < L ? p.delta[idx] : 0.f;
  }
  float dq_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { dq_acc[i][0] = dq_acc[i][1] = dq_acc[i][2] = dq_acc[i][3] = 0.f; }

  const int kv_end = p.causal ? min(L, q0 + BQ) : WIN ? min(L, q0 + BQ - 1 + p.window) : L;
  for (int kv0 = win_begin<WIN, BKV>(q0, p.window); kv0 < kv_end; kv0 += BKV) {
    __syncthreads();
    const int nvalid = min(BKV, L - kv0);
    load_tile<BKV, D, 128>(sK, p.k + (tok0 + kv0) * p.ldk + (size_t)hk * D, p.ldk, nvalid);
    load_tile<BKV, D, 128>(sV, p.v + (tok0 + kv0) * p.ldv + (size_t)hk * D, p.ldv, nvalid);
    if (threadIdx.x < BKV) {
      const int key = kv0 + threadIdx.x;
      bool keep = key < L;
      if (keep && p.mask) keep = p.mask[tok0 + key] != 0;
      sMask[threadIdx.x] = keep ? 0.f : -INFINITY;
    }
    __syncthreads();

    float s[BKV / 8][4], dp[BKV / 8][4];
#pragma unroll
    for (int i = 0; i < BKV / 8; ++i) {
      s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    }
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      uint32_t a[4], ad[4];
      load_a_frag<D>(a, sQ, warp * 16, kk * 16, lane);
      load_a_frag<D>(ad, sdO, warp * 16, kk * 16, lane);
#pragma unroll
      for (int nt = 0; nt < BKV / 16; ++nt) {
        uint32_t bf[4];
        load_b_frag_nk<D>(bf, sK, nt * 16, kk * 16, lane);
        mma16816(s[2 * nt], a, bf[0], bf[1]);
        mma16816(s[2 * nt + 1], a, bf[2], bf[3]);
        load_b_frag_nk<D>(bf, sV, nt * 16, kk * 16, lane);
        mma16816(dp[2 * nt], ad, bf[0], bf[1]);
        mma16816(dp[2 * nt + 1], ad, bf[2], bf[3]);
      }
    }
    float msq[DROP ? BKV / 8 : 1][4];
    if (DROP) {
      const unsigned long long dstream = drop_stream(p.drop);
      const unsigned long long rbase = ((unsigned long long)b * p.Hq + h) * L;
      const int lp8 = (L + 7) >> 3;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int qr = r == 0 ? row_a : row_b;
          float sc[8];
          drop_scale8(p.drop, dstream, (rbase + qr) * lp8 + ((kv0 >> 3) + nt), sc);
          float s0 = sc[0], s1 = sc[1];
#pragma unroll
          for (int j = 1; j < 4; ++j) if (t == j) { s0 = sc[2 * j]; s1 = sc[2 * j + 1]; }
          msq[nt][2 * r] = s0; msq[nt][2 * r + 1] = s1;
        }
      }
    }
    // dS = P * (dP - delta) * scale
#pragma unroll
    for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kc = nt * 8 + t * 2 + (e & 1);
        const int qr = (e < 2) ? row_a : row_b;
        float val = s[nt][e] * sl2 + sMask[kc];
        if (p.causal && (kv0 + kc) > qr) val = -INFINITY;
        if (WIN && (kv0 + kc) <= qr - p.window) val = -INFINITY;
        if (WIN && (kv0 + kc) >= qr + p.window) val = -INFINITY;
        const float pv = exp2f(val - lse2[e >> 1]);
        float dpv = dp[nt][e];
        if (DROP) dpv *= msq[nt][e];
        s[nt][e] = pv * (dpv - dl[e >> 1]) * p.scale;
      }
    }
    // dQ += dS K
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
      a[1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
      a[2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int nt = 0; nt < D / 16; ++nt) {
        uint32_t bf[4];
        load_b_frag_kn<D>(bf, sK, kk * 16, nt * 16, lane);
        mma16816(dq_acc[2 * nt], a, bf[0], bf[1]);
        mma16816(dq_acc[2 * nt + 1], a, bf[2], bf[3]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r == 0 ? row_a : row_b;
    if (row < L) {
      __nv_bfloat16* dqrow = p.dq + (tok0 + row) * p.lddq + (size_t)h * D;
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt)
        *reinterpret_cast<uint32_t*>(dqrow + nt * 8 + t * 2) = pack_bf16(dq_acc[nt][2 * r], dq_acc[nt][2 * r + 1]);
    }
  }
}

template <int D> static size_t fwd_smem() { return (size_t)(64 * 3) * (D + 8) * 2 + 64 * 4; }
template <int D> static size_t dkv_smem() { return (size_t)(64 * 2 + 32 * 2) * (D + 8) * 2 + (32 + 32 + 64) * 4; }
template <int D> static size_t dq_smem()  { return (size_t)(64 * 4) * (D + 8) * 2 + 64 * 4; }

template <int D, bool DROP, bool WIN> static int launch_fwd(const AttnParams& p, cudaStream_t st) {
  static bool attr = false;
  if (!attr) { DALM_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<D, DROP, WIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<D>())); attr = true; }
  dim3 grid((p.L + 63) / 64, p.Hq, p.B);
  attn_fwd_kernel<D, DROP, WIN><<<grid, 128, fwd_smem<D>(), st>>>(p);
  count_launch();
  return check_launch("attn_fwd_kernel");
}
template <int D, bool DROP, bool WIN> static int launch_bwd(const AttnParams& p, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    DALM_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_kernel<D, DROP, WIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dkv_smem<D>()));
    DALM_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel<D, DROP, WIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dq_smem<D>()));
    attr = true;
  }
  const int total_warps = p.B * p.L * p.Hq;
  attn_delta_kernel<<<(total_warps * 32 + 255) / 256, 256, 0, st>>>(p.o, p.ldo, p.d_o, p.lddo, p.delta, p.B, p.L, p.Hq, D);
  if (int e = check_launch("attn_delta_kernel")) return e;
  dim3 gkv((p.L + 63) / 64, p.Hkv, p.B);
  attn_bwd_dkv_kernel<D, DROP, WIN><<<gkv, 128, dkv_smem<D>(), st>>>(p);
  if (int e = check_launch("attn_bwd_dkv_kernel")) return e;
  dim3 gq((p.L + 63) / 64, p.Hq, p.B);
  attn_bwd_dq_kernel<D, DROP, WIN><<<gq, 128, dq_smem<D>(), st>>>(p);
  count_launch(3);
  return check_launch("attn_bwd_dq_kernel");
}

// ============================================================================================================
// wgmma kernels (head_dim 64 / 128). One warpgroup per CTA = 64 rows; warp w holds rows 16w + g and 16w + g + 8, exactly
// the rows and columns it holds in the mma.sync kernels above (the wgmma accumulator and register-A fragments coincide
// with the m16n8k16 ones), so the softmax / dropout / dS code is the same. Streamed tiles are double-buffered: the TMA
// load of tile i+1 is in flight while tile i is computed.
// ============================================================================================================
namespace wg {
using namespace ptx;
__device__ __forceinline__ unsigned char* align1024(unsigned char* p) {
  return reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}
// [R rows x D] bf16 tile as D/64 TMA boxes of [R rows x 128 B], 128B-swizzled
template <int R, int D> __device__ __forceinline__ void load_tile(unsigned char* dst, const CUtensorMap* m, uint64_t* bar, int col0, int row0) {
#pragma unroll
  for (int c = 0; c < D / 64; ++c) tma_load_2d(dst + c * R * 128, m, bar, col0 + c * 64, row0);
}
// descriptor of k-step kk: K-major tile (contraction over its D columns) / MN-major tile (contraction over its R rows)
template <int R> __device__ __forceinline__ uint64_t kdesc(uint32_t base, int kk) {
  return make_sw128_kmajor_desc(base + (uint32_t)(kk >> 2) * (R * 128) + (uint32_t)(kk & 3) * 32);
}
template <int R> __device__ __forceinline__ uint64_t mndesc(uint32_t base, int kk) {
  return make_sw128_mnmajor_desc(base + (uint32_t)kk * 2048, R * 128, 1024);
}
template <int D> __device__ __forceinline__ void mma_rs(float* acc, const uint32_t* a, uint64_t db) {
  if constexpr (D == 128) wgmma_m64n128k16_rs<1>(acc, a, db, 1);
  else wgmma_m64n64k16_rs<1>(acc, a, db, 1);
}
}  // namespace wg

template <int D> constexpr int wg_tile() { return 64 * D * 2; }
template <int D> constexpr int wg_fwd_smem() { return 5 * wg_tile<D>() + 64 * 4 + 64 + 1024; }
template <int D> constexpr int wg_dq_smem() { return 6 * wg_tile<D>() + 64 * 4 + 64 + 1024; }
template <int D> constexpr int wg_dkv_smem() { return 2 * wg_tile<D>() + 4 * (wg_tile<D>() / 2) + (64 + 32 + 32) * 4 + 64 + 1024; }

template <int D, bool DROP, bool WIN>
__global__ void __launch_bounds__(128) attn_fwd_wg_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                                                          const __grid_constant__ CUtensorMap tv, AttnParams p) {
  using namespace wg;
  constexpr int BQ = 64, BKV = 64, TILE = wg_tile<D>();
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sQ = align1024(smem_raw);
  unsigned char* sKV = sQ + TILE;                               // buffer j: K at sKV + 2j TILE, V right after it
  float* sMask = reinterpret_cast<float*>(sKV + 4 * TILE);      // [BKV] additive 0 / -inf
  uint64_t* bar = reinterpret_cast<uint64_t*>(sMask + BKV);     // [0] Q, [1 + j] K/V buffer j

  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (p.Hq / p.Hkv);
  const int L = p.L, q0 = qb * BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t tok0 = (size_t)b * L;
  const int kv_end = p.causal ? min(L, q0 + BQ) : WIN ? min(L, q0 + BQ - 1 + p.window) : L;
  const int kv_begin = win_begin<WIN, BKV>(q0, p.window);       // tile `it` starts at kv_begin + it * BKV
  const int ntile = (kv_end - kv_begin + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(&bar[0], TILE);
    load_tile<64, D>(sQ, &tq, &bar[0], h * D, (int)(tok0 + q0));
    mbar_arrive_expect_tx(&bar[1], 2 * TILE);
    load_tile<64, D>(sKV, &tk, &bar[1], hk * D, (int)(tok0 + kv_begin));
    load_tile<64, D>(sKV + TILE, &tv, &bar[1], hk * D, (int)(tok0 + kv_begin));
  }
  __syncthreads();

  float o_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float sl2 = p.scale * 1.4426950408889634f;
  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const uint32_t qbase = smem_u32(sQ);
  mbar_wait(&bar[0], 0);

  for (int it = 0; it < ntile; ++it) {
    const int kv0 = kv_begin + it * BKV, cb = it & 1;
    if (threadIdx.x == 0 && it + 1 < ntile) {                   // buffer cb^1 was released by the barrier closing it - 1
      unsigned char* nb = sKV + (cb ^ 1) * 2 * TILE;
      mbar_arrive_expect_tx(&bar[1 + (cb ^ 1)], 2 * TILE);
      load_tile<64, D>(nb, &tk, &bar[1 + (cb ^ 1)], hk * D, (int)(tok0 + kv0 + BKV));
      load_tile<64, D>(nb + TILE, &tv, &bar[1 + (cb ^ 1)], hk * D, (int)(tok0 + kv0 + BKV));
    }
    if (threadIdx.x < BKV) {
      const int key = kv0 + threadIdx.x;
      bool keep = key < L;
      if (keep && p.mask) keep = p.mask[tok0 + key] != 0;
      sMask[threadIdx.x] = keep ? 0.f : -INFINITY;
    }
    __syncthreads();
    mbar_wait(&bar[1 + cb], (uint32_t)(it >> 1) & 1u);
    const uint32_t kbase = smem_u32(sKV + cb * 2 * TILE), vbase = kbase + TILE;

    // ---- S = Q K^T (64 x 64) ----
    float s[BKV / 8][4];
#pragma unroll
    for (int i = 0; i < BKV / 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64k16<0, 0>(&s[0][0], kdesc<64>(qbase, kk), kdesc<64>(kbase, kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
    // ---- mask + online softmax (base-2) ----
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kc = nt * 8 + t * 2 + (e & 1);
        const int qr = (e < 2) ? row_a : row_b;
        float val = s[nt][e] * sl2 + sMask[kc];
        if (p.causal && (kv0 + kc) > qr) val = -INFINITY;
        if (WIN && (kv0 + kc) <= qr - p.window) val = -INFINITY;
        if (WIN && (kv0 + kc) >= qr + p.window) val = -INFINITY;
        s[nt][e] = val;
        mx[e >> 1] = fmaxf(mx[e >> 1], val);
      }
    }
    float corr[2], mnew[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      mnew[r] = fmaxf(m_run[r], mx[r]);
      const float msafe = (mnew[r] == -INFINITY) ? 0.f : mnew[r];
      corr[r] = exp2f(m_run[r] - msafe);
      m_run[r] = mnew[r];
      mnew[r] = msafe;
    }
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f(s[nt][e] - mnew[e >> 1]);
        s[nt][e] = pv;
        rs[e >> 1] += pv;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
      rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
      l_run[r] = l_run[r] * corr[r] + rs[r];
    }
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      o_acc[i][0] *= corr[0]; o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1]; o_acc[i][3] *= corr[1];
    }
    if (DROP) {
      const unsigned long long dstream = drop_stream(p.drop);
      const unsigned long long rbase = ((unsigned long long)b * p.Hq + h) * L;
      const int lp8 = (L + 7) >> 3;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int qr = r == 0 ? row_a : row_b;
          float sc[8];
          drop_scale8(p.drop, dstream, (rbase + qr) * lp8 + ((kv0 >> 3) + nt), sc);
          float s0 = sc[0], s1 = sc[1];
#pragma unroll
          for (int j = 1; j < 4; ++j) if (t == j) { s0 = sc[2 * j]; s1 = sc[2 * j + 1]; }
          s[nt][2 * r] *= s0; s[nt][2 * r + 1] *= s1;
        }
      }
    }
    // ---- O += P V (P from registers, V MN-major) ----
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      pa[kk][0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
      pa[kk][1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
      pa[kk][2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      pa[kk][3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) mma_rs<D>(&o_acc[0][0], pa[kk], mndesc<64>(vbase, kk));
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();                                            // K/V buffer cb and sMask may be overwritten
  }

  const float inv_l[2] = {l_run[0] > 0.f ? 1.f / l_run[0] : 0.f, l_run[1] > 0.f ? 1.f / l_run[1] : 0.f};
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r == 0 ? row_a : row_b;
    if (row < L) {
      __nv_bfloat16* orow = p.o + (tok0 + row) * p.ldo + (size_t)h * D;
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt) {
        const uint32_t pk = pack_bf16(o_acc[nt][2 * r] * inv_l[r], o_acc[nt][2 * r + 1] * inv_l[r]);
        *reinterpret_cast<uint32_t*>(orow + nt * 8 + t * 2) = pk;
      }
      if (t == 0) {
        const float lse = l_run[r] > 0.f ? (m_run[r] + log2f(l_run[r])) * 0.6931471805599453f : INFINITY;
        p.lse[((size_t)b * p.Hq + h) * L + row] = lse;
      }
    }
  }
}

// dK, dV: grid (ceil(L/64), Hkv, B); the warpgroup owns 64 keys (K, V resident), query tiles of 32 rows streamed over
// the q heads of the group
template <int D, bool DROP, bool WIN>
__global__ void __launch_bounds__(128) attn_bwd_dkv_wg_kernel(const __grid_constant__ CUtensorMap tk, const __grid_constant__ CUtensorMap tv,
                                                              const __grid_constant__ CUtensorMap tq32, const __grid_constant__ CUtensorMap tdo32,
                                                              AttnParams p) {
  using namespace wg;
  constexpr int BKV = 64, BQ = 32, TILE = wg_tile<D>(), TQ = TILE / 2;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sK = align1024(smem_raw);
  unsigned char* sV = sK + TILE;
  unsigned char* sQD = sV + TILE;                               // buffer j: Q at sQD + 2j TQ, dO right after it
  float* sMask  = reinterpret_cast<float*>(sQD + 4 * TQ);       // [BKV]
  float* sLse   = sMask + BKV;                                  // [BQ]
  float* sDelta = sLse + BQ;                                    // [BQ]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sDelta + BQ);     // [0] K/V, [1 + j] Q/dO buffer j

  const int kb = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int group = p.Hq / p.Hkv;
  const int L = p.L, kv0 = kb * BKV;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t tok0 = (size_t)b * L;
  const float sl2 = p.scale * 1.4426950408889634f;
  const int q_begin = p.causal ? (kv0 / BQ) * BQ : win_begin<WIN, BQ>(kv0, p.window);
  const int q_end = WIN ? min(L, kv0 + BKV - 1 + p.window) : L;
  const int nqt = (q_end - q_begin + BQ - 1) / BQ;
  const int nit = group * nqt;                                   // (q head, query tile) pairs, head-major

  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(&bar[0], 2 * TILE);
    load_tile<64, D>(sK, &tk, &bar[0], hk * D, (int)(tok0 + kv0));
    load_tile<64, D>(sV, &tv, &bar[0], hk * D, (int)(tok0 + kv0));
    if (nit > 0) {
      mbar_arrive_expect_tx(&bar[1], 2 * TQ);
      load_tile<32, D>(sQD, &tq32, &bar[1], hk * group * D, (int)(tok0 + q_begin));
      load_tile<32, D>(sQD + TQ, &tdo32, &bar[1], hk * group * D, (int)(tok0 + q_begin));
    }
  }
  if (threadIdx.x < BKV) {
    const int key = kv0 + threadIdx.x;
    bool keep = key < L;
    if (keep && p.mask) keep = p.mask[tok0 + key] != 0;
    sMask[threadIdx.x] = keep ? 0.f : -INFINITY;
  }
  __syncthreads();

  float dk_acc[D / 8][4], dv_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) {
    dk_acc[i][0] = dk_acc[i][1] = dk_acc[i][2] = dk_acc[i][3] = 0.f;
    dv_acc[i][0] = dv_acc[i][1] = dv_acc[i][2] = dv_acc[i][3] = 0.f;
  }
  const int key_a = kv0 + warp * 16 + g, key_b = key_a + 8;
  const float mk_a = sMask[warp * 16 + g], mk_b = sMask[warp * 16 + g + 8];
  const uint32_t kbase = smem_u32(sK), vbase = smem_u32(sV);
  mbar_wait(&bar[0], 0);

  for (int it = 0; it < nit; ++it) {
    const int hq = hk * group + it / nqt, q0 = q_begin + (it % nqt) * BQ, cb = it & 1;
    if (threadIdx.x == 0 && it + 1 < nit) {
      const int hq1 = hk * group + (it + 1) / nqt, q1 = q_begin + ((it + 1) % nqt) * BQ;
      unsigned char* nb = sQD + (cb ^ 1) * 2 * TQ;
      mbar_arrive_expect_tx(&bar[1 + (cb ^ 1)], 2 * TQ);
      load_tile<32, D>(nb, &tq32, &bar[1 + (cb ^ 1)], hq1 * D, (int)(tok0 + q1));
      load_tile<32, D>(nb + TQ, &tdo32, &bar[1 + (cb ^ 1)], hq1 * D, (int)(tok0 + q1));
    }
    if (threadIdx.x < BQ) {
      const int qi = q0 + threadIdx.x;
      const size_t idx = ((size_t)b * p.Hq + hq) * L + qi;
      sLse[threadIdx.x]   = qi < L ? p.lse[idx] * 1.4426950408889634f : INFINITY;
      sDelta[threadIdx.x] = qi < L ? p.delta[idx] : 0.f;
    }
    __syncthreads();
    mbar_wait(&bar[1 + cb], (uint32_t)(it >> 1) & 1u);
    const uint32_t qbase = smem_u32(sQD + cb * 2 * TQ), dobase = qbase + TQ;

    // ---- S^T = K Q^T and dP^T = V dO^T : 64 keys x 32 queries ----
    float st[BQ / 8][4], dpt[BQ / 8][4];
#pragma unroll
    for (int i = 0; i < BQ / 8; ++i) {
      st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f;
      dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f;
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n32k16<0, 0>(&st[0][0], kdesc<64>(kbase, kk), kdesc<32>(qbase, kk), 1);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n32k16<0, 0>(&dpt[0][0], kdesc<64>(vbase, kk), kdesc<32>(dobase, kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
    // ---- P^T = exp2(S^T * sl2 - lse2[q]) with masks ----
#pragma unroll
    for (int nt = 0; nt < BQ / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qc = nt * 8 + t * 2 + (e & 1);
        const int key = (e < 2) ? key_a : key_b;
        float val = st[nt][e] * sl2 + ((e < 2) ? mk_a : mk_b);
        if (p.causal && key > (q0 + qc)) val = -INFINITY;
        if (WIN && key <= (q0 + qc) - p.window) val = -INFINITY;
        if (WIN && key >= (q0 + qc) + p.window) val = -INFINITY;
        st[nt][e] = exp2f(val - sLse[qc]);
      }
    }
    float ms[DROP ? BQ / 8 : 1][4];
    if (DROP) {
      const unsigned long long dstream = drop_stream(p.drop);
      const unsigned long long rbase = ((unsigned long long)b * p.Hq + hq) * L;
      const int lp8 = (L + 7) >> 3;
      const int kg = (kv0 >> 3) + warp * 2;
#pragma unroll
      for (int nt = 0; nt < BQ / 8; ++nt) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int qi = q0 + nt * 8 + t * 2 + c;
          float sa[8], sb[8];
          drop_scale8(p.drop, dstream, (rbase + qi) * lp8 + kg, sa);
          drop_scale8(p.drop, dstream, (rbase + qi) * lp8 + kg + 1, sb);
          float va = sa[0], vb = sb[0];
#pragma unroll
          for (int j = 1; j < 8; ++j) if (g == j) { va = sa[j]; vb = sb[j]; }
          ms[nt][c] = va; ms[nt][2 + c] = vb;
        }
      }
    }
    // ---- dS^T = P^T * (dP^T - delta[q]) * scale ----
    uint32_t pa[BQ / 16][4], da[BQ / 16][4];
#pragma unroll
    for (int kk = 0; kk < BQ / 16; ++kk) {
      float pd[2][4], ds[2][4];
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int nt = 2 * kk + half;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = nt * 8 + t * 2 + (e & 1);
          pd[half][e] = DROP ? st[nt][e] * ms[nt][e] : st[nt][e];
          const float dpv = DROP ? dpt[nt][e] * ms[nt][e] : dpt[nt][e];
          ds[half][e] = st[nt][e] * (dpv - sDelta[qc]) * p.scale;
        }
      }
      pa[kk][0] = pack_bf16(pd[0][0], pd[0][1]); pa[kk][1] = pack_bf16(pd[0][2], pd[0][3]);
      pa[kk][2] = pack_bf16(pd[1][0], pd[1][1]); pa[kk][3] = pack_bf16(pd[1][2], pd[1][3]);
      da[kk][0] = pack_bf16(ds[0][0], ds[0][1]); da[kk][1] = pack_bf16(ds[0][2], ds[0][3]);
      da[kk][2] = pack_bf16(ds[1][0], ds[1][1]); da[kk][3] = pack_bf16(ds[1][2], ds[1][3]);
    }
    // ---- dV += P_drop^T dO ; dK += dS^T Q (both B operands MN-major over the 32 query rows) ----
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BQ / 16; ++kk) mma_rs<D>(&dv_acc[0][0], pa[kk], mndesc<32>(dobase, kk));
#pragma unroll
    for (int kk = 0; kk < BQ / 16; ++kk) mma_rs<D>(&dk_acc[0][0], da[kk], mndesc<32>(qbase, kk));
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();                                            // Q/dO buffer cb, sLse and sDelta may be overwritten
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = r == 0 ? key_a : key_b;
    if (key < L) {
      __nv_bfloat16* dkrow = p.dk + (tok0 + key) * p.lddk + (size_t)hk * D;
      __nv_bfloat16* dvrow = p.dv + (tok0 + key) * p.lddv + (size_t)hk * D;
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt) {
        *reinterpret_cast<uint32_t*>(dkrow + nt * 8 + t * 2) = pack_bf16(dk_acc[nt][2 * r], dk_acc[nt][2 * r + 1]);
        *reinterpret_cast<uint32_t*>(dvrow + nt * 8 + t * 2) = pack_bf16(dv_acc[nt][2 * r], dv_acc[nt][2 * r + 1]);
      }
    }
  }
}

// dQ: grid (ceil(L/64), Hq, B); the warpgroup owns 64 queries (Q, dO resident), key tiles of 64 streamed
template <int D, bool DROP, bool WIN>
__global__ void __launch_bounds__(128) attn_bwd_dq_wg_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tdo,
                                                             const __grid_constant__ CUtensorMap tk, const __grid_constant__ CUtensorMap tv,
                                                             AttnParams p) {
  using namespace wg;
  constexpr int BQ = 64, BKV = 64, TILE = wg_tile<D>();
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sQ = align1024(smem_raw);
  unsigned char* sdO = sQ + TILE;
  unsigned char* sKV = sdO + TILE;                              // buffer j: K at sKV + 2j TILE, V right after it
  float* sMask = reinterpret_cast<float*>(sKV + 4 * TILE);
  uint64_t* bar = reinterpret_cast<uint64_t*>(sMask + BKV);

  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (p.Hq / p.Hkv);
  const int L = p.L, q0 = qb * BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t tok0 = (size_t)b * L;
  const float sl2 = p.scale * 1.4426950408889634f;
  const int kv_end = p.causal ? min(L, q0 + BQ) : WIN ? min(L, q0 + BQ - 1 + p.window) : L;
  const int kv_begin = win_begin<WIN, BKV>(q0, p.window);       // tile `it` starts at kv_begin + it * BKV
  const int ntile = (kv_end - kv_begin + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(&bar[0], 2 * TILE);
    load_tile<64, D>(sQ, &tq, &bar[0], h * D, (int)(tok0 + q0));
    load_tile<64, D>(sdO, &tdo, &bar[0], h * D, (int)(tok0 + q0));
    mbar_arrive_expect_tx(&bar[1], 2 * TILE);
    load_tile<64, D>(sKV, &tk, &bar[1], hk * D, (int)(tok0 + kv_begin));
    load_tile<64, D>(sKV + TILE, &tv, &bar[1], hk * D, (int)(tok0 + kv_begin));
  }
  __syncthreads();

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  float lse2[2], dl[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r == 0 ? row_a : row_b;
    const size_t idx = ((size_t)b * p.Hq + h) * L + row;
    lse2[r] = row < L ? p.lse[idx] * 1.4426950408889634f : INFINITY;
    dl[r]   = row < L ? p.delta[idx] : 0.f;
  }
  float dq_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { dq_acc[i][0] = dq_acc[i][1] = dq_acc[i][2] = dq_acc[i][3] = 0.f; }
  const uint32_t qbase = smem_u32(sQ), dobase = smem_u32(sdO);
  mbar_wait(&bar[0], 0);

  for (int it = 0; it < ntile; ++it) {
    const int kv0 = kv_begin + it * BKV, cb = it & 1;
    if (threadIdx.x == 0 && it + 1 < ntile) {
      unsigned char* nb = sKV + (cb ^ 1) * 2 * TILE;
      mbar_arrive_expect_tx(&bar[1 + (cb ^ 1)], 2 * TILE);
      load_tile<64, D>(nb, &tk, &bar[1 + (cb ^ 1)], hk * D, (int)(tok0 + kv0 + BKV));
      load_tile<64, D>(nb + TILE, &tv, &bar[1 + (cb ^ 1)], hk * D, (int)(tok0 + kv0 + BKV));
    }
    if (threadIdx.x < BKV) {
      const int key = kv0 + threadIdx.x;
      bool keep = key < L;
      if (keep && p.mask) keep = p.mask[tok0 + key] != 0;
      sMask[threadIdx.x] = keep ? 0.f : -INFINITY;
    }
    __syncthreads();
    mbar_wait(&bar[1 + cb], (uint32_t)(it >> 1) & 1u);
    const uint32_t kbase = smem_u32(sKV + cb * 2 * TILE), vbase = kbase + TILE;

    float s[BKV / 8][4], dp[BKV / 8][4];
#pragma unroll
    for (int i = 0; i < BKV / 8; ++i) {
      s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64k16<0, 0>(&s[0][0], kdesc<64>(qbase, kk), kdesc<64>(kbase, kk), 1);
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) wgmma_m64n64k16<0, 0>(&dp[0][0], kdesc<64>(dobase, kk), kdesc<64>(vbase, kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
    float msq[DROP ? BKV / 8 : 1][4];
    if (DROP) {
      const unsigned long long dstream = drop_stream(p.drop);
      const unsigned long long rbase = ((unsigned long long)b * p.Hq + h) * L;
      const int lp8 = (L + 7) >> 3;
#pragma unroll
      for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int qr = r == 0 ? row_a : row_b;
          float sc[8];
          drop_scale8(p.drop, dstream, (rbase + qr) * lp8 + ((kv0 >> 3) + nt), sc);
          float s0 = sc[0], s1 = sc[1];
#pragma unroll
          for (int j = 1; j < 4; ++j) if (t == j) { s0 = sc[2 * j]; s1 = sc[2 * j + 1]; }
          msq[nt][2 * r] = s0; msq[nt][2 * r + 1] = s1;
        }
      }
    }
#pragma unroll
    for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kc = nt * 8 + t * 2 + (e & 1);
        const int qr = (e < 2) ? row_a : row_b;
        float val = s[nt][e] * sl2 + sMask[kc];
        if (p.causal && (kv0 + kc) > qr) val = -INFINITY;
        if (WIN && (kv0 + kc) <= qr - p.window) val = -INFINITY;
        if (WIN && (kv0 + kc) >= qr + p.window) val = -INFINITY;
        const float pv = exp2f(val - lse2[e >> 1]);
        float dpv = dp[nt][e];
        if (DROP) dpv *= msq[nt][e];
        s[nt][e] = pv * (dpv - dl[e >> 1]) * p.scale;
      }
    }
    // ---- dQ += dS K (K MN-major over its 64 key rows) ----
    uint32_t da[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      da[kk][0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
      da[kk][1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
      da[kk][2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      da[kk][3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) mma_rs<D>(&dq_acc[0][0], da[kk], mndesc<64>(kbase, kk));
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r == 0 ? row_a : row_b;
    if (row < L) {
      __nv_bfloat16* dqrow = p.dq + (tok0 + row) * p.lddq + (size_t)h * D;
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt)
        *reinterpret_cast<uint32_t*>(dqrow + nt * 8 + t * 2) = pack_bf16(dq_acc[nt][2 * r], dq_acc[nt][2 * r + 1]);
    }
  }
}

template <int D, bool DROP, bool WIN> static int launch_fwd_wg(const AttnParams& p, int qcols, int kvcols, cudaStream_t st) {
  static bool attr = false;
  if (!attr) { DALM_CUDA(cudaFuncSetAttribute(attn_fwd_wg_kernel<D, DROP, WIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_fwd_smem<D>())); attr = true; }
  const long long rows = (long long)p.B * p.L;
  CUtensorMap tq, tk, tv;
  if (int e = get_tmap(p.q, rows, qcols, p.ldq, 64, &tq)) return e;
  if (int e = get_tmap(p.k, rows, kvcols, p.ldk, 64, &tk)) return e;
  if (int e = get_tmap(p.v, rows, kvcols, p.ldv, 64, &tv)) return e;
  dim3 grid((p.L + 63) / 64, p.Hq, p.B);
  attn_fwd_wg_kernel<D, DROP, WIN><<<grid, 128, wg_fwd_smem<D>(), st>>>(tq, tk, tv, p);
  count_launch();
  return check_launch("attn_fwd_wg_kernel");
}
template <int D, bool DROP, bool WIN> static int launch_bwd_wg(const AttnParams& p, int qcols, int kvcols, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    DALM_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_wg_kernel<D, DROP, WIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_dkv_smem<D>()));
    DALM_CUDA(cudaFuncSetAttribute(attn_bwd_dq_wg_kernel<D, DROP, WIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, wg_dq_smem<D>()));
    attr = true;
  }
  const long long rows = (long long)p.B * p.L;
  CUtensorMap tq, tdo, tq32, tdo32, tk, tv;
  if (int e = get_tmap(p.q, rows, qcols, p.ldq, 64, &tq)) return e;
  if (int e = get_tmap(p.d_o, rows, qcols, p.lddo, 64, &tdo)) return e;
  if (int e = get_tmap(p.q, rows, qcols, p.ldq, 32, &tq32)) return e;
  if (int e = get_tmap(p.d_o, rows, qcols, p.lddo, 32, &tdo32)) return e;
  if (int e = get_tmap(p.k, rows, kvcols, p.ldk, 64, &tk)) return e;
  if (int e = get_tmap(p.v, rows, kvcols, p.ldv, 64, &tv)) return e;
  const int total_warps = p.B * p.L * p.Hq;
  attn_delta_kernel<<<(total_warps * 32 + 255) / 256, 256, 0, st>>>(p.o, p.ldo, p.d_o, p.lddo, p.delta, p.B, p.L, p.Hq, D);
  if (int e = check_launch("attn_delta_kernel")) return e;
  dim3 gkv((p.L + 63) / 64, p.Hkv, p.B);
  attn_bwd_dkv_wg_kernel<D, DROP, WIN><<<gkv, 128, wg_dkv_smem<D>(), st>>>(tk, tv, tq32, tdo32, p);
  if (int e = check_launch("attn_bwd_dkv_wg_kernel")) return e;
  dim3 gq((p.L + 63) / 64, p.Hq, p.B);
  attn_bwd_dq_wg_kernel<D, DROP, WIN><<<gq, 128, wg_dq_smem<D>(), st>>>(tq, tdo, tk, tv, p);
  count_launch(3);
  return check_launch("attn_bwd_dq_wg_kernel");
}

static int check_common(const AttnParams& p, int D) {
  DALM_REQUIRE(D == 32 || D == 64 || D == 128, "attention: head_dim %d unsupported (32/64/128)", D);
  DALM_REQUIRE(p.B > 0 && p.L > 0 && p.Hq > 0 && p.Hkv > 0 && p.Hq % p.Hkv == 0, "attention: bad shape B=%d L=%d Hq=%d Hkv=%d", p.B, p.L, p.Hq, p.Hkv);
  DALM_REQUIRE(p.B <= 65535 && p.Hq <= 65535, "attention: B=%d sequences / Hq=%d heads past 65535 (grid extents)", p.B, p.Hq);
  DALM_REQUIRE(p.ldq % 8 == 0 && p.ldk % 8 == 0 && p.ldv % 8 == 0 && p.ldo % 2 == 0, "attention: strides must keep 16-byte row alignment");
  DALM_REQUIRE(((uintptr_t)p.q & 15) == 0 && ((uintptr_t)p.k & 15) == 0 && ((uintptr_t)p.v & 15) == 0, "attention: q/k/v must be 16-byte aligned");
  DALM_REQUIRE(p.window >= 0, "attention: window %d must be >= 0", p.window);
  DALM_REQUIRE(p.window == 0 || p.drop.p == 0.f, "attention: probability dropout with a sliding window is not built");
  return 0;
}

// window > 0 runs the WIN instances (window clamped to L: a wider window masks nothing more); window 0 runs the
// instances that were built before the window existed, unchanged
static bool set_window(AttnParams& p, int window) {
  p.window = window > 0 ? min(window, p.L) : window;        // a negative window stays negative: check_common refuses it
  return window > 0;
}
}  // namespace dalm

using namespace dalm;

// q/k/v: bf16 token-major views (row b*L+l, head h at column h*D); mask: int64 [B,L] or NULL; out: bf16; lse: fp32 [B,Hq,L]
extern "C" int dalm_b200_attention_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                       long long ldv, const int64_t* mask, void* out, long long ldo, float* lse, int B,
                                       int L, int Hq, int Hkv, int D, float scale, int causal, int window, float drop_p,
                                       unsigned long long drop_seed, unsigned long long drop_stream_id,
                                       const void* drop_offset, void* stream) {
  AttnParams p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.mask = mask; p.o = (__nv_bfloat16*)out; p.ldo = ldo; p.lse = lse;
  p.B = B; p.L = L; p.Hq = Hq; p.Hkv = Hkv; p.scale = scale; p.causal = causal;
  p.drop = make_drop(drop_p, drop_seed, drop_stream_id, drop_offset);
  const bool win = set_window(p, window);
  if (int e = check_common(p, D)) return e;
  DALM_REQUIRE(drop_p >= 0.f && drop_p < 1.f, "attention: dropout p must be in [0,1)");
  DALM_REQUIRE(drop_p == 0.f || D <= 64, "attention: probability dropout is built for head_dim <= 64 (encoder); Llama has attention_dropout = 0");
  cudaStream_t st = (cudaStream_t)stream;
  if (drop_p > 0.f) return D == 32 ? launch_fwd<32, true, false>(p, st) : launch_fwd<64, true, false>(p, st);
  if (win) return D == 32 ? launch_fwd<32, false, true>(p, st) : D == 64 ? launch_fwd<64, false, true>(p, st) : launch_fwd<128, false, true>(p, st);
  if (D == 32) return launch_fwd<32, false, false>(p, st);
  if (D == 64) return launch_fwd<64, false, false>(p, st);
  return launch_fwd<128, false, false>(p, st);
}

// delta: fp32 workspace [B,Hq,L]; dq/dk/dv: bf16 token-major outputs (dk/dv have Hkv heads)
extern "C" int dalm_b200_attention_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                       long long ldv, const int64_t* mask, const void* out, long long ldo,
                                       const float* lse, const void* d_out, long long lddo, float* delta, void* dq,
                                       long long lddq, void* dk, long long lddk, void* dv, long long lddv, int B, int L,
                                       int Hq, int Hkv, int D, float scale, int causal, int window, float drop_p,
                                       unsigned long long drop_seed, unsigned long long drop_stream_id,
                                       const void* drop_offset, void* stream) {
  AttnParams p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.mask = mask; p.o = (__nv_bfloat16*)const_cast<void*>(out); p.ldo = ldo;
  p.lse = const_cast<float*>(lse); p.d_o = (const __nv_bfloat16*)d_out; p.lddo = lddo; p.delta = delta;
  p.dq = (__nv_bfloat16*)dq; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv;
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
  p.B = B; p.L = L; p.Hq = Hq; p.Hkv = Hkv; p.scale = scale; p.causal = causal;
  p.drop = make_drop(drop_p, drop_seed, drop_stream_id, drop_offset);
  const bool win = set_window(p, window);
  if (int e = check_common(p, D)) return e;
  DALM_REQUIRE(lddo % 8 == 0 && ((uintptr_t)d_out & 15) == 0, "attention_bwd: d_out alignment");
  DALM_REQUIRE(drop_p >= 0.f && drop_p < 1.f && (drop_p == 0.f || D <= 64), "attention_bwd: dropout needs p in [0,1) and head_dim <= 64");
  cudaStream_t st = (cudaStream_t)stream;
  if (drop_p > 0.f) return D == 32 ? launch_bwd<32, true, false>(p, st) : launch_bwd<64, true, false>(p, st);
  if (win) return D == 32 ? launch_bwd<32, false, true>(p, st) : D == 64 ? launch_bwd<64, false, true>(p, st) : launch_bwd<128, false, true>(p, st);
  if (D == 32) return launch_bwd<32, false, false>(p, st);
  if (D == 64) return launch_bwd<64, false, false>(p, st);
  return launch_bwd<128, false, false>(p, st);
}

// the wgmma kernels: same contract as dalm_b200_attention_fwd, head_dim 64 or 128 (dropout at 64)
extern "C" int dalm_b200_attention_tc_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                          long long ldv, const int64_t* mask, void* out, long long ldo, float* lse, int B,
                                          int L, int Hq, int Hkv, int D, float scale, int causal, int window, float drop_p,
                                          unsigned long long drop_seed, unsigned long long drop_stream_id,
                                          const void* drop_offset, void* stream) {
  AttnParams p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.mask = mask; p.o = (__nv_bfloat16*)out; p.ldo = ldo; p.lse = lse;
  p.B = B; p.L = L; p.Hq = Hq; p.Hkv = Hkv; p.scale = scale; p.causal = causal;
  p.drop = make_drop(drop_p, drop_seed, drop_stream_id, drop_offset);
  const bool win = set_window(p, window);
  if (int e = check_common(p, D)) return e;
  DALM_REQUIRE(D == 64 || D == 128, "attention_tc: head_dim %d unsupported (64/128)", D);
  DALM_REQUIRE(drop_p >= 0.f && drop_p < 1.f && (drop_p == 0.f || D == 64), "attention_tc: dropout needs p in [0,1) and head_dim 64");
  cudaStream_t st = (cudaStream_t)stream;
  if (drop_p > 0.f) return launch_fwd_wg<64, true, false>(p, Hq * D, Hkv * D, st);
  if (win) return D == 64 ? launch_fwd_wg<64, false, true>(p, Hq * D, Hkv * D, st) : launch_fwd_wg<128, false, true>(p, Hq * D, Hkv * D, st);
  if (D == 64) return launch_fwd_wg<64, false, false>(p, Hq * D, Hkv * D, st);
  return launch_fwd_wg<128, false, false>(p, Hq * D, Hkv * D, st);
}

// the wgmma kernels: same contract as dalm_b200_attention_bwd, head_dim 64 or 128 (dropout at 64)
extern "C" int dalm_b200_attention_tc_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                          long long ldv, const int64_t* mask, const void* out, long long ldo,
                                          const float* lse, const void* d_out, long long lddo, float* delta, void* dq,
                                          long long lddq, void* dk, long long lddk, void* dv, long long lddv, int B, int L,
                                          int Hq, int Hkv, int D, float scale, int causal, int window, float drop_p,
                                          unsigned long long drop_seed, unsigned long long drop_stream_id,
                                          const void* drop_offset, void* stream) {
  AttnParams p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.mask = mask; p.o = (__nv_bfloat16*)const_cast<void*>(out); p.ldo = ldo;
  p.lse = const_cast<float*>(lse); p.d_o = (const __nv_bfloat16*)d_out; p.lddo = lddo; p.delta = delta;
  p.dq = (__nv_bfloat16*)dq; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv;
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
  p.B = B; p.L = L; p.Hq = Hq; p.Hkv = Hkv; p.scale = scale; p.causal = causal;
  p.drop = make_drop(drop_p, drop_seed, drop_stream_id, drop_offset);
  const bool win = set_window(p, window);
  if (int e = check_common(p, D)) return e;
  DALM_REQUIRE(D == 64 || D == 128, "attention_tc: head_dim %d unsupported (64/128)", D);
  DALM_REQUIRE(lddo % 8 == 0 && ((uintptr_t)d_out & 15) == 0, "attention_tc_bwd: d_out alignment");
  DALM_REQUIRE(drop_p >= 0.f && drop_p < 1.f && (drop_p == 0.f || D == 64), "attention_tc_bwd: dropout needs p in [0,1) and head_dim 64");
  cudaStream_t st = (cudaStream_t)stream;
  if (drop_p > 0.f) return launch_bwd_wg<64, true, false>(p, Hq * D, Hkv * D, st);
  if (win) return D == 64 ? launch_bwd_wg<64, false, true>(p, Hq * D, Hkv * D, st) : launch_bwd_wg<128, false, true>(p, Hq * D, Hkv * D, st);
  if (D == 64) return launch_bwd_wg<64, false, false>(p, Hq * D, Hkv * D, st);
  return launch_bwd_wg<128, false, false>(p, Hq * D, Hkv * D, st);
}
