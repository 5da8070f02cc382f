// dalm_b200 — bf16 GEMM on the Hopper tensor cores (wgmma, accumulators in registers, operands fed by TMA).
//
//     D[M,N] = epilogue( alpha * A[M,K] . B[N,K]^T )            A, B bf16 row-major ("TN": both K-contiguous)
//
// This single kernel is every dense contraction of the training step: the linear layers of the encoder / decoder
// forward (B = W[out,in]), their dgrad (B = W^T[in,out], kept as a resident transposed copy - weights are frozen in
// PEFT mode), the LoRA adapters (folded into the K dimension: A = [x | x A_l^T], B = [W | s B_l]) and the lm_head. It
// replaces the cuBLAS calls made by HF modeling code under dalm/models/rag_e2e_base_model.py:93,105 (reference) and the
// autograd backward of those. The kernel structure is described above gemm_bf16_tn_kernel.
#include "common.cuh"
#include "ptx.cuh"
#include <cudaTypedefs.h>
#include <mutex>
#include <unordered_map>

namespace dalm {
using namespace ptx;

// Epilogue kind, a template parameter of the kernel: each fused entry point launches its own instance, and the plain
// instances carry no fused code.
enum class Epi {
  Plain,     // out = act(alpha * acc + bias) (+ dropout) + resid                                        (gemm_bf16)
  SwiGLU,    // tile columns [0,128) = gate, [128,256) = up of the same 128 features (weight rows interleaved); besides
             // `out` (gate|up, the backward's input) the tile's silu(gate) * up goes to tmap_out2        (gemm_bf16_swiglu)
  RoPE,      // rotary position embedding (head_dim 128, HF rotate_half) on output columns < rope_cols    (gemm_bf16_rope)
  GeluPair,  // `out` = pre-activation (bf16, what the backward needs), tmap_out2 = gelu(pre) (bf16, the next GEMM's
             // operand): one launch instead of GEMM + a 2-pass kernel                                     (gemm_bf16_gelu)
  NormRoPE,  // RoPE after a per-head RMSNorm (Qwen3 q_norm / k_norm); tmap_out2 = the pre-norm q|k columns (bf16), and
             // the per-head rstd to ep.norm_rstd (fp32): what the backward needs                        (gemm_bf16_rope)
};

struct GemmEpilogue {
  void* out;            // [M, ldo]
  long long ldo;
  int out_f32;          // 0: bf16, 1: fp32
  const float* bias;    // [N] fp32 or nullptr
  const void* resid;    // [M, ldr] added after activation, or nullptr (may alias out)
  long long ldr;
  int resid_f32;
  int act;              // 0: none, 1: GELU(erf), 2: GELU backward - out = bf16(alpha*acc + bias) * gelu'(resid) (resid = the bf16
                        //    pre-activation; multiplied, not added): the dgrad GEMM of the FFN output projection emits d(pre) directly
  float alpha;
  int M, N, K;
  DropCfg drop;         // dropout on act(alpha*acc+bias) BEFORE the residual add (BertSelfOutput / BertOutput); p = 0 => off
  int group_m;          // tile rasterisation: bands of group_m m-tiles, n-tiles walked serpentine inside a band (0 = m-fastest)
  const float* rope_cos; const float* rope_sin;   // Epi::RoPE: fp32 [rope_L, 64]; the position of output row m is m % rope_L
  int rope_L, rope_cols;
  const float* q_norm; const float* k_norm;       // Epi::NormRoPE: fp32 [128] weights of the q heads / of the k heads
  int nq_heads;                                   //   heads [0, nq_heads) of the rope columns are q heads, the rest k heads
  float norm_eps;
  float* norm_rstd; long long ld_rstd;            //   fp32 [M, rope_cols / 128] or nullptr
  int norm_pre;                                   //   1: tmap_out2 receives the pre-norm q|k columns [M, rope_cols]
  int l2_hints;         // TMA L2 eviction priorities: bit 0 = A loads evict_last (the panel the resident CTAs share across waves),
                        // bit 1 = B loads evict_first (streamed once per band), bit 2 = output stores evict_first
};

// Tile rasterisation. Persistent CTA i works on tiles i, i + grid, ...: the tiles resident at one moment are ~132 consecutive
// indices, and (L2 serving the CTAs that share a panel) DRAM sees each A panel / B panel of that footprint once per wave.
// m-fastest order makes the footprint num_m x 4 tiles: all of A is re-read by every wave. Bands of group_m m-tiles make it
// ~square (group_m x 132/group_m), which minimises
// rows-of-A + rows-of-B per wave, and the serpentine n order lets consecutive waves of a band re-use its A panel from L2.
__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int gm, int& m_blk, int& n_blk) {
  if (gm <= 0) { m_blk = tile % num_m; n_blk = tile / num_m; return; }
  const int band_tiles = gm * num_n;
  const int band = tile / band_tiles;
  const int r = tile - band * band_tiles;
  const int m0 = band * gm;
  const int h = min(gm, num_m - m0);                            // the last band may be shorter
  const int n = r / h;
  m_blk = m0 + (r - n * h);
  n_blk = (band & 1) ? (num_n - 1 - n) : n;
}

// The epilogue runs on the accumulator registers, in the wgmma fragment layout. In a consumer warpgroup (64 rows of the tile),
// thread (warp q, lane) holds acc[4 j + 2 h + e] = row 16 q + lane / 4 + 8 h, column 8 j + 2 (lane & 3) + e of the tile,
// for j < BN / 8, h, e in {0, 1}. Each warpgroup drains its own 64 rows through a 128B-swizzled staging box and TMA stores:
// 128 bytes of columns per store block (64 bf16 or 32 fp32). HBM sees full 128-byte lines, and the TMA unit clips ragged
// M / N edges. Nothing goes through the stage ring, so the producer loads the next tile while this one is stored.
constexpr int kBoxRows = 64;                                    // output tensor maps: [64 rows x 128 bytes] boxes
constexpr int kBoxBytes = kBoxRows * 128;                       // one staging box
constexpr int kStageTileBytes = 2 * kBoxBytes;                  // per consumer warpgroup: two boxes used in turn
constexpr int kEpiGroups = 2;                                   // the two consumer warpgroups, each its own epilogue
constexpr int kGemmThreads = 128 + kEpiGroups * 128;            // warpgroup 0: TMA producer ; warpgroups 1-2: wgmma + epilogue

// A consumer warpgroup's staging: two boxes used in turn, so that the math of one store block overlaps the TMA unit reading
// the previous one. begin() hands out the box once its last store has read it; end() stores it as a [64 rows x 128 B] box.
struct EpiStage {
  unsigned char* boxes;                                         // 1024-aligned, 2 x kBoxBytes
  int bar;                                                      // named barrier of the warpgroup's 128 threads
  bool issuer;                                                  // the warpgroup's first thread issues and waits for the stores
  int buf;
  __device__ __forceinline__ unsigned char* begin() {
    if (issuer) bulk_wait_read<1>();                            // the store issued two blocks ago has finished reading this box
    named_bar_sync(bar, 128);
    return boxes + buf * kBoxBytes;
  }
  __device__ __forceinline__ void end(const CUtensorMap* tm, int col, int row, bool evict_first) {
    fence_proxy_async();                                        // generic-proxy smem writes -> visible to the TMA unit
    named_bar_sync(bar, 128);
    if (issuer) {
      const unsigned char* box = boxes + buf * kBoxBytes;
      if (evict_first) tma_store_2d_hint(tm, box, col, row, l2_policy_evict_first());
      else             tma_store_2d(tm, box, col, row);
      bulk_commit();
    }
    buf ^= 1;
  }
};

// Box row r, byte b of the row: 16-byte pieces XOR-swizzled by r % 8, the layout CU_TENSOR_MAP_SWIZZLE_128B expects. A warp's
// 8 rows (r % 8 all different) x 4 lanes fill all 32 banks: conflict-free.
__device__ __forceinline__ void box_st_bf16x2(unsigned char* box, int r, int b, float lo, float hi) {
  *reinterpret_cast<__nv_bfloat162*>(box + r * 128 + ((((b >> 4) ^ (r & 7)) << 4) | (b & 15))) = __floats2bfloat162_rn(lo, hi);
}
__device__ __forceinline__ void box_st_f32x2(unsigned char* box, int r, int b, float lo, float hi) {
  *reinterpret_cast<float2*>(box + r * 128 + ((((b >> 4) ^ (r & 7)) << 4) | (b & 15))) = make_float2(lo, hi);
}

// The plain epilogue on the 8 values a thread holds of fragment columns j0, j0 + 1: x[4 jj + 2 h + e] is row `row` + 8 h,
// column `col` + 8 jj + e (col = 8 j0 + 2 (lane & 3) in output columns). Per element, in this order: alpha, + bias, act 1
// (GELU), dropout, then the residual (act 2: the value rounded to bf16, times gelu'(resid)). resid_loaded: the caller adds
// an fp32 residual it has already loaded, so it is not read here.
__device__ __forceinline__ void epilogue_math(const GemmEpilogue& ep, float* x, int row, int col, bool ok0, bool ok1,
                                              unsigned long long dstream, bool resid_loaded = false) {
  const int N = ep.N;
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] *= ep.alpha;
  if (ep.bias) {
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      if (col + 8 * jj < N) {                                   // N % 8 == 0: both columns of the pair are in or out
        const float b0 = __ldg(ep.bias + col + 8 * jj), b1 = __ldg(ep.bias + col + 8 * jj + 1);
        x[4 * jj + 0] += b0; x[4 * jj + 1] += b1; x[4 * jj + 2] += b0; x[4 * jj + 3] += b1;
      }
    }
  }
  if (ep.act == 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = gelu_erf(x[i]);
  }
  if (ep.drop.p > 0.f) {
    // The values lie in 4 groups of 8 columns, g = 2 jj + h, and every lane of the quad holds 2 columns of each: word k of
    // the group's Philox output (k = lane & 3). Lane k draws group k, and the quad transposes the words with shuffles.
    const int k = threadIdx.x & 3;
    const unsigned long long idx8 = ((unsigned long long)(row + 8 * (k & 1)) * (unsigned long long)N +
                                     (unsigned long long)(col - 2 * k + 8 * (k >> 1))) >> 3;
    const uint4 r = drop_bits8(ep.drop, dstream, idx8);
    unsigned int m0 = 0u, m1 = 0u, m2 = 0u, m3 = 0u;            // word k of groups 0..3 (scalars: no local-memory array)
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      // send word k ^ s of this lane's group (what lane k ^ s needs), receive word k of group k ^ s
      const int t = k ^ s;
      const unsigned int v = t == 0 ? r.x : t == 1 ? r.y : t == 2 ? r.z : r.w;
      const unsigned int got = s ? __shfl_xor_sync(0xffffffffu, v, s) : v;
      m0 = t == 0 ? got : m0; m1 = t == 1 ? got : m1; m2 = t == 2 ? got : m2; m3 = t == 3 ? got : m3;
    }
    const unsigned int m[4] = {m0, m1, m2, m3};
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      x[2 * g + 0] *= (m[g] & 0xFFFFu) >= ep.drop.thresh ? ep.drop.inv_keep : 0.f;
      x[2 * g + 1] *= (m[g] >> 16) >= ep.drop.thresh ? ep.drop.inv_keep : 0.f;
    }
  }
  if (ep.resid && !resid_loaded) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!(h ? ok1 : ok0)) continue;
      const size_t roff = (size_t)(row + 8 * h) * ep.ldr;
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int c = col + 8 * jj;
        if (c >= N) continue;
        float* v = x + 4 * jj + 2 * h;
        if (ep.resid_f32) {
          const float2 t = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(ep.resid) + roff + c);
          v[0] += t.x; v[1] += t.y;
        } else {
          const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(reinterpret_cast<const __nv_bfloat16*>(ep.resid) + roff + c));
          if (ep.act == 2) {     // same roundings as the un-fused pair (bf16 dgrad output, then gelu_bwd_kernel): bit-identical results
            v[0] = __bfloat162float(__float2bfloat16_rn(v[0])) * gelu_erf_grad(t.x);
            v[1] = __bfloat162float(__float2bfloat16_rn(v[1])) * gelu_erf_grad(t.y);
          } else {
            v[0] += t.x; v[1] += t.y;
          }
        }
      }
    }
  }
}

// Drains this warpgroup's 64 x BN accumulator (rows row0 .., tile columns tile_col0 ..) to HBM; see above for the layout.
// The plain store blocks run as a loop that is not unrolled: each iteration reads the 8 fragment columns at the front of acc
// (static indices, so acc stays in registers) and then shifts the rest down, which consumes acc. Unrolled, the epilogue is
// straight-line code several times the size of the instruction cache, and its GELU and dropout variants ran slower than
// the loop over an accumulator parked in shared memory that they replace.
template <int BN, Epi EPI>
__device__ __forceinline__ void epilogue_tile(const GemmEpilogue& ep, const CUtensorMap* tmap_out, const CUtensorMap* tmap_out2,
                                              EpiStage& sg, float (&acc)[BN / 2], int row0, int tile_col0) {
  static_assert(BN == 256 || EPI == Epi::Plain || EPI == Epi::GeluPair, "the SwiGLU and RoPE epilogues need 256-wide tiles");
  const int N = ep.N;
  const int lane = threadIdx.x & 31, k = lane & 3;
  const int rb = 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2);  // box row of the thread's first row; the second is rb + 8
  const int row = row0 + rb;
  const bool ok0 = row < ep.M, ok1 = row + 8 < ep.M;
  const int cq = tile_col0 + 2 * k;                             // output column of x[0] of fragment column 0
  const bool hint = (ep.l2_hints & 4) != 0;
  const unsigned long long dstream = ep.drop.p > 0.f ? drop_stream(ep.drop) : 0ull;
  auto frag8 = [&](float* x, int j0) {                          // fragment columns j0, j0 + 1 (j0 a constant once unrolled)
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = acc[4 * j0 + i];
  };
  auto shift8 = [&]() {                                         // fragment columns 8.. to the front
#pragma unroll
    for (int i = 0; i + 32 < BN / 2; ++i) acc[i] = acc[i + 32];
  };

  if (EPI == Epi::Plain && ep.out_f32) {
    // fp32 out: 32 columns = fragment columns 4 b .. 4 b + 3 of the front per store block, two blocks per iteration. An
    // fp32 residual (o_proj / down-projection: x_out = x + y) is fetched one block ahead, so its HBM latency is not in the
    // block's serial chain.
    const bool rpf = ep.resid != nullptr && ep.resid_f32;
    float2 rn[8];                                               // [4 u + 2 jj + h]: the next block's residual
    auto fetch_resid = [&](int c) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int h = i & 1, cc = cq + c + 8 * (i >> 1);
        rn[i] = ((h ? ok1 : ok0) && c < BN && cc < N)
                    ? *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(ep.resid) + (size_t)(row + 8 * h) * ep.ldr + cc)
                    : make_float2(0.f, 0.f);
      }
    };
    if (rpf) fetch_resid(0);
#pragma unroll 1
    for (int c = 0; c < BN && tile_col0 + c < N; c += 64) {    // uniform across the warpgroup
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int cb = c + 32 * b;
        if (tile_col0 + cb >= N) break;
        unsigned char* box = sg.begin();
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          float x[8];
          frag8(x, 4 * b + 2 * u);
          epilogue_math(ep, x, row, cq + cb + 16 * u, ok0, ok1, dstream, rpf);
#pragma unroll
          for (int i = 0; i < 4; ++i) {                       // the residual, last (zero where out of bounds)
            if (rpf) { x[2 * i] += rn[4 * u + i].x; x[2 * i + 1] += rn[4 * u + i].y; }
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) box_st_f32x2(box, rb + 8 * (i & 1), 64 * u + 32 * (i >> 1) + 8 * k, x[2 * i], x[2 * i + 1]);
        }
        if (rpf) fetch_resid(cb + 32);
        sg.end(tmap_out, tile_col0 + cb, row0, hint);
      }
      shift8();
    }
    return;
  }

  if constexpr (EPI == Epi::SwiGLU) {
    // SwiGLU forward: act[:, 128 n_blk + 64 b + ...] = silu(gate) * up from the fp32 accumulators (gate columns 64 b.., up
    // columns 128 + 64 b..: fragment columns j and j + 16 of the same thread), two more store blocks per tile. Replaces a
    // separate pass that re-read the 203 MB gate|up buffer. First, while acc is whole.
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      unsigned char* box = sg.begin();
#pragma unroll
      for (int jl = 0; jl < 8; ++jl) {
        const int j = 8 * b + jl;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float f[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float g = acc[4 * j + 2 * h + e];
            f[e] = g / (1.f + __expf(-g)) * acc[4 * (j + 16) + 2 * h + e];
          }
          box_st_bf16x2(box, rb + 8 * h, 16 * jl + 4 * k, f[0], f[1]);
        }
      }
      sg.end(tmap_out2, (tile_col0 >> 1) + 64 * b, row0, hint);
    }
  }
  // bf16 out: 64 columns = fragment columns 8 b .. 8 b + 7 per store block
  const bool rope_tile = (EPI == Epi::RoPE || EPI == Epi::NormRoPE) && tile_col0 < ep.rope_cols;   // rope_cols % 256 == 0
  float rstd[2][2];                                             // NormRoPE: [head of the tile][h]
  const float* nwt[2];
  if (EPI == Epi::NormRoPE && rope_tile) {
    // per-head RMSNorm (Qwen3 q_norm / k_norm over each head's 128 columns, weight [128]): a thread holds 32 of a head's
    // columns in each of its two rows; the quad's partial sums of squares are combined with a butterfly, so all 4 lanes
    // (and both halves of the head) use the same rstd.
#pragma unroll
    for (int hd = 0; hd < 2; ++hd) {
      const int head = (tile_col0 >> 7) + hd;
      nwt[hd] = head < ep.nq_heads ? ep.q_norm : ep.k_norm;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float ss = 0.f;
#pragma unroll
        for (int jl = 0; jl < 16; ++jl) {
          const int j = 16 * hd + jl;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float x = acc[4 * j + 2 * h + e];
            if (ep.bias) x += __ldg(ep.bias + cq + 8 * j + e);
            ss = fmaf(x, x, ss);
          }
        }
        ss += __shfl_xor_sync(0xffffffffu, ss, 1);
        ss += __shfl_xor_sync(0xffffffffu, ss, 2);
        rstd[hd][h] = rsqrtf(ss * (1.f / 128.f) + ep.norm_eps);
        if (ep.norm_rstd && (h ? ok1 : ok0) && k == 0) ep.norm_rstd[(size_t)(row + 8 * h) * ep.ld_rstd + head] = rstd[hd][h];
      }
    }
  }
  if ((EPI == Epi::RoPE || EPI == Epi::NormRoPE) && rope_tile) {
#pragma unroll
    for (int c = 0; c < BN; c += 64) {                         // rope tiles lie inside N
      const int col0 = tile_col0 + c;
      const int jb = c / 8;
      // RoPE in the QKV epilogue (head_dim 128, HF rotate_half): this 64-column block is one half of a head (x1 = columns
      // 0..63, x2 = 64..127; tiles are 256 columns = two whole heads). Its partner half is fragment column j -+ 8, in the
      // same thread.    x1' = x1 cos - x2 sin ,  x2' = x2 cos + x1 sin    (cos / sin of the row's position, index column % 64)
      // A q/k/v bias (Qwen2) is added to both halves in fp32 before the rotation; NormRoPE (Qwen3) then applies
      // x * rstd * w. The only rounding is the final bf16 store.
      const bool second = ((c >> 6) & 1) != 0;
      const int jp = second ? -8 : 8;
      const int hd = c >> 7;
      const int io = (c & 64) + 2 * k, ip = ((c & 64) ^ 64) + 2 * k;   // in-head index of the own / partner value of jl = 0
      unsigned char* box = sg.begin();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int pos = (h ? ok1 : ok0) ? (row + 8 * h) % ep.rope_L : 0;
        const float* cs = ep.rope_cos + (size_t)pos * 64 + 2 * k;
        const float* sn = ep.rope_sin + (size_t)pos * 64 + 2 * k;
#pragma unroll
        for (int jl = 0; jl < 8; ++jl) {
          const int j = jb + jl;
          const float2 cc = __ldg(reinterpret_cast<const float2*>(cs + 8 * jl));
          const float2 s2 = __ldg(reinterpret_cast<const float2*>(sn + 8 * jl));
          float f[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float own = acc[4 * j + 2 * h + e], oth = acc[4 * (j + jp) + 2 * h + e];
            if (ep.bias) {
              own += __ldg(ep.bias + cq + 8 * j + e);
              oth += __ldg(ep.bias + cq + 8 * (j + jp) + e);
            }
            if constexpr (EPI == Epi::NormRoPE) {
              own = own * rstd[hd][h] * __ldg(nwt[hd] + io + 8 * jl + e);
              oth = oth * rstd[hd][h] * __ldg(nwt[hd] + ip + 8 * jl + e);
            }
            const float cv = e ? cc.y : cc.x, sv = e ? s2.y : s2.x;
            f[e] = second ? fmaf(own, cv, oth * sv) : fmaf(own, cv, -oth * sv);
          }
          box_st_bf16x2(box, rb + 8 * h, 16 * jl + 4 * k, f[0], f[1]);
        }
      }
      sg.end(tmap_out, col0, row0, hint);
      if (EPI == Epi::NormRoPE && ep.norm_pre) {
        // the pre-norm block (+ bias, rounded once to bf16) for the backward
        box = sg.begin();
#pragma unroll
        for (int jl = 0; jl < 8; ++jl) {
          const int j = jb + jl;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float f[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              f[e] = acc[4 * j + 2 * h + e];
              if (ep.bias) f[e] += __ldg(ep.bias + cq + 8 * j + e);
            }
            box_st_bf16x2(box, rb + 8 * h, 16 * jl + 4 * k, f[0], f[1]);
          }
        }
        sg.end(tmap_out2, col0, row0, false);
      }
    }
    return;
  }
  // plain math, bf16 out: fragment columns 0..7 of the front per store block; GeluPair also writes gelu() of the ROUNDED
  // values (exactly what gelu_fwd_kernel would read back from HBM) to tmap_out2
#pragma unroll 1
  for (int c = 0; c < BN && tile_col0 + c < N; c += 64) {      // uniform across the warpgroup
    const int col0 = tile_col0 + c;
    __nv_bfloat162 pk[16];                                      // [4 u + 2 jj + h]
    unsigned char* box = sg.begin();
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float x[8];
      frag8(x, 2 * u);
      epilogue_math(ep, x, row, cq + c + 16 * u, ok0, ok1, dstream);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        pk[4 * u + i] = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
        *reinterpret_cast<__nv_bfloat162*>(box + (rb + 8 * (i & 1)) * 128 +
                                           ((((2 * u + (i >> 1)) ^ (rb & 7)) << 4) | (4 * k))) = pk[4 * u + i];
      }
    }
    sg.end(tmap_out, col0, row0, hint);
    if constexpr (EPI == Epi::GeluPair) {
      box = sg.begin();
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float2 p = __bfloat1622float2(pk[i]);
        box_st_bf16x2(box, rb + 8 * (i & 1), 16 * (i >> 1) + 4 * k, gelu_erf(p.x), gelu_erf(p.y));
      }
      sg.end(tmap_out2, col0, row0, false);
    }
    shift8();
  }
}

template <int BN> struct GemmCfg {
  static constexpr int BM = 128, BK = 64;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + kEpiGroups * kStageTileBytes + 1024 /*alignment slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "exceeds 227 KB of shared memory per block");
};

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t da, uint64_t db, int scale_d) {
  if constexpr (BN == 256) wgmma_m64n256k16<TA, TB>(d, da, db, scale_d);
  else if constexpr (BN == 128) wgmma_m64n128k16<TA, TB>(d, da, db, scale_d);
  else wgmma_m64n64k16<TA, TB>(d, da, db, scale_d);
}

// LAYOUT selects how the two bf16 operands lie in HBM (wgmma reads either major directly; nothing is transposed):
//   0  "TN"  A[M,K], B[N,K]  both K-contiguous                 forward y = x W^T, and PEFT dgrad against resident W^T copies
//   1  "NN"  A[M,K], B[K,N]  B is MN-major (N-contiguous)      dgrad dx = dy W straight from W[out,in] (full fine-tuning:
//                                                              weights change every step, so no transposed copy is kept)
//   2  "wgrad" A[K,M], B[K,N] both MN-major                    dW[out,in] = dy^T x : contraction over the token rows
// MN-major stage tiles are stored [64 k-rows][64 elements = 128 B] per 64-wide chunk (8 KB, chunks LBO = 8 KB apart,
// 8-row groups SBO = 1 KB apart), each chunk one TMA box of the row-major source.
//
// Structure (persistent CTAs, 384 threads = three warpgroups):
//   warpgroup 0 : TMA producer (one thread) - 128B-swizzled tiles into a STAGES-deep shared-memory ring
//   warpgroups 1, 2 : consumers - each issues m64 x BN x 16 wgmma for its 64 rows of the 128-row tile, accumulators in
//                 registers; after the k loop each runs epilogue_tile on its own accumulator registers and stores its
//                 64 rows through its own staging boxes.
// The consumers release a stage as soon as the wgmmas reading it have retired, at the end of a tile as inside it, and the
// producer refills it at once: while the consumers run a tile's epilogue, the next tile's first STAGES k-blocks load.
// CL = 2: a cluster of two CTAs computes a 256 x BN tile (128 rows each); each CTA loads half of the shared B tile and
// multicasts it to both, so every B panel is read from L2 once per two CTAs (block_n 2128 / 2256).
template <int BN, int LAYOUT, Epi EPI, int CL>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                    const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_out2, const GemmEpilogue ep) {
  using Cfg = GemmCfg<BN>;
  constexpr int BM = Cfg::BM, BK = Cfg::BK, STAGES = Cfg::STAGES;
  static_assert(CL == 1 || (LAYOUT == 0 && EPI == Epi::Plain), "the cluster kernel takes the plain TN layout");
  extern __shared__ unsigned char smem_raw[];
  // 128B swizzle atoms need 1024-byte aligned tile bases
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* staging = smem + STAGES * Cfg::STAGE_BYTES;             // per consumer warpgroup 2 x [64 rows x 128 B], 1024-aligned
  uint64_t* full_bar  = reinterpret_cast<uint64_t*>(staging + kEpiGroups * kStageTileBytes);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = CL == 2 ? cluster_ctarank() : 0u;
  const int M = ep.M, N = ep.N, K = ep.K;
  const int num_m = (M + CL * BM - 1) / (CL * BM), num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (K + BK - 1) / BK;
  const int unit = blockIdx.x / CL, num_units = gridDim.x / CL;
  const int group_m = CL == 2 ? 0 : ep.group_m;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    prefetch_tmap(&tmap_out);
    if constexpr (EPI == Epi::SwiGLU || EPI == Epi::GeluPair || EPI == Epi::NormRoPE) prefetch_tmap(&tmap_out2);
  }
  if (threadIdx.x == 32) {
    // consumer releases: one arrive per consumer warp, of every CTA whose producer writes into this stage
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8 * CL); }
    fence_mbar_init();
  }
  if constexpr (CL == 2) cluster_sync_all();
  else __syncthreads();

  if (warp < 4) {
    // =============================== TMA producer ===============================
    // registers go to the consumers: 40 x 128 + 232 x 256 <= 64 K
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      const bool hint_a = (ep.l2_hints & 1) != 0, hint_b = (ep.l2_hints & 2) != 0;
      const uint64_t pol_a = hint_a ? l2_policy_evict_last() : 0ull, pol_b = hint_b ? l2_policy_evict_first() : 0ull;
      auto load = [](void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, bool hinted, uint64_t pol) {
        if (hinted) tma_load_2d_hint(dst, tm, bar, c0, c1, pol);
        else        tma_load_2d(dst, tm, bar, c0, c1);
      };
      for (int tile = unit; tile < num_tiles; tile += num_units) {
        int m_blk, n_blk;
        tile_coords(tile, num_m, num_n, group_m, m_blk, n_blk);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          unsigned char* sa = smem + stage * Cfg::STAGE_BYTES;
          unsigned char* sb = sa + Cfg::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          if constexpr (CL == 2) {
            load(sa, &tmap_a, &full_bar[stage], kb * BK, (m_blk * CL + (int)rank) * BM, hint_a, pol_a);
            tma_load_2d_multicast(sb + rank * (Cfg::B_BYTES / 2), &tmap_b, &full_bar[stage], kb * BK, n_blk * BN + (int)rank * (BN / 2), 0x3);
          } else {
            if constexpr (LAYOUT == 2) {
#pragma unroll
              for (int c = 0; c < BM / 64; ++c) load(sa + c * 8192, &tmap_a, &full_bar[stage], m_blk * BM + c * 64, kb * BK, hint_a, pol_a);
            } else {
              load(sa, &tmap_a, &full_bar[stage], kb * BK, m_blk * BM, hint_a, pol_a);
            }
            if constexpr (LAYOUT >= 1) {
#pragma unroll
              for (int c = 0; c < BN / 64; ++c) load(sb + c * 8192, &tmap_b, &full_bar[stage], n_blk * BN + c * 64, kb * BK, hint_b, pol_b);
            } else {
              load(sb, &tmap_b, &full_bar[stage], kb * BK, n_blk * BN, hint_b, pol_b);
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // =============================== consumers: wgmma, then epilogue ===============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int grp = (warp - 4) >> 2;                            // warpgroup 0 / 1 = rows [64 grp, 64 grp + 64) of the tile
    EpiStage sg{staging + grp * kStageTileBytes, 1 + grp, (threadIdx.x & 127) == 0, 0};
    constexpr int TA = LAYOUT == 2 ? 1 : 0, TB = LAYOUT >= 1 ? 1 : 0;
    // k-step (16 elements of K) in 16-byte units of the descriptor start address: K-major +32 B inside the swizzle atom,
    // MN-major +16 rows * 128 B
    constexpr uint64_t a_step = TA ? 128 : 2, b_step = TB ? 128 : 2;
    // this warpgroup's 64 rows of A: K-major rows 64 grp.. (8 KB in), MN-major the second 64-element chunk (8 KB in)
    const uint32_t a_off = (uint32_t)grp * 8192u;
    int stage = 0; uint32_t phase = 0;
    for (int tile = unit; tile < num_tiles; tile += num_units) {
      int m_blk, n_blk;
      tile_coords(tile, num_m, num_n, group_m, m_blk, n_blk);
      float acc[BN / 2];
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);                     // TMA bytes have landed
        const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
        const uint32_t sb = sa + Cfg::A_BYTES;
        const uint64_t adesc = TA ? make_sw128_mnmajor_desc(sa + a_off, 8192, 1024) : make_sw128_kmajor_desc(sa + a_off);
        const uint64_t bdesc = TB ? make_sw128_mnmajor_desc(sb, 8192, 1024) : make_sw128_kmajor_desc(sb);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_tile<BN, TA, TB>(acc, adesc + a_step * (uint64_t)k, bdesc + b_step * (uint64_t)k, (kb | k) != 0 ? 1 : 0);
        wgmma_commit();
        wgmma_wait<1>();                                        // the previous k-block's wgmmas have retired
        if (prev >= 0 && lane == 0) {
          mbar_arrive(&empty_bar[prev]);
          if constexpr (CL == 2) mbar_arrive_remote(&empty_bar[prev], rank ^ 1u);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (lane == 0) {
        mbar_arrive(&empty_bar[prev]);
        if constexpr (CL == 2) mbar_arrive_remote(&empty_bar[prev], rank ^ 1u);
      }
      epilogue_tile<BN, EPI>(ep, &tmap_out, &tmap_out2, sg, acc, (m_blk * CL + (int)rank) * BM + grp * 64, n_blk * BN);
    }
    if (sg.issuer) bulk_wait<0>();                              // staging boxes must outlive their TMA reads
  }
  if constexpr (CL == 2) cluster_sync_all();                    // the peer may still multicast into / signal this CTA
}

// ------------------------------------------------------------------------------------------------------------
// host side: tensor-map construction (driver entry point fetched at run time, no libcuda link dependency) + cache
// ------------------------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  return fn;
}

struct TmapKey {
  const void* ptr; long long rows, cols, ld; int box_rows; int f32;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && f32 == o.f32;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h = h * 1000003u ^ (size_t)k.rows; h = h * 1000003u ^ (size_t)k.cols;
    h = h * 1000003u ^ (size_t)k.ld;   h = h * 1000003u ^ (size_t)(k.box_rows * 2 + k.f32);
    return h;
  }
};
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmaps;
static std::mutex g_tmap_mu;

// row-major [rows, cols] (bf16, or fp32 when f32 != 0) with row stride ld (elements);
// box = {128 bytes of columns, box_rows}, 128B swizzle, OOB loads -> 0, OOB stores clipped
int get_tmap(const void* ptr, long long rows, long long cols, long long ld, int box_rows, CUtensorMap* out, int f32) {
  TmapKey key{ptr, rows, cols, ld, box_rows, f32};
  {
    std::lock_guard<std::mutex> g(g_tmap_mu);
    auto it = g_tmaps.find(key);
    if (it != g_tmaps.end()) { *out = it->second; return 0; }
  }
  auto fn = get_encode_fn();
  DALM_REQUIRE(fn != nullptr, "gemm: cuTensorMapEncodeTiled driver entry point unavailable");
  DALM_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "gemm: operand base %p is not 16-byte aligned", ptr);
  DALM_REQUIRE((ld % (f32 ? 4 : 8)) == 0, "gemm: row stride %lld is not a multiple of 16 bytes", ld);
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * (f32 ? 4 : 2)};
  cuuint32_t box[2] = {f32 ? 32u : 64u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUtensorMap m;
  CUresult r = fn(&m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DALM_REQUIRE(r == CUDA_SUCCESS, "gemm: cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld box_rows=%d",
               (int)r, rows, cols, ld, box_rows);
  {
    std::lock_guard<std::mutex> g(g_tmap_mu);
    if (g_tmaps.size() > 8192) g_tmaps.clear();
    g_tmaps[key] = m;
  }
  *out = m;
  return 0;
}

template <int BN, int LAYOUT, Epi EPI>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const GemmEpilogue& ep,
                       int max_ctas, cudaStream_t stream, const CUtensorMap* to2) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    DALM_CUDA(cudaFuncSetAttribute(gemm_bf16_tn_kernel<BN, LAYOUT, EPI, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  const int num_tiles = ((ep.M + 127) / 128) * ((ep.N + BN - 1) / BN);
  int grid = num_tiles < num_sms() ? num_tiles : num_sms();
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  gemm_bf16_tn_kernel<BN, LAYOUT, EPI, 1><<<grid, kGemmThreads, Cfg::SMEM_BYTES, stream>>>(ta, tb, to, to2 ? *to2 : to, ep);
  count_launch();
  return check_launch("gemm_bf16_tn_kernel");
}

// block_n (64 / 128 / 256) -> the single-CTA kernel of that tile width
template <int LAYOUT, Epi EPI>
static int launch_gemm_bn(int bn, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const GemmEpilogue& ep,
                          int max_ctas, cudaStream_t stream, const CUtensorMap* to2 = nullptr) {
  if (bn == 256) return launch_gemm<256, LAYOUT, EPI>(ta, tb, to, ep, max_ctas, stream, to2);
  if (bn == 128) return launch_gemm<128, LAYOUT, EPI>(ta, tb, to, ep, max_ctas, stream, to2);
  return launch_gemm<64, LAYOUT, EPI>(ta, tb, to, ep, max_ctas, stream, to2);
}

template <int BN>
static int launch_gemm_cluster(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const GemmEpilogue& ep,
                               int max_ctas, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_bf16_tn_kernel<BN, 0, Epi::Plain, 2>;
  static bool attr_set = false;
  if (!attr_set) {
    DALM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  const int num_tiles = ((ep.M + 255) / 256) * ((ep.N + BN - 1) / BN);
  int clusters = num_tiles < num_sms() / 2 ? num_tiles : num_sms() / 2;
  if (max_ctas > 0 && clusters > max_ctas / 2) clusters = max_ctas / 2 > 0 ? max_ctas / 2 : 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * clusters);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  DALM_CUDA(cudaLaunchKernelEx(&cfg, kern, ta, tb, to, to, ep));
  count_launch();
  return check_launch("gemm_bf16_tn_kernel (cluster of 2)");
}

}  // namespace dalm

using namespace dalm;

// tile rasterisation override: -1 = m-fastest order everywhere, 0 = automatic (default: pick_group_m below), -2 = bands
// (bands for every multi-wave problem), > 0 = that many m-tiles per band. Initial value: env DALM_B200_GEMM_RASTER.
static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}
static int g_group_m_override = env_int("DALM_B200_GEMM_RASTER", 0);
extern "C" void dalm_b200_gemm_set_raster(int group_m) { g_group_m_override = group_m; }
// TMA L2 eviction hints (GemmEpilogue::l2_hints bit mask): -1 = automatic (default), 0..7 = that mask on every launch.
// Initial value: env DALM_B200_GEMM_L2_HINTS.
static int g_l2_hints = env_int("DALM_B200_GEMM_L2_HINTS", -1);
// largest A operand (bytes) treated as L2-resident across tile waves: a third of the L2 (16.7 MB on an H100), the rest
// serving the streamed B panels and output tiles. An estimate scaled from the rule's original derivation, not an H100
// measurement; the hints and the raster never change results.
static double l2_resident_a() { return (double)l2_bytes() / 3.0; }
extern "C" void dalm_b200_gemm_set_l2_hints(int mask) { g_l2_hints = mask < 0 ? -1 : (mask & 7); }
// Automatic choice: in the m-fastest regime (A [M,K] small enough to stay in L2, bf16 output) "A evict_last, B and stores
// evict_first" keeps the A panel resident while B and the output stream through; with banded rasters no hint is set.
static int pick_l2_hints(int M, int N, int K, int tile_n, int group_m, bool stream_out) {
  if (g_l2_hints >= 0) return g_l2_hints;
  const long long tiles = (long long)((M + 127) / 128) * ((N + tile_n - 1) / tile_n);
  return (group_m == 0 && tiles > num_sms() && 2.0 * M * K <= l2_resident_a() && !stream_out) ? 7 : 0;
}

// tile-shape heuristic: estimated time = waves of num_sms() CTAs x tile width x an efficiency penalty for narrow tiles (a
// 128 x BN tile re-reads its A operand from shared memory for every BN columns). The cluster kernel (block_n 2128/2256)
// is selected only explicitly.
static int pick_block_n(int M, int N) {
  const long long m1 = (M + 127) / 128;
  double best = 1e30;
  int bn = 64;
  const int cand[3] = {256, 128, 64};
  const double penalty[3] = {1.0, 1.55, 2.7};      // relative time per output column of 128x256 / 128x128 / 128x64 tiles
  for (int i = 0; i < 3; ++i) {
    if (cand[i] > 64 && N < cand[i]) continue;                // do not pad N by more than one tile
    const long long tiles = m1 * ((N + cand[i] - 1) / cand[i]);
    const double cost = (double)((tiles + num_sms() - 1) / num_sms()) * cand[i] * penalty[i];
    if (cost < best) { best = cost; bn = cand[i]; }
  }
  return bn;
}

// Band height of the tile rasterisation (0 = m-fastest). One wave = the num_sms() tiles resident at a time.
//  * m-fastest: a wave spans every m-tile of ~num_sms()/num_m n-tiles, so all of A is touched by every wave. When A [M,K] is small
//    enough to stay in L2 across waves (l2_resident_a(), next to a bf16 output stream) DRAM sees A once and every B panel
//    once - the algorithmic minimum.
//  * bands of g m-tiles walked serpentine in n: only the band's rows of A have to stay resident, B is streamed once per band:
//    traffic ~ A + B * nbands. Wins when A does not fit (down-projection, K = 11008) or when fp32 output + residual streams
//    push A out of L2 anyway (o_proj).
static int pick_group_m(int M, int N, int K, int tile_n, bool stream_out) {
  const int num_m = (M + 127) / 128, num_n = (N + tile_n - 1) / tile_n;
  int group_m = 0;
  if (g_group_m_override > 0) return g_group_m_override;
  if (g_group_m_override == -1 || (long long)num_m * num_n <= num_sms()) return 0;
  const double a_bytes = 2.0 * M * K;
  if (g_group_m_override == 0 && a_bytes <= l2_resident_a() && !stream_out) return 0;
  const double ideal = sqrt((double)num_sms() * tile_n / 128.0);   // footprint of a wave ~square: min rows-of-A + rows-of-B
  int nbands = (int)(num_m / ideal + 0.5);
  if (nbands < 1) nbands = 1;
  group_m = (num_m + nbands - 1) / nbands;                        // bands equalised over num_m
  if (group_m >= num_m) group_m = 0;                              // one band == m-fastest
  return group_m;
}

// The epilogue of one launch over an M x N x K problem in tiles tile_n wide, writing `out`, with the plain epilogue's
// defaults (alpha 1, no bias, activation, dropout or residual): callers set what their entry point adds. The raster and
// the L2 hints are chosen here for every entry point; an fp32 output or a residual read counts as streamed output.
static GemmEpilogue gemm_epilogue(int M, int N, int K, int tile_n, void* out, long long ldo, int out_f32 = 0,
                                  const void* resid = nullptr, long long ldr = 0, int resid_f32 = 0) {
  GemmEpilogue ep{};
  ep.out = out; ep.ldo = ldo; ep.out_f32 = out_f32;
  ep.resid = resid; ep.ldr = ldr; ep.resid_f32 = resid_f32;
  ep.alpha = 1.f;
  ep.M = M; ep.N = N; ep.K = K;
  ep.drop = make_drop(0.f, 0, 0, nullptr);
  const bool stream_out = out_f32 != 0 || resid != nullptr;
  ep.group_m = pick_group_m(M, N, K, tile_n, stream_out);
  ep.l2_hints = pick_l2_hints(M, N, K, tile_n, ep.group_m, stream_out);
  return ep;
}

// D[M,N] = act(alpha * A[M,K] B[N,K]^T + bias) + resid, out: bf16|fp32 [M,N] row stride ldo
// layout 0: A[M,K] B[N,K] (TN)   1: A[M,K] B[K,N] (NN, dgrad from W[out,in])   2: A[K,M] B[K,N] (wgrad, contraction over rows)
// block_n: 0 = auto, 64/128/256, or 2128/2256 (cluster of two CTAs).   max_ctas: 0 = all SMs (used by tests to force
// multi-tile-per-CTA paths)
extern "C" int dalm_b200_gemm_bf16(int layout, const void* A, long long lda, const void* B, long long ldb, void* out,
                                   long long ldo, int out_f32, int M, int N, int K, float alpha, const float* bias,
                                   int act, const void* resid, long long ldr, int resid_f32, int block_n,
                                   int max_ctas, float drop_p, unsigned long long drop_seed,
                                   unsigned long long drop_stream_id, const void* drop_offset, void* stream) {
  DALM_REQUIRE(layout >= 0 && layout <= 2, "gemm: layout must be 0 (TN), 1 (NN) or 2 (wgrad)");
  DALM_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  DALM_REQUIRE((N % 8) == 0, "gemm: N=%d must be a multiple of 8", N);
  DALM_REQUIRE((K % 8) == 0 || layout == 2, "gemm: K=%d must be a multiple of 8", K);
  DALM_REQUIRE((M % 8) == 0 || layout != 2, "gemm: M=%d must be a multiple of 8 for the wgrad layout", M);
  DALM_REQUIRE(lda >= (layout == 2 ? M : K) && ldb >= (layout >= 1 ? N : K) && ldo >= N, "gemm: leading dimensions too small");
  DALM_REQUIRE((ldo % (out_f32 ? 4 : 8)) == 0, "gemm: ldo=%lld breaks 16-byte row alignment", ldo);
  DALM_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "gemm: out is not 16-byte aligned");
  if (resid) {
    DALM_REQUIRE((ldr % (resid_f32 ? 4 : 8)) == 0, "gemm: ldr=%lld breaks 16-byte row alignment", ldr);
    DALM_REQUIRE((reinterpret_cast<uintptr_t>(resid) & 15) == 0, "gemm: resid is not 16-byte aligned");
  }
  DALM_REQUIRE(act == 0 || act == 1 || act == 2, "gemm: act must be 0 (none), 1 (gelu) or 2 (gelu backward: multiply by gelu'(resid))");
  DALM_REQUIRE(act != 2 || (resid != nullptr && !resid_f32 && !out_f32 && drop_p == 0.f),
               "gemm: act 2 (gelu backward) needs a bf16 `resid` (the pre-activation), a bf16 output and no dropout");
  int bn = block_n;
  if (bn == 0) bn = pick_block_n(M, N);
  DALM_REQUIRE(bn == 64 || bn == 128 || bn == 256 || bn == 2128 || bn == 2256,
               "gemm: block_n must be 0, 64/128/256 (single CTA) or 2128/2256 (cluster of two CTAs)");
  const bool pair = bn > 1000;
  DALM_REQUIRE(!(pair && layout != 0), "gemm: the cluster kernel only takes the TN layout");
  const int tile_n = pair ? bn % 1000 : bn;
  CUtensorMap ta, tb, to;
  if (layout == 2) { if (int e = get_tmap(A, K, M, lda, 64, &ta)) return e; }
  else             { if (int e = get_tmap(A, M, K, lda, 128, &ta)) return e; }
  if (layout >= 1) { if (int e = get_tmap(B, K, N, ldb, 64, &tb)) return e; }
  else             { if (int e = get_tmap(B, N, K, ldb, pair ? tile_n / 2 : tile_n, &tb)) return e; }
  if (int e = get_tmap(out, M, N, ldo, kBoxRows, &to, out_f32)) return e;
  DALM_REQUIRE(drop_p >= 0.f && drop_p < 1.f, "gemm: dropout p must be in [0,1)");
  GemmEpilogue ep = gemm_epilogue(M, N, K, tile_n, out, ldo, out_f32, resid, ldr, resid_f32);
  ep.bias = bias; ep.act = act; ep.alpha = alpha;
  ep.drop = make_drop(drop_p, drop_seed, drop_stream_id, drop_offset);
  cudaStream_t st = (cudaStream_t)stream;
  if (bn == 2256) return launch_gemm_cluster<256>(ta, tb, to, ep, max_ctas, st);
  if (bn == 2128) return launch_gemm_cluster<128>(ta, tb, to, ep, max_ctas, st);
  if (layout == 1) return launch_gemm_bn<1, Epi::Plain>(bn, ta, tb, to, ep, max_ctas, st);
  if (layout == 2) return launch_gemm_bn<2, Epi::Plain>(bn, ta, tb, to, ep, max_ctas, st);
  return launch_gemm_bn<0, Epi::Plain>(bn, ta, tb, to, ep, max_ctas, st);
}

// gate|up projection of LlamaMLP with SiLU(gate) * up fused into the epilogue (see include/dalm_b200.h)
extern "C" int dalm_b200_gemm_bf16_swiglu(const void* A, long long lda, const void* B, long long ldb, void* gu, long long ldgu,
                                          void* act, long long ldact, int M, int N, int K, void* stream) {
  DALM_REQUIRE(M > 0 && K > 0 && N >= 256 && (N % 256) == 0, "gemm_swiglu: N=%d must be a positive multiple of 256 (128-feature gate / up blocks)", N);
  DALM_REQUIRE((K % 8) == 0 && lda >= K && ldb >= K && ldgu >= N && ldact >= N / 2, "gemm_swiglu: bad K / leading dimensions");
  DALM_REQUIRE((ldgu % 8) == 0 && (ldact % 8) == 0 && ((uintptr_t)gu & 15) == 0 && ((uintptr_t)act & 15) == 0, "gemm_swiglu: output alignment");
  CUtensorMap ta, tb, to, to2;
  if (int e = get_tmap(A, M, K, lda, 128, &ta)) return e;
  if (int e = get_tmap(B, N, K, ldb, 256, &tb)) return e;
  if (int e = get_tmap(gu, M, N, ldgu, kBoxRows, &to, 0)) return e;
  if (int e = get_tmap(act, M, N / 2, ldact, kBoxRows, &to2, 0)) return e;
  const GemmEpilogue ep = gemm_epilogue(M, N, K, 256, gu, ldgu);
  return launch_gemm<256, 0, Epi::SwiGLU>(ta, tb, to, ep, 0, (cudaStream_t)stream, &to2);
}

// intermediate projection of a GELU MLP (BertIntermediate, Falcon dense_h_to_4h) with the activation fused into the epilogue and
// BOTH tensors written: pre = A B^T + bias (bf16; gelu_bwd needs it) and act = gelu(pre) (bf16; the output projection's operand).
extern "C" int dalm_b200_gemm_bf16_gelu(const void* A, long long lda, const void* B, long long ldb, void* pre, long long ldpre,
                                        void* act, long long ldact, int M, int N, int K, const float* bias, void* stream) {
  DALM_REQUIRE(M > 0 && N > 0 && K > 0 && (N % 8) == 0 && (K % 8) == 0, "gemm_gelu: bad shape M=%d N=%d K=%d", M, N, K);
  DALM_REQUIRE(lda >= K && ldb >= K && ldpre >= N && ldact >= N, "gemm_gelu: leading dimensions too small");
  DALM_REQUIRE((ldpre % 8) == 0 && (ldact % 8) == 0 && ((uintptr_t)pre & 15) == 0 && ((uintptr_t)act & 15) == 0, "gemm_gelu: output alignment");
  const int bn = pick_block_n(M, N);
  CUtensorMap ta, tb, to, to2;
  if (int e = get_tmap(A, M, K, lda, 128, &ta)) return e;
  if (int e = get_tmap(B, N, K, ldb, bn, &tb)) return e;
  if (int e = get_tmap(pre, M, N, ldpre, kBoxRows, &to, 0)) return e;
  if (int e = get_tmap(act, M, N, ldact, kBoxRows, &to2, 0)) return e;
  GemmEpilogue ep = gemm_epilogue(M, N, K, bn, pre, ldpre);
  ep.bias = bias;
  return launch_gemm_bn<0, Epi::GeluPair>(bn, ta, tb, to, ep, 0, (cudaStream_t)stream, &to2);
}

// fused q|k|v projection + rotary embedding: out[M,N] = A[M,K] B[N,K]^T + bias with HF's rotate_half RoPE (head_dim 128) applied to
// the output columns [0, rope_cols) in the epilogue. cos / sin: fp32 [L, 64]; row m sits at position m % L (token-major [B*L] rows).
// bias: fp32 [N] or NULL, added before the rotation on every column.
// q_norm != NULL (Qwen3): each 128-column head of [0, rope_cols) is RMS-normalised before the rotation, with weight q_norm on heads
// [0, nq_heads) and k_norm on the rest; pre_out (bf16 [M, rope_cols], ld_pre) receives the pre-norm columns and rstd_out (fp32
// [M, rope_cols / 128], ld_rstd) the heads' rstd, each when non-NULL. q_norm == NULL launches the plain RoPE instance.
extern "C" int dalm_b200_gemm_bf16_rope(const void* A, long long lda, const void* B, long long ldb, void* out, long long ldo, int M,
                                        int N, int K, const float* bias, const float* cos_t, const float* sin_t, int L, int rope_cols,
                                        const float* q_norm, const float* k_norm, int nq_heads, float eps, void* pre_out,
                                        long long ld_pre, float* rstd_out, long long ld_rstd, void* stream) {
  DALM_REQUIRE(M > 0 && N > 0 && K > 0 && (N % 8) == 0 && (K % 8) == 0, "gemm_rope: bad shape M=%d N=%d K=%d", M, N, K);
  DALM_REQUIRE(rope_cols > 0 && rope_cols <= N && (rope_cols % 256) == 0, "gemm_rope: rope_cols=%d must be a multiple of 256 (whole 128-wide heads per tile)", rope_cols);
  DALM_REQUIRE(L > 0 && cos_t != nullptr && sin_t != nullptr && ((uintptr_t)cos_t & 15) == 0 && ((uintptr_t)sin_t & 15) == 0, "gemm_rope: cos / sin tables");
  DALM_REQUIRE(lda >= K && ldb >= K && ldo >= N && (ldo % 8) == 0 && ((uintptr_t)out & 15) == 0, "gemm_rope: leading dimensions / alignment");
  CUtensorMap ta, tb, to;
  if (int e = get_tmap(A, M, K, lda, 128, &ta)) return e;
  if (int e = get_tmap(B, N, K, ldb, 256, &tb)) return e;
  if (int e = get_tmap(out, M, N, ldo, kBoxRows, &to, 0)) return e;
  GemmEpilogue ep = gemm_epilogue(M, N, K, 256, out, ldo);
  ep.bias = bias;
  ep.rope_cos = cos_t; ep.rope_sin = sin_t; ep.rope_L = L; ep.rope_cols = rope_cols;
  if (q_norm == nullptr) {
    DALM_REQUIRE(k_norm == nullptr && pre_out == nullptr && rstd_out == nullptr, "gemm_rope: k_norm / pre_out / rstd_out need q_norm");
    return launch_gemm<256, 0, Epi::RoPE>(ta, tb, to, ep, 0, (cudaStream_t)stream, nullptr);
  }
  DALM_REQUIRE(k_norm != nullptr && nq_heads >= 0 && nq_heads <= rope_cols / 128 && eps >= 0.f, "gemm_rope: norm weights / nq_heads=%d", nq_heads);
  DALM_REQUIRE(rstd_out == nullptr || ld_rstd >= rope_cols / 128, "gemm_rope: ld_rstd=%lld < %d heads", ld_rstd, rope_cols / 128);
  CUtensorMap to2 = to;
  if (pre_out != nullptr) {
    DALM_REQUIRE(ld_pre >= rope_cols && (ld_pre % 8) == 0 && ((uintptr_t)pre_out & 15) == 0, "gemm_rope: pre_out leading dimension / alignment");
    if (int e = get_tmap(pre_out, M, rope_cols, ld_pre, kBoxRows, &to2, 0)) return e;
  }
  ep.q_norm = q_norm; ep.k_norm = k_norm; ep.nq_heads = nq_heads; ep.norm_eps = eps;
  ep.norm_rstd = rstd_out; ep.ld_rstd = ld_rstd; ep.norm_pre = pre_out != nullptr;
  return launch_gemm<256, 0, Epi::NormRoPE>(ta, tb, to, ep, 0, (cudaStream_t)stream, &to2);
}

// drop cached tensor maps (call when operand buffers are freed / re-allocated at the same address with other shapes)
extern "C" void dalm_b200_gemm_clear_cache() {
  std::lock_guard<std::mutex> g(g_tmap_mu);
  g_tmaps.clear();
}
