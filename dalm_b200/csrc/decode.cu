// dalm_b200 — autoregressive greedy decoding for the evaluation path (reference dalm/eval/eval_rag.py:126-140:
// `model.generate(**inputs, max_length=max_length, early_stopping=True)` on the generator, then exact match :268-277).
//
//   rope_pos_kernel      : RoPE at explicit per-token position ids (HF generate derives them from the attention mask:
//                          cumsum(mask) - 1, so left / right padded prompts rotate differently from arange)
//   attn_decode_kernel   : one query token per sequence against the KV cache. HBM-bound: reads the cached K and V of
//                          one (sequence, kv head) once = 2 * T * D * 2 bytes; the current token's K / V rows are
//                          appended to the cache by the same launch (no separate copy kernel)
//   greedy_step_kernel   : argmax over the vocabulary row + HF's finished-sequence bookkeeping (pad after EOS), writes
//                          the token, its attention-mask bit and its position id for the next step
//   sample_step_kernel   : the same step with the token drawn from HF's temperature -> top-k -> top-p warpers
//
// All state a step needs (next token ids, position ids, finished flags, per-step alive counts, and — in device-column mode —
// each row's current column) lives in device memory: a decode step is then the SAME launch sequence with the same
// arguments for every token and can be captured once as a CUDA graph and replayed (292 launches per token at Llama-2-7B).
// The host reads back one "is anyone still generating" counter every few steps.
#include "common.cuh"
#include <limits.h>
#include <stdlib.h>

namespace dalm {

__global__ void rope_pos_kernel(__nv_bfloat16* __restrict__ buf, long long ld, int col0, int nheads, int D,
                                const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                const int64_t* __restrict__ pos, int T) {
  // one CTA per token row; HF rotate_half convention, same arithmetic as rope_kernel (rowwise.cu)
  const size_t r = blockIdx.x;
  long long p = pos[r];
  p = p < 0 ? 0 : (p >= T ? T - 1 : p);
  const int half = D / 2;
  __nv_bfloat16* base = buf + r * ld + col0;
  for (int i = threadIdx.x; i < nheads * half; i += blockDim.x) {
    const int h = i / half, j = i - h * half;
    __nv_bfloat16* q = base + h * D + j;
    const float x1 = __bfloat162float(q[0]), x2 = __bfloat162float(q[half]);
    const float c = cos_t[(size_t)p * half + j], s = sin_t[(size_t)p * half + j];
    q[0] = __float2bfloat16(x1 * c - x2 * s);
    q[half] = __float2bfloat16(x2 * c + x1 * s);
  }
}

// one explicit 16-byte read-only load -> 8 floats (struct-typed bf16x8 loads are split into 32-bit loads by the compiler)
__device__ __forceinline__ void load8_nc(const __nv_bfloat16* p, float* f) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x; f[2 * i + 1] = t.y;
  }
}

// grid (Hq, B), 128 threads. Shared memory: q[D] | p[sp_cap] | red[32] | part[1024] floats.
//   pass 1: thread-per-key scores (each thread reads whole K rows with 16-byte loads, q broadcast from smem)
//   pass 2: block max / exp / sum
//   pass 3: PV with 128 threads = KG key groups x D/8 lanes; every lane loads 16 bytes of V unconditionally (masked keys
//           carry p = 0; their cache rows are initialised memory) and the KG partial rows meet in shared memory
// With a sliding window (window > 0) all three passes run over columns max(0, cur - window + 1) .. cur only; while
// cur < window that is every column, in the same order, so the result is bit-identical to window = 0.
template <int D>
__global__ void __launch_bounds__(128) attn_decode_kernel(const __nv_bfloat16* __restrict__ qkv, long long ldq, int q_col,
                                                          int k_col, int v_col, __nv_bfloat16* __restrict__ cache_k,
                                                          __nv_bfloat16* __restrict__ cache_v, long long cache_sb,
                                                          long long cache_st, const int64_t* __restrict__ mask,
                                                          long long ldm, __nv_bfloat16* __restrict__ out, long long ldo,
                                                          int Hq, int Hkv, int cur_host, const int* __restrict__ cur_dev,
                                                          int sp_cap, float scale, int window) {
  extern __shared__ float sm[];
  float* sq = sm;
  float* sp = sm + D;
  float* red = sp + sp_cap;                      // sp_cap >= cur + 1, a multiple of 4 (host-side: the cache length in
  float* part = red + 32;                        // device-column mode, so one captured launch serves every step)
                                                 // part = [KG][D] = 1024 floats for every supported D
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int cur = cur_dev ? min(cur_dev[b], sp_cap - 1) : cur_host;
  const int t0 = window > 0 ? max(0, cur - window + 1) : 0;   // first visible column
  const int group = Hq / Hkv, kvh = h / group;
  const __nv_bfloat16* qrow = qkv + (size_t)b * ldq + q_col + h * D;
  const __nv_bfloat16* krow = qkv + (size_t)b * ldq + k_col + kvh * D;
  const __nv_bfloat16* vrow = qkv + (size_t)b * ldq + v_col + kvh * D;
  __nv_bfloat16* ck = cache_k + (size_t)b * cache_sb + kvh * D;
  __nv_bfloat16* cv = cache_v + (size_t)b * cache_sb + kvh * D;
  if (tid < D) {
    sq[tid] = __bfloat162float(qrow[tid]) * scale;
    if (h % group == 0) {                       // the first query head of each kv group appends this token's K / V
      ck[(size_t)cur * cache_st + tid] = krow[tid];
      cv[(size_t)cur * cache_st + tid] = vrow[tid];
    }
  }
  __syncthreads();

  float lmax = -INFINITY;
  for (int t = t0 + tid; t <= cur; t += 128) {
    // column `cur` is the token being decoded: always visible, read from the qkv row (its cache slot is written above
    // by ANOTHER CTA of this launch, so nobody reads it back here)
    const bool valid = (t == cur) || mask[(size_t)b * ldm + t] != 0;
    const __nv_bfloat16* kp = (t == cur) ? krow : ck + (size_t)t * cache_st;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < D; j += 8) {
      float f[8];
      load8_nc(kp + j, f);
#pragma unroll
      for (int e = 0; e < 8; ++e) s += sq[j + e] * f[e];
    }
    s = valid ? s : -INFINITY;
    sp[t] = s;
    lmax = fmaxf(lmax, s);
  }
  const float m = block_max(lmax, red);         // finite: column `cur` is always valid
  float lsum = 0.f;
  for (int t = t0 + tid; t <= cur; t += 128) {
    const float s = sp[t];
    const float p = (s == -INFINITY) ? 0.f : __expf(s - m);
    sp[t] = p;
    lsum += p;
  }
  const float sum = block_sum(lsum, red);
  __syncthreads();

  constexpr int LPK = D / 8, KG = 128 / LPK;    // lanes per key (16 bytes each), key groups: 16 x 8, 8 x 16, 4 x 32
  const int kg = tid / LPK, dl = tid % LPK;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll 4
  for (int t = t0 + kg; t <= cur; t += KG) {
    const __nv_bfloat16* vp = (t == cur) ? vrow : cv + (size_t)t * cache_st;
    float f[8];
    load8_nc(vp + 8 * dl, f);
    const float p = sp[t];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += p * f[e];
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) part[kg * D + 8 * dl + e] = acc[e];
  __syncthreads();
  if (tid < D) {
    float o = 0.f;
#pragma unroll
    for (int k = 0; k < KG; ++k) o += part[k * D + tid];
    out[(size_t)b * ldo + h * D + tid] = __float2bfloat16(o / sum);
  }
}

// HF's per-token bookkeeping (transformers generation/utils.py _sample), run by one thread per row after the token is chosen:
// finished rows emit pad, a row finishes when it emits an EOS id, the new column joins the attention mask, the position id
// advances, alive[col] counts the rows still generating, and in device-column mode the row's column counter advances.
__device__ __forceinline__ void finish_token(int b, int col, long long cand, const int64_t* __restrict__ eos_ids, int n_eos,
                                             long long pad_id, int* __restrict__ unfinished, int64_t* __restrict__ tokens,
                                             long long ldt, int64_t* __restrict__ mask, long long ldm, int* __restrict__ cur_dev,
                                             int64_t* __restrict__ next_ids, int64_t* __restrict__ pos, int* __restrict__ alive) {
  int unf = unfinished[b];
  const long long tok = unf ? cand : pad_id;
  tokens[(size_t)b * ldt + col] = tok;
  mask[(size_t)b * ldm + col] = 1;               // HF appends ones to the attention mask for every generated column
  next_ids[b] = tok;
  pos[b] += 1;                                   // position id of the new token = cumsum(mask) - 1
  if (unf)
    for (int e = 0; e < n_eos; ++e)
      if (tok == eos_ids[e]) unf = 0;
  unfinished[b] = unf;
  if (unf) atomicAdd(alive + col, 1);
  if (cur_dev) cur_dev[b] = col;
}

// grid B, 256 threads. argmax over logits[b, 0..V) (ties -> lowest index, like torch.argmax), then HF's greedy bookkeeping
// (transformers generation/utils.py _sample, do_sample=False): finished rows emit pad, a row finishes when it emits an EOS id.
__global__ void __launch_bounds__(256) greedy_step_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V,
                                                          const int64_t* __restrict__ eos_ids, int n_eos, long long pad_id,
                                                          int* __restrict__ unfinished, int64_t* __restrict__ tokens,
                                                          long long ldt, int64_t* __restrict__ mask, long long ldm,
                                                          int col_host, int* __restrict__ cur_dev, int T,
                                                          int64_t* __restrict__ next_ids, int64_t* __restrict__ pos,
                                                          int* __restrict__ alive) {
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // device-column mode (CUDA-graph replays): this row's new token goes one column after the token just decoded, and the
  // row's own counter advances — no cross-CTA state, so no ordering between the CTAs of this launch is needed
  const int col = cur_dev ? cur_dev[b] + 1 : col_host;
  if (col >= T) return;                          // a replay past the end of the buffers is a no-op
  const __nv_bfloat16* row = logits + (size_t)b * ld;
  float best = -INFINITY;
  int bi = INT_MAX;
  for (int i = tid; i < V; i += 256) {
    const float v = __bfloat162float(row[i]);
    if (bi == INT_MAX || v > best) { best = v; bi = i; }      // ascending i: strict > keeps the lowest index
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi != INT_MAX && (bi == INT_MAX || ov > best || (ov == best && oi < bi))) { best = ov; bi = oi; }
  }
  __shared__ float sv[8];
  __shared__ int si[8];
  if (lane == 0) { sv[warp] = best; si[warp] = bi; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w) {
      const float ov = sv[w];
      const int oi = si[w];
      if (oi != INT_MAX && (bi == INT_MAX || ov > best || (ov == best && oi < bi))) { best = ov; bi = oi; }
    }
    finish_token(b, col, (long long)bi, eos_ids, n_eos, pad_id, unfinished, tokens, ldt, mask, ldm, cur_dev, next_ids, pos, alive);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Sampling step: HF's _sample with do_sample=True and its warper stack, temperature -> top-k -> top-p, then one draw.
// grid B, 1024 threads, one CTA per row; the row is re-read from L2 by every pass (V up to SAMPLE_MAX_V).
//   keys      every pass works on the 16-bit order-preserving key of the bf16 logit (-0 folded onto +0). x = logit / T is
//             strictly increasing over bf16 logits as long as it does not underflow, so ties and order of x are those of
//             the keys
//   top-k     radix select (two 8-bit digits) of the k-th largest key; survivors are the keys >= it (ties all kept)
//   top-p     mass-weighted radix search over the survivors' keys, ascending: the first key at which the cumulative mass
//             exceeds (1 - top_p) * Z. Masses are exp(x - max) in 2^-40 fixed point (64-bit integer sums are exact and
//             order-independent; the quantisation moves a cumulative share by < 1e-7). Inside the tie group at the cut,
//             tokens are removed in ascending index order, i.e. the order is (x, index): our deterministic rule where
//             HF's unstable sort leaves it open. The largest (x, index) always stays (min_tokens_to_keep = 1)
//   draw      u in [0, 1) from Philox keyed by the seed with counter (column, row): the same column gives the same draw
//             whether the step is launched eagerly or replayed from a CUDA graph. The token is the first kept index,
//             ascending, whose inclusive prefix sum of exp(x - max) exceeds u * Z; prefix sums and Z in fp64, in a fixed
//             order (warp segments of consecutive indices)
// ------------------------------------------------------------------------------------------------------------
constexpr int SAMPLE_THREADS = 1024;
constexpr int SAMPLE_MAX_V = 1 << 20;            // 2^20 * 2^40 fits the 64-bit mass sums; indices fit 3 radix digits

__device__ __forceinline__ unsigned int bf16_key(unsigned short b) {
  if (b == 0x8000u) b = 0;                       // -0 == +0
  return (b & 0x8000u) ? (~b & 0xFFFFu) : (b | 0x8000u);
}
__device__ __forceinline__ float key_logit(unsigned int k) {
  const unsigned int b = (k & 0x8000u) ? (k & 0x7FFFu) : (~k & 0xFFFFu);
  return __uint_as_float(b << 16);
}
// exp(x - m) with the difference carried past fp32: d = x - m is exact in fp64; exp(hi + lo) ~ expf(hi) * (1 + lo)
__device__ __forceinline__ double mass_of(float x, float m) {
  const double d = (double)x - (double)m;
  const float hi = (float)d;
  return (double)expf(hi) * (1.0 + (d - (double)hi));
}
__device__ __forceinline__ double sample_uniform(unsigned long long seed, int col, int row) {
  const uint4 r = philox4x32_7(make_uint2((unsigned int)seed, (unsigned int)(seed >> 32)),
                               make_uint4((unsigned int)col, 0u, (unsigned int)row, 0u));
  return (double)(((unsigned long long)r.x << 21) | (r.y >> 11)) * 0x1p-53;    // 53 random bits
}

// k-th largest (k >= 1) of key(i) over the i < V with pred(i, key), by `levels` 8-bit radix digits (most significant first).
// cnt: 256 shared counters, bc: 2 shared words.
template <class KeyF, class PredF>
__device__ unsigned int radix_kth_largest(int V, int levels, KeyF key, PredF pred, unsigned int k, unsigned int* cnt,
                                          unsigned int* bc) {
  unsigned int prefix = 0, hmask = 0;
  for (int lv = levels - 1; lv >= 0; --lv) {
    const int shift = 8 * lv;
    for (int j = threadIdx.x; j < 256; j += blockDim.x) cnt[j] = 0;
    __syncthreads();
    for (int i0 = threadIdx.x & ~31; i0 < V; i0 += blockDim.x) {          // warp-uniform trip count
      const int i = i0 + (threadIdx.x & 31);
      unsigned int kk = 0;
      bool want = i < V;
      if (want) { kk = key(i); want = (kk & hmask) == prefix && pred(i, kk); }
      const unsigned int act = __ballot_sync(0xffffffffu, want);
      if (want) {                                // one atomic per distinct bin of the warp: few bins hold most keys
        const unsigned int d = (kk >> shift) & 255u;
        const unsigned int peers = __match_any_sync(act, d);
        if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&cnt[d], (unsigned int)__popc(peers));
      }
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      unsigned int c[8], s = 0;
#pragma unroll
      for (int e = 0; e < 8; ++e) { c[e] = cnt[255 - 8 * lane - e]; s += c[e]; }      // lane 0 holds the top bins
      unsigned int inc = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      unsigned int run = inc - s;
      if (run < k && k <= inc) {
        for (int e = 0; e < 8; ++e) {
          if (run + c[e] >= k) { bc[0] = 255 - 8 * lane - e; bc[1] = k - run; break; }
          run += c[e];
        }
      }
    }
    __syncthreads();
    prefix |= bc[0] << shift;
    hmask |= 255u << shift;
    k = bc[1];
  }
  return prefix;
}

__global__ void __launch_bounds__(SAMPLE_THREADS) sample_step_kernel(
    const __nv_bfloat16* __restrict__ logits, long long ld, int V, const int64_t* __restrict__ eos_ids, int n_eos,
    long long pad_id, int* __restrict__ unfinished, int64_t* __restrict__ tokens, long long ldt, int64_t* __restrict__ mask,
    long long ldm, int col_host, int* __restrict__ cur_dev, int T, int64_t* __restrict__ next_ids, int64_t* __restrict__ pos,
    int* __restrict__ alive, float temperature, int top_k, float top_p, unsigned long long seed,
    const double* __restrict__ u_in, float* __restrict__ scores_out) {
  __shared__ unsigned int cnt[256];
  __shared__ unsigned long long qmass[256];
  __shared__ unsigned int bc[4];
  __shared__ unsigned long long bcl[2];
  __shared__ double wtot[32], bcd[2];
  __shared__ int wlast[32], chosen;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int col = cur_dev ? cur_dev[b] + 1 : col_host;
  if (col >= T) return;                          // a replay past the end of the buffers is a no-op
  if (unfinished[b]) {                           // finished rows emit pad: nothing to choose
    const unsigned short* row = reinterpret_cast<const unsigned short*>(logits + (size_t)b * ld);
    auto lkey = [&](int i) { return bf16_key(row[i]); };
    auto xval = [&](int i) { return __fdiv_rn(__bfloat162float(__ushort_as_bfloat16(row[i])), temperature); };

    // ---- max key (the largest x, the softmax shift) ----
    unsigned int mk = 0;
    for (int i = tid; i < V; i += SAMPLE_THREADS) mk = max(mk, lkey(i));
    mk = __reduce_max_sync(0xffffffffu, mk);
    if (lane == 0) cnt[warp] = mk;
    __syncthreads();
    if (warp == 0) {
      const unsigned int v = __reduce_max_sync(0xffffffffu, cnt[lane]);
      if (lane == 0) bc[2] = v;
    }
    __syncthreads();
    mk = bc[2];
    const float mx = __fdiv_rn(key_logit(mk), temperature);

    // ---- top-k: survivors are the keys >= the k-th largest ----
    unsigned int kthr = 0;
    if (top_k > 0 && top_k < V)
      kthr = radix_kth_largest(V, 2, lkey, [](int, unsigned int) { return true; }, (unsigned int)top_k, cnt, bc);

    // ---- top-p: kept = (key, index) >= (kp, icut) ----
    unsigned int kp = kthr, icut = 0;
    if (top_p < 1.f) {
      unsigned int prefix = 0, hmask = 0;
      unsigned long long below = 0;              // fixed-point mass of the survivors below the current prefix
      double c = 0.0;                            // (1 - top_p) * Z, warp 0 only
      for (int lv = 1; lv >= 0; --lv) {
        const int shift = 8 * lv;
        for (int j = tid; j < 256; j += SAMPLE_THREADS) { cnt[j] = 0; qmass[j] = 0; }
        __syncthreads();
        for (int i0 = tid - lane; i0 < V; i0 += SAMPLE_THREADS) {          // warp-uniform trip count
          const int i = i0 + lane;
          unsigned int kk = 0;
          bool want = i < V;
          if (want) { kk = lkey(i); want = kk >= kthr && (kk & hmask) == prefix; }
          const unsigned int act = __ballot_sync(0xffffffffu, want);
          if (want) {                            // the warp's tokens of one bin are summed first: one atomic per bin
            const unsigned int d = (kk >> shift) & 255u;
            const unsigned long long q = __double2ull_rn(mass_of(xval(i), mx) * 0x1p40);
            const unsigned int peers = __match_any_sync(act, d);
            unsigned long long sum = 0;
            for (unsigned int p = peers; p; p &= p - 1) sum += __shfl_sync(peers, q, __ffs(p) - 1);
            if (lane == __ffs(peers) - 1) {
              atomicAdd(&qmass[d], sum);
              atomicAdd(&cnt[d], (unsigned int)__popc(peers));
            }
          }
        }
        __syncthreads();
        if (warp == 0) {
          unsigned long long m8[8], s = 0;
          unsigned int any = 0;
#pragma unroll
          for (int e = 0; e < 8; ++e) { m8[e] = qmass[8 * lane + e]; s += m8[e]; any |= cnt[8 * lane + e]; }   // ascending bins
          unsigned long long inc = s;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
          }
          if (lv == 1) c = (1.0 - (double)top_p) * (double)__shfl_sync(0xffffffffu, inc, 31);
          const unsigned int cross = __ballot_sync(0xffffffffu, (double)(below + inc) > c);
          // no bin crosses only when rounding ate the last (1 - top_p) share: keep the largest key, as HF keeps one token
          const int src = cross ? __ffs(cross) - 1 : 31 - __clz(__ballot_sync(0xffffffffu, any != 0));
          if (lane == src) {
            int e = 0;
            if (cross)
              while (e < 7 && !((double)(below + inc - s + m8[e]) > c)) s -= m8[e++];    // s: mass from bin e to the lane's end
            else
              for (int f = 7; f >= 0; --f)
                if (cnt[8 * lane + f]) { e = f; break; }
            unsigned long long run = below + inc - s;                                      // mass below bin e
            if (!cross)
              for (int f = 0; f < e; ++f) run += m8[f];
            const int d = 8 * lane + e;
            bc[0] = d; bc[1] = cnt[d]; bcl[0] = run; bcl[1] = qmass[d];
            if (lv == 0) {
              // tie group at the cut: n tokens of mass w each, cumulative run + (r + 1) w; the first r0 (by index) have
              // a cumulative share <= 1 - top_p and go; at least one of the group stays
              const unsigned int n = cnt[d];
              const double w = (double)(qmass[d] / n);
              double r0 = floor((c - (double)run) / w);
              r0 = r0 < 0.0 ? 0.0 : (r0 > (double)(n - 1) ? (double)(n - 1) : r0);
              bc[2] = (unsigned int)r0;
            }
          }
        }
        __syncthreads();
        prefix |= bc[0] << shift;
        hmask |= 255u << shift;
        below = bcl[0];
      }
      kp = prefix;
      const unsigned int nt = bc[1], r0 = bc[2];
      if (r0 > 0)                                // the (nt - r0)-th largest index of the tie group is the first one kept
        icut = radix_kth_largest(V, 3, [](int i) { return (unsigned int)i; },
                                 [&](int i, unsigned int) { return lkey(i) == kp; }, nt - r0, cnt, bc);
    }
    auto kept = [&](int i, unsigned int kk) { return kk > kp || (kk == kp && (unsigned int)i >= icut); };

    // ---- draw: per-warp segments of consecutive indices, fp64 sums in a fixed order ----
    const double u = u_in ? u_in[b] : sample_uniform(seed, col, b);
    const int seg = (((V + 31) / 32) + 31) & ~31;
    const int s0 = warp * seg, s1 = min(V, s0 + seg);
    double acc = 0.0;
    int last = -1;
    for (int i = s0 + lane; i < s1; i += 32) {
      const unsigned int kk = lkey(i);
      const float x = xval(i);
      const bool k_ = kept(i, kk);
      if (k_) {
        const double w = mass_of(x, mx);
        acc += w;
        if (w > 0.0) last = i;
      }
      if (scores_out) scores_out[(size_t)b * ld + i] = k_ ? x : -INFINITY;
    }
    acc = warp_sum_d(acc);
    last = __reduce_max_sync(0xffffffffu, last);
    if (lane == 0) { wtot[warp] = acc; wlast[warp] = last; }
    __syncthreads();
    if (warp == 0) {
      const double t = wtot[lane];
      double inc = t;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
      }
      const double target = u * __shfl_sync(0xffffffffu, inc, 31);
      const unsigned int cross = __ballot_sync(0xffffffffu, inc > target);
      const int glast = __reduce_max_sync(0xffffffffu, wlast[lane]);
      const int wc = cross ? __ffs(cross) - 1 : -1;
      const double base = __shfl_sync(0xffffffffu, inc - t, wc < 0 ? 0 : wc);
      if (lane == 0) { bc[3] = (unsigned int)wc; bcd[0] = base; bcd[1] = target; chosen = glast; }
    }
    __syncthreads();
    if (warp == (int)bc[3]) {                    // the warp whose segment holds the crossing walks it 32 tokens at a time
      double run = bcd[0];
      const double target = bcd[1];
      int pick = wlast[warp];                    // rounding fallback: the segment's last kept token
      for (int j = s0; j < s1; j += 32) {
        const int i = j + lane;
        double w = 0.0;
        if (i < s1 && kept(i, lkey(i))) w = mass_of(xval(i), mx);
        double inc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const double v = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += v;
        }
        const unsigned int hit = __ballot_sync(0xffffffffu, w > 0.0 && run + inc > target);
        if (hit) { pick = j + __ffs(hit) - 1; break; }
        run += __shfl_sync(0xffffffffu, inc, 31);
      }
      if (lane == 0) chosen = pick;
    }
    __syncthreads();
  }
  if (tid == 0)
    finish_token(b, col, (long long)chosen, eos_ids, n_eos, pad_id, unfinished, tokens, ldt, mask, ldm, cur_dev, next_ids, pos,
                 alive);
}

// ------------------------------------------------------------------------------------------------------------
// Weight-streaming GEMM for the decode step: out[m, n] = act(sum_k A[m,k] W[n,k] + bias[n]) + resid[m,n] with M <= 16 token rows.
// HBM-bound: every weight is read exactly once (N*K*2 bytes), the activations (16 x K bf16) stay in L2. The 128-row wgmma
// tile of the training GEMM wastes 7/8 of its A tile here and runs N = 4096 on 64 CTAs, so this path uses one `mma.sync.m16n8k16` row tile = the whole batch instead:
//   CTA = 16 output columns (2 n-tiles) x all of K, 256 threads; the 8 warps interleave over 32-wide k-chunks (split-K inside
//   the CTA), partial sums meet in shared memory. Each lane loads 16 bytes (8 consecutive k) of one weight row and of two
//   activation rows per chunk straight from global memory into MMA fragments: lane (g, t) takes k = chunk*32 + 8t .. +7, and
//   the SAME permutation of k inside the chunk is applied to A and W (a contraction does not care about the order), so no
//   cross-lane exchange or ldmatrix is needed. The pieces travel through a per-lane cp.async ring (6 chunks deep).
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// 16-byte asynchronous global -> shared copy (zero-fill when !ok). L1-allocating for the activations (every CTA of an SM
// reads the same 16 x K block), L2-only for the weight stream.
__device__ __forceinline__ void cp_async16_ca(void* smem, const void* gmem, bool ok) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async16_cg(void* smem, const void* gmem, bool ok) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit_group() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

constexpr int DG_NT = 2;                 // 8-column n-tiles per CTA
constexpr int DG_STAGES = 6;             // k-chunks in flight per lane (each: 2 activation + DG_NT weight 16-byte pieces)
constexpr int DG_SLOTS = 2 + DG_NT;
constexpr int DG_SMEM = DG_STAGES * 8 * DG_SLOTS * 32 * 16;     // 96 KB: [stage][warp][slot][lane] of 16 bytes

// Every lane prefetches ITS OWN fragment pieces through a private ring in shared memory (it reads back exactly the 16-byte
// slots it copied), so the ring needs no barrier at all: `cp.async.wait_group` orders a thread's own copies. Plain register
// loads were tried first: ptxas sank each load next to its MMA (3 loads in flight per lane instead of 16).
__global__ void __launch_bounds__(256) decode_gemm_kernel(const __nv_bfloat16* __restrict__ A, long long lda,
                                                          const __nv_bfloat16* __restrict__ W, long long ldw,
                                                          void* __restrict__ out, long long ldo, int out_f32,
                                                          const float* __restrict__ bias,
                                                          const void* __restrict__ resid, long long ldr, int resid_f32, int act,
                                                          int M, int N, int K) {
  extern __shared__ __align__(16) unsigned char dg_smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int n0 = blockIdx.x * (DG_NT * 8);
  const int nchunks = (K + 31) / 32;
  const int my_chunks = nchunks > warp ? (nchunks - warp + 7) / 8 : 0;    // this warp takes chunks warp, warp + 8, ...
  uint4* ring = reinterpret_cast<uint4*>(dg_smem) + (size_t)warp * DG_SLOTS * 32 + lane;   // + stage*8*SLOTS*32 + slot*32
  constexpr int STAGE_STRIDE = 8 * DG_SLOTS * 32;
  float acc[DG_NT][4];
#pragma unroll
  for (int i = 0; i < DG_NT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
  const bool row_lo = g < M, row_hi = g + 8 < M;
  const __nv_bfloat16* a_lo_p = A + (size_t)(row_lo ? g : 0) * lda;
  const __nv_bfloat16* a_hi_p = A + (size_t)(row_hi ? g + 8 : 0) * lda;
  const __nv_bfloat16* w_p[DG_NT];
  bool w_ok[DG_NT];
#pragma unroll
  for (int i = 0; i < DG_NT; ++i) {
    const int n = n0 + i * 8 + g;
    w_ok[i] = n < N;
    w_p[i] = W + (size_t)(w_ok[i] ? n : 0) * ldw;
  }
  auto issue = [&](int i) {                              // i-th chunk of this warp -> ring stage i % DG_STAGES
    if (i < my_chunks) {
      const int k = (warp + 8 * i) * 32 + 8 * t;         // K % 8 == 0: a lane's 8 elements are all inside or all outside K
      const bool kin = k < K;
      const int ks = kin ? k : 0;
      uint4* st = ring + (size_t)(i % DG_STAGES) * STAGE_STRIDE;
      cp_async16_ca(st, a_lo_p + ks, kin && row_lo);
      cp_async16_ca(st + 32, a_hi_p + ks, kin && row_hi);
#pragma unroll
      for (int j = 0; j < DG_NT; ++j) cp_async16_cg(st + (2 + j) * 32, w_p[j] + ks, kin && w_ok[j]);
    }
    cp_async_commit_group();                             // one group per call, empty or not: the wait below counts groups
  };
#pragma unroll
  for (int i = 0; i < DG_STAGES - 1; ++i) issue(i);
  for (int i = 0; i < my_chunks; ++i) {
    issue(i + DG_STAGES - 1);                            // refills the stage this lane consumed in the previous iteration
    cp_async_wait_group<DG_STAGES - 1>();                // chunk i has landed
    const uint4* st = ring + (size_t)(i % DG_STAGES) * STAGE_STRIDE;
    const uint4 alo = st[0], ahi = st[32];
#pragma unroll
    for (int j = 0; j < DG_NT; ++j) {
      const uint4 b = st[(2 + j) * 32];
      // fragment k-slots (2t,2t+1) and (2t+8,2t+9) are fed actual k (8t+0,1),(8t+2,3), then (8t+4,5),(8t+6,7), for A and W alike
      mma16816(acc[j], alo.x, ahi.x, alo.y, ahi.y, b.x, b.y);
      mma16816(acc[j], alo.z, ahi.z, alo.w, ahi.w, b.z, b.w);
    }
  }
  cp_async_wait_group<0>();
  __syncthreads();                                       // every warp is done with its ring: reuse the memory for the partials
  float(*part)[16][DG_NT * 8 + 1] = reinterpret_cast<float(*)[16][DG_NT * 8 + 1]>(dg_smem);
  // accumulator fragment: c0,c1 = (row g, cols 2t, 2t+1), c2,c3 = (row g+8, same cols)
#pragma unroll
  for (int i = 0; i < DG_NT; ++i) {
    part[warp][g][i * 8 + 2 * t] = acc[i][0];
    part[warp][g][i * 8 + 2 * t + 1] = acc[i][1];
    part[warp][g + 8][i * 8 + 2 * t] = acc[i][2];
    part[warp][g + 8][i * 8 + 2 * t + 1] = acc[i][3];
  }
  __syncthreads();
  const int m = tid >> 4, nn = tid & 15, n = n0 + nn;   // 256 threads = 16 rows x 16 columns
  if (m < M && n < N) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += part[w][m][nn];
    if (bias) v += bias[n];
    if (act == 1) v = gelu_erf(v);
    if (resid) v += resid_f32 ? static_cast<const float*>(resid)[(size_t)m * ldr + n]
                              : __bfloat162float(static_cast<const __nv_bfloat16*>(resid)[(size_t)m * ldr + n]);
    if (out_f32) static_cast<float*>(out)[(size_t)m * ldo + n] = v;
    else static_cast<__nv_bfloat16*>(out)[(size_t)m * ldo + n] = __float2bfloat16(v);
  }
}

}  // namespace dalm

using namespace dalm;
#define ST(s) ((cudaStream_t)(s))

extern "C" int dalm_b200_decode_gemm(const void* A, long long lda, const void* W, long long ldw, void* out, long long ldo,
                                     int out_f32, const float* bias, const void* resid, long long ldr, int resid_f32, int act,
                                     int M, int N, int K, void* stream) {
  DALM_REQUIRE(M > 0 && M <= 16 && N > 0 && K > 0, "decode_gemm: needs 1 <= M <= 16 token rows (got M=%d N=%d K=%d)", M, N, K);
  DALM_REQUIRE((K % 8) == 0 && (lda % 8) == 0 && (ldw % 8) == 0 && lda >= K && ldw >= K && ldo >= N,
               "decode_gemm: K and the operand row strides must be multiples of 8 elements");
  DALM_REQUIRE(((uintptr_t)A & 15) == 0 && ((uintptr_t)W & 15) == 0, "decode_gemm: operands must be 16-byte aligned");
  DALM_REQUIRE(act == 0 || act == 1, "decode_gemm: act must be 0 (none) or 1 (gelu)");
  DALM_REQUIRE(resid == nullptr || ldr >= N, "decode_gemm: residual row stride");
  static bool attr = false;
  if (!attr) { DALM_CUDA(cudaFuncSetAttribute(decode_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DG_SMEM)); attr = true; }
  decode_gemm_kernel<<<(N + DG_NT * 8 - 1) / (DG_NT * 8), 256, DG_SMEM, ST(stream)>>>(
      (const __nv_bfloat16*)A, lda, (const __nv_bfloat16*)W, ldw, out, ldo, out_f32, bias, resid, ldr, resid_f32, act, M, N, K);
  count_launch();
  return check_launch("decode_gemm_kernel");
}

extern "C" int dalm_b200_rope_pos(void* buf, long long ld, int col0, int nheads, int D, const float* cos_t,
                                  const float* sin_t, const int64_t* pos, int M, int T, void* stream) {
  DALM_REQUIRE(M > 0 && T > 0 && nheads > 0 && (D % 2) == 0, "rope_pos: bad shape M=%d T=%d heads=%d D=%d", M, T, nheads, D);
  DALM_REQUIRE(pos != nullptr && cos_t != nullptr && sin_t != nullptr, "rope_pos: null table / positions");
  rope_pos_kernel<<<M, 256, 0, ST(stream)>>>((__nv_bfloat16*)buf, ld, col0, nheads, D, cos_t, sin_t, pos, T);
  count_launch();
  return check_launch("rope_pos_kernel");
}

extern "C" int dalm_b200_attention_decode(const void* qkv, long long ldq, int q_col, int k_col, int v_col, void* cache_k,
                                          void* cache_v, long long cache_sb, long long cache_st, const int64_t* mask,
                                          long long ldm, void* out, long long ldo, int B, int Hq, int Hkv, int D, int cur,
                                          const int* cur_dev, int T, float scale, int window, void* stream) {
  DALM_REQUIRE(B > 0 && Hq > 0 && Hkv > 0 && (Hq % Hkv) == 0, "attention_decode: bad heads B=%d Hq=%d Hkv=%d", B, Hq, Hkv);
  DALM_REQUIRE(D == 32 || D == 64 || D == 128, "attention_decode: head_dim %d unsupported (32/64/128)", D);
  DALM_REQUIRE(T > 0 && T <= 8192 && (cur_dev != nullptr || (cur >= 0 && cur < T)),
               "attention_decode: column %d outside the cache of %d tokens (max 8192)", cur, T);
  DALM_REQUIRE((ldq % 8) == 0 && (q_col % 8) == 0 && (k_col % 8) == 0 && (v_col % 8) == 0 && (cache_st % 8) == 0 &&
                   (cache_sb % 8) == 0, "attention_decode: rows must be 16-byte aligned");
  DALM_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)cache_k & 15) == 0 && ((uintptr_t)cache_v & 15) == 0,
               "attention_decode: pointers must be 16-byte aligned");
  DALM_REQUIRE(mask != nullptr && cache_st >= (long long)Hkv * D && cache_sb >= cache_st * T, "attention_decode: cache layout");
  DALM_REQUIRE(window >= 0, "attention_decode: window %d must be >= 0 (0 = no window)", window);
  const int sp_cap = ((cur_dev ? T : cur + 1) + 3) & ~3;
  const size_t smem = (size_t)(D + sp_cap + 32 + 1024) * sizeof(float);
  dim3 grid(Hq, B);
#define DALM_DECODE(DD)                                                                                                  \
  attn_decode_kernel<DD><<<grid, 128, smem, ST(stream)>>>((const __nv_bfloat16*)qkv, ldq, q_col, k_col, v_col,           \
                                                          (__nv_bfloat16*)cache_k, (__nv_bfloat16*)cache_v, cache_sb,    \
                                                          cache_st, mask, ldm, (__nv_bfloat16*)out, ldo, Hq, Hkv, cur,     \
                                                          cur_dev, sp_cap, scale, window)
  if (D == 128) DALM_DECODE(128); else if (D == 64) DALM_DECODE(64); else DALM_DECODE(32);
#undef DALM_DECODE
  count_launch();
  return check_launch("attn_decode_kernel");
}

extern "C" int dalm_b200_greedy_step(const void* logits, long long ld, int B, int V, const int64_t* eos_ids, int n_eos,
                                     long long pad_id, int* unfinished, int64_t* tokens, long long ldt, int64_t* mask,
                                     long long ldm, int col, int* cur_dev, int T, int64_t* next_ids, int64_t* pos, int* alive,
                                     void* stream) {
  DALM_REQUIRE(B > 0 && V > 0 && T > 0 && T <= ldt && T <= ldm, "greedy_step: bad shape B=%d V=%d T=%d", B, V, T);
  DALM_REQUIRE(cur_dev != nullptr || (col >= 0 && col < T), "greedy_step: column %d outside the %d-token buffers", col, T);
  DALM_REQUIRE(n_eos >= 0 && (n_eos == 0 || eos_ids != nullptr), "greedy_step: eos list");
  DALM_REQUIRE(unfinished && tokens && mask && next_ids && pos && alive, "greedy_step: null state pointer");
  greedy_step_kernel<<<B, 256, 0, ST(stream)>>>((const __nv_bfloat16*)logits, ld, V, eos_ids, n_eos, pad_id, unfinished, tokens,
                                                ldt, mask, ldm, col, cur_dev, T, next_ids, pos, alive);
  count_launch();
  return check_launch("greedy_step_kernel");
}

extern "C" int dalm_b200_sample_step(const void* logits, long long ld, int B, int V, const int64_t* eos_ids, int n_eos,
                                     long long pad_id, int* unfinished, int64_t* tokens, long long ldt, int64_t* mask,
                                     long long ldm, int col, int* cur_dev, int T, int64_t* next_ids, int64_t* pos, int* alive,
                                     float temperature, int top_k, float top_p, unsigned long long seed, const double* u,
                                     float* scores_out, void* stream) {
  DALM_REQUIRE(B > 0 && V > 0 && T > 0 && T <= ldt && T <= ldm && ld >= V, "sample_step: bad shape B=%d V=%d T=%d", B, V, T);
  DALM_REQUIRE(V <= SAMPLE_MAX_V, "sample_step: vocabulary of %d exceeds the kernel's limit of %d", V, SAMPLE_MAX_V);
  DALM_REQUIRE(cur_dev != nullptr || (col >= 0 && col < T), "sample_step: column %d outside the %d-token buffers", col, T);
  DALM_REQUIRE(n_eos >= 0 && (n_eos == 0 || eos_ids != nullptr), "sample_step: eos list");
  DALM_REQUIRE(unfinished && tokens && mask && next_ids && pos && alive, "sample_step: null state pointer");
  DALM_REQUIRE(temperature > 0.f && isfinite(temperature), "sample_step: temperature must be positive and finite (got %g)",
               (double)temperature);
  DALM_REQUIRE(top_p > 0.f && top_p <= 1.f, "sample_step: top_p must be in (0, 1] (got %g)", (double)top_p);
  DALM_REQUIRE(top_k >= 0, "sample_step: top_k must be >= 0 (0 or >= V: off), got %d", top_k);
  sample_step_kernel<<<B, SAMPLE_THREADS, 0, ST(stream)>>>((const __nv_bfloat16*)logits, ld, V, eos_ids, n_eos, pad_id, unfinished,
                                                           tokens, ldt, mask, ldm, col, cur_dev, T, next_ids, pos, alive,
                                                           temperature, top_k, top_p, seed, u, scores_out);
  count_launch();
  return check_launch("sample_step_kernel");
}
