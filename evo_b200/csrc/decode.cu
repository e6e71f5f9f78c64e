// Decode-step kernels (one new token per sequence): everything a CUDA-graph replay of the
// step needs, with the sequence position read from DEVICE memory so the same captured graph
// serves every step (the reference re-launches ~20 tiny kernels per layer per token from
// Python, SURVEY.md 8a row a9/a12).
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/evo_b200.h"

using namespace evo;

namespace {

constexpr int HD = 128;

// out[m, g*128 + c] = gelu_gate(t[m, g*256 + c], t[m, g*256 + 128 + c])   (t = [l1 | l2] interleaved GEMM output)
__global__ void gelu_gate_kernel(const bf16* __restrict__ t, bf16* __restrict__ out, long long M, int ipad) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // (m, pair of columns)
  long long total = M * (ipad / 2);
  if (idx >= total) return;
  int c2 = (int)(idx % (ipad / 2)) * 2;
  long long m = idx / (ipad / 2);
  int g = c2 / 128, c = c2 % 128;
  const uint32_t a = *reinterpret_cast<const uint32_t*>(t + m * 2 * ipad + g * 256 + c);
  const uint32_t b = *reinterpret_cast<const uint32_t*>(t + m * 2 * ipad + g * 256 + 128 + c);
  *reinterpret_cast<uint32_t*>(out + m * ipad + c2) = pack_bf16(gelu_gate(bf_lo(a), bf_lo(b)), gelu_gate(bf_hi(a), bf_hi(b)));
}

// Rotary on element pair (i, i + 64) of q,k of row b, head h at position `pos`; k,v appended at cache row `row`.
__device__ __forceinline__ void qkv_prep_pair(bf16* __restrict__ qkv, bf16* __restrict__ cache, const bf16* __restrict__ cos, const bf16* __restrict__ sin,
                                              long long pos, long long row, int b, int h, int i, int H, long long max_seqlen) {
  const float c = __bfloat162float(cos[pos * 64 + i]), s = __bfloat162float(sin[pos * 64 + i]);
  bf16* q = qkv + ((long long)(b * 3 + 0) * H + h) * HD;
  bf16* k = qkv + ((long long)(b * 3 + 1) * H + h) * HD;
  const bf16* v = qkv + ((long long)(b * 3 + 2) * H + h) * HD;
  float q0 = __bfloat162float(q[i]), q1 = __bfloat162float(q[i + 64]);
  float k0 = __bfloat162float(k[i]), k1 = __bfloat162float(k[i + 64]);
  bf16 kr0, kr1;
  rope_rotate(k0, k1, c, s, kr0, kr1);
  rope_rotate(q0, q1, c, s, q[i], q[i + 64]);
  k[i] = kr0; k[i + 64] = kr1;
  bf16* ck = cache + (((long long)b * max_seqlen + row) * 2 + 0) * H * HD + (long long)h * HD;
  bf16* cv = ck + (long long)H * HD;
  ck[i] = kr0; ck[i + 64] = kr1;
  cv[i] = v[i]; cv[i + 64] = v[i + 64];
}

// L == 1: rotary on q,k at position pos_ptr[b * pos_stride], k,v appended to the cache at that row.  pos_stride 0 = one
// position shared by the batch, 1 = one position per row (prompts of different lengths decoded together).
// qkv (B, 3, H, 128) in place; cos/sin tables indexed by absolute position.
__global__ void decode_qkv_prep_kernel(bf16* __restrict__ qkv, bf16* __restrict__ cache, const bf16* __restrict__ cos, const bf16* __restrict__ sin,
                                       const long long* __restrict__ pos_ptr, int pos_stride, int B, int H, long long max_seqlen) {
  pdl_launch_dependents(); pdl_wait();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;       // (b, h, i) i in [0, 64)
  if (idx >= B * H * 64) return;
  int i = idx % 64, h = (idx / 64) % H, b = idx / (64 * H);
  const long long pos = pos_ptr[(long long)b * pos_stride];
  if (pos >= max_seqlen) return;
  qkv_prep_pair(qkv, cache, cos, sin, pos, pos, b, h, i, H, max_seqlen);
}

// Shared-prefix decode: rotary at the absolute position pos[b], k,v appended at row spos[b] of the row's own suffix cache
// (B, S, 2, H, 128) that holds the generated tokens only.
__global__ void decode_qkv_prep_shared_kernel(bf16* __restrict__ qkv, bf16* __restrict__ cache, const bf16* __restrict__ cos, const bf16* __restrict__ sin,
                                              const long long* __restrict__ pos_ptr, const long long* __restrict__ spos_ptr, int B, int H, long long S) {
  pdl_launch_dependents(); pdl_wait();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * H * 64) return;
  int i = idx % 64, h = (idx / 64) % H, b = idx / (64 * H);
  const long long pos = pos_ptr[b], row = spos_ptr[b];
  if (row < 0 || row >= S || pos < 0) return;
  qkv_prep_pair(qkv, cache, cos, sin, pos, row, b, h, i, H, S);
}

// Single-query attention over the KV cache, keys [0, pos_ptr[b * pos_stride]].  grid (H, B, nsplit); each CTA scans a
// contiguous key range: thread t owns keys t, t+128, ... of the range (one 256-byte K row and one
// V row per key), keeps an online-softmax state and a 128-wide fp32 accumulator in registers, and the
// 128 partial states are merged through shared memory; splits are merged by the last kernel.
constexpr int DT = 128;
__global__ void __launch_bounds__(DT) decode_attn_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ cache, float* __restrict__ part_o,
                                                         float* __restrict__ part_ml, const long long* __restrict__ pos_ptr, int pos_stride,
                                                         int H, long long max_seqlen, int nsplit, float scale) {
  pdl_launch_dependents(); pdl_wait();
  const int h = blockIdx.x, b = blockIdx.y, sp = blockIdx.z, tid = threadIdx.x;
  const long long nk = min(pos_ptr[(long long)b * pos_stride] + 1, max_seqlen);   // per row: a split past the row's keys stays empty
  const long long per = (nk + nsplit - 1) / nsplit;
  const long long k0 = (long long)sp * per, k1 = min(nk, k0 + per);
  __shared__ float qs[HD];
  __shared__ float red_m[DT], red_l[DT];
  __shared__ float red_o[32][HD + 1];
  qs[tid] = __bfloat162float(qkv[((long long)(b * 3) * H + h) * HD + tid]) * scale;
  __syncthreads();
  float m = -INFINITY, l = 0.f, o[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) o[d] = 0.f;
  const long long row_stride = 2LL * H * HD;
  const bf16* kb = cache + ((long long)b * max_seqlen) * row_stride + (long long)h * HD;
  for (long long j = k0 + tid; j < k1; j += DT) {
    const uint4* kr = reinterpret_cast<const uint4*>(kb + j * row_stride);
    const uint4* vr = reinterpret_cast<const uint4*>(kb + j * row_stride + (long long)H * HD);
    float sdot = 0.f;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      uint4 kv = __ldg(kr + c);
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&kv);
#pragma unroll
      for (int e = 0; e < 4; ++e) { sdot = fmaf(qs[c * 8 + 2 * e], bf_lo(w[e]), sdot); sdot = fmaf(qs[c * 8 + 2 * e + 1], bf_hi(w[e]), sdot); }
    }
    const float mn = fmaxf(m, sdot);
    const float alpha = __expf(m - mn), p = __expf(sdot - mn);
    const float pb = rbf(p);                      // P rounded to bf16 before the PV product, like the prefill kernel
    l = l * alpha + p;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      uint4 vv = __ldg(vr + c);
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&vv);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        o[c * 8 + 2 * e] = fmaf(pb, bf_lo(w[e]), o[c * 8 + 2 * e] * alpha);
        o[c * 8 + 2 * e + 1] = fmaf(pb, bf_hi(w[e]), o[c * 8 + 2 * e + 1] * alpha);
      }
    }
    m = mn;
  }
  // merge the 128 per-thread states: common max, rescale, then reduce 32 threads at a time through smem
  red_m[tid] = m;
  __syncthreads();
  float M = -INFINITY;
  for (int i = 0; i < DT; ++i) M = fmaxf(M, red_m[i]);
  const float sc = (m == -INFINITY) ? 0.f : __expf(m - M);
  red_l[tid] = l * sc;
  __syncthreads();
  float acc = 0.f;                                 // thread tid owns output dim tid
  for (int round = 0; round < DT / 32; ++round) {
    if (tid / 32 == round) {
#pragma unroll
      for (int d = 0; d < HD; ++d) red_o[tid % 32][d] = o[d] * sc;
    }
    __syncthreads();
    for (int i = 0; i < 32; ++i) acc += red_o[i][tid];
    __syncthreads();
  }
  float L = 0.f;
  for (int i = 0; i < DT; ++i) L += red_l[i];
  const long long pidx = ((long long)b * H + h) * nsplit + sp;
  part_o[pidx * HD + tid] = acc;
  if (tid == 0) { part_ml[pidx * 2] = M; part_ml[pidx * 2 + 1] = L; }
}

// ---- decode attention, TMA-fed (default when max_seqlen % 64 == 0) ----
// The per-thread-row kernel above issues 16-byte loads whose 32 lanes touch 32 different 128-byte lines (K rows of
// one head are 16 KB apart): the L1 tag stage caps it near 3 TB/s.  Here a producer warp streams 64-key K and V tiles
// of one (b, h) into a 3-stage shared-memory ring with TMA (box {128, 1, 64} of the cache viewed as
// (hd, 2H, B*S)), and four independent compute warps each own 16 keys of every tile: QK with lane = (key, half
// row) reading rotated 16-byte chunks (conflict-free), a warp-local online softmax, PV with lane = 4 output dims.
// The warps' (m, l, o) states are merged once at the end; splits are merged by decode_attn_merge_kernel.
constexpr int TK = 64;                 // keys per tile
constexpr int AST = 3;                 // ring stages
constexpr int TILE_BYTES = TK * HD * 2;          // 16 KB (K) + 16 KB (V) per stage
constexpr int ATT2_SMEM = AST * 2 * TILE_BYTES + 1024;
__global__ void __launch_bounds__(160, 2) decode_attn_tma_kernel(const __grid_constant__ CUtensorMap tm, const bf16* __restrict__ qkv,
                                                                 float* __restrict__ part_o, float* __restrict__ part_ml,
                                                                 const long long* __restrict__ pos_ptr, int pos_stride, int H, long long S, int nsplit,
                                                                 float scale) {
  pdl_launch_dependents(); pdl_wait();
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + AST * 2 * TILE_BYTES);
  uint64_t* empty = full + AST;
  bf16* qb = reinterpret_cast<bf16*>(empty + AST);                   // 256 B
  float* red = reinterpret_cast<float*>(qb + HD);                      // [4][2] (m, l) then [4][128] o, overlaid on stage 0 after the loop
  const int h = blockIdx.x, b = blockIdx.y, sp = blockIdx.z, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long nk = min(pos_ptr[(long long)b * pos_stride] + 1, S);   // keys, splits and tiles are per row
  long long per = (nk + nsplit - 1) / nsplit;
  per = (per + TK - 1) / TK * TK;                                      // splits start on tile boundaries
  const long long k0 = (long long)sp * per, k1 = min(nk, k0 + per);
  const int ntiles = k1 > k0 ? (int)((k1 - k0 + TK - 1) / TK) : 0;
  if (tid == 0) {
    for (int i = 0; i < AST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4); }
    fence_barrier_init();
  }
  if (tid < HD) qb[tid] = qkv[((long long)(b * 3) * H + h) * HD + tid];
  __syncthreads();

  float m = -INFINITY, l = 0.f, o0 = 0.f, o1 = 0.f, o2 = 0.f, o3 = 0.f;
  if (warp == 4) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int t = 0; t < ntiles; ++t) {
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full[stage], 2 * TILE_BYTES);
        const int row = (int)((long long)b * S + k0 + (long long)t * TK);
        tma_load_3d(smem + stage * 2 * TILE_BYTES, &tm, &full[stage], 0, h, row);
        tma_load_3d(smem + stage * 2 * TILE_BYTES + TILE_BYTES, &tm, &full[stage], 0, H + h, row);
        if (++stage == AST) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const int key = lane & 15, half = lane >> 4;
    int stage = 0; uint32_t phase = 0;
    for (int t = 0; t < ntiles; ++t) {
      mbar_wait(&full[stage], phase);
      const uint8_t* Ks = smem + stage * 2 * TILE_BYTES;
      const uint8_t* Vs = Ks + TILE_BYTES;
      const long long jg = k0 + (long long)t * TK + warp * 16 + key;
      float sd = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int cc = (c + lane) & 7;                                 // rotated: a quarter-warp covers all 32 banks
        const uint4 kv = *reinterpret_cast<const uint4*>(Ks + (warp * 16 + key) * (HD * 2) + half * 128 + cc * 16);
        const uint4 qv = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(qb) + half * 128 + cc * 16);
        const uint32_t* kw = reinterpret_cast<const uint32_t*>(&kv);
        const uint32_t* qw = reinterpret_cast<const uint32_t*>(&qv);
#pragma unroll
        for (int e = 0; e < 4; ++e) { sd = fmaf(bf_lo(qw[e]), bf_lo(kw[e]), sd); sd = fmaf(bf_hi(qw[e]), bf_hi(kw[e]), sd); }
      }
      sd += __shfl_xor_sync(0xffffffffu, sd, 16);
      sd = jg < k1 ? sd * scale : -INFINITY;
      float mx = sd;
#pragma unroll
      for (int x = 8; x > 0; x >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, x));
      const float mn = fmaxf(m, mx);
      if (mn != -INFINITY) {                                           // warp-uniform
        const float alpha = __expf(m - mn), pe = __expf(sd - mn);
        l = l * alpha + (half == 0 ? pe : 0.f);
        const float pb = rbf(pe);                                      // P rounded to bf16 before the PV product, like the prefill kernel
        o0 *= alpha; o1 *= alpha; o2 *= alpha; o3 *= alpha;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float pj = __shfl_sync(0xffffffffu, pb, j);
          if (pj != 0.f) {                                             // masked keys (and underflowed ones) contribute nothing; garbage rows never reach the FMA
            const uint2 vv = *reinterpret_cast<const uint2*>(Vs + (warp * 16 + j) * (HD * 2) + lane * 8);
            o0 = fmaf(pj, bf_lo(vv.x), o0); o1 = fmaf(pj, bf_hi(vv.x), o1);
            o2 = fmaf(pj, bf_lo(vv.y), o2); o3 = fmaf(pj, bf_hi(vv.y), o3);
          }
        }
        m = mn;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == AST) { stage = 0; phase ^= 1; }
    }
#pragma unroll
    for (int x = 16; x > 0; x >>= 1) l += __shfl_xor_sync(0xffffffffu, l, x);
  }
  __syncthreads();                                                      // every tile consumed: stage 0 is free for the merge
  float* red_o = reinterpret_cast<float*>(smem);                       // [4][128]
  if (warp < 4) {
    if (lane == 0) { red[warp * 2] = m; red[warp * 2 + 1] = l; }
    *reinterpret_cast<float4*>(red_o + warp * HD + lane * 4) = make_float4(o0, o1, o2, o3);
  }
  __syncthreads();
  if (tid < HD) {
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < 4; ++w) M = fmaxf(M, red[w * 2]);
    float acc = 0.f, L = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float sc = red[w * 2] == -INFINITY ? 0.f : __expf(red[w * 2] - M);
      acc += red_o[w * HD + tid] * sc;
      L += red[w * 2 + 1] * sc;
    }
    const long long pidx = ((long long)b * H + h) * nsplit + sp;
    part_o[pidx * HD + tid] = acc;
    if (tid == 0) { part_ml[pidx * 2] = M; part_ml[pidx * 2 + 1] = L; }
  }
}

__global__ void decode_attn_merge_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml, bf16* __restrict__ out,
                                         int H, int nsplit) {
  pdl_launch_dependents(); pdl_wait();
  const int h = blockIdx.x, b = blockIdx.y, d = threadIdx.x;
  const long long base = ((long long)b * H + h) * nsplit;
  float M = -INFINITY;
  for (int s = 0; s < nsplit; ++s) M = fmaxf(M, part_ml[(base + s) * 2]);
  float L = 0.f, acc = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    const float ms = part_ml[(base + s) * 2];
    const float w = (ms == -INFINITY) ? 0.f : __expf(ms - M);
    L += part_ml[(base + s) * 2 + 1] * w;
    acc += part_o[(base + s) * HD + d] * w;
  }
  out[((long long)b * H + h) * HD + d] = __float2bfloat16_rn(acc / L);
}

// ---- shared-prefix decode attention: the prefix part ----
// Rows of a group (samples of one prompt) are contiguous in the batch and share one prefix of K,V in a (G, P, 2, H, 128) cache.
// One CTA = one head, one chunk of <= 64 rows of one group, one key split: the chunk's query rows are one m64 wgmma tile loaded
// once by TMA straight from qkv (B, 3, H, 128); the split's keys stream through a 3-stage ring of 128-key K and V tiles, each read
// once for all the chunk's rows.  S = Q K^T (wgmma m64n128k16, both operands in shared memory), an online softmax on the
// fragments (fp32, exact running max), P rounded to bf16 straight into the A fragment of O += P V (V read in place as the
// MN-major operand).  Every prefix key is visible (no causal mask); keys at or past prefix_len[g] are masked, and the V rows of
// a tile past that point are zeroed in shared memory before the PV product, so whatever the cache holds there (NaN included)
// cannot reach the output.  Output: unnormalised (m, l, o) per (row, head, split), m in natural-log units like the other
// decode partials; rows of the tile outside the chunk are never stored.  warps 0-3: the consumer warpgroup; warp 4: producer.
constexpr int SP_ROWS = 64;
constexpr int SP_KEYS = 128;
constexpr int SP_STAGES = 3;
constexpr int SP_Q_BYTES = SP_ROWS * HD * 2;           // 2 x 64-column halves of 8 KB
constexpr int SP_KV_BYTES = SP_KEYS * HD * 2;          // 2 x 64-column halves of 16 KB
constexpr int SP_SMEM = SP_Q_BYTES + 2 * SP_STAGES * SP_KV_BYTES + 256;
static_assert(SP_SMEM <= 232448, "exceeds the 227 KB dynamic shared memory limit");

__device__ __forceinline__ float ex2f(float x) { float y; asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

__global__ void __launch_bounds__(160, 1) decode_attn_prefix_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                                                                    const long long* __restrict__ grp, const long long* __restrict__ plen_ptr,
                                                                    int G, long long P, int B, int H, int nsplit, float scale_log2,
                                                                    float* __restrict__ part_o, float* __restrict__ part_ml) {
  pdl_launch_dependents(); pdl_wait();
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();                         // 128B-swizzled tiles need 1024-byte alignment
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + SP_Q_BYTES;
  uint8_t* sV = sK + SP_STAGES * SP_KV_BYTES;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + SP_STAGES * SP_KV_BYTES);
  uint64_t* k_full = q_full + 1;
  uint64_t* k_empty = k_full + SP_STAGES;
  uint64_t* v_full = k_empty + SP_STAGES;
  uint64_t* v_empty = v_full + SP_STAGES;
  const int h = blockIdx.x, sp = blockIdx.z, tid = threadIdx.x;

  // blockIdx.y -> (group, 64-row chunk of it); offsets are clamped to [0, B] so a malformed array cannot move a load or store
  int c = blockIdx.y, g = 0;
  long long r0 = 0, nrows = 0;
  for (; g < G; ++g) {
    const long long a = min(max(grp[g], 0LL), (long long)B), e = min(max(grp[g + 1], a), (long long)B);
    const long long nch = (e - a + SP_ROWS - 1) / SP_ROWS;
    if (c < nch) { r0 = a + (long long)c * SP_ROWS; nrows = min((long long)SP_ROWS, e - r0); break; }
    c -= (int)nch;
  }
  if (g == G) return;                                                   // past the last chunk: the grid is an upper bound
  const long long plen = min(max(plen_ptr[g], 0LL), P);
  long long per = (plen + nsplit - 1) / nsplit;
  per = (per + SP_KEYS - 1) / SP_KEYS * SP_KEYS;                         // splits start on tile boundaries
  const long long k0 = (long long)sp * per, k1 = min(plen, k0 + per);
  const int ntiles = k1 > k0 ? (int)((k1 - k0 + SP_KEYS - 1) / SP_KEYS) : 0;

  if (tid == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < SP_STAGES; ++i) { mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], 4); mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (tid >= 128) {
    if (tid == 128 && ntiles > 0) {
      tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmKV);
      mbar_arrive_expect_tx(q_full, SP_Q_BYTES);
      tma_load_3d(sQ, &tmQ, q_full, 0, h, (int)r0);
      tma_load_3d(sQ + SP_Q_BYTES / 2, &tmQ, q_full, 64, h, (int)r0);
      for (int t = 0; t < ntiles; ++t) {
        const int st = t % SP_STAGES;
        const uint32_t ph = (uint32_t)(t / SP_STAGES) & 1;
        const int row = (int)((long long)g * P + k0 + (long long)t * SP_KEYS);
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&k_full[st], SP_KV_BYTES);
        tma_load_3d(sK + st * SP_KV_BYTES, &tmKV, &k_full[st], 0, h, row);
        tma_load_3d(sK + st * SP_KV_BYTES + SP_KV_BYTES / 2, &tmKV, &k_full[st], 64, h, row);
        mbar_wait(&v_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&v_full[st], SP_KV_BYTES);
        tma_load_3d(sV + st * SP_KV_BYTES, &tmKV, &v_full[st], 0, H + h, row);
        tma_load_3d(sV + st * SP_KV_BYTES + SP_KV_BYTES / 2, &tmKV, &v_full[st], 64, H + h, row);
      }
    }
    return;
  }
  const int warp = tid >> 5, lane = tid & 31, quad = lane & 3;
  const int r = warp * 16 + (lane >> 2);                                // this thread's rows of the tile: r and r + 8
  float o[HD / 2];
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  if (ntiles > 0) mbar_wait(q_full, 0);
  const uint32_t qa = smem_u32(sQ);
  for (int t = 0; t < ntiles; ++t) {
    const int st = t % SP_STAGES;
    const uint32_t ph = (uint32_t)(t / SP_STAGES) & 1;
    const long long key0 = k0 + (long long)t * SP_KEYS;
    float s[SP_KEYS / 2];
    mbar_wait(&k_full[st], ph);
    const uint32_t ka = smem_u32(sK + st * SP_KV_BYTES);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      wgmma_m64n128k16_ss(s, wgmma_desc_k_sw128(qa + (kk >> 2) * (SP_Q_BYTES / 2) + (kk & 3) * 32),
                          wgmma_desc_k_sw128(ka + (kk >> 2) * (SP_KV_BYTES / 2) + (kk & 3) * 32), kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    if (lane == 0) mbar_arrive(&k_empty[st]);
    const bool partial = key0 + SP_KEYS > k1;                           // the split's last tile: keys at or past k1 are masked
    if (partial) {
#pragma unroll
      for (int i = 0; i < SP_KEYS / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (key0 + 8 * i + 2 * quad + e >= k1) { s[4 * i + e] = -INFINITY; s[4 * i + 2 + e] = -INFINITY; }
    }
    uint32_t pf[SP_KEYS / 16][4];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < SP_KEYS / 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * hr], s[4 * i + 2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2)) * scale_log2;
      const float mn = fmaxf(m[hr], mx);                                // finite: every tile holds at least one visible key
      const float alpha = ex2f(m[hr] - mn);
      m[hr] = mn; l[hr] *= alpha;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) { o[4 * i + 2 * hr] *= alpha; o[4 * i + 2 * hr + 1] *= alpha; }
      float ls = 0.f;
#pragma unroll
      for (int i = 0; i < SP_KEYS / 8; ++i) {
        const float p0 = ex2f(fmaf(s[4 * i + 2 * hr], scale_log2, -mn));
        const float p1 = ex2f(fmaf(s[4 * i + 2 * hr + 1], scale_log2, -mn));
        ls += p0 + p1;
        pf[i >> 1][(i & 1) * 2 + hr] = pack_bf16(p0, p1);               // P rounded to bf16 before the PV product
      }
      l[hr] += ls;
    }
    mbar_wait(&v_full[st], ph);
    uint8_t* vs = sV + st * SP_KV_BYTES;
    if (partial) {                                                      // zero V rows [k1 - key0, 128): a 128-byte swizzled row stays one row
      const int nvalid = (int)(k1 - key0);
      for (int idx = tid; idx < (SP_KEYS - nvalid) * 16; idx += 128) {
        const int row = nvalid + idx / 16, chunk = idx % 16;
        *reinterpret_cast<uint4*>(vs + (chunk / 8) * (SP_KV_BYTES / 2) + row * 128 + (chunk % 8) * 16) = make_uint4(0, 0, 0, 0);
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
    }
    const uint32_t va = smem_u32(vs);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < SP_KEYS / 16; ++kk)
      wgmma_m64n128k16_rs<1>(o, pf[kk], wgmma_desc_sw128(va + kk * 16 * 128, SP_KV_BYTES / 2, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if (lane == 0) mbar_arrive(&v_empty[st]);
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float lt = l[hr];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    if (r + 8 * hr >= nrows) continue;
    const long long pidx = ((r0 + r + 8 * hr) * H + h) * nsplit + sp;
    float* po = part_o + pidx * HD;
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) *reinterpret_cast<float2*>(po + 8 * i + 2 * quad) = make_float2(o[4 * i + 2 * hr], o[4 * i + 2 * hr + 1]);
    if (quad == 0) { part_ml[pidx * 2] = m[hr] * 0.69314718055994531f; part_ml[pidx * 2 + 1] = lt; }
  }
}

// Two-source form of decode_attn_merge_kernel: the prefix partials (np splits) and the suffix partials (ns splits) of row b.
__global__ void decode_attn_merge2_kernel(const float* __restrict__ p_o, const float* __restrict__ p_ml, int np,
                                          const float* __restrict__ s_o, const float* __restrict__ s_ml, int ns, bf16* __restrict__ out, int H) {
  pdl_launch_dependents(); pdl_wait();
  const int h = blockIdx.x, b = blockIdx.y, d = threadIdx.x;
  const long long bp = ((long long)b * H + h) * np, bs = ((long long)b * H + h) * ns;
  float M = -INFINITY;
  for (int s = 0; s < np; ++s) M = fmaxf(M, p_ml[(bp + s) * 2]);
  for (int s = 0; s < ns; ++s) M = fmaxf(M, s_ml[(bs + s) * 2]);
  float L = 0.f, acc = 0.f;
  for (int s = 0; s < np; ++s) {
    const float ms = p_ml[(bp + s) * 2];
    const float w = (ms == -INFINITY) ? 0.f : __expf(ms - M);
    L += p_ml[(bp + s) * 2 + 1] * w;
    acc += p_o[(bp + s) * HD + d] * w;
  }
  for (int s = 0; s < ns; ++s) {
    const float ms = s_ml[(bs + s) * 2];
    const float w = (ms == -INFINITY) ? 0.f : __expf(ms - M);
    L += s_ml[(bs + s) * 2 + 1] * w;
    acc += s_o[(bs + s) * HD + d] * w;
  }
  out[((long long)b * H + h) * HD + d] = __float2bfloat16_rn(acc / L);
}

__global__ void add_i64_rows_kernel(long long* p, int n, long long v) {
  pdl_launch_dependents(); pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] += v;
}

}  // namespace

extern "C" int evo_gelu_gate_interleaved(const void* t, void* out, int64_t M, int ipad, void* stream) {
  EVO_REQUIRE(ipad % 128 == 0, "evo_gelu_gate_interleaved: ipad must be a multiple of 128");
  long long total = M * (ipad / 2);
  if (total == 0) return 0;
  gelu_gate_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)t, (bf16*)out, M, ipad);
  return check_launch("evo_gelu_gate_interleaved");
}

static int decode_qkv_prep(const char* what, void* qkv, void* cache, const void* cos, const void* sin, const int64_t* pos, int pos_stride,
                           int B, int H, int hd, int64_t max_seqlen, void* stream) {
  EVO_REQUIRE(hd == HD, "%s: head_dim %d unsupported", what, hd);
  int n = B * H * 64;
  EVO_CUDA(launch_pdl(decode_qkv_prep_kernel, dim3((n + 127) / 128), dim3(128), 0, (cudaStream_t)stream, (bf16*)qkv, (bf16*)cache, (const bf16*)cos, (const bf16*)sin,
                      (const long long*)pos, pos_stride, B, H, max_seqlen));
  return check_launch(what);
}

extern "C" int evo_decode_qkv_prep(void* qkv, void* cache, const void* cos, const void* sin, const int64_t* pos,
                                   int B, int H, int hd, int64_t max_seqlen, void* stream) {
  return decode_qkv_prep("evo_decode_qkv_prep", qkv, cache, cos, sin, pos, 0, B, H, hd, max_seqlen, stream);
}

extern "C" int evo_decode_qkv_prep_rows(void* qkv, void* cache, const void* cos, const void* sin, const int64_t* pos,
                                        int B, int H, int hd, int64_t max_seqlen, void* stream) {
  return decode_qkv_prep("evo_decode_qkv_prep_rows", qkv, cache, cos, sin, pos, 1, B, H, hd, max_seqlen, stream);
}

extern "C" size_t evo_decode_attn_workspace(int B, int H, int nsplit) { return (size_t)B * H * nsplit * (HD + 2) * sizeof(float); }

// the split partials of one query per row over cache keys [0, pos[b * pos_stride]]: the TMA-fed kernel when the cache length is a
// multiple of 64, the per-thread-row kernel otherwise
static int decode_attn_partials(const char* what, const void* qkv, const void* cache, float* part_o, float* part_ml, const int64_t* pos, int pos_stride,
                                int B, int H, int64_t max_seqlen, int nsplit, float softmax_scale, void* stream) {
  int rc;
  if (max_seqlen % TK == 0 && (long long)B * max_seqlen < (1LL << 31)) {
    CUtensorMap tm;
    const uint64_t dims[3] = {(uint64_t)HD, (uint64_t)(2 * H), (uint64_t)B * (uint64_t)max_seqlen};
    const uint64_t str[2] = {(uint64_t)HD * 2, (uint64_t)2 * H * HD * 2};
    const uint32_t box[3] = {(uint32_t)HD, 1, (uint32_t)TK};
    rc = make_tmap_nd_bf16(&tm, cache, 3, dims, str, box, false);
    if (rc) return rc;
    static unsigned long long attr_done = 0;
    if ((rc = ensure_dyn_smem(decode_attn_tma_kernel, ATT2_SMEM, attr_done))) return rc;
    EVO_CUDA(launch_pdl(decode_attn_tma_kernel, dim3(H, B, nsplit), dim3(160), (size_t)ATT2_SMEM, (cudaStream_t)stream, tm, (const bf16*)qkv, part_o, part_ml,
                        (const long long*)pos, pos_stride, H, (long long)max_seqlen, nsplit, softmax_scale));
  } else {
    EVO_CUDA(launch_pdl(decode_attn_kernel, dim3(H, B, nsplit), dim3(DT), 0, (cudaStream_t)stream, (const bf16*)qkv, (const bf16*)cache, part_o, part_ml,
                        (const long long*)pos, pos_stride, H, max_seqlen, nsplit, softmax_scale));
  }
  return check_launch(what);
}

static int decode_attn(const char* what, const void* qkv, const void* cache, void* out, const int64_t* pos, int pos_stride, int B, int H, int hd,
                       int64_t max_seqlen, int nsplit, float softmax_scale, void* workspace, size_t workspace_bytes, void* stream) {
  EVO_REQUIRE(hd == HD, "%s: head_dim %d unsupported", what, hd);
  EVO_REQUIRE(nsplit >= 1 && nsplit <= 64, "%s: bad nsplit %d", what, nsplit);
  EVO_REQUIRE(workspace && workspace_bytes >= evo_decode_attn_workspace(B, H, nsplit), "%s: workspace too small", what);
  float* part_o = (float*)workspace;
  float* part_ml = part_o + (size_t)B * H * nsplit * HD;
  int rc;
  if ((rc = decode_attn_partials(what, qkv, cache, part_o, part_ml, pos, pos_stride, B, H, max_seqlen, nsplit, softmax_scale, stream))) return rc;
  EVO_CUDA(launch_pdl(decode_attn_merge_kernel, dim3(H, B), dim3(HD), 0, (cudaStream_t)stream, (const float*)part_o, (const float*)part_ml, (bf16*)out, H, nsplit));
  return check_launch("evo_decode_attn_merge");
}

extern "C" int evo_decode_attn(const void* qkv, const void* cache, void* out, const int64_t* pos, int B, int H, int hd,
                               int64_t max_seqlen, int nsplit, float softmax_scale, void* workspace, size_t workspace_bytes, void* stream) {
  return decode_attn("evo_decode_attn", qkv, cache, out, pos, 0, B, H, hd, max_seqlen, nsplit, softmax_scale, workspace, workspace_bytes, stream);
}

extern "C" int evo_decode_attn_rows(const void* qkv, const void* cache, void* out, const int64_t* pos, int B, int H, int hd,
                                    int64_t max_seqlen, int nsplit, float softmax_scale, void* workspace, size_t workspace_bytes, void* stream) {
  return decode_attn("evo_decode_attn_rows", qkv, cache, out, pos, 1, B, H, hd, max_seqlen, nsplit, softmax_scale, workspace, workspace_bytes, stream);
}

extern "C" int evo_advance_positions(int64_t* pos, int B, int64_t delta, void* stream) {
  EVO_REQUIRE(B >= 1, "evo_advance_positions: bad batch %d", B);
  EVO_CUDA(launch_pdl(add_i64_rows_kernel, dim3((B + 127) / 128), dim3(128), 0, (cudaStream_t)stream, (long long*)pos, B, (long long)delta));
  return check_launch("evo_advance_positions");
}

extern "C" int evo_decode_qkv_prep_shared(void* qkv, void* suffix_cache, const void* cos, const void* sin, const int64_t* pos, const int64_t* spos,
                                          int B, int H, int hd, int64_t suffix_len, void* stream) {
  EVO_REQUIRE(hd == HD, "evo_decode_qkv_prep_shared: head_dim %d unsupported", hd);
  EVO_REQUIRE(B >= 1 && H >= 1 && suffix_len >= 1, "evo_decode_qkv_prep_shared: bad batch %d, heads %d or suffix length %lld", B, H, (long long)suffix_len);
  int n = B * H * 64;
  EVO_CUDA(launch_pdl(decode_qkv_prep_shared_kernel, dim3((n + 127) / 128), dim3(128), 0, (cudaStream_t)stream, (bf16*)qkv, (bf16*)suffix_cache,
                      (const bf16*)cos, (const bf16*)sin, (const long long*)pos, (const long long*)spos, B, H, (long long)suffix_len));
  return check_launch("evo_decode_qkv_prep_shared");
}

extern "C" size_t evo_decode_attn_shared_workspace(int B, int H, int nsplit_prefix, int nsplit_suffix) {
  return (size_t)B * H * (nsplit_prefix + nsplit_suffix) * (HD + 2) * sizeof(float);
}

extern "C" int evo_decode_attn_shared(const void* qkv, const void* prefix_cache, const int64_t* group_offsets, const int64_t* prefix_len, int G,
                                      int64_t prefix_cache_len, const void* suffix_cache, const int64_t* spos, int64_t suffix_len, void* out,
                                      int B, int H, int hd, int nsplit_prefix, int nsplit_suffix, float softmax_scale,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  const char* what = "evo_decode_attn_shared";
  EVO_REQUIRE(hd == HD, "%s: head_dim %d unsupported", what, hd);
  EVO_REQUIRE(B >= 1 && G >= 1 && G <= B && H >= 1 && H <= 65535, "%s: bad batch %d, group count %d or head count %d", what, B, G, H);
  EVO_REQUIRE(nsplit_prefix >= 1 && nsplit_prefix <= 64 && nsplit_suffix >= 1 && nsplit_suffix <= 64, "%s: bad nsplit %d / %d", what, nsplit_prefix, nsplit_suffix);
  EVO_REQUIRE(prefix_cache_len >= 1 && (long long)G * prefix_cache_len < (1LL << 31) && suffix_len >= 1,
              "%s: bad cache lengths (prefix %lld x %d groups, suffix %lld)", what, (long long)prefix_cache_len, G, (long long)suffix_len);
  EVO_REQUIRE(group_offsets && prefix_len && spos, "%s: needs group_offsets, prefix_len and spos", what);
  EVO_REQUIRE(workspace && workspace_bytes >= evo_decode_attn_shared_workspace(B, H, nsplit_prefix, nsplit_suffix), "%s: workspace too small", what);
  float* pre_o = (float*)workspace;
  float* pre_ml = pre_o + (size_t)B * H * nsplit_prefix * HD;
  float* suf_o = pre_ml + (size_t)B * H * nsplit_prefix * 2;
  float* suf_ml = suf_o + (size_t)B * H * nsplit_suffix * HD;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  CUtensorMap tmQ, tmKV;
  {
    const uint64_t dims[3] = {(uint64_t)HD, (uint64_t)H, (uint64_t)B};                 // q of qkv (B, 3, H, 128)
    const uint64_t str[2] = {(uint64_t)HD * 2, (uint64_t)3 * H * HD * 2};
    const uint32_t box[3] = {64, 1, (uint32_t)SP_ROWS};
    if ((rc = make_tmap_nd_bf16(&tmQ, qkv, 3, dims, str, box, true))) return rc;
  }
  {
    const uint64_t dims[3] = {(uint64_t)HD, (uint64_t)(2 * H), (uint64_t)G * (uint64_t)prefix_cache_len};   // (G * P, 2H, 128)
    const uint64_t str[2] = {(uint64_t)HD * 2, (uint64_t)2 * H * HD * 2};
    const uint32_t box[3] = {64, 1, (uint32_t)SP_KEYS};
    if ((rc = make_tmap_nd_bf16(&tmKV, prefix_cache, 3, dims, str, box, true))) return rc;
  }
  static unsigned long long attr_done = 0;
  if ((rc = ensure_dyn_smem(decode_attn_prefix_kernel, SP_SMEM, attr_done))) return rc;
  // every group has ceil(rows / 64) chunks, so G + B / 64 bounds their number; CTAs past the last chunk exit at once
  EVO_CUDA(launch_pdl(decode_attn_prefix_kernel, dim3(H, G + B / SP_ROWS, nsplit_prefix), dim3(160), (size_t)SP_SMEM, st, tmQ, tmKV,
                      (const long long*)group_offsets, (const long long*)prefix_len, G, (long long)prefix_cache_len, B, H, nsplit_prefix,
                      softmax_scale * 1.4426950408889634f, pre_o, pre_ml));
  if ((rc = check_launch(what))) return rc;
  if ((rc = decode_attn_partials(what, qkv, suffix_cache, suf_o, suf_ml, spos, 1, B, H, suffix_len, nsplit_suffix, softmax_scale, stream))) return rc;
  EVO_CUDA(launch_pdl(decode_attn_merge2_kernel, dim3(H, B), dim3(HD), 0, st, (const float*)pre_o, (const float*)pre_ml, nsplit_prefix,
                      (const float*)suf_o, (const float*)suf_ml, nsplit_suffix, (bf16*)out, H));
  return check_launch("evo_decode_attn_shared_merge");
}
