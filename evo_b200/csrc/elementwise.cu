// Memory-bound glue kernels: embedding gather, RMSNorm, rotary tables / application,
// KV-cache append, residual add, fused log-softmax + gather.  All 128-bit coalesced.
#include "common.cuh"
#include "../../include/evo_b200.h"

using namespace evo;

// ------------------------------------------------------------------ embed
// VocabParallelEmbedding.embed: out[t, :] = table[ids[t], :]
template <typename IdT>
__global__ void embed_kernel(const IdT* __restrict__ ids, const uint4* __restrict__ table, uint4* __restrict__ out,
                             int64_t n_tokens, int row_vec, int vocab) {
  pdl_launch_dependents(); pdl_wait();
  int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (warp >= n_tokens) return;
  long long id = (long long)ids[warp];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  const uint4* src = table + (int64_t)id * row_vec;
  uint4* dst = out + warp * row_vec;
  for (int i = lane_id(); i < row_vec; i += 32) dst[i] = __ldg(src + i);
}

extern "C" int evo_embed(const void* ids, int ids_are_i64, const void* table, void* out,
                         int64_t n_tokens, int D, int vocab, void* stream) {
  EVO_REQUIRE(D % 8 == 0, "evo_embed: D (%d) must be a multiple of 8", D);
  if (n_tokens == 0) return 0;
  int wpb = 8;
  dim3 grid((unsigned)((n_tokens + wpb - 1) / wpb)), block(wpb * 32);
  if (ids_are_i64)
    EVO_CUDA(launch_pdl(embed_kernel<long long>, grid, block, 0, (cudaStream_t)stream, (const long long*)ids, (const uint4*)table, (uint4*)out, n_tokens, D / 8, vocab));
  else
    EVO_CUDA(launch_pdl(embed_kernel<int>, grid, block, 0, (cudaStream_t)stream, (const int*)ids, (const uint4*)table, (uint4*)out, n_tokens, D / 8, vocab));
  return check_launch("evo_embed");
}

// ------------------------------------------------------------------ RMSNorm
// One warp per row; the row stays in registers between the reduction and the scale.  The rounding chain is rms_rinv and
// rms_word (common.cuh).
template <int MAXV>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const uint4* __restrict__ x, const uint4* __restrict__ scale,
                                                      uint4* __restrict__ out, int64_t rows, int nvec_per_lane,
                                                      float inv_sqrt_d, float eps) {
  pdl_launch_dependents(); pdl_wait();
  int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = lane_id();
  const int row_vec = nvec_per_lane * 32;
  const uint4* xr = x + row * row_vec;
  uint4 v[MAXV];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    if (i < nvec_per_lane) {
      v[i] = __ldg(xr + i * 32 + lane);
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&v[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) { float a = bf_lo(w[j]), b = bf_hi(w[j]); ss = fmaf(a, a, ss); ss = fmaf(b, b, ss); }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rinv = rms_rinv(ss, inv_sqrt_d, eps);
  uint4* orow = out + row * row_vec;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    if (i < nvec_per_lane) {
      uint4 s = __ldg(scale + i * 32 + lane);
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&v[i]);
      const uint32_t* sw = reinterpret_cast<const uint32_t*>(&s);
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) ow[j] = rms_word(w[j], sw[j], rinv);
      orow[i * 32 + lane] = o;
    }
  }
}

// Few rows (decode step): one 256-thread CTA per row instead of one warp per row -- the row and the scale are fetched
// by 8 warps at once (the warp-per-row kernel is a 5 us latency chain on 2 CTAs at 16 rows).
__global__ void __launch_bounds__(256) rmsnorm_row_kernel(const uint4* __restrict__ x, const uint4* __restrict__ scale,
                                                          uint4* __restrict__ out, int row_vec, float inv_sqrt_d, float eps) {
  pdl_launch_dependents(); pdl_wait();
  __shared__ float red[8];
  const int tid = threadIdx.x;
  const uint4* xr = x + (int64_t)blockIdx.x * row_vec;
  uint4 v[4], sc[4];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid + i * 256;
    if (idx < row_vec) { v[i] = __ldg(xr + idx); sc[i] = __ldg(scale + idx); }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (tid + i * 256 < row_vec) {
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&v[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) { float a = bf_lo(w[j]), b = bf_hi(w[j]); ss = fmaf(a, a, ss); ss = fmaf(b, b, ss); }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];
  const float rinv = rms_rinv(tot, inv_sqrt_d, eps);
  uint4* orow = out + (int64_t)blockIdx.x * row_vec;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid + i * 256;
    if (idx < row_vec) {
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&v[i]);
      const uint32_t* sw = reinterpret_cast<const uint32_t*>(&sc[i]);
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) ow[j] = rms_word(w[j], sw[j], rinv);
      orow[idx] = o;
    }
  }
}

extern "C" int evo_rmsnorm(const void* x, const void* scale, void* out, int64_t rows, int D, float eps, void* stream) {
  EVO_REQUIRE(D % 256 == 0 && D <= 8192, "evo_rmsnorm: D (%d) must be a multiple of 256 and <= 8192", D);
  if (rows == 0) return 0;
  if (rows <= 64) {
    EVO_CUDA(launch_pdl_light(rmsnorm_row_kernel, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream, (const uint4*)x, (const uint4*)scale, (uint4*)out,
                        D / 8, (float)(1.0 / sqrt((double)D)), eps));
    return check_launch("evo_rmsnorm");
  }
  int nvec = D / 256;
  dim3 grid((unsigned)((rows + 7) / 8)), block(256);
  float isd = (float)(1.0 / sqrt((double)D));
  if (nvec <= 16)
    EVO_CUDA(launch_pdl(rmsnorm_kernel<16>, grid, block, 0, (cudaStream_t)stream, (const uint4*)x, (const uint4*)scale, (uint4*)out, rows, nvec, isd, eps));
  else
    EVO_CUDA(launch_pdl(rmsnorm_kernel<32>, grid, block, 0, (cudaStream_t)stream, (const uint4*)x, (const uint4*)scale, (uint4*)out, rows, nvec, isd, eps));
  return check_launch("evo_rmsnorm");
}

// ------------------------------------------------------------------ rotary
__global__ void rope_table_kernel(bf16* __restrict__ cos_out, bf16* __restrict__ sin_out, const float* __restrict__ inv_freq,
                                  int64_t pos0, int64_t n_pos, int half, float scaling) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_pos * half) return;
  int i = (int)(idx % half);
  int64_t p = idx / half;
  float t = (float)(pos0 + p);
  if (scaling != 1.0f) t = __fdiv_rn(t, scaling);   // LinearlyScaledRotaryEmbedding: t /= scaling_factor
  float f = t * inv_freq[i];                        // torch.outer(t, inv_freq), fp32
  float s, c;
  sincosf(f, &s, &c);
  cos_out[idx] = __float2bfloat16_rn(c);
  sin_out[idx] = __float2bfloat16_rn(s);
}

extern "C" int evo_rope_tables(void* cos_out, void* sin_out, const float* inv_freq, int64_t pos0, int64_t n_pos,
                               int half_dim, float scaling_factor, void* stream) {
  if (n_pos == 0) return 0;
  int64_t n = n_pos * half_dim;
  rope_table_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((bf16*)cos_out, (bf16*)sin_out, inv_freq, pos0, n_pos, half_dim, scaling_factor);
  return check_launch("evo_rope_tables");
}

// In-place NeoX rotary on q and k.  One thread rotates 8 (x0, x1) pairs: 2x16 B in, 2x16 B out.
__global__ void rotary_qk_kernel(uint4* __restrict__ qkv, const uint4* __restrict__ cos, const uint4* __restrict__ sin,
                                 int64_t n_tok, int64_t L, int H, int hd) {
  const int vec_per_half = hd / 16;                 // uint4 per 64 bf16 = 8 for hd 128
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = n_tok * 2 * H * vec_per_half;
  if (idx >= total) return;
  int c = (int)(idx % vec_per_half);
  int64_t r = idx / vec_per_half;
  int h = (int)(r % H); r /= H;
  int which = (int)(r % 2); r /= 2;                 // 0 = q, 1 = k
  int64_t tok = r;
  int64_t l = tok % L;
  uint4* base = qkv + ((tok * 3 + which) * H + h) * (hd / 8);
  uint4 a = base[c], b = base[c + vec_per_half];
  uint4 cv = __ldg(cos + l * vec_per_half + c), sv = __ldg(sin + l * vec_per_half + c);
  const uint32_t *aw = (const uint32_t*)&a, *bw = (const uint32_t*)&b, *cw = (const uint32_t*)&cv, *sw = (const uint32_t*)&sv;
  uint4 oa, ob;
  uint32_t *oaw = (uint32_t*)&oa, *obw = (uint32_t*)&ob;
#pragma unroll
  for (int j = 0; j < 4; ++j) rope_words(bf_lo(aw[j]), bf_hi(aw[j]), bf_lo(bw[j]), bf_hi(bw[j]), cw[j], sw[j], oaw[j], obw[j]);
  base[c] = oa;
  base[c + vec_per_half] = ob;
}

extern "C" int evo_rotary_qk(void* qkv, const void* cos, const void* sin, int B, int64_t L, int H, int hd, void* stream) {
  EVO_REQUIRE(hd % 16 == 0, "evo_rotary_qk: head_dim (%d) must be a multiple of 16", hd);
  int64_t total = (int64_t)B * L * 2 * H * (hd / 16);
  if (total == 0) return 0;
  rotary_qk_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((uint4*)qkv, (const uint4*)cos, (const uint4*)sin, (int64_t)B * L, L, H, hd);
  return check_launch("evo_rotary_qk");
}

// ------------------------------------------------------------------ KV cache append
__global__ void kv_append_kernel(const uint4* __restrict__ qkv, uint4* __restrict__ cache, int64_t L, int row_vec,
                                 int64_t pos0, int64_t max_seqlen, int64_t total) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  int c = (int)(idx % (2 * row_vec));
  int64_t tok = idx / (2 * row_vec);
  int64_t b = tok / L, l = tok % L;
  cache[(b * max_seqlen + pos0 + l) * (2 * row_vec) + c] = qkv[tok * (3 * row_vec) + row_vec + c];
}

extern "C" int evo_kv_append(const void* qkv, void* cache, int B, int64_t L, int H, int hd,
                             int64_t pos0, int64_t max_seqlen, void* stream) {
  EVO_REQUIRE(pos0 + L <= max_seqlen, "evo_kv_append: sequence length %lld exceeds the KV cache (%lld)", (long long)(pos0 + L), (long long)max_seqlen);
  int row_vec = H * hd / 8;
  int64_t total = (int64_t)B * L * 2 * row_vec;
  if (total == 0) return 0;
  kv_append_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint4*)qkv, (uint4*)cache, L, row_vec, pos0, max_seqlen, total);
  return check_launch("evo_kv_append");
}

// packed sequences: grid row b copies sequence b's rows [cu[b], cu[b+1]) to cache rows [0, len) of batch row b
__global__ void kv_append_varlen_kernel(const uint4* __restrict__ qkv, uint4* __restrict__ cache, const long long* __restrict__ cu,
                                        long long T, long long max_len, int row_vec, int64_t cache_len) {
  const int b = blockIdx.y;
  const long long row0 = min(max(cu[b], 0LL), T);
  const long long len = min(min(cu[b + 1], T) - row0, max_len);
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c = (int)(idx % (2 * row_vec));
  const int64_t l = idx / (2 * row_vec);
  if (l >= len) return;
  cache[((int64_t)b * cache_len + l) * (2 * row_vec) + c] = qkv[(row0 + l) * (3 * row_vec) + row_vec + c];
}

extern "C" int evo_kv_append_varlen(const void* qkv, void* cache, const int64_t* cu_seqlens, int n_seq, int64_t T, int64_t max_seqlen,
                                    int H, int hd, int64_t cache_len, void* stream) {
  EVO_REQUIRE(n_seq > 0 && n_seq <= 65535 && cu_seqlens != nullptr, "evo_kv_append_varlen: bad sequence count %d or no cu_seqlens", n_seq);
  EVO_REQUIRE(max_seqlen > 0 && max_seqlen <= T && max_seqlen <= cache_len,
              "evo_kv_append_varlen: longest sequence %lld must be in (0, min(T %lld, cache %lld)]", (long long)max_seqlen, (long long)T, (long long)cache_len);
  EVO_REQUIRE((H * hd) % 8 == 0, "evo_kv_append_varlen: H * hd must be a multiple of 8");
  const int row_vec = H * hd / 8;
  const int64_t per_seq = max_seqlen * 2 * row_vec;
  kv_append_varlen_kernel<<<dim3((unsigned)((per_seq + 255) / 256), n_seq), 256, 0, (cudaStream_t)stream>>>(
      (const uint4*)qkv, (uint4*)cache, (const long long*)cu_seqlens, T, max_seqlen, row_vec, cache_len);
  return check_launch("evo_kv_append_varlen");
}

// ------------------------------------------------------------------ scoring epilogue
// out[r] = log_softmax(logits[r, :])[target[r]], fp32 statistics; one warp per row.
__global__ void logprobs_kernel(const bf16* __restrict__ logits, const long long* __restrict__ targets, float* __restrict__ out,
                                int64_t rows, int V) {
  int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const bf16* lr = logits + row * V;
  const int lane = lane_id();
  float m = -INFINITY;
  for (int i = lane; i < V; i += 32) m = fmaxf(m, __bfloat162float(lr[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int i = lane; i < V; i += 32) s += expf(__bfloat162float(lr[i]) - m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    long long t = targets[row];
    out[row] = (t < 0 || t >= V) ? 0.f : (__bfloat162float(lr[t]) - m - logf(s));
  }
}
extern "C" int evo_logprobs(const void* logits, const int64_t* targets, float* out, int64_t rows, int V, void* stream) {
  if (rows == 0) return 0;
  logprobs_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>((const bf16*)logits, (const long long*)targets, out, rows, V);
  return check_launch("evo_logprobs");
}
