// Sequence pooling over packed rows (embeddings): one fp32 vector per sequence from the (T, D) bf16 rows of a packed forward.
//
// A sequence's kept rows are cut into POOL_CHUNK-row chunks counted from its first kept row; every (chunk, 256-column slice)
// pair is one CTA.  A sequence of one chunk is finished by that CTA.  A longer one writes one fp32 partial row per chunk to
// the workspace and pool_combine_kernel folds them in chunk order.  No atomics: each output is a fixed sum tree that depends
// only on the sequence's kept-row count, so the bits do not depend on where the sequence sits in the pack.
//
// Chunk c of sequence b owns work slot s(b, c) = b + floor(cu[b] / POOL_CHUNK) + c.  The slots of one sequence are consecutive,
// s(b, last) < s(b + 1, 0) (its chunk count is at most ceil(len_b / POOL_CHUNK)), and s < n_seq + T / POOL_CHUNK + 1, so the
// grid and the workspace are sized from T and n_seq on the host while the lengths stay on the device.  A CTA finds its
// sequence by binary search over cu; slots between two sequences exit at once.
#include "common.cuh"
#include "../../include/evo_b200.h"

using namespace evo;

namespace {

constexpr int POOL_CHUNK = 512;      // rows per chunk
constexpr int POOL_THREADS = 256;    // 8 row groups x 32 lanes; a lane holds 8 columns (one 16-byte vector)
constexpr int POOL_GROUPS = POOL_THREADS / 32;
constexpr int POOL_COLS = 256;       // columns per CTA

struct SeqRows {
  int64_t first, n;                  // first kept row, kept-row count
  int64_t slot0;                     // work slot of chunk 0
  int nc;                            // chunks (0 when no row is kept)
};

__device__ __forceinline__ int64_t clamp64(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Sequence b's rows, clamped to [0, T) and to max_seqlen so a malformed device array cannot move a load out of bounds.
__device__ __forceinline__ SeqRows seq_rows(const int64_t* __restrict__ cu, int b, int64_t T, int64_t max_seqlen, int skip) {
  const int64_t a = clamp64(cu[b], 0, T);
  const int64_t e = clamp64(cu[b + 1], a, a + max_seqlen < T ? a + max_seqlen : T);
  SeqRows s;
  s.first = a + skip;
  s.n = e - s.first > 0 ? e - s.first : 0;
  s.slot0 = b + a / POOL_CHUNK;
  s.nc = (int)((s.n + POOL_CHUNK - 1) / POOL_CHUNK);
  return s;
}

__device__ __forceinline__ float combine(float a, float b, int mode) { return mode == EVO_POOL_MAX ? fmaxf(a, b) : __fadd_rn(a, b); }

__global__ void __launch_bounds__(POOL_THREADS) pool_rows_kernel(const uint4* __restrict__ x, int64_t ldx_vec, const int64_t* __restrict__ cu,
                                                                 int n_seq, int64_t T, int64_t max_seqlen, int D, int skip, int mode,
                                                                 float* __restrict__ out, int64_t ldo, float* __restrict__ ws) {
  const int64_t j = blockIdx.x;
  // the last sequence whose chunk-0 slot is <= j
  int lo = 0, hi = n_seq - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (mid + clamp64(cu[mid], 0, T) / POOL_CHUNK <= j) lo = mid; else hi = mid - 1;
  }
  const int b = lo;
  const SeqRows s = seq_rows(cu, b, T, max_seqlen, skip);
  const int64_t c = j - s.slot0;
  if (c < 0 || c >= (s.nc > 0 ? s.nc : 1)) return;

  const int tid = threadIdx.x, lane = tid & 31, g = tid >> 5;
  const int col0 = blockIdx.y * POOL_COLS;
  const int vcol = blockIdx.y * (POOL_COLS / 8) + lane;    // this lane's 16-byte vector of the row
  const bool live = vcol * 8 < D;
  float* orow = out + (int64_t)b * ldo;

  if (s.n == 0) {                                          // no kept row: NaN in every mode
    for (int k = tid; k < POOL_COLS && col0 + k < D; k += POOL_THREADS) orow[col0 + k] = __int_as_float(0x7fffffff);
    return;
  }
  if (mode == EVO_POOL_LAST) {                             // the last kept row, widened
    if (g == 0 && live) {
      const uint4 v = __ldg(x + (s.first + s.n - 1) * ldx_vec + vcol);
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int k = 0; k < 4; ++k) { orow[vcol * 8 + 2 * k] = bf_lo(w[k]); orow[vcol * 8 + 2 * k + 1] = bf_hi(w[k]); }
    }
    return;
  }

  // rows r0 + g, r0 + g + 8, ... of this chunk, in row order, per lane; then the 8 row groups in order
  __shared__ __align__(16) float red[POOL_GROUPS][POOL_COLS];
  const int64_t r0 = s.first + c * POOL_CHUNK;
  const int64_t r1 = r0 + POOL_CHUNK < s.first + s.n ? r0 + POOL_CHUNK : s.first + s.n;
  const float init = mode == EVO_POOL_MAX ? -INFINITY : 0.f;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = init;
  if (live) {
    const uint4* p = x + vcol;
    int64_t r = r0 + g;
    constexpr int U = 4;
    for (; r + (U - 1) * POOL_GROUPS < r1; r += U * POOL_GROUPS) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = __ldg(p + (r + u * POOL_GROUPS) * ldx_vec);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&v[u]);
#pragma unroll
        for (int k = 0; k < 4; ++k) { acc[2 * k] = combine(acc[2 * k], bf_lo(w[k]), mode); acc[2 * k + 1] = combine(acc[2 * k + 1], bf_hi(w[k]), mode); }
      }
    }
    for (; r < r1; r += POOL_GROUPS) {
      const uint4 v = __ldg(p + r * ldx_vec);
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int k = 0; k < 4; ++k) { acc[2 * k] = combine(acc[2 * k], bf_lo(w[k]), mode); acc[2 * k + 1] = combine(acc[2 * k + 1], bf_hi(w[k]), mode); }
    }
  }
  float4* dst = reinterpret_cast<float4*>(&red[g][lane * 8]);
  dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  __syncthreads();
  const int col = col0 + tid;
  if (col >= D) return;
  float t = red[0][tid];
#pragma unroll
  for (int q = 1; q < POOL_GROUPS; ++q) t = combine(t, red[q][tid], mode);
  if (s.nc == 1)
    orow[col] = mode == EVO_POOL_MEAN ? __fdiv_rn(t, (float)s.n) : t;
  else
    ws[j * D + col] = t;
}

// Sequences of more than one chunk: fold the chunk partials in chunk order.
__global__ void __launch_bounds__(POOL_THREADS) pool_combine_kernel(const int64_t* __restrict__ cu, int64_t T, int64_t max_seqlen, int D,
                                                                    int skip, int mode, float* __restrict__ out, int64_t ldo,
                                                                    const float* __restrict__ ws, int64_t n_slots) {
  const int b = blockIdx.x;
  const SeqRows s = seq_rows(cu, b, T, max_seqlen, skip);
  const int col = blockIdx.y * POOL_COLS + threadIdx.x;
  if (s.nc <= 1 || col >= D) return;
  const int nc = (int)(s.slot0 + s.nc <= n_slots ? s.nc : n_slots - s.slot0);
  const float* p = ws + s.slot0 * D + col;
  float t = p[0];
  int c = 1;
  constexpr int U = 8;
  for (; c + U <= nc; c += U) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = p[(int64_t)(c + u) * D];
#pragma unroll
    for (int u = 0; u < U; ++u) t = combine(t, v[u], mode);
  }
  for (; c < nc; ++c) t = combine(t, p[(int64_t)c * D], mode);
  out[(int64_t)b * ldo + col] = mode == EVO_POOL_MEAN ? __fdiv_rn(t, (float)s.n) : t;
}

int64_t pool_slots(const evo_pool_varlen_params* p) { return (int64_t)p->n_seq + p->T / POOL_CHUNK + 1; }

// Only a sequence of more than one chunk needs the workspace, and none has more rows than max_seqlen.
bool pool_needs_combine(const evo_pool_varlen_params* p) {
  return p->mode != EVO_POOL_LAST && p->max_seqlen - (p->skip_first > 0 ? p->skip_first : 0) > POOL_CHUNK;
}

}  // namespace

extern "C" size_t evo_pool_varlen_workspace(const evo_pool_varlen_params* p) {
  if (p == nullptr || p->n_seq < 1 || p->T < 1 || p->D < 1 || !pool_needs_combine(p)) return 0;
  return (size_t)pool_slots(p) * (size_t)p->D * sizeof(float);
}

extern "C" int evo_pool_varlen(const evo_pool_varlen_params* p, void* workspace, size_t workspace_bytes, void* stream) {
  EVO_REQUIRE(p != nullptr, "evo_pool_varlen: params is NULL");
  EVO_REQUIRE(p->x != nullptr && p->cu_seqlens != nullptr && p->out != nullptr, "evo_pool_varlen: x, cu_seqlens and out must be non-NULL");
  EVO_REQUIRE(p->D > 0 && p->D % 8 == 0, "evo_pool_varlen: D (%d) must be a positive multiple of 8", p->D);
  EVO_REQUIRE(p->ldx >= p->D && p->ldx % 8 == 0, "evo_pool_varlen: ldx (%lld) must be >= D (%d) and a multiple of 8",
              (long long)p->ldx, p->D);
  EVO_REQUIRE(((uintptr_t)p->x & 15) == 0, "evo_pool_varlen: x must be 16-byte aligned");
  EVO_REQUIRE(p->ldo >= p->D, "evo_pool_varlen: ldo (%lld) must be >= D (%d)", (long long)p->ldo, p->D);
  EVO_REQUIRE(p->n_seq >= 1 && p->n_seq <= 65535, "evo_pool_varlen: n_seq (%d) must be in [1, 65535]", p->n_seq);
  EVO_REQUIRE(p->T >= 1, "evo_pool_varlen: T (%lld) must be >= 1", (long long)p->T);
  EVO_REQUIRE(p->max_seqlen >= 1 && p->max_seqlen <= p->T, "evo_pool_varlen: max_seqlen (%lld) must be in [1, T = %lld]",
              (long long)p->max_seqlen, (long long)p->T);
  EVO_REQUIRE(p->skip_first >= 0, "evo_pool_varlen: skip_first (%d) must be >= 0", p->skip_first);
  EVO_REQUIRE(p->mode == EVO_POOL_MEAN || p->mode == EVO_POOL_MAX || p->mode == EVO_POOL_LAST,
              "evo_pool_varlen: unknown mode %d", p->mode);
  const size_t need = evo_pool_varlen_workspace(p);
  EVO_REQUIRE(workspace_bytes >= need && (need == 0 || workspace != nullptr),
              "evo_pool_varlen: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  const int64_t n_slots = pool_slots(p);
  const unsigned slices = (unsigned)((p->D + POOL_COLS - 1) / POOL_COLS);
  cudaStream_t st = (cudaStream_t)stream;
  pool_rows_kernel<<<dim3((unsigned)n_slots, slices), POOL_THREADS, 0, st>>>(
      (const uint4*)p->x, p->ldx / 8, p->cu_seqlens, p->n_seq, p->T, p->max_seqlen, p->D, p->skip_first, p->mode, p->out, p->ldo,
      (float*)workspace);
  int rc = check_launch("evo_pool_varlen");
  if (rc != 0 || need == 0) return rc;
  pool_combine_kernel<<<dim3((unsigned)p->n_seq, slices), POOL_THREADS, 0, st>>>(
      p->cu_seqlens, p->T, p->max_seqlen, p->D, p->skip_first, p->mode, p->out, p->ldo, (const float*)workspace, n_slots);
  return check_launch("evo_pool_varlen(combine)");
}
