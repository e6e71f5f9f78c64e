// Weight-streaming linear layer for the decode step (M <= 64 rows): C[M,N] = epilogue(A[M,K] . W[N,K]^T).
//
// At M = 16 the layer is a pure HBM stream of W (2*N*K bytes against 32*N*K flops), so the kernel is built
// around keeping all SMs pulling weights at an equal rate:
//   * swap-AB: 128 rows of W are the MMA M dimension (two m64 wgmma row halves, one per consumer warpgroup) and
//     the (padded) M activation rows are the MMA N dimension (16..64), so the tensor pipe never limits the stream;
//   * stream-K: the (N/128) x (K/64) k-block iterations are cut into gridDim.x equal contiguous ranges, one
//     per SM, so every shape (N = 4096 .. 22016) loads the machine evenly -- no wave quantisation;
//   * a range that covers only part of a tile's K leaves its 128 x Mb fp32 partial in a workspace slot; the
//     LAST contributor to arrive (per-tile counter) sums the slots in slot order -- deterministic, no spin
//     wait, no co-residency requirement -- and applies the epilogue;
//   * programmatic dependent launch: the producer prefetches its first ring of W tiles (weights never depend
//     on the previous kernel) BEFORE griddepcontrol.wait, so the pipeline fill overlaps the tail of whatever
//     ran before; everything that reads activations / residuals or writes happens after the wait.
// Roles: warpgroup 0 TMA producer; warpgroups 1-2 issue the wgmma for W rows [0, 64) / [64, 128) of the tile, park the
// accumulator fragments in shared memory as [column][W row], and run the epilogue (thread = one W row = one output
// column, 16 batch values per pass; the two warpgroups take alternate 16-row batch chunks).
// EVO_EPI_GELU_GATE: a tile is 256 packed rows [l1 | l2] (two MMA row groups), the epilogue thread holds l1[b] and
// l2[b] of its column: gelu(l1)*l2 is fused.
//
// FP8 weights (evo_gemm_smallm_fp8, template flag FP8): W is stored as E4M3 q[n, k] with a power-of-two scale 2^e[n] per row,
// W'[n, k] = q[n, k] 2^e[n], and the kernel streams q (one byte per weight) instead of the bf16 W'.  Only the path of the W operand
// changes: one 1-D bulk copy per stage of a block laid out in the order of the wgmma A register fragments (the FP8 decode layout below), two
// 16-byte shared loads per thread and k-block, an exact E4M3 -> bf16 conversion, and wgmma with A from registers.  The cut rule,
// the grid, the fix-up order, the PDL prefetch and finalize16 are the bf16 kernel's; the scale 2^e[n] multiplies the fp32 sum of
// column n once, after the fix-up's slot sum and before the epilogue.  A power-of-two scale commutes exactly with every fp32
// partial sum (no under- or overflow at weight magnitudes), so the output is bit-identical to evo_gemm_smallm on W'.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/evo_b200.h"
#include <cuda_fp8.h>
#include <algorithm>
#include <cmath>
#include <cstring>

using namespace evo;

namespace {

constexpr int BK = 64;              // bf16 per k-block = one 128-byte swizzle row
constexpr int UK = 16;
constexpr int WROWS = 128;          // W rows per MMA row group (UMMA M)
constexpr int MAXST = 12;           // ring depth upper bound (barrier array size)
constexpr int NTHREADS = 384;
constexpr int CONSUMER_WARPS = 8;
constexpr int STG_LD = WROWS + 4;      // staging row stride (floats): conflict-free fragment stores
constexpr int MAX_MB = 64;
constexpr int RING_BYTES = 104 * 1024;  // shared memory for the W + A ring (152 KB measured the same, 208 KB slower)

struct SmArgs {
  bf16* C; long long ldc;
  const bf16* bias;
  const bf16* resid; long long ldr;
  int M, Mb;                        // rows of A; rows staged / UMMA N (multiple of 16)
  int n_tiles, KB;                  // tiles of (128*R) W rows; k-blocks per tile
  int n_stages;
  int* counters;                    // [n_tiles], zero between launches
  float* slots;                     // [2 * gridDim.x][R * Mb][128] fp32 partials
  const uint8_t* Wq;                // FP8 form: E4M3 weights in the FP8 decode layout
  const int8_t* Wexp;               // FP8 form: (N) row exponents
};

// FP8 decode layout.  One contiguous block of 128 x 64 bytes per (tile, row group r, k-block) in iteration order (tile, k-block,
// r), so a CTA's stream-K range is one contiguous run of DRAM.  Inside a block, consumer thread t of warpgroup cw (W rows
// cw*64 + 16*(t/32) + (t%32)/4 [+8]) owns 32 bytes: its wgmma A fragments for the four k16 steps, split into two 16-byte halves
// (k16 steps {0,1} and {2,3}) that lie 512 bytes apart, so that each quarter-warp's 16-byte loads cover 128 contiguous bytes
// (no bank conflict).  Byte order inside a half: k16 step, fragment register a[0..3], low k of the pair first.  fp8_quantize_kernel
// writes it (and is its one definition); the model's fp8_layout() is the host reference.
constexpr int FP8_BLOCK = WROWS * BK;

// four E4M3 values (bytes 0..3) -> two bf16 pairs: exact (f16 holds every E4M3 value as a normal number or zero, and bf16 every f16
// with a 4-bit significand in E4M3's exponent range)
__device__ __forceinline__ void e4m3x4_to_bf16x2(uint32_t v, uint32_t& lo, uint32_t& hi) {
  uint32_t h0, h1;
  asm("{\n\t.reg .b16 a, b;\n\tmov.b32 {a, b}, %2;\n\t"
      "cvt.rn.f16x2.e4m3x2 %0, a;\n\tcvt.rn.f16x2.e4m3x2 %1, b;\n\t}\n" : "=r"(h0), "=r"(h1) : "r"(v));
  const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&h0)), f1 = __half22float2(*reinterpret_cast<const __half2*>(&h1));
  lo = __byte_perm(__float_as_uint(f0.x), __float_as_uint(f0.y), 0x7632);
  hi = __byte_perm(__float_as_uint(f1.x), __float_as_uint(f1.y), 0x7632);
}
__device__ __forceinline__ float pow2f(int e) { return __int_as_float((e + 127) << 23); }   // e in [-126, 127]

// first k-block iteration of CTA c when `total` iterations are cut into `parts` contiguous ranges.  32-bit on purpose
// (the host checks total * parts < 2^31): 64-bit division is a ~100-instruction subroutine and this sits in the tail.
__device__ __forceinline__ uint32_t range_start(uint32_t c, uint32_t total, uint32_t parts) { return c * total / parts; }
__device__ __forceinline__ int cta_of(uint32_t it, uint32_t total, uint32_t parts) {
  uint32_t c = it * parts / total;
  while (c + 1 < parts && range_start(c + 1, total, parts) <= it) ++c;
  while (c > 0 && range_start(c, total, parts) > it) --c;
  return (int)c;
}

// residual values of 16 batch rows of output column n, fetched BEFORE the accumulators are needed (one round trip
// for all 16 instead of a load -> store chain the compiler may not reorder)
template <int EPI>
__device__ __forceinline__ void load_resid16(const SmArgs& g, long long n, int b0, float (&rv)[16]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    rv[j] = 0.f;
    if constexpr (EPI == EVO_EPI_BIAS_RESID || EPI == EVO_EPI_RESID)
      if (b0 + j < g.M) rv[j] = __bfloat162float(g.resid[(long long)(b0 + j) * g.ldr + n]);
  }
}

// epilogue of 16 batch rows [b0, b0+16) of output column n; v0 (and v1 for the gate) are fp32 sums
template <int EPI>
__device__ __forceinline__ void finalize16(const SmArgs& g, long long n, int b0, float bias, const float (&rv)[16],
                                           const float (&v0)[16], const float (&v1)[16]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int b = b0 + j;
    const float o = EPI == EVO_EPI_GELU_GATE ? gelu_gate_acc(v0[j], v1[j])
                                             : linear_out<EPI == EVO_EPI_BIAS || EPI == EVO_EPI_BIAS_RESID,
                                                          EPI == EVO_EPI_BIAS_RESID || EPI == EVO_EPI_RESID>(v0[j], bias, rv[j]);
    if (b < g.M) g.C[(long long)b * g.ldc + n] = __float2bfloat16_rn(o);
  }
}

template <int EPI> struct RowGroups { static constexpr int R = EPI == EVO_EPI_GELU_GATE ? 2 : 1; };

template <int MB>
__device__ __forceinline__ void wgmma_ss_n(float (&d)[MB / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (MB == 16) wgmma_m64n16k16_ss(d, da, db, scale_d);
  else if constexpr (MB == 32) wgmma_m64n32k16_ss(d, da, db, scale_d);
  else if constexpr (MB == 48) wgmma_m64n48k16_ss(d, da, db, scale_d);
  else wgmma_m64n64k16_ss(d, da, db, scale_d);
}

template <int MB>
__device__ __forceinline__ void wgmma_rs_n(float (&d)[MB / 2], const uint32_t (&a)[4], uint64_t db, int scale_d) {
  if constexpr (MB == 16) wgmma_m64n16k16_rs(d, a, db, scale_d);
  else if constexpr (MB == 32) wgmma_m64n32k16_rs(d, a, db, scale_d);
  else if constexpr (MB == 48) wgmma_m64n48k16_rs(d, a, db, scale_d);
  else wgmma_m64n64k16_rs(d, a, db, scale_d);
}

template <int EPI, int MB, bool FP8 = false>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_smallm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmA, const SmArgs g) {
  constexpr int R = RowGroups<EPI>::R;                         // MMA row groups per tile
  constexpr int WBOX = R == 2 ? 2 * WROWS : WROWS;             // W rows per TMA box (a box dimension is at most 256)
  constexpr int NBOX = R * WROWS / WBOX;
  constexpr int W_STAGE = FP8 ? R * FP8_BLOCK : R * WROWS * BK * 2;
  constexpr int A_STAGE = MB * BK * 2;
  constexpr int ACC_COLS = R * MB;                             // fp32 columns of one accumulator
  extern __shared__ __align__(1024) uint8_t smem[];
  const int NST = g.n_stages, KB = g.KB;
  uint8_t* smW = smem;
  uint8_t* smA = smem + NST * W_STAGE;
  float* stg = reinterpret_cast<float*>(smA + NST * A_STAGE);  // [ACC_COLS][STG_LD]: accumulator of the current range
  uint64_t* full = reinterpret_cast<uint64_t*>(stg + ACC_COLS * STG_LD);
  uint64_t* empty = full + MAXST;
  int* flag = reinterpret_cast<int*>(empty + MAXST);

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  pdl_launch_dependents();
  if ((smem_u32(smem) & 1023u) != 0) __trap();

  if (threadIdx.x == 0) {
    if constexpr (!FP8) tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmA);
    for (int i = 0; i < MAXST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  const uint32_t total = (uint32_t)g.n_tiles * KB, parts = gridDim.x;
  const int it_begin = (int)range_start(blockIdx.x, total, parts), it_end = (int)range_start(blockIdx.x + 1, total, parts);
  const int n_it = it_end - it_begin;
  const uint32_t STAGE_TX = (uint32_t)(W_STAGE + A_STAGE);

  if (wg == 0) {
    // ------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (tid == 0) {
      const int tile_b = it_begin / KB, kb_b = it_begin - tile_b * KB;
      const int pre = min(NST, n_it);
      int tile = tile_b, kb = kb_b;
      for (int i = 0; i < pre; ++i) {                         // weights first: they do not depend on the previous kernel
        mbar_arrive_expect_tx(&full[i], STAGE_TX);
        if constexpr (FP8) {
          bulk_load(smW + i * W_STAGE, g.Wq + (size_t)(it_begin + i) * W_STAGE, W_STAGE, &full[i]);
        } else {
#pragma unroll
          for (int bx = 0; bx < NBOX; ++bx) tma_load_2d(smW + i * W_STAGE + bx * (WBOX * BK * 2), &tmW, &full[i], kb * BK, tile * (R * WROWS) + bx * WBOX);
        }
        if (++kb == KB) { kb = 0; ++tile; }
      }
      pdl_wait();
      tile = tile_b; kb = kb_b;
      for (int i = 0; i < pre; ++i) {
        tma_load_2d(smA + i * A_STAGE, &tmA, &full[i], kb * BK, 0);
        if (++kb == KB) { kb = 0; ++tile; }
      }
      int stage = pre == NST ? 0 : pre; uint32_t phase = pre == NST ? 1 : 0;
      for (int i = pre; i < n_it; ++i) {
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full[stage], STAGE_TX);
        if constexpr (FP8) {
          bulk_load(smW + stage * W_STAGE, g.Wq + (size_t)(it_begin + i) * W_STAGE, W_STAGE, &full[stage]);
        } else {
#pragma unroll
          for (int bx = 0; bx < NBOX; ++bx) tma_load_2d(smW + stage * W_STAGE + bx * (WBOX * BK * 2), &tmW, &full[stage], kb * BK, tile * (R * WROWS) + bx * WBOX);
        }
        tma_load_2d(smA + stage * A_STAGE, &tmA, &full[stage], kb * BK, 0);
        if (++kb == KB) { kb = 0; ++tile; }
        if (++stage == NST) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ------------------------------------------------ consumers: MMA, then epilogue / stream-K fix-up
    setmaxnreg_inc<232>();
    pdl_wait();
    const int cw = wg - 1, warp = tid >> 5, lane = tid & 31;
    const int row = tid;                                      // epilogue: W row inside the row group == output column inside the tile
    const int slot_floats = ACC_COLS * WROWS;
    float acc[R][MB / 2];
    int stage = 0; uint32_t phase = 0;
    int it = it_begin;
    const int my_first_tile = it_begin / KB;
    while (it < it_end) {
      const int tile = it / KB, k0 = it - tile * KB;
      const int k1 = min(KB, k0 + (it_end - it));
      const bool whole = k0 == 0 && k1 == KB;
      int prev = -1;
      for (int kb = k0; kb < k1; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t b0 = smem_u32(smA + stage * A_STAGE);
        if constexpr (FP8) {
          uint32_t af[R][BK / UK][4];
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const uint8_t* q = smW + stage * W_STAGE + r * FP8_BLOCK + cw * 4096 + warp * 1024 + lane * 16;
            const uint4 h0 = *reinterpret_cast<const uint4*>(q), h1 = *reinterpret_cast<const uint4*>(q + 512);
            e4m3x4_to_bf16x2(h0.x, af[r][0][0], af[r][0][1]); e4m3x4_to_bf16x2(h0.y, af[r][0][2], af[r][0][3]);
            e4m3x4_to_bf16x2(h0.z, af[r][1][0], af[r][1][1]); e4m3x4_to_bf16x2(h0.w, af[r][1][2], af[r][1][3]);
            e4m3x4_to_bf16x2(h1.x, af[r][2][0], af[r][2][1]); e4m3x4_to_bf16x2(h1.y, af[r][2][2], af[r][2][3]);
            e4m3x4_to_bf16x2(h1.z, af[r][3][0], af[r][3][1]); e4m3x4_to_bf16x2(h1.w, af[r][3][2], af[r][3][3]);
          }
          wgmma_fence();
#pragma unroll
          for (int r = 0; r < R; ++r)
#pragma unroll
            for (int k = 0; k < BK / UK; ++k) wgmma_rs_n<MB>(acc[r], af[r][k], wgmma_desc_k_sw128(b0 + k * 32), (kb != k0 || k != 0));
        } else {
          wgmma_fence();
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const uint32_t a0 = smem_u32(smW + stage * W_STAGE + r * (WROWS * BK * 2) + cw * 64 * 128);
#pragma unroll
            for (int k = 0; k < BK / UK; ++k)
              wgmma_ss_n<MB>(acc[r], wgmma_desc_k_sw128(a0 + k * 32), wgmma_desc_k_sw128(b0 + k * 32), (kb != k0 || k != 0));
          }
        }
        wgmma_commit();
        // FP8: the next k-block's conversion rewrites the A fragment registers, which an unfinished register-A wgmma may
        // still read (undefined in PTX; at the gate's register pressure it gave wrong and launch-dependent sums): wait for it
        if constexpr (FP8) wgmma_wait<0>();
        else wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == NST) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int r = 0; r < R; ++r) wgmma_fence_regs(acc[r]);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      // fragments -> stg[r * MB + b][W row]
      {
        const int wr = cw * 64 + warp * 16 + (lane >> 2), bq = 2 * (lane & 3);
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
          for (int i = 0; i < MB / 8; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) stg[(r * MB + 8 * i + bq + (e & 1)) * STG_LD + wr + 8 * (e >> 1)] = acc[r][4 * i + e];
      }
      named_bar_sync(1, 256);
      const long long n = (long long)tile * WROWS + row;      // output column (gate: of the N/2-wide output)
      float bias = 0.f;
      if constexpr (EPI == EVO_EPI_BIAS || EPI == EVO_EPI_BIAS_RESID) bias = __bfloat162float(g.bias[n]);
      float s0 = 1.f, s1 = 1.f;                               // FP8: 2^e of the column's W row (gate: of its l1 and l2 rows)
      if constexpr (FP8) {
        s0 = pow2f(g.Wexp[(long long)tile * R * WROWS + row]);
        if constexpr (R >= 2) s1 = pow2f(g.Wexp[(long long)tile * R * WROWS + WROWS + row]);
      }
      if (whole) {
        for (int c = cw * 16; c < MB; c += 32) {
          float rv[16], v0[16], v1[16];
          load_resid16<EPI>(g, n, c, rv);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            v0[j] = stg[(c + j) * STG_LD + row];
            v1[j] = R >= 2 ? stg[(MB + c + j) * STG_LD + row] : 0.f;
            if constexpr (FP8) { v0[j] *= s0; v1[j] *= s1; }
          }
          finalize16<EPI>(g, n, c, bias, rv, v0, v1);
        }
      } else {
        float* slot = g.slots + (size_t)(2 * blockIdx.x + (tile == my_first_tile ? 0 : 1)) * slot_floats;
        for (int c = cw * 16; c < ACC_COLS; c += 32)
#pragma unroll
          for (int j = 0; j < 16; ++j) slot[(c + j) * WROWS + row] = stg[(c + j) * STG_LD + row];
      }
      named_bar_sync(1, 256);                                 // stg is free for the next range
      if (!whole) {
        // publication: the barrier above orders every thread's partial stores before thread 0's acq_rel atomic (release
        // is cumulative), whose acquire half orders the finisher's slot reads after the other contributors' releases
        const int c_first = cta_of((uint32_t)tile * KB, total, parts), c_last = cta_of((uint32_t)(tile + 1) * KB - 1, total, parts);
        if (threadIdx.x == 128) {
          int old;
          asm volatile("atom.add.acq_rel.gpu.global.s32 %0, [%1], 1;" : "=r"(old) : "l"(g.counters + tile) : "memory");
          *flag = old;
        }
        named_bar_sync(1, 256);
        const bool last = *flag == c_last - c_first;
        if (last) {
          for (int c = cw * 16; c < MB; c += 32) {
            float v0[16], v1[16], rv[16];
            load_resid16<EPI>(g, n, c, rv);
#pragma unroll
            for (int j = 0; j < 16; ++j) { v0[j] = 0.f; v1[j] = 0.f; }
            // slots are summed in contributor order (deterministic); the loads of FX contributors are in flight together
            constexpr int FX = R == 2 ? 2 : 4;
            for (int cb = c_first; cb <= c_last; cb += FX) {
              float t0v[FX][16], t1v[FX][16];
#pragma unroll
              for (int u = 0; u < FX; ++u) {
                const int cc = min(cb + u, c_last);
                const int first_tile_cc = (int)(range_start((uint32_t)cc, total, parts) / (uint32_t)KB);
                const float* s = g.slots + (size_t)(2 * cc + (first_tile_cc == tile ? 0 : 1)) * slot_floats;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                  t0v[u][j] = __ldcg(s + (c + j) * WROWS + row);
                  if constexpr (R >= 2) t1v[u][j] = __ldcg(s + (MB + c + j) * WROWS + row);
                }
              }
#pragma unroll
              for (int u = 0; u < FX; ++u) {
                if (cb + u <= c_last) {
#pragma unroll
                  for (int j = 0; j < 16; ++j) { v0[j] += t0v[u][j]; if constexpr (R >= 2) v1[j] += t1v[u][j]; }
                }
              }
            }
            if constexpr (FP8) {
#pragma unroll
              for (int j = 0; j < 16; ++j) { v0[j] *= s0; v1[j] *= s1; }
            }
            finalize16<EPI>(g, n, c, bias, rv, v0, v1);
          }
          if (threadIdx.x == 128) g.counters[tile] = 0;      // self-cleaning for the next launch
        }
        named_bar_sync(1, 256);                               // *flag is reused by the next range
      }
      it += k1 - k0;
    }
  }
}

template <int EPI, int MB, bool FP8>
int launch(const evo_gemm_smallm_params* p, const void* w_exp, cudaStream_t st) {
  constexpr int R = RowGroups<EPI>::R;
  CUtensorMap tmW, tmA;
  int rc;
  if constexpr (FP8) memset(&tmW, 0, sizeof(tmW));            // the FP8 form streams W by 1-D bulk copies
  else if ((rc = make_tmap_2d_bf16(&tmW, p->W, (uint64_t)p->K, (uint64_t)p->N, (uint64_t)p->K * 2, BK, R == 2 ? 2 * WROWS : WROWS, true))) return rc;
  if ((rc = make_tmap_2d_bf16(&tmA, p->A, (uint64_t)p->K, (uint64_t)p->M, (uint64_t)p->lda * 2, BK, (uint32_t)MB, true))) return rc;
  SmArgs g;
  g.Wq = (const uint8_t*)p->W; g.Wexp = (const int8_t*)w_exp;
  g.C = (bf16*)p->C; g.ldc = p->ldc; g.bias = (const bf16*)p->bias; g.resid = (const bf16*)p->residual; g.ldr = p->ldr;
  g.M = (int)p->M; g.Mb = MB;
  g.n_tiles = (int)(p->N / (R * WROWS));
  g.KB = (int)(p->K / BK);
  const int stage_bytes = (FP8 ? R * FP8_BLOCK : R * WROWS * BK * 2) + MB * BK * 2;
  const int tail = R * MB * STG_LD * 4 + 2 * MAXST * 8 + 16;
  const int budget = std::min(RING_BYTES, 227 * 1024 - tail);
  g.n_stages = std::max(2, std::min(MAXST, budget / stage_bytes));
  const int smem_bytes = g.n_stages * stage_bytes + tail;
  const long long total = (long long)g.n_tiles * g.KB;
  EVO_REQUIRE(total * device_sm_count() < (1LL << 31), "evo_gemm_smallm: N * K too large (%lld k-block iterations)", total);
  // one range per SM, but at least 8 k-blocks per range (bounds the contributors per tile for tiny layers)
  const int grid = (int)std::max<long long>(1, std::min<long long>(device_sm_count(), total / 8));
  const size_t need = evo_gemm_smallm_workspace(p->M, p->N, p->K, p->epilogue);
  EVO_REQUIRE(p->workspace != nullptr && p->workspace_bytes >= need, "evo_gemm_smallm: workspace too small (%zu < %zu)", p->workspace_bytes, need);
  g.counters = (int*)p->workspace;
  g.slots = (float*)((uint8_t*)p->workspace + 16384);
  static unsigned long long attr_done = 0;
  auto kern = gemm_smallm_kernel<EPI, MB, FP8>;
  { int rc_ = ensure_dyn_smem(kern, 227 * 1024, attr_done); if (rc_) return rc_; }
  EVO_CUDA(launch_pdl_at(1, kern, dim3(grid), dim3(NTHREADS), smem_bytes, st, tmW, tmA, g));
  return check_launch(FP8 ? "evo_gemm_smallm_fp8" : "evo_gemm_smallm");
}

template <int EPI, bool FP8>
int launch_mb(const evo_gemm_smallm_params* p, const void* w_exp, cudaStream_t st) {
  switch ((p->M + 15) / 16) {
    case 1: return launch<EPI, 16, FP8>(p, w_exp, st);
    case 2: return launch<EPI, 32, FP8>(p, w_exp, st);
    case 3: return launch<EPI, 48, FP8>(p, w_exp, st);
    default: return launch<EPI, 64, FP8>(p, w_exp, st);
  }
}

// the argument checks of both forms, under the entry point's name
int check_smallm(const char* what, const evo_gemm_smallm_params* p) {
  EVO_REQUIRE(p->M >= 0 && p->M <= MAX_MB, "%s: M (%lld) must be in [0, %d]", what, (long long)p->M, MAX_MB);
  EVO_REQUIRE(p->N > 0 && p->K > 0 && p->K % BK == 0, "%s: K (%lld) must be a positive multiple of %d", what, (long long)p->K, BK);
  EVO_REQUIRE(p->N % 256 == 0 && p->N / WROWS <= 4096, "%s: N (%lld) must be a multiple of 256 (and <= 524288)", what, (long long)p->N);
  EVO_REQUIRE(p->lda % 8 == 0, "%s: lda must be a multiple of 8 elements", what);
  EVO_REQUIRE(((uintptr_t)p->A % 16) == 0 && ((uintptr_t)p->W % 16) == 0, "%s: A and W must be 16-byte aligned", what);
  if (p->epilogue == EVO_EPI_BIAS || p->epilogue == EVO_EPI_BIAS_RESID) EVO_REQUIRE(p->bias != nullptr, "%s: bias epilogue without bias", what);
  if (p->epilogue == EVO_EPI_RESID || p->epilogue == EVO_EPI_BIAS_RESID) EVO_REQUIRE(p->residual != nullptr, "%s: residual epilogue without residual", what);
  return 0;
}

template <bool FP8>
int dispatch(const char* what, const evo_gemm_smallm_params* p, const void* w_exp, cudaStream_t st) {
  switch (p->epilogue) {
    case EVO_EPI_NONE: return launch_mb<EVO_EPI_NONE, FP8>(p, w_exp, st);
    case EVO_EPI_BIAS: return launch_mb<EVO_EPI_BIAS, FP8>(p, w_exp, st);
    case EVO_EPI_BIAS_RESID: return launch_mb<EVO_EPI_BIAS_RESID, FP8>(p, w_exp, st);
    case EVO_EPI_RESID: return launch_mb<EVO_EPI_RESID, FP8>(p, w_exp, st);
    case EVO_EPI_GELU_GATE: return launch_mb<EVO_EPI_GELU_GATE, FP8>(p, w_exp, st);
  }
  set_error("%s: unknown epilogue %d", what, p->epilogue);
  return -1;
}

// ---- quantizer of the FP8 decode weights
// e[n] = ceil(log2(amax_n / 448)), at least -124 (so that every q 2^e is a bf16 number and 2^e a normal fp32 one); 0 for an all-zero
// row.  amax = m 2^p with m in [0.5, 1) and 448 = 0.875 2^9: amax / 448 lies in (2^(p-10), 2^(p-9)] when m <= 0.875.
__global__ void fp8_row_exp_kernel(const bf16* __restrict__ W, int K, int8_t* __restrict__ w_exp, int* status) {
  const long long n = blockIdx.x;
  float amax = 0.f;
  bool bad = false;
  for (int k = threadIdx.x * 8; k < K; k += blockDim.x * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(W + n * K + k);
    const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = fabsf(bf_lo(w4[j])), b = fabsf(bf_hi(w4[j]));
      bad |= !(a <= 3.0e38f) || !(b <= 3.0e38f);
      amax = fmaxf(amax, fmaxf(a, b));
    }
  }
  __shared__ float red[32];
  __shared__ int red_bad[32];
  for (int o = 16; o; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  bad = __any_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = amax; red_bad[threadIdx.x >> 5] = bad; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) { amax = fmaxf(amax, red[i]); bad |= red_bad[i] != 0; }
    int e = 0;
    if (amax > 0.f) {
      int p;
      const float m = frexpf(amax, &p);
      e = max(m <= 0.875f ? p - 9 : p - 8, -124);
    }
    w_exp[n] = (int8_t)e;
    if (bad) atomicOr(status, 1);
  }
}

// one thread per 16 bytes of the layout: q = E4M3(w 2^-e) (round to nearest even; |w 2^-e| <= 448), W' = q 2^e over w in place.
// Does nothing when any weight of the matrix was not finite.
__global__ void fp8_quantize_kernel(bf16* W, long long K, int KB, int R, const int8_t* __restrict__ w_exp, uint8_t* __restrict__ q,
                                    const int* status, long long n_chunks) {
  if (*status) return;
  for (long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x; c < n_chunks; c += (long long)gridDim.x * blockDim.x) {
    // chunk c = (block of R*8192 bytes, r, warpgroup, warp, half, lane), the FP8 decode layout
    const long long blk = c / (R * 512);
    int rem = (int)(c - blk * R * 512);
    const int r = rem / 512, cw = (rem / 256) % 2, warp = (rem / 64) % 4, h = (rem / 32) % 2, lane = rem % 32;
    const long long tile = blk / KB;
    const int kb = (int)(blk - tile * KB);
    uint32_t out[4];
#pragma unroll
    for (int b = 0; b < 16; b += 2) {
      const int ks = 2 * h + b / 8, reg = (b % 8) / 2;
      const long long n = tile * R * WROWS + r * WROWS + cw * 64 + warp * 16 + (reg % 2) * 8 + lane / 4;
      const long long k = (long long)kb * BK + ks * UK + (reg / 2) * 8 + (lane % 4) * 2;
      const int e = w_exp[n];
      bf16* wp = W + n * K + k;
      const uint32_t wv = *reinterpret_cast<const uint32_t*>(wp);
      const float inv = pow2f(-e), sc = pow2f(e);
      __nv_fp8x2_storage_t q2 = __nv_cvt_float2_to_fp8x2(make_float2(bf_lo(wv) * inv, bf_hi(wv) * inv), __NV_SATFINITE, __NV_E4M3);
      // the conversion returns +0 for a negative value that rounds to zero; round to nearest keeps the sign (-0)
      if ((q2 & 0x007f) == 0 && (wv & 0x8000u)) q2 |= 0x0080;
      if ((q2 & 0x7f00) == 0 && (wv & 0x80000000u)) q2 |= 0x8000;
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2(q2, __NV_E4M3);
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
      *reinterpret_cast<uint32_t*>(wp) = pack_bf16(f.x * sc, f.y * sc);
      const uint32_t q16 = (uint32_t)q2;
      if (b % 4 == 0) out[b / 4] = q16; else out[b / 4] |= q16 << 16;
    }
    *reinterpret_cast<uint4*>(q + c * 16) = make_uint4(out[0], out[1], out[2], out[3]);
  }
}

// dequantizer of the FP8 decode weights: W' = q 2^e, row-major, from the layout fp8_quantize_kernel wrote, through that kernel's
// conversion and scaling (so the bits are those it left in W).  One CTA per (tile, k-block) block of R * 8192 bytes: the block is
// read whole with 16-byte loads into shared memory; then each thread gathers 8 consecutive columns of one row (the pair of bytes
// at the same place in four consecutive 16-byte chunks: lanes 4j .. 4j + 3 of the fragment layout) and stores them as one
// 16-byte segment, so a warp writes four whole 128-byte row pieces.
constexpr int DQ_THREADS = 256;

__global__ void __launch_bounds__(DQ_THREADS) fp8_dequant_kernel(const uint8_t* __restrict__ q, const int8_t* __restrict__ w_exp,
                                                                 bf16* __restrict__ W, long long K, int KB, int R) {
  __shared__ __align__(16) uint8_t blk[2 * FP8_BLOCK];
  const long long b = blockIdx.x, tile = b / KB;
  const int kb = (int)(b - tile * KB);
  const uint4* src = reinterpret_cast<const uint4*>(q + b * (long long)(R * FP8_BLOCK));
  for (int c = threadIdx.x; c < R * FP8_BLOCK / 16; c += DQ_THREADS) reinterpret_cast<uint4*>(blk)[c] = src[c];
  __syncthreads();
  for (int s = threadIdx.x; s < R * WROWS * (BK / 8); s += DQ_THREADS) {
    // row nr of the tile = (r, warpgroup, warp, register % 2, lane / 4); columns 8 seg .. 8 seg + 7 = (k16 step, register / 2)
    const int nr = s / (BK / 8), seg = s % (BK / 8);
    const int r = nr / WROWS, rr = nr % WROWS;
    const int cw = rr / 64, warp = (rr % 64) / 16, reg = 2 * (seg % 2) + (rr % 16) / 8, ks = seg / 2;
    const int at = (r * 512 + cw * 256 + warp * 64 + (ks / 2) * 32 + (rr % 8) * 4) * 16 + (ks % 2) * 8 + reg * 2;
    const long long n = tile * R * WROWS + nr;
    const float sc = pow2f(w_exp[n]);
    uint32_t out[4];
#pragma unroll
    for (int l = 0; l < 4; ++l) {                            // lane % 4 = l: columns 2l, 2l + 1 of the segment
      const __nv_fp8x2_storage_t q2 = *reinterpret_cast<const __nv_fp8x2_storage_t*>(blk + at + l * 16);
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2(q2, __NV_E4M3);
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
      out[l] = pack_bf16(f.x * sc, f.y * sc);
    }
    *reinterpret_cast<uint4*>(W + n * K + (long long)kb * BK + seg * 8) = make_uint4(out[0], out[1], out[2], out[3]);
  }
}

}  // namespace

extern "C" size_t evo_gemm_smallm_workspace(int64_t M, int64_t N, int64_t K, int epilogue) {
  (void)K;
  const int R = epilogue == EVO_EPI_GELU_GATE ? 2 : 1;
  const size_t Mb = (size_t)((M + 15) / 16 * 16);
  if (N / (R * WROWS) > 4096) return 0;
  return 16384 + (size_t)2 * device_sm_count() * R * Mb * WROWS * sizeof(float);
}

extern "C" int evo_gemm_smallm(const evo_gemm_smallm_params* p, void* stream) {
  if (check_smallm("evo_gemm_smallm", p)) return -1;
  if (p->M == 0) return 0;
  return dispatch<false>("evo_gemm_smallm", p, nullptr, (cudaStream_t)stream);
}

extern "C" int evo_gemm_smallm_fp8(const evo_gemm_smallm_fp8_params* p, void* stream) {
  if (check_smallm("evo_gemm_smallm_fp8", &p->base)) return -1;
  EVO_REQUIRE(p->W_exp != nullptr, "evo_gemm_smallm_fp8: W_exp is required");
  if (p->base.M == 0) return 0;
  return dispatch<true>("evo_gemm_smallm_fp8", &p->base, p->W_exp, (cudaStream_t)stream);
}

extern "C" size_t evo_fp8_weight_bytes(int64_t N, int64_t K, int epilogue) {
  const int R = epilogue == EVO_EPI_GELU_GATE ? 2 : 1;
  if (N <= 0 || K <= 0 || K % BK != 0 || N % (R * WROWS) != 0) {
    set_error("evo_fp8_weight_bytes: needs K a positive multiple of %d and N a positive multiple of %d (N %lld, K %lld)", BK, R * WROWS,
              (long long)N, (long long)K);
    return 0;
  }
  return (size_t)N * (size_t)K;
}

extern "C" int evo_fp8_quantize_rows(void* W, int64_t N, int64_t K, int epilogue, void* W_q, void* W_exp, int* status, void* stream) {
  EVO_REQUIRE(evo_fp8_weight_bytes(N, K, epilogue) != 0, "evo_fp8_quantize_rows: needs K a positive multiple of %d and N a positive multiple of %d "
              "(N %lld, K %lld)", BK, epilogue == EVO_EPI_GELU_GATE ? 2 * WROWS : WROWS, (long long)N, (long long)K);
  EVO_REQUIRE(N <= (1LL << 31) - 1, "evo_fp8_quantize_rows: N (%lld) too large", (long long)N);
  EVO_REQUIRE(W != nullptr && W_q != nullptr && W_exp != nullptr && status != nullptr, "evo_fp8_quantize_rows: W, W_q, W_exp and status are required");
  EVO_REQUIRE(((uintptr_t)W % 16) == 0 && ((uintptr_t)W_q % 16) == 0, "evo_fp8_quantize_rows: W and W_q must be 16-byte aligned");
  const cudaStream_t st = (cudaStream_t)stream;
  const int R = epilogue == EVO_EPI_GELU_GATE ? 2 : 1;
  EVO_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  fp8_row_exp_kernel<<<(unsigned)N, 256, 0, st>>>((const bf16*)W, (int)K, (int8_t*)W_exp, status);
  if (int rc = check_launch("evo_fp8_quantize_rows")) return rc;
  const long long n_chunks = N * K / 16;
  const int grid = (int)std::min<long long>((n_chunks + 255) / 256, 64LL * std::max(1, device_sm_count()));
  fp8_quantize_kernel<<<grid, 256, 0, st>>>((bf16*)W, K, (int)(K / BK), R, (const int8_t*)W_exp, (uint8_t*)W_q, status, n_chunks);
  return check_launch("evo_fp8_quantize_rows");
}

extern "C" int evo_fp8_dequant_rows(const void* W_q, const void* W_exp, int64_t N, int64_t K, int epilogue, void* W_out, void* stream) {
  EVO_REQUIRE(evo_fp8_weight_bytes(N, K, epilogue) != 0, "evo_fp8_dequant_rows: needs K a positive multiple of %d and N a positive multiple of %d "
              "(N %lld, K %lld)", BK, epilogue == EVO_EPI_GELU_GATE ? 2 * WROWS : WROWS, (long long)N, (long long)K);
  EVO_REQUIRE(N <= (1LL << 31) - 1 && N / WROWS * (K / BK) <= (1LL << 31) - 1, "evo_fp8_dequant_rows: N * K (%lld x %lld) too large",
              (long long)N, (long long)K);
  EVO_REQUIRE(W_q != nullptr && W_exp != nullptr && W_out != nullptr, "evo_fp8_dequant_rows: W_q, W_exp and W_out are required");
  EVO_REQUIRE(((uintptr_t)W_q % 16) == 0 && ((uintptr_t)W_out % 16) == 0, "evo_fp8_dequant_rows: W_q and W_out must be 16-byte aligned");
  const int R = epilogue == EVO_EPI_GELU_GATE ? 2 : 1;
  const long long blocks = N / (R * WROWS) * (K / BK);
  fp8_dequant_kernel<<<(unsigned)blocks, DQ_THREADS, 0, (cudaStream_t)stream>>>((const uint8_t*)W_q, (const int8_t*)W_exp, (bf16*)W_out, K,
                                                                                 (int)(K / BK), R);
  return check_launch("evo_fp8_dequant_rows");
}
