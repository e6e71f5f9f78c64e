// Tensor-core linear layers for sm_90a: C[M,N] = epilogue(A[M,K] . W[N,K]^T).
//
// Persistent, warp-specialised wgmma kernel, one CTA per SM walking 128 x BN output tiles:
//   warpgroup 0      TMA producer  (one thread: cp.async.bulk.tensor, 128B-swizzled K-major tiles, mbarrier ring)
//   warpgroups 1-2   consumers     (64 rows each: wgmma.mma_async m64nBNk16, fp32 accumulators in registers,
//                                   then the fused epilogue straight from the accumulator fragments)
// The producer runs ahead into the next tile while the consumers finish the epilogue of the current one.  On the 256-column
// tile the consumers stage C in shared memory and hand it to TMA stores that drain behind the next tile's MMAs.
//
// BN = 256: the throughput tile (variants 0 and 1).  BN = 64: the small-M weight-streaming tile (variants 2 and 3;
// variant 3 reads W tile-major, [N/64][K/64][64][64]), N/64 CTAs keep every SM pulling weights.
//
// Epilogues reproduce the reference's bf16 rounding points (include/evo_b200.h) through the chain helpers of common.cuh.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/evo_b200.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>

using namespace evo;

namespace {

constexpr int BM = 128;            // rows of C per tile (two consumer warpgroups of 64)
constexpr int BN_BIG = 256;        // columns of C per tile for the throughput tiles
constexpr int BN_SMALL = 64;       // weight-streaming tiles for small M (decode)
constexpr int BK = 64;             // bf16 elements per k-block = one 128-byte swizzle row
constexpr int UK = 16;             // wgmma K for 16-bit inputs
constexpr int NTHREADS = 384;
constexpr int CONSUMER_WARPS = 8;

// TMA-store epilogue (256-column tile): each consumer warpgroup stages its 64 rows in two 128-column halves of its own, each
// two 128B-swizzled 64 x 64 boxes (the swizzle caps a box row at 64 bf16): 64 KB for the two warpgroups.
constexpr int EPI_BOX_BYTES = 64 * 64 * 2;
constexpr int EPI_HALF_BYTES = 2 * EPI_BOX_BYTES;

template <int BN, bool TMA_C = false> struct Cfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // 192 KB of ring for the direct-store kernels; the TMA-store kernel gives a fourth stage to the staging (measured faster
  // than 4 stages with one 16 KB staging half per warpgroup: DESIGN 3.2)
  static constexpr int STAGES = BN == BN_SMALL ? 8 : (TMA_C ? 3 : 4);
  static constexpr int STAGING_BYTES = TMA_C ? 4 * EPI_HALF_BYTES : 0;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

struct GemmArgs {
  bf16* C; long long ldc;
  const bf16* bias;
  const bf16* resid; long long ldr;
  long long M, N, K;
  int m_blocks, n_blocks, group_m;
  int b_tiled;           // small-M tile only: W is tile-major [N/64][K/64][64][64] (contiguous 8 KB tiles: every DRAM page opened is fully used)
  // peer-scattered output (sequence-parallel Ulysses re-shard fused into the Wqkv epilogue): column n of row m goes to
  // c_peer[(n % peer_period) / peer_inner] at [(peer_row0 + m) * ldc + (n / peer_period) * peer_inner + n % peer_inner]
  bf16* c_peer[8]; int n_peers; int peer_period, peer_inner; long long peer_row0;
  const bf16* rope_cos; const bf16* rope_sin;   // EVO_EPI_BIAS_ROPE: (positions, 64) bf16 tables, row l = position of token row l
  long long rope_L, rope_cols;                  //   rows repeat with period rope_L (tokens per sequence); columns < rope_cols (q and k) are rotated
  const long long* targets;   // EPI_LSE only: (M) target token per row (-1: none)
  float4* part;               // EPI_LSE only: (M, n_blocks) per-row partial statistics {max, sum e^(x-max), sum e^(x-max) x, target logit}
  int raster_n;          // 0: groups of `group_m` row-blocks sweep all of N (A stays in L2); 1: groups of `group_m` column-blocks sweep all of M (W stays in L2)
};

constexpr int EPI_LSE = 5;     // internal: scoring epilogue (evo_unembed_score); no C is written (EVO_EPI_BIAS_ROPE is 6)

// grouped rasterisation: GROUP_M row-blocks share the sweep over n so their A tiles stay in L2
__device__ __forceinline__ void tile_coords(int tile, const GemmArgs& g, int& m_blk, int& n_blk) {
  const int major = g.raster_n ? g.n_blocks : g.m_blocks;     // the grouped dimension
  const int minor = g.raster_n ? g.m_blocks : g.n_blocks;     // the swept dimension
  int per_group = g.group_m * minor;
  int grp = tile / per_group;
  int first = grp * g.group_m;
  int gsz = min(g.group_m, major - first);
  int in = tile - grp * per_group;
  int a = first + in % gsz, b = in / gsz;
  m_blk = g.raster_n ? b : a;
  n_blk = g.raster_n ? a : b;
}

// address of C[row, col] (four adjacent columns from a multiple of 4 never straddle a head)
__device__ __forceinline__ bf16* c_ptr(const GemmArgs& g, long long row, int col) {
  if (g.n_peers == 0) return g.C + row * g.ldc + col;
  const int t = col / g.peer_period, rem = col - t * g.peer_period;
  const int p = rem / g.peer_inner;
  return g.c_peer[p] + (g.peer_row0 + row) * g.ldc + t * g.peer_inner + (rem - p * g.peer_inner);
}

// columns (col, col + 1) of one row
template <bool BIAS, bool RESID>
__device__ __forceinline__ void store_pair(const GemmArgs& g, long long row, int col, float v0, float v1) {
  *reinterpret_cast<uint32_t*>(c_ptr(g, row, col)) =
      linear_word<BIAS, RESID>(v0, v1, BIAS ? ld_pair(g.bias + col) : 0u, [&] { return ld_pair(g.resid + row * g.ldr + col); });
}

// Quad exchange for full-sector stores.  Lane q of a quad holds bf16 pairs `lo` (columns 8i + 2q + {0, 1}) and `hi` (columns
// 8(i+1) + 2q + {0, 1}) of one row.  One shuffle leaves every lane four adjacent columns: even lanes 8i + 2q + {0..3}, odd lanes
// 8(i+1) + 2(q-1) + {0..3} (`quad_cols` gives the offset from 8i).  A warp then writes each of its 8 rows as one whole 32-byte
// sector with 8-byte stores, instead of two half-filled sectors with 4-byte stores.  Every lane of the warp must call it.
__device__ __forceinline__ int quad_cols(int quad) { return (quad & 1) ? 8 + 2 * (quad - 1) : 2 * quad; }
__device__ __forceinline__ uint2 quad_pair(uint32_t lo, uint32_t hi, int quad) {
  const bool odd = quad & 1;
  const uint32_t got = __shfl_xor_sync(0xffffffffu, odd ? lo : hi, 1);
  return odd ? make_uint2(got, hi) : make_uint2(lo, got);
}
__device__ __forceinline__ void st_quad(bf16* p, uint2 v) { *reinterpret_cast<uint2*>(p) = v; }

// fold (m2, s2, w2) into (m, s, w): running max, sum e^(x-max), sum e^(x-max) x
__device__ __forceinline__ void lse_merge(float& m, float& s, float& w, float m2, float s2, float w2) {
  const float M = fmaxf(m, m2);
  const float a = m == -INFINITY ? 0.f : __expf(m - M), b = m2 == -INFINITY ? 0.f : __expf(m2 - M);
  s = s * a + s2 * b; w = w * a + w2 * b; m = M;
}

// byte offset of the bf16 pair (r, c), c even, in a staged 64 x 128 half: box c / 64, 128 B rows whose 16-byte chunks are
// XOR-swizzled by r % 8 (the TMA SWIZZLE_128B layout).  The 8 rows a warp writes per column pair fall in 8 distinct chunks.
__device__ __forceinline__ int stage_off(int r, int c) {
  return (c >> 6) * EPI_BOX_BYTES + r * 128 + ((((c >> 3) & 7) ^ (r & 7)) << 4) + (c & 7) * 2;
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// TMA_C: the C-writing epilogues of the 256-column tile go through shared memory and TMA stores (tmC), and the residual
// arrives by TMA (tmR).  Otherwise every thread stores its fragments itself (the small-M tile, the scoring statistics and the
// peer-scattered output, whose column -> peer mapping is not one tensor map); tmC and tmR are then unused.
template <int EPI, int BN, bool TMA_C>
__device__ __forceinline__ void gemm_body(const CUtensorMap* tmA, const CUtensorMap* tmB, const CUtensorMap* tmC, const CUtensorMap* tmR,
                                          const GemmArgs& g) {
  using C_ = Cfg<BN, TMA_C>;
  static_assert(EPI != EVO_EPI_GELU_GATE || BN == BN_BIG, "the gate epilogue needs [l1 | l2] halves of a 256-column tile");
  static_assert(!TMA_C || (BN == BN_BIG && EPI != EPI_LSE), "TMA stores: the 256-column tile's C-writing epilogues");
  constexpr bool BIAS = EPI == EVO_EPI_BIAS || EPI == EVO_EPI_BIAS_RESID;
  constexpr bool RESID = EPI == EVO_EPI_BIAS_RESID || EPI == EVO_EPI_RESID;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smA = smem;
  uint8_t* smB = smem + C_::STAGES * C_::A_BYTES;
  uint8_t* staging = smB + C_::STAGES * C_::B_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(staging + C_::STAGING_BYTES);
  uint64_t* empty = full + C_::STAGES;
  uint64_t* rfull = empty + C_::STAGES;     // TMA_C with a residual: one per staging half of each consumer warpgroup

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tmA); tma_prefetch_desc(tmB);
    for (int i = 0; i < C_::STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONSUMER_WARPS); }
    if constexpr (TMA_C && RESID) for (int i = 0; i < 4; ++i) mbar_init(&rfull[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int n_tiles = g.m_blocks * g.n_blocks;
  const int nkb = (int)(g.K / BK);

  if (wg == 0) {
    // ------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (tid == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int m_blk, n_blk; tile_coords(tile, g, m_blk, n_blk);
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], C_::STAGE_BYTES);
          tma_load_2d(smA + stage * C_::A_BYTES, tmA, &full[stage], kb * BK, m_blk * BM);
          if (BN == BN_SMALL && g.b_tiled) tma_load_4d(smB + stage * C_::B_BYTES, tmB, &full[stage], 0, 0, kb, n_blk);
          else tma_load_2d(smB + stage * C_::B_BYTES, tmB, &full[stage], kb * BK, n_blk * BN);
          if (++stage == C_::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------ consumers: mainloop + epilogue
    setmaxnreg_inc<232>();
    const int cw = wg - 1, warp = tid >> 5, lane = tid & 31;
    const int quad = lane & 3;
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    [[maybe_unused]] uint8_t* stg = staging + cw * 2 * EPI_HALF_BYTES;   // this warpgroup's two staging halves
    [[maybe_unused]] uint32_t rphase = 0;                                // parity of rfull, one bit per half
#ifdef EVO_GEMM_NO_STORE
    constexpr bool STORE = false;     // experiment builds only: the epilogue arithmetic without residual loads or C stores
#else
    constexpr bool STORE = true;
#endif
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      int m_blk, n_blk; tile_coords(tile, g, m_blk, n_blk);
      [[maybe_unused]] const int row_g = m_blk * BM + cw * 64;     // first row of this warpgroup's 64
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t a0 = smem_u32(smA + stage * C_::A_BYTES + cw * 64 * 128), b0 = smem_u32(smB + stage * C_::B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / UK; ++k) {     // +32 B per k16 step inside the 128B swizzle row
          if constexpr (BN == BN_BIG) wgmma_m64n256k16_ss(acc, wgmma_desc_k_sw128(a0 + k * 32), wgmma_desc_k_sw128(b0 + k * 32), (kb | k) != 0);
          else                        wgmma_m64n64k16_ss(acc, wgmma_desc_k_sw128(a0 + k * 32), wgmma_desc_k_sw128(b0 + k * 32), (kb | k) != 0);
        }
        wgmma_commit();
        if constexpr (TMA_C) {
          // behind the MMAs of the tile's first k-blocks: wait until the previous tile's stores have read the staging, then
          // fetch this tile's residual into it (rows >= M arrive as zeros)
          if (kb == (nkb > 1 ? 1 : 0) && tid == 0) {
            tma_store_wait_read<0>();
            if constexpr (RESID && STORE) {
              for (int hf = 0; hf < 2; ++hf) {
                uint64_t* bar = &rfull[cw * 2 + hf];
                uint8_t* dst = stg + hf * EPI_HALF_BYTES;
                const int col = n_blk * BN + hf * 128;
                mbar_arrive_expect_tx(bar, EPI_HALF_BYTES);
                tma_load_2d(dst, tmR, bar, col, row_g);
                tma_load_2d(dst + EPI_BOX_BYTES, tmR, bar, col + 64, row_g);
              }
            }
          }
        }
        wgmma_wait<1>();                        // the previous k-block's MMAs are done: its stage can be refilled
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == C_::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

      // thread (warp, lane) holds rows r0 = 16 warp + lane/4 and r0 + 8 of its 64, columns 8i + 2 (lane%4) + {0, 1}
      const long long row0 = (long long)m_blk * BM + cw * 64 + warp * 16 + (lane >> 2);
      if constexpr (TMA_C) {
        // The direct-store epilogues below, written as bf16 pairs into the staging; the TMA store clips rows >= M.  C may
        // alias the residual: each element is read before its own store is issued.
        constexpr int HALVES = EPI == EVO_EPI_GELU_GATE ? 1 : 2;      // the gate tile writes 128 columns
        const int rl0 = warp * 16 + (lane >> 2);
        if constexpr (!(RESID && STORE)) named_bar_sync(1 + cw, 128);  // after tid 0's wait for the previous stores
#pragma unroll
        for (int hf = 0; hf < HALVES; ++hf) {
          uint8_t* buf = stg + hf * EPI_HALF_BYTES;
          if constexpr (RESID && STORE) { mbar_wait(&rfull[cw * 2 + hf], (rphase >> hf) & 1); rphase ^= 1u << hf; }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int rl = rl0 + 8 * h;
            if constexpr (EPI == EVO_EPI_BIAS_ROPE) {
              const bool rotate = (long long)n_blk * BN + 128 * hf < g.rope_cols;     // per 128-column head
              const long long l = row0 + 8 * h < g.M ? (row0 + 8 * h) % g.rope_L : 0;   // rows >= M: any row in the tables
#pragma unroll
              for (int j = 0; j < 8; ++j) {      // columns c and c + 64 of the head in this half
                const int i = 16 * hf + j, c = 8 * j + 2 * quad, col = n_blk * BN + 128 * hf + c;
                uint32_t o1, o2;
                bias_rope_words(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], acc[4 * (i + 8) + 2 * h], acc[4 * (i + 8) + 2 * h + 1],
                                g.bias, col, rotate, g.rope_cos, g.rope_sin, l, c, o1, o2);
                *reinterpret_cast<uint32_t*>(buf + stage_off(rl, c)) = o1;
                *reinterpret_cast<uint32_t*>(buf + stage_off(rl, c + 64)) = o2;
              }
            } else if constexpr (EPI == EVO_EPI_GELU_GATE) {
#pragma unroll
              for (int i = 0; i < BN / 16; ++i) {
                const float a0 = rbf(acc[4 * i + 2 * h]), a1 = rbf(acc[4 * i + 2 * h + 1]);
                const float b0 = rbf(acc[4 * (i + BN / 16) + 2 * h]), b1 = rbf(acc[4 * (i + BN / 16) + 2 * h + 1]);
                *reinterpret_cast<uint32_t*>(buf + stage_off(rl, 8 * i + 2 * quad)) = pack_bf16(gelu_gate(a0, b0), gelu_gate(a1, b1));
              }
            } else {
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const int i = 16 * hf + j;
                const uint32_t b = BIAS ? ld_pair(g.bias + n_blk * BN + 8 * i + 2 * quad) : 0u;
                uint32_t* p = reinterpret_cast<uint32_t*>(buf + stage_off(rl, 8 * j + 2 * quad));
                *p = linear_word<BIAS, RESID>(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], b, [&] { return *p; });
              }
            }
          }
          fence_proxy_async_smem();           // the staging writes become visible to the TMA unit
          named_bar_sync(1 + cw, 128);
          if (STORE && tid == 0) {
            const int col = EPI == EVO_EPI_GELU_GATE ? n_blk * (BN / 2) : n_blk * BN + 128 * hf;
            tma_store_2d(tmC, buf, col, row_g);
            tma_store_2d(tmC, buf + EPI_BOX_BYTES, col + 64, row_g);
            tma_store_commit();
          }
        }
      } else if constexpr (EPI == EPI_LSE) {
        // scoring epilogue: the 256 logits of this row's half never leave the SM.  Max / sum-exp / sum-exp-times-logit over the
        // bf16-rounded logits (the reference's logits tensor is bf16), plus the target's logit if it is in this half.
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = row0 + 8 * h;
          const long long tgt = row < g.M && g.targets ? g.targets[row] - (long long)n_blk * BN : -1;
          float mx = -INFINITY, s = 0.f, w = 0.f, t_logit = 0.f;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) mx = fmaxf(mx, fmaxf(rbf(acc[4 * i + 2 * h]), rbf(acc[4 * i + 2 * h + 1])));
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float v = rbf(acc[4 * i + 2 * h + e]);
              const float x = __expf(v - mx);
              s += x; w = fmaf(x, v, w);
              if (tgt == 8 * i + 2 * quad + e) t_logit = v;
            }
          }
#pragma unroll
          for (int o = 1; o < 4; o <<= 1) {
            const float m2 = __shfl_xor_sync(0xffffffffu, mx, o), s2 = __shfl_xor_sync(0xffffffffu, s, o), w2 = __shfl_xor_sync(0xffffffffu, w, o);
            t_logit += __shfl_xor_sync(0xffffffffu, t_logit, o);
            lse_merge(mx, s, w, m2, s2, w2);
          }
          if (quad == 0 && row < g.M) g.part[row * g.n_blocks + n_blk] = make_float4(mx, s, w, t_logit);
        }
      } else if constexpr (EPI == EVO_EPI_BIAS_ROPE && BN == BN_BIG) {
        // columns c and c + 64 of one 128-wide head
        const int qc = quad_cols(quad);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = row0 + 8 * h;      // rows >= M (a ragged last block) compute and exchange, but store nothing
          const long long l = row < g.M ? row % g.rope_L : 0;   // and read table row 0: the tables need only cover rows < M
#pragma unroll
          for (int hc = 0; hc < BN; hc += 128) {
            const bool rotate = (long long)n_blk * BN + hc < g.rope_cols;             // per 128-column head
#pragma unroll
            for (int i8 = 0; i8 < 8; i8 += 2) {
              uint32_t o1[2], o2[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int i = hc / 8 + i8 + e, c = 8 * (i8 + e) + 2 * quad, col = n_blk * BN + hc + c;
                bias_rope_words(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], acc[4 * (i + 8) + 2 * h], acc[4 * (i + 8) + 2 * h + 1],
                                g.bias, col, rotate, g.rope_cos, g.rope_sin, l, c, o1[e], o2[e]);
              }
              const uint2 w1 = quad_pair(o1[0], o1[1], quad), w2 = quad_pair(o2[0], o2[1], quad);
              const int col = n_blk * BN + hc + 8 * i8 + qc;
              if (row < g.M) { st_quad(c_ptr(g, row, col), w1); st_quad(c_ptr(g, row, col + 64), w2); }
            }
          }
        }
      } else if constexpr (EPI == EVO_EPI_GELU_GATE && BN == BN_BIG) {
        // packed [l1 | l2] tile: output column n_blk * 128 + c from tile columns c and c + 128
        const int qc = quad_cols(quad);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = row0 + 8 * h;
#pragma unroll
          for (int i = 0; i < BN / 16; i += 2) {
            uint32_t o[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float a0 = rbf(acc[4 * (i + e) + 2 * h]), a1 = rbf(acc[4 * (i + e) + 2 * h + 1]);
              const float b0 = rbf(acc[4 * (i + e + BN / 16) + 2 * h]), b1 = rbf(acc[4 * (i + e + BN / 16) + 2 * h + 1]);
              o[e] = pack_bf16(gelu_gate(a0, b0), gelu_gate(a1, b1));
            }
            const uint2 w = quad_pair(o[0], o[1], quad);
            if (row < g.M) st_quad(c_ptr(g, row, n_blk * (BN / 2) + 8 * i + qc), w);
          }
        }
      } else if constexpr (BN == BN_BIG) {
        // the linear output is rounded before the exchange (the exchanged bf16 pairs hold it exactly), the residual added after
        // it.  The residual of half a row is loaded ahead of its stores (one load latency per half row, not one per column pair);
        // C may alias it, since every element is read before the same thread writes it.
        const int qc = quad_cols(quad);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = row0 + 8 * h;
          const bool live = row < g.M;
          constexpr int CH = BN / 32;              // residual words loaded ahead per chunk (half a row: no register spills)
#pragma unroll
          for (int i0 = 0; i0 < BN / 16; i0 += CH) {
            uint2 r[CH];
            if constexpr (RESID) {
#pragma unroll
              for (int j = 0; j < CH; ++j)
                r[j] = live ? __ldg(reinterpret_cast<const uint2*>(g.resid + row * g.ldr + n_blk * BN + 16 * (i0 + j) + qc)) : make_uint2(0u, 0u);
            }
#pragma unroll
            for (int j = 0; j < CH; ++j) {
              const int i = i0 + j;
              uint32_t o[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const uint32_t b = BIAS ? ld_pair(g.bias + n_blk * BN + 8 * (2 * i + e) + 2 * quad) : 0u;
                o[e] = linear_word<BIAS, false>(acc[4 * (2 * i + e) + 2 * h], acc[4 * (2 * i + e) + 2 * h + 1], b, 0);
              }
              uint2 w = quad_pair(o[0], o[1], quad);
              if constexpr (RESID) { w.x = resid_word(w.x, r[j].x); w.y = resid_word(w.y, r[j].y); }
              if (live) st_quad(c_ptr(g, row, n_blk * BN + 16 * i + qc), w);
            }
          }
        }
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = row0 + 8 * h;
          if (row >= g.M) continue;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) store_pair<BIAS, RESID>(g, row, n_blk * BN + 8 * i + 2 * quad, acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
        }
      }
    }
    if constexpr (TMA_C) {
      if (tid == 0) tma_store_wait_all();     // the staging must outlive the last stores' reads
    }
  }
}

template <int EPI, int BN>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmArgs g) {
  gemm_body<EPI, BN, false>(&tmA, &tmB, nullptr, nullptr, g);
}

template <int EPI>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_wgmma_tma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
                      const __grid_constant__ CUtensorMap tmR, const GemmArgs g) {
  gemm_body<EPI, BN_BIG, true>(&tmA, &tmB, &tmC, &tmR, g);
}

template <int EPI, int BN>
int launch(const evo_gemm_params* p, cudaStream_t st, const long long* targets = nullptr, float4* part = nullptr) {
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_tmap_2d_bf16(&tmA, p->A, (uint64_t)p->K, (uint64_t)p->M, (uint64_t)p->lda * 2, BK, BM, true))) return rc;
  const bool b_tiled = BN == BN_SMALL && p->variant == 3;
  if (b_tiled) {
    uint64_t dims[4] = {(uint64_t)BK, (uint64_t)BN, (uint64_t)(p->K / BK), (uint64_t)(p->N / BN)};
    uint64_t str[3] = {(uint64_t)BK * 2, (uint64_t)BK * BN * 2, (uint64_t)(p->K / BK) * BK * BN * 2};
    uint32_t box[4] = {(uint32_t)BK, (uint32_t)BN, 1, 1};
    if ((rc = make_tmap_nd_bf16(&tmB, p->W, 4, dims, str, box, true))) return rc;
  } else if ((rc = make_tmap_2d_bf16(&tmB, p->W, (uint64_t)p->K, (uint64_t)p->N, (uint64_t)p->K * 2, BK, BN, true))) return rc;
  GemmArgs g;
  g.C = (bf16*)p->C; g.ldc = p->ldc; g.bias = (const bf16*)p->bias; g.resid = (const bf16*)p->residual; g.ldr = p->ldr;
  g.M = p->M; g.N = p->N; g.K = p->K;
  g.targets = targets; g.part = part;
  g.n_peers = p->n_c_peers; g.peer_period = (int)p->peer_period; g.peer_inner = (int)p->peer_inner; g.peer_row0 = p->peer_row0;
  for (int i = 0; i < 8; ++i) g.c_peer[i] = i < p->n_c_peers ? (bf16*)p->c_peers[i] : nullptr;
  g.rope_cos = (const bf16*)p->rope_cos; g.rope_sin = (const bf16*)p->rope_sin; g.rope_L = p->rope_L > 0 ? p->rope_L : 1; g.rope_cols = p->rope_cols;
  g.b_tiled = b_tiled;
  g.m_blocks = (int)((p->M + BM - 1) / BM);
  g.n_blocks = (int)(p->N / BN);
  // Rasterisation: keep the smaller operand slab resident in L2 while the other one streams.
  //   grouped along M: GM row-blocks (GM * rows * K * 2 bytes of A) stay hot, W streams once per group;
  //   grouped along N: GN column-blocks of W stay hot, A streams once per group.
  // Pick the variant with the lower DRAM traffic estimate for a resident slab of about a third of the 50 MB L2.
  {
    const double a_blk = (double)BM * p->K * 2, w_blk = (double)BN * p->K * 2;
    const double a_tot = (double)p->M * p->K * 2, w_tot = (double)p->N * p->K * 2, budget = 16e6;
    // a short last group sweeps the other operand almost unshared: use one group fewer when that stretches the slab by
    // <= 20 %, else spread the blocks evenly
    auto balanced = [](int blocks, int gmax) {
      const int groups = (blocks + gmax - 1) / gmax, last = blocks - (groups - 1) * gmax;
      if (groups == 1 || 2 * last >= gmax) return gmax;
      const int fewer = (blocks + groups - 2) / (groups - 1);
      return 5 * fewer <= 6 * gmax ? fewer : (blocks + groups - 1) / groups;
    };
    int gm = balanced(g.m_blocks, (int)std::max(1.0, std::min((double)g.m_blocks, budget / a_blk)));
    int gn = balanced(g.n_blocks, (int)std::max(1.0, std::min((double)g.n_blocks, budget / w_blk)));
    const double traffic_m = a_tot + w_tot * std::ceil((double)g.m_blocks / gm);
    const double traffic_n = w_tot + a_tot * std::ceil((double)g.n_blocks / gn);
    g.raster_n = traffic_n < traffic_m;
    g.group_m = g.raster_n ? gn : gm;
    const char* env_g = getenv("EVO_B200_GEMM_GROUP");      // experiments only (read per launch)
    const char* env_r = getenv("EVO_B200_GEMM_RASTER_N");
    if (env_r) g.raster_n = atoi(env_r);
    if (env_g) g.group_m = std::max(1, atoi(env_g));
  }
  const int grid = std::min(g.m_blocks * g.n_blocks, device_sm_count());
  // attr_done: one bit per device, a separate copy for each kernel instance
  auto run = [&](auto kern, int smem_bytes, unsigned long long& attr_done, auto... args) {
    if (int rc_ = ensure_dyn_smem(kern, smem_bytes, attr_done)) return rc_;
    kern<<<grid, NTHREADS, smem_bytes, st>>>(args...);
    return check_launch("evo_gemm");
  };
  if constexpr (BN == BN_BIG && EPI != EPI_LSE) {
    // C by TMA stores unless it is peer-scattered; EVO_B200_GEMM_DIRECT_STORE=1 keeps the per-thread stores (the tests'
    // reference for the staged path)
    const char* env_d = getenv("EVO_B200_GEMM_DIRECT_STORE");
    if (p->n_c_peers == 0 && !(env_d && atoi(env_d))) {
      constexpr bool RESID = EPI == EVO_EPI_BIAS_RESID || EPI == EVO_EPI_RESID;
      const uint64_t n_out = EPI == EVO_EPI_GELU_GATE ? p->N / 2 : p->N;
      CUtensorMap tmC, tmR;
      if ((rc = make_tmap_2d_bf16(&tmC, p->C, n_out, (uint64_t)p->M, (uint64_t)p->ldc * 2, 64, 64, true))) return rc;
      if (RESID) { if ((rc = make_tmap_2d_bf16(&tmR, p->residual, n_out, (uint64_t)p->M, (uint64_t)p->ldr * 2, 64, 64, true))) return rc; }
      else tmR = tmC;
      static unsigned long long attr_done = 0;
      return run(gemm_wgmma_tma_kernel<EPI>, Cfg<BN, true>::SMEM_BYTES, attr_done, tmA, tmB, tmC, tmR, g);
    }
  }
  static unsigned long long attr_done = 0;
  return run(gemm_wgmma_kernel<EPI, BN>, Cfg<BN>::SMEM_BYTES, attr_done, tmA, tmB, g);
}

template <int BN>
int dispatch_epi(const evo_gemm_params* p, cudaStream_t st) {
  switch (p->epilogue) {
    case EVO_EPI_NONE: return launch<EVO_EPI_NONE, BN>(p, st);
    case EVO_EPI_BIAS: return launch<EVO_EPI_BIAS, BN>(p, st);
    case EVO_EPI_BIAS_RESID: return launch<EVO_EPI_BIAS_RESID, BN>(p, st);
    case EVO_EPI_RESID: return launch<EVO_EPI_RESID, BN>(p, st);
    case EVO_EPI_BIAS_ROPE:
      if constexpr (BN == BN_BIG) return launch<EVO_EPI_BIAS_ROPE, BN>(p, st);
      else { set_error("evo_gemm: the rotary epilogue is not available on the small-M tile (variant 2)"); return -1; }
    case EVO_EPI_GELU_GATE:
      if constexpr (BN == BN_BIG) return launch<EVO_EPI_GELU_GATE, BN>(p, st);
      else { set_error("evo_gemm: the GELU-gate epilogue is not available on the small-M tile (variant 2)"); return -1; }
  }
  set_error("evo_gemm: unknown epilogue %d", p->epilogue);
  return -1;
}

}  // namespace

extern "C" int evo_gemm(const evo_gemm_params* p, void* stream) {
  EVO_REQUIRE(p->M >= 0 && p->N > 0 && p->K > 0, "evo_gemm: bad shape");
  EVO_REQUIRE(p->variant >= 0 && p->variant <= 3, "evo_gemm: unknown variant %d", p->variant);
  EVO_REQUIRE(p->K % BK == 0, "evo_gemm: K (%lld) must be a multiple of %d", (long long)p->K, BK);
  EVO_REQUIRE(p->N % BN_BIG == 0, "evo_gemm: N (%lld) must be a multiple of %d (pack weights at load time)", (long long)p->N, BN_BIG);
  EVO_REQUIRE(p->lda % 8 == 0 && p->ldc % 8 == 0, "evo_gemm: lda/ldc must be multiples of 8 elements");
  EVO_REQUIRE(((uintptr_t)p->A % 16) == 0 && ((uintptr_t)p->W % 16) == 0 && ((uintptr_t)p->C % 16) == 0, "evo_gemm: pointers must be 16-byte aligned");
  if (p->epilogue == EVO_EPI_BIAS || p->epilogue == EVO_EPI_BIAS_RESID || p->epilogue == EVO_EPI_BIAS_ROPE) EVO_REQUIRE(p->bias != nullptr, "evo_gemm: bias epilogue without bias");
  if (p->epilogue == EVO_EPI_BIAS_ROPE)
    EVO_REQUIRE(p->rope_cos && p->rope_sin && p->rope_L > 0 && p->rope_cols % 128 == 0 && p->rope_cols <= p->N && ((uintptr_t)p->rope_cos % 16) == 0 && ((uintptr_t)p->rope_sin % 16) == 0,
                "evo_gemm: rotary epilogue needs 16-byte aligned cos/sin tables, rope_L > 0 and rope_cols a multiple of the head width (128)");
  if (p->epilogue == EVO_EPI_RESID || p->epilogue == EVO_EPI_BIAS_RESID)
    EVO_REQUIRE(p->residual != nullptr && p->ldr % 8 == 0 && ((uintptr_t)p->residual % 16) == 0, "evo_gemm: residual epilogue without a valid residual");
  if (p->n_c_peers != 0) {
    EVO_REQUIRE(p->n_c_peers > 0 && p->n_c_peers <= 8 && p->c_peers != nullptr, "evo_gemm: 1..8 peer destinations");
    EVO_REQUIRE(p->peer_inner > 0 && p->peer_inner % 128 == 0 && p->peer_period == p->peer_inner * p->n_c_peers && p->N % p->peer_period == 0,
                "evo_gemm: peer scatter needs peer_inner %% 128 == 0, peer_period = n_peers * peer_inner, N %% peer_period == 0");
    EVO_REQUIRE(p->epilogue == EVO_EPI_BIAS || p->epilogue == EVO_EPI_NONE || p->epilogue == EVO_EPI_BIAS_ROPE, "evo_gemm: peer scatter supports the none / bias / rotary epilogues");
    EVO_REQUIRE(p->variant == 0 || p->variant == 1, "evo_gemm: peer scatter needs the 256-column tiles");
  }
  if (p->M == 0) return 0;
  if (p->variant == 2 || p->variant == 3) return dispatch_epi<BN_SMALL>(p, (cudaStream_t)stream);
  return dispatch_epi<BN_BIG>(p, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------
// Fused scoring head (SURVEY 8f-1): unembed GEMM + log-softmax + gather (+ entropy); the (M, V) logits never reach HBM.
// The GEMM's epilogue leaves one float4 of statistics per (row, 256-column half); the finish kernel folds the halves:
//   lse = M + log(sum_j s_j e^(m_j - M)),  logprob = x_target - lse,  entropy = lse - (sum_j w_j e^(m_j - M)) / S.
// ---------------------------------------------------------------------------------------------
namespace {
__global__ void score_finish_kernel(const float4* __restrict__ part, int n_blocks, long long M, const long long* __restrict__ targets, int V,
                                    float* __restrict__ logprobs, float* __restrict__ entropy) {
  const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= M) return;
  float mx = -INFINITY;
  for (int j = 0; j < n_blocks; ++j) mx = fmaxf(mx, part[row * n_blocks + j].x);
  float S = 0.f, W = 0.f;
  for (int j = 0; j < n_blocks; ++j) {
    const float4 q = part[row * n_blocks + j];
    const float sc = expf(q.x - mx);
    S = fmaf(q.y, sc, S); W = fmaf(q.z, sc, W);
  }
  const float lse = mx + logf(S);
  if (logprobs) {
    const long long t = targets ? targets[row] : -1;
    logprobs[row] = (t < 0 || t >= V) ? 0.f : part[row * n_blocks + (int)(t / BN_BIG)].w - lse;
  }
  if (entropy) entropy[row] = lse - W / S;
}
}  // namespace

extern "C" size_t evo_unembed_score_workspace(int64_t M, int V) { return (size_t)M * (size_t)(V / BN_BIG) * sizeof(float4); }

extern "C" int evo_unembed_score(const evo_score_params* p, void* stream) {
  EVO_REQUIRE(p->M >= 0 && p->V > 0 && p->V % BN_BIG == 0, "evo_unembed_score: vocabulary (%d) must be a multiple of %d", p->V, BN_BIG);
  EVO_REQUIRE(p->K > 0 && p->K % BK == 0, "evo_unembed_score: K (%lld) must be a multiple of %d", (long long)p->K, BK);
  EVO_REQUIRE(((uintptr_t)p->x % 16) == 0 && ((uintptr_t)p->W % 16) == 0, "evo_unembed_score: pointers must be 16-byte aligned");
  EVO_REQUIRE(p->logprobs == nullptr || p->targets != nullptr, "evo_unembed_score: logprobs need targets");
  if (p->M == 0) return 0;
  const size_t need = evo_unembed_score_workspace(p->M, p->V);
  EVO_REQUIRE(p->workspace != nullptr && p->workspace_bytes >= need, "evo_unembed_score: workspace too small (%zu < %zu)", p->workspace_bytes, need);
  evo_gemm_params gp = {};
  gp.A = p->x; gp.lda = p->K; gp.W = p->W; gp.C = nullptr; gp.ldc = p->V; gp.M = p->M; gp.N = p->V; gp.K = p->K; gp.epilogue = EPI_LSE; gp.variant = 0;
  int rc = launch<EPI_LSE, BN_BIG>(&gp, (cudaStream_t)stream, (const long long*)p->targets, (float4*)p->workspace);
  if (rc) return rc;
  score_finish_kernel<<<(unsigned)((p->M + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const float4*)p->workspace, p->V / BN_BIG, p->M, (const long long*)p->targets, p->V,
                                                                                       p->logprobs, p->entropy);
  return check_launch("evo_unembed_score");
}
