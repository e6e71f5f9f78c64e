// Hyena scan, mode-split TMA kernel: the production path for head_dim 128 / D % 256 == 0.
//
// Same operator and rounding points as hyena_scan_kernel (hyena.cu); what changes is how the machine is driven:
//   * a CTA owns two heads (256 channels) of one batch row and walks its L segment in tiles of T2 tokens; a producer
//     warp keeps an mbarrier ring of z tiles ([x2|x1|v] x 2 heads = six 128-column boxes, 24 KB per stage) in flight
//     by TMA, so HBM latency is never exposed to the scan;
//   * a thread carries a channel PAIR (fp32 pair arithmetic, fadd2 / fmul2 / ffma2, one rounding per lane), but only
//     FOUR of the eight modal states: lanes l and l^16 of a warp share a pair.  A thread that carried all eight states
//     needed ~214 registers and left one warp per SM sub-partition, latency-starved; here a 256-channel CTA has
//     8 compute warps = two per sub-partition, so a dependent FMA chain in one warp is covered by the other;
//   * the element-wise work is split between the two halves instead of duplicated: half 0 runs the x1 FIR, half 1
//     the v FIR (one shuffle exchanges the bf16x2 results); half 0 gates tokens 0..3 of a group of eight, half 1
//     tokens 4..7 (one shuffle per fp32 word moves the partial residue sums to the half that needs them);
//   * every bf16 (x) bf16 -> bf16 tensor op of the reference (bias add, x1*v, D*x1v, +conv, *x2) is ONE packed
//     add.rn.bf16x2 / mul.rn.bf16x2 instead of unpack + fp32 op + pack: the product of two bf16 is exact in fp32 and
//     the sum of two bf16 is exact in fp32 or rounds to the larger operand either way, so a single rounding of the
//     exact result is bit-identical to the reference's "compute in fp32, round to bf16".
#pragma once
#include "common.cuh"
#include <type_traits>

namespace evo_hy3 {

using namespace evo;

constexpr int NS = 8;
constexpr int NSH = 4;                       // modal states per thread
constexpr int T2 = 16;                       // tokens per stage
constexpr int STAGES = 8;                    // maximum ring depth (barriers); the launch uses 4
constexpr int CH_PER_CTA = 256;              // two heads of 128
constexpr int SUB_BYTES = T2 * 128 * 2;      // one 128-column box
constexpr int STAGE_BYTES = 6 * SUB_BYTES;   // [head0: x2 x1 v][head1: x2 x1 v]
constexpr int CWARPS = 8;                    // compute warps: 4 per head, 16 channel pairs x 2 halves each
constexpr int THREADS = (CWARPS + 1) * 32;   // + 1 TMA producer warp
constexpr int G = 8;                         // tokens per group
constexpr int smem_bytes(int nst) { return nst * STAGE_BYTES + 128 + 1024; }

struct Args2 {                               // batched sequences
  bf16* y;
  const bf16* z;
  const bf16* fir_w; const bf16* fir_b; const bf16* Dskip;
  const float* poles; const float* residues;
  const bf16* halo; const float* state_in;
  float* state_out;
  float* seg_states;                         // (B, nseg, D, NS, 2) zero-start end states of each segment
  int B, D, nseg, nst;
  long long L, seg_len;
};
struct Args2V : Args2 {                      // packed sequences (VARLEN)
  const long long* cu_seqlens;               // (B + 1) row offsets; Args2::L is the longest length
  long long T;                               // packed rows
};
struct Args2R : Args2V {                     // checkpoint emission and resumed starts (RESUME)
  // emission: the output pass stores the running state after row k*ckpt_stride - 1 of sequence b at table row ckpt_base[b] + k - 1
  // (k >= 1, k*ckpt_stride < its length; ckpt_stride a multiple of 128, seg_len a multiple of the 16-token stage), NULL = none
  float* ckpt_out; const long long* ckpt_base; long long ckpt_stride, n_ckpt;
  // resumed start: sequence b starts from state_table[start_idx[b]] and FIR history halo_table[start_idx[b]] (-1 = zero start)
  const long long* start_idx; const float* state_table; const bf16* halo_table; long long n_table;
};

__device__ __forceinline__ float2 unpack2(uint32_t v) { return make_float2(bf_lo(v), bf_hi(v)); }
__device__ __forceinline__ uint32_t lds32(uint32_t addr) { uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr)); return v; }

struct C2 { float2 r, i; };                  // two complex numbers (one per channel of the pair)
__device__ __forceinline__ C2 cmul2(C2 a, C2 b) {
  C2 o;
  o.r = ffma2(a.r, b.r, fmul2(make_float2(-a.i.x, -a.i.y), b.i));
  o.i = ffma2(a.r, b.i, fmul2(a.i, b.r));
  return o;
}
__device__ __forceinline__ C2 cpow2(C2 p, long long n) {
  C2 acc; acc.r = make_float2(1.f, 1.f); acc.i = make_float2(0.f, 0.f);
  while (n > 0) { if (n & 1) acc = cmul2(acc, p); p = cmul2(p, p); n >>= 1; }
  return acc;
}

__device__ __forceinline__ uint32_t mul_bf2(uint32_t a, uint32_t b) { uint32_t d; asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ uint32_t add_bf2(uint32_t a, uint32_t b) { uint32_t d; asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ uint32_t ldg32(const bf16* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); }

// VARLEN: packed sequences (evo_hyena_fwd_varlen).  Grid row b is sequence b = rows [cu[b], cu[b+1]) of a (3D, T, 1) tensor map;
// a.L is the longest length.  Every segment but a sequence's last is full (one seg_len for all), so the carry below holds unchanged;
// a tile that reaches into the next sequence goes through the ragged-tile path (n_valid), so no foreign token enters the scan.
// RESUME (implies VARLEN; evo_hyena_fwd_varlen_ckpt): a sequence may start from a checkpoint table row instead of zero -- the
// state_in / halo of the batched kernel, indexed per sequence -- and the output pass may store checkpoints as it goes.
template <bool STATE_ONLY, bool VARLEN = false, bool RESUME = false>
__global__ void __launch_bounds__(THREADS, 1)
hyena_scan_ms_kernel(const __grid_constant__ CUtensorMap tmZ, const std::conditional_t<RESUME, Args2R, std::conditional_t<VARLEN, Args2V, Args2>> a) {
  static_assert(!RESUME || VARLEN, "the resumed form is a packed-sequence form");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  const int NST = a.nst;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + NST * STAGE_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cb = blockIdx.x, b = blockIdx.y, seg = blockIdx.z;
  const long long t0 = (long long)seg * a.seg_len;
  long long row0 = 0, len = a.L;
  if constexpr (VARLEN) {          // clamped, so that a malformed cu_seqlens cannot move a load or store outside [0, T)
    row0 = min(max(a.cu_seqlens[b], 0LL), a.T);
    len = min(min(a.cu_seqlens[b + 1], a.T) - row0, a.L);
    if (t0 >= len) return;
  }
  const long long t1 = min(len, t0 + a.seg_len);
  const int n_tiles = t1 > t0 ? (int)((t1 - t0 + T2 - 1) / T2) : 0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CWARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == CWARPS) {
    // ------------------------------------------------ TMA producer (one lane)
    if (lane == 0) {
      tma_prefetch_desc(&tmZ);
      for (int k = 0; k < n_tiles; ++k) {
        const int st = k % NST;
        mbar_wait(&empty[st], ((uint32_t)(k / NST) & 1) ^ 1);
        uint8_t* dst = smem + st * STAGE_BYTES;
        const int row = (int)(row0 + t0 + (long long)k * T2);
        const int zb3 = VARLEN ? 0 : b;
        if (STATE_ONLY) {
          mbar_arrive_expect_tx(&full[st], 4 * SUB_BYTES);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
#pragma unroll
            for (int w = 1; w < 3; ++w)
              tma_load_3d(dst + (hh * 3 + w) * SUB_BYTES, &tmZ, &full[st], cb * 768 + hh * 384 + w * 128, row, zb3);
        } else {
          mbar_arrive_expect_tx(&full[st], STAGE_BYTES);
#pragma unroll
          for (int s6 = 0; s6 < 6; ++s6)
            tma_load_3d(dst + s6 * SUB_BYTES, &tmZ, &full[st], cb * 768 + s6 * 128, row, zb3);
        }
      }
    }
    return;
  }

  // ------------------------------------------------ compute warps: thread = (channel pair, half of the modes)
  const int hh = warp >> 2;                               // head within the CTA
  const int half = lane >> 4;                             // 0: modes 0..3, x1 FIR, tokens 0..3 | 1: modes 4..7, v FIR, tokens 4..7
  const int j2 = ((warp & 3) * 16 + (lane & 15)) * 2;     // first channel of the pair inside the head
  const int ch = cb * CH_PER_CTA + hh * 128 + j2;         // global channel (of D)
  const int zc = cb * 768 + hh * 384 + j2;                // z column of x2; x1 = +128, v = +256
  const int own = 1 + half;                               // sub-box this thread's FIR reads: 1 = x1, 2 = v
  const int m0 = half * NSH;
  const long long C3 = 3LL * a.D;

  float2 pr[NSH], pi[NSH], npi[NSH], rr[NSH], ri[NSH], sr[NSH], si[NSH];
#pragma unroll
  for (int s = 0; s < NSH; ++s) {
    const float2 p0 = __ldg(reinterpret_cast<const float2*>(a.poles) + (long long)ch * NS + m0 + s);
    const float2 p1 = __ldg(reinterpret_cast<const float2*>(a.poles) + (long long)(ch + 1) * NS + m0 + s);
    const float2 r0 = __ldg(reinterpret_cast<const float2*>(a.residues) + (long long)ch * NS + m0 + s);
    const float2 r1 = __ldg(reinterpret_cast<const float2*>(a.residues) + (long long)(ch + 1) * NS + m0 + s);
    pr[s] = make_float2(p0.x, p1.x); pi[s] = make_float2(p0.y, p1.y); npi[s] = make_float2(-p0.y, -p1.y);
    rr[s] = make_float2(r0.x, r1.x); ri[s] = make_float2(-r0.y, -r1.y);      // Re(R s) = Rr sr - Ri si
    sr[s] = make_float2(0.f, 0.f); si[s] = make_float2(0.f, 0.f);
  }
  // FIR taps of the owned channel pair and of x2; biases / skip stay packed bf16x2
  float2 wo[3], w2[3];
  {
    const bf16* p0 = a.fir_w + (long long)(zc + own * 128) * 3;
    const bf16* q0 = a.fir_w + (long long)zc * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      wo[k] = make_float2(__bfloat162float(p0[k]), __bfloat162float(p0[3 + k]));
      w2[k] = make_float2(__bfloat162float(q0[k]), __bfloat162float(q0[3 + k]));
    }
  }
  const uint32_t boq = ldg32(a.fir_b + zc + own * 128);
  const uint32_t b2q = ldg32(a.fir_b + zc);
  const uint32_t dskq = ldg32(a.Dskip + ch);

  long long sidx = -1;                                    // RESUME: checkpoint row this sequence starts from (clamped to the table)
  if constexpr (RESUME) {
    if (a.start_idx) { sidx = a.start_idx[b]; if (sidx >= a.n_table) sidx = -1; }
  }
  if (!STATE_ONLY) {
    if constexpr (RESUME) {
      if (sidx >= 0) {
#pragma unroll
        for (int s = 0; s < NSH; ++s) {
          const float2 v0 = __ldg(reinterpret_cast<const float2*>(a.state_table) + (sidx * a.D + ch) * NS + m0 + s);
          const float2 v1 = __ldg(reinterpret_cast<const float2*>(a.state_table) + (sidx * a.D + ch + 1) * NS + m0 + s);
          sr[s] = make_float2(v0.x, v1.x); si[s] = make_float2(v0.y, v1.y);
        }
      }
    } else if (a.state_in) {
#pragma unroll
      for (int s = 0; s < NSH; ++s) {
        const float2 v0 = __ldg(reinterpret_cast<const float2*>(a.state_in) + ((long long)b * a.D + ch) * NS + m0 + s);
        const float2 v1 = __ldg(reinterpret_cast<const float2*>(a.state_in) + ((long long)b * a.D + ch + 1) * NS + m0 + s);
        sr[s] = make_float2(v0.x, v1.x); si[s] = make_float2(v0.y, v1.y);
      }
    }
    if (seg > 0) {      // carry entering this segment: S_j = p^len S_{j-1} + E_{j-1} over the zero-start end states
#pragma unroll
      for (int s = 0; s < NSH; ++s) {
        C2 p; p.r = pr[s]; p.i = pi[s];
        const C2 pl = cpow2(p, a.seg_len);
        C2 acc; acc.r = sr[s]; acc.i = si[s];
        for (int q = 0; q < seg; ++q) {
          const float2* e = reinterpret_cast<const float2*>(a.seg_states) + (((long long)b * a.nseg + q) * a.D + ch) * NS + m0 + s;
          const float2 e0 = e[0], e1 = e[NS];
          acc = cmul2(pl, acc);
          acc.r = fadd2(acc.r, make_float2(e0.x, e1.x));
          acc.i = fadd2(acc.i, make_float2(e0.y, e1.y));
        }
        sr[s] = acc.r; si[s] = acc.i;
      }
    }
  }

  // FIR history z[t0-2], z[t0-1]: fp32 pair for the owned channel, packed words for x2 (half 0 only uses them)
  const long long seq_row = VARLEN ? row0 : (long long)b * a.L;      // z / y row of the sequence's token 0
  const bf16* zb = a.z + seq_row * C3;
  float2 ho[2];
  uint32_t h2q[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    ho[k] = make_float2(0.f, 0.f); h2q[k] = 0u;
    const long long t = t0 - 2 + k;
    const bf16* row = nullptr;
    if (t >= 0) row = zb + t * C3;
    else if constexpr (RESUME) { if (sidx >= 0) row = a.halo_table + (sidx * 2 + (t + 2)) * C3; }
    else if (a.halo) row = a.halo + ((long long)b * 2 + (t + 2)) * C3;
    if (row) { ho[k] = unpack2(ldg32(row + zc + own * 128)); if (!STATE_ONLY) h2q[k] = ldg32(row + zc); }
  }

  const long long ystride = a.D / 2;        // in 32-bit words
  uint32_t* yrow = STATE_ONLY ? nullptr : reinterpret_cast<uint32_t*>(a.y + (seq_row + t0) * a.D + ch) + (long long)(4 * half) * ystride;

  auto do_group = [&](uint32_t tile, int j0, int n_valid, uint32_t* ydst) {
    // ---- stage A: the owned short FIR (fp32 accumulate, rp) + bias (rp) for all G tokens
    float2 zo[G];
#pragma unroll
    for (int g = 0; g < G; ++g) zo[g] = unpack2(lds32(tile + own * SUB_BYTES + (j0 + g) * 256));
    uint32_t xq[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const float2 a_ = g >= 2 ? zo[g - 2] : ho[g], b_ = g >= 1 ? zo[g - 1] : ho[1];
      const float2 acc = ffma2(wo[2], zo[g], ffma2(wo[1], b_, fmul2(wo[0], a_)));
      const uint32_t f = add_bf2(pack_bf16(acc.x, acc.y), boq);
      xq[g] = mul_bf2(f, __shfl_xor_sync(0xffffffffu, f, 16));          // x1v = x1 * v (rp): the partner holds the other factor
    }
    if (n_valid == G) { ho[0] = zo[G - 2]; ho[1] = zo[G - 1]; }
    // ---- stage A2: x2 FIR for the four tokens this half gates (window = 6 consecutive z2 rows)
    uint32_t f2q[4];
    if (!STATE_ONLY) {
      uint32_t l2[6];
#pragma unroll
      for (int i = 0; i < 4; ++i) l2[i] = lds32(tile + half * 512 + (j0 + i) * 256);      // tokens i (half 0) / i + 2 (half 1)
      l2[4] = lds32(tile + (j0 + 6) * 256); l2[5] = lds32(tile + (j0 + 7) * 256);
      float2 wf[6];
      wf[0] = unpack2(half ? l2[0] : h2q[0]); wf[1] = unpack2(half ? l2[1] : h2q[1]);
#pragma unroll
      for (int i = 2; i < 6; ++i) wf[i] = unpack2(half ? l2[i] : l2[i - 2]);
      if (n_valid == G) { h2q[0] = l2[4]; h2q[1] = l2[5]; }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 acc = ffma2(w2[2], wf[k + 2], ffma2(w2[1], wf[k + 1], fmul2(w2[0], wf[k])));
        f2q[k] = add_bf2(pack_bf16(acc.x, acc.y), b2q);
      }
    }
    // ---- stage B: modal recurrence on this half's four states, sequential in t; partial residue sums
    float2 pc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (g < n_valid) {
        const float2 x = unpack2(xq[g]);
        float2 ar = make_float2(0.f, 0.f), ai = ar;
#pragma unroll
        for (int s = 0; s < NSH; ++s) {
          const float2 t_ = ffma2(npi[s], si[s], x);
          const float2 nr = ffma2(pr[s], sr[s], t_);
          const float2 ni = ffma2(pr[s], si[s], fmul2(pi[s], sr[s]));
          sr[s] = nr; si[s] = ni;
          if (!STATE_ONLY) { ar = s ? ffma2(rr[s], nr, ar) : fmul2(rr[s], nr); ai = s ? ffma2(ri[s], ni, ai) : fmul2(ri[s], ni); }
        }
        if (!STATE_ONLY) pc[g] = fadd2(ar, ai);
      }
    }
    // ---- stage C: conv = partial(modes 0..3) + partial(modes 4..7) (rp to bf16); y = (conv + x1v*D) * x2 with the reference's roundings
    if (!STATE_ONLY) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 mine = half ? pc[4 + k] : pc[k];
        const float2 send = half ? pc[k] : pc[4 + k];
        const float2 recv = make_float2(__shfl_xor_sync(0xffffffffu, send.x, 16), __shfl_xor_sync(0xffffffffu, send.y, 16));
        const float2 c = fadd2(mine, recv);
        const uint32_t xk = half ? xq[4 + k] : xq[k];
        const uint32_t u = add_bf2(pack_bf16(c.x, c.y), mul_bf2(xk, dskq));
        if (4 * half + k < n_valid) ydst[(long long)k * ystride] = mul_bf2(u, f2q[k]);
      }
    }
  };

  // RESUME emission: the next checkpoint row count this segment reaches (t0 is a multiple of the stage, so every checkpoint
  // ends a full tile)
  long long next_ck = 0;
  if constexpr (RESUME && !STATE_ONLY) { if (a.ckpt_out) next_ck = (t0 / a.ckpt_stride + 1) * a.ckpt_stride; }
  for (int k = 0; k < n_tiles; ++k) {
    const int st = k % NST;
    mbar_wait(&full[st], (uint32_t)(k / NST) & 1);
    const uint32_t tile = smem_u32(smem) + st * STAGE_BYTES + hh * 3 * SUB_BYTES + j2 * 2;
    const int n_tok = (int)min((long long)T2, t1 - (t0 + (long long)k * T2));
    uint32_t* ytile = STATE_ONLY ? nullptr : yrow + (long long)k * T2 * ystride;
    if (n_tok == T2) {
#pragma unroll
      for (int j0 = 0; j0 < T2; j0 += G) do_group(tile, j0, G, STATE_ONLY ? nullptr : ytile + (long long)j0 * ystride);
    } else {                                   // ragged last tile of the segment
      for (int j0 = 0; j0 < n_tok; j0 += G) do_group(tile, j0, min(G, n_tok - j0), STATE_ONLY ? nullptr : ytile + (long long)j0 * ystride);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
    if constexpr (RESUME && !STATE_ONLY) {
      if (a.ckpt_out && t0 + (long long)(k + 1) * T2 == next_ck) {     // the state after row next_ck - 1: 16 floats per thread
        const long long row = a.ckpt_base[b] + next_ck / a.ckpt_stride - 1;
        if (next_ck < len && row >= 0 && row < a.n_ckpt) {
          float2* e = reinterpret_cast<float2*>(a.ckpt_out + ((row * a.D + ch) * NS) * 2) + m0;
#pragma unroll
          for (int s = 0; s < NSH; ++s) { e[s] = make_float2(sr[s].x, si[s].x); e[NS + s] = make_float2(sr[s].y, si[s].y); }
        }
        next_ck += a.ckpt_stride;
      }
    }
  }

  float* dst = nullptr;
  if (STATE_ONLY) dst = a.seg_states + ((((long long)b * a.nseg + seg) * a.D + ch) * NS) * 2;
  else if (a.state_out && (VARLEN ? t1 == len : seg == a.nseg - 1)) dst = a.state_out + (((long long)b * a.D + ch) * NS) * 2;
  if (dst) {
    float2* e = reinterpret_cast<float2*>(dst) + m0;
#pragma unroll
    for (int s = 0; s < NSH; ++s) { e[s] = make_float2(sr[s].x, si[s].x); e[NS + s] = make_float2(sr[s].y, si[s].y); }
  }
}

}  // namespace evo_hy3
