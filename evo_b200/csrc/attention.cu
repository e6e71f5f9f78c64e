// Causal rotary attention core for sm_90a (head_dim 128): softmax(Q K^T / sqrt(d)) V.
// Replaces flash_attn_qkvpacked_func (flash_attn/modules/mha.py:122) with a wgmma kernel:
//
//   one CTA = 128 query rows of one (batch, head); 3 warpgroups:
//     warpgroup 0     TMA producer: Q once, K and V tiles (128 keys) through 2-deep mbarrier rings
//     warpgroups 1-2  64 query rows each: S = Q K^T (wgmma m64n128k16, both operands in shared memory) into
//                     registers, online softmax on the fragments (a row lives in the 4 threads of a quad),
//                     then O += P V with P taken from registers as the A operand and V read in place as an
//                     MN-major B operand.  O stays in registers across KV tiles and is rescaled lazily (only
//                     when the running max grows by more than 2^8); the 1/l normalisation happens in the epilogue.
//   The two consumer warpgroups work on the same K / V tiles, so while one runs its softmax the other keeps the
//   tensor cores busy.
//
// Rounding points match FlashAttention's: fp32 scores and statistics, P rounded to bf16 for the
// PV product, fp32 accumulation, single bf16 rounding of the output.  The running max does not: P
// is taken against a reference that may lag the row's max by up to 2^8, so P in (1, 2^8] is
// rounded to bf16 (same relative error as P <= 1), and alpha = ex2(m_ref - mx) flushes to 0 after
// a jump past 2^126.  tests/test_gpu_attention_peaked.py holds rows with a moving max to the fp64
// and bf16-oracle bars of the other attention tests, and one-hot and tied rows bit for bit.
#include "common.cuh"
#include "wgmma.cuh"
#include <type_traits>
#include "../../include/evo_b200.h"

using namespace evo;

namespace {

constexpr int HD = 128;          // head dim
constexpr int BQ = 128;          // query rows per CTA
constexpr int BKV = 128;         // keys per tile
constexpr int TILE_BYTES = 128 * 128 * 2;          // any 128x128 bf16 tile = 2 x (128 rows x 64) swizzled halves
constexpr int HALF_BYTES = TILE_BYTES / 2;
constexpr int ATT_THREADS = 384;
constexpr int CONSUMER_WARPS = 8;
constexpr int KV_STAGES = 2;
constexpr int ATT_SMEM = TILE_BYTES * (1 + 2 * KV_STAGES) + 256;
static_assert(ATT_SMEM <= 232448, "exceeds the 227 KB dynamic shared memory limit");

struct AttArgs {
  bf16* out;
  bf16* out_peer[8]; int n_out_peers; long long out_rows_per_peer, out_row_stride, out_col0;   // peer-scattered output (evo_attn_params)
  int B, H;
  long long Lq, Lk, q_pos0;
  float scale_log2;              // softmax_scale * log2(e)
};
struct AttArgsV : AttArgs {      // packed sequences (VARLEN); AttArgs itself stays as it is, and so does its kernel
  const long long* cu_seqlens;   // (B + 1) row offsets; Lq = Lk = the longest length
  long long T;                   // packed rows
};
struct AttArgsP : AttArgsV {     // packed queries behind a cached prefix (PREFIX); AttArgsV and its kernels stay as they are
  const long long* prefix_seq;   // (B) batch row of the cache holding sequence b's prefix
  const long long* prefix_len;   // (B) prefix keys of sequence b: cache rows [0, prefix_len[b]); its rows sit at positions prefix_len[b] + t
  long long cache_len;           // rows per batch row of the cache
  int n_cache;                   // batch rows of the cache
};

// PREFIX: sequence b's prefix keys, clamped to the cache; 0 in every other form
template <bool PREFIX, typename A>
__device__ __forceinline__ long long prefix_keys(const A& a, int b) {
  if constexpr (PREFIX) return min(max(a.prefix_len[b], 0LL), a.cache_len);
  else return 0;
}

__device__ __forceinline__ float ex2(float x) { float y; asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// VARLEN: grid row b is packed sequence b = rows [cu[b], cu[b+1]) of (HD, H, T, 1) maps.  Query and key tiles start at the
// sequence's first row, exactly as in a batch-1 call on it; keys past its end are hidden by the causal mask and query rows past
// its end are not stored, so the output is that call's bits.
// PREFIX (implies VARLEN; evo_attn_fwd_varlen_prefix): tmQ maps the packed qkv as (HD, 3H, T, 1) -- q, k, v are heads h, H + h,
// 2H + h -- and tmK maps a KV cache as (HD, 2H, cache_len, n_cache) -- k, v are heads h, H + h.  Sequence b's rows sit at positions
// P = prefix_len[b] + t: the key tiles are first the prefix tiles of cache row prefix_seq[b], keys [0, P) from key 0 (no causal
// mask; keys at or past P masked, and their V rows zeroed in shared memory so that nothing the cache holds there reaches the
// output), then the sequence's own tiles from its first row, causally.  One online softmax runs over both, so with P % 128 == 0
// the tiles, masks and bits are those of a batch-1 evo_attn_fwd_ws call with q_pos0 = P on one cache holding both.
template <bool VARLEN, bool PREFIX = false>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const std::conditional_t<PREFIX, AttArgsP, std::conditional_t<VARLEN, AttArgsV, AttArgs>> a) {
  static_assert(!PREFIX || VARLEN, "the prefix form is a packed-sequence form");
  extern __shared__ __align__(1024) uint8_t smem[];            // 128B-swizzled tiles need 1024-byte alignment
  if ((smem_u32(smem) & 1023u) != 0) __trap();               // fail loudly, never compute on a misaligned tile
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + TILE_BYTES;
  uint8_t* sV = sK + KV_STAGES * TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KV_STAGES * TILE_BYTES);
  uint64_t* q_full = bars;                 // 1
  uint64_t* k_full = bars + 1;             // KV_STAGES
  uint64_t* k_empty = k_full + KV_STAGES;
  uint64_t* v_full = k_empty + KV_STAGES;
  uint64_t* v_empty = v_full + KV_STAGES;

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int h = blockIdx.y, b = blockIdx.z;
  long long Lq = a.Lq, Lk = a.Lk, row0 = 0;
  if constexpr (VARLEN) {          // clamped, so that a malformed cu_seqlens cannot move a load or store outside [0, T)
    row0 = min(max(a.cu_seqlens[b], 0LL), a.T);
    Lq = Lk = min(min(a.cu_seqlens[b + 1], a.T) - row0, a.Lq);
  }
  const int n_qblk = (int)((Lq + BQ - 1) / BQ);
  const int qblk = n_qblk - 1 - (int)blockIdx.x;      // longest (latest) blocks first
  if (VARLEN && qblk < 0) return;                     // past this sequence's last query block
  const int zb = VARLEN ? 0 : b;
  const long long q0 = (long long)qblk * BQ;
  // keys visible to this block: j <= q_pos0 + q0 + 127, j < Lk
  const long long last_key = min(Lk - 1, a.q_pos0 + q0 + BQ - 1);
  const long long plen = prefix_keys<PREFIX>(a, b);   // PREFIX: prefix keys (0 otherwise) and the tiles that hold them
  const int n_pre = (int)((plen + BKV - 1) / BKV);
  const int n_kv = (int)(last_key / BKV) + 1 + n_pre;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_STAGES; ++i) { mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], CONSUMER_WARPS); mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (tid == 0) {
      mbar_arrive_expect_tx(q_full, TILE_BYTES);
      tma_load_4d(sQ, &tmQ, q_full, 0, h, (int)(row0 + q0), zb);
      tma_load_4d(sQ + HALF_BYTES, &tmQ, q_full, 64, h, (int)(row0 + q0), zb);
      for (int j = 0; j < n_kv; ++j) {
        const int st = j % KV_STAGES;
        const uint32_t ph = (uint32_t)(j / KV_STAGES) & 1;
        if constexpr (PREFIX) {                // cache tile (k, v = heads h, H + h of tmK) or own tile (k, v = heads H + h, 2H + h of tmQ)
          const bool pre = j < n_pre;
          const CUtensorMap* m = pre ? &tmK : &tmQ;
          const int key0 = pre ? j * BKV : (int)row0 + (j - n_pre) * BKV, kh = pre ? h : a.H + h, vh = kh + a.H;
          const int zz = pre ? (int)min(max(a.prefix_seq[b], 0LL), (long long)a.n_cache - 1) : 0;
          mbar_wait(&k_empty[st], ph ^ 1);
          mbar_arrive_expect_tx(&k_full[st], TILE_BYTES);
          tma_load_4d(sK + st * TILE_BYTES, m, &k_full[st], 0, kh, key0, zz);
          tma_load_4d(sK + st * TILE_BYTES + HALF_BYTES, m, &k_full[st], 64, kh, key0, zz);
          mbar_wait(&v_empty[st], ph ^ 1);
          mbar_arrive_expect_tx(&v_full[st], TILE_BYTES);
          tma_load_4d(sV + st * TILE_BYTES, m, &v_full[st], 0, vh, key0, zz);
          tma_load_4d(sV + st * TILE_BYTES + HALF_BYTES, m, &v_full[st], 64, vh, key0, zz);
          continue;
        }
        const int key0 = (int)row0 + j * BKV;
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&k_full[st], TILE_BYTES);
        tma_load_4d(sK + st * TILE_BYTES, &tmK, &k_full[st], 0, h, key0, zb);
        tma_load_4d(sK + st * TILE_BYTES + HALF_BYTES, &tmK, &k_full[st], 64, h, key0, zb);
        mbar_wait(&v_empty[st], ph ^ 1);       // (d, H, key, B): two d-halves of 128 keys x 64 d
        mbar_arrive_expect_tx(&v_full[st], TILE_BYTES);
        tma_load_4d(sV + st * TILE_BYTES, &tmV, &v_full[st], 0, h, key0, zb);
        tma_load_4d(sV + st * TILE_BYTES + HALF_BYTES, &tmV, &v_full[st], 64, h, key0, zb);
      }
    }
  } else {
    // ------------------------------------------------ consumers: 64 query rows each
    setmaxnreg_inc<232>();
    const int cw = wg - 1, warp = tid >> 5, lane = tid & 31, quad = lane & 3;
    const int r0 = cw * 64 + warp * 16 + (lane >> 2);        // this thread's rows: r0 and r0 + 8 of the block
    const long long pos[2] = {a.q_pos0 + q0 + r0 + plen, a.q_pos0 + q0 + r0 + 8 + plen};
    float o[HD / 2];
    float m_ref[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    mbar_wait(q_full, 0);
    const uint32_t qa = smem_u32(sQ) + cw * 64 * 128;
    for (int j = 0; j < n_kv; ++j) {
      const int st = j % KV_STAGES;
      const uint32_t ph = (uint32_t)(j / KV_STAGES) & 1;
      float s[BKV / 2];
      mbar_wait(&k_full[st], ph);
      const uint32_t ka = smem_u32(sK + st * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        const uint32_t off = (kk >> 2) * HALF_BYTES + (kk & 3) * 32;
        wgmma_m64n128k16_ss(s, wgmma_desc_k_sw128(qa + off), wgmma_desc_k_sw128(ka + off), kk != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      if (lane == 0) mbar_arrive(&k_empty[st]);
      // causal / length mask on tiles that reach past a row's position
      const bool pre_tile = PREFIX && j < n_pre;
      if constexpr (PREFIX) {      // a prefix tile's keys run from 0 and stop at plen; own keys run from position plen
        const long long key0 = (pre_tile ? (long long)j * BKV : plen + (long long)(j - n_pre) * BKV) + 2 * quad;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const long long lim = pre_tile ? plen - 1 : pos[hr];
          if (key0 + BKV - 1 - 2 * quad > lim) {
#pragma unroll
            for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
              for (int e = 0; e < 2; ++e) if (key0 + 8 * i + e > lim) s[4 * i + 2 * hr + e] = -INFINITY;
          }
        }
      } else {
        const long long key0 = (long long)j * BKV + 2 * quad;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          if (key0 + BKV - 1 - 2 * quad > pos[hr]) {
#pragma unroll
            for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
              for (int e = 0; e < 2; ++e) if (key0 + 8 * i + e > pos[hr]) s[4 * i + 2 * hr + e] = -INFINITY;
          }
        }
      }
      uint32_t pf[BKV / 16][4];                                 // P as the A operand of the PV product, bf16 pairs
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < BKV / 8; ++i) mx = fmaxf(mx, fmaxf(s[4 * i + 2 * hr], s[4 * i + 2 * hr + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2)) * a.scale_log2;
        // lazy rescale: keep the old reference unless the max grew by more than 2^8
        if (j == 0) m_ref[hr] = (mx == -INFINITY) ? 0.f : mx;
        else if (mx > m_ref[hr] + 8.f) {
          const float alpha = ex2(m_ref[hr] - mx);
          m_ref[hr] = mx; l[hr] *= alpha;
#pragma unroll
          for (int i = 0; i < HD / 8; ++i) { o[4 * i + 2 * hr] *= alpha; o[4 * i + 2 * hr + 1] *= alpha; }
        }
        float ls = 0.f;
#pragma unroll
        for (int i = 0; i < BKV / 8; ++i) {
          const float p0 = ex2(fmaf(s[4 * i + 2 * hr], a.scale_log2, -m_ref[hr]));
          const float p1 = ex2(fmaf(s[4 * i + 2 * hr + 1], a.scale_log2, -m_ref[hr]));
          ls += p0 + p1;
          pf[i >> 1][(i & 1) * 2 + hr] = pack_bf16(p0, p1);
        }
        l[hr] += ls;
      }
      mbar_wait(&v_full[st], ph);
      if constexpr (PREFIX) {
        if (pre_tile && (long long)(j + 1) * BKV > plen) {   // zero V rows [plen - 128 j, 128): a 128-byte swizzled row stays one row
          const int nvalid = (int)(plen - (long long)j * BKV);
          uint8_t* vs = sV + st * TILE_BYTES;
          for (int idx = threadIdx.x - 128; idx < (BKV - nvalid) * 16; idx += 256) {
            const int row = nvalid + idx / 16, chunk = idx % 16;
            *reinterpret_cast<uint4*>(vs + (chunk / 8) * HALF_BYTES + row * 128 + (chunk % 8) * 16) = make_uint4(0, 0, 0, 0);
          }
          fence_proxy_async_smem();
          named_bar_sync(1, 256);
        }
      }
      const uint32_t va = smem_u32(sV + st * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk)
        wgmma_m64n128k16_rs<1>(o, pf[kk], wgmma_desc_sw128(va + kk * 16 * 128, HALF_BYTES, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      if (lane == 0) mbar_arrive(&v_empty[st]);
    }
    // epilogue: O / l -> bf16 -> out[b, q0 + r, h*128 : +128]; l = sum over the quad
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float lt = l[hr];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const float inv_l = 1.f / lt;
      const long long tok = q0 + r0 + 8 * hr;
      if (tok >= Lq) continue;
      bf16* orow = a.out + (((VARLEN ? row0 : (long long)b * a.Lq) + tok) * a.H + h) * HD;
      if (a.n_out_peers > 0) {
        const long long pr = tok / a.out_rows_per_peer;
        orow = a.out_peer[pr < a.n_out_peers ? pr : 0] + (tok - pr * a.out_rows_per_peer) * a.out_row_stride + a.out_col0 + (long long)h * HD;
      }
#pragma unroll
      for (int i = 0; i < HD / 8; ++i)
        *reinterpret_cast<uint32_t*>(orow + 8 * i + 2 * quad) = pack_bf16(o[4 * i + 2 * hr] * inv_l, o[4 * i + 2 * hr + 1] * inv_l);
    }
  }
}

// (HD, heads, rows, batches) map of bf16 rows of `heads` x 128 elements, tok_stride / batch_stride elements apart, read in
// 128B-swizzled {64, 1, rows_box, 1} boxes
int make_head_map(CUtensorMap* m, const void* base, long long heads, long long rows, long long batches, long long tok_stride,
                  long long batch_stride, uint32_t rows_box) {
  uint64_t dims[4] = {(uint64_t)HD, (uint64_t)heads, (uint64_t)rows, (uint64_t)batches};
  uint64_t str[3] = {(uint64_t)HD * 2, (uint64_t)tok_stride * 2, (uint64_t)batch_stride * 2};
  uint32_t box[4] = {64, 1, rows_box, 1};
  return make_tmap_nd_bf16(m, base, 4, dims, str, box, true);
}

// one CTA per (128 query rows, head, sequence); A is the argument struct of the <VARLEN, PREFIX> form
template <bool VARLEN, bool PREFIX, typename A>
int launch_attn(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const A& a, cudaStream_t st, const char* what) {
  static unsigned long long done = 0;      // one mask per kernel: the limit is an attribute of each kernel
  int rc;
  if ((rc = ensure_dyn_smem(attn_fwd_kernel<VARLEN, PREFIX>, ATT_SMEM, done))) return rc;
  dim3 grid((unsigned)((a.Lq + BQ - 1) / BQ), a.H, a.B);
  attn_fwd_kernel<VARLEN, PREFIX><<<grid, ATT_THREADS, ATT_SMEM, st>>>(tmQ, tmK, tmV, a);
  return check_launch(what);
}

}  // namespace

// Variants 0-3 of the C ABI select among kernels of earlier hardware generations; every variant runs the one kernel above
// (peer-scattered output stays limited to variants 2 and 3, as the ABI documents).
extern "C" size_t evo_attn_fwd_workspace(const evo_attn_params* p, int variant) {
  (void)p; (void)variant;
  return 0;
}

extern "C" int evo_attn_fwd_ws(const evo_attn_params* p, int variant, void* workspace, size_t workspace_bytes, void* stream) {
  (void)workspace; (void)workspace_bytes;
  EVO_REQUIRE(p->hd == HD, "evo_attn_fwd: head_dim %d unsupported (kernel is specialised for 128)", p->hd);
  EVO_REQUIRE(p->q_tok_stride % 8 == 0 && p->kv_tok_stride % 8 == 0 && p->q_batch_stride % 8 == 0 && p->kv_batch_stride % 8 == 0,
              "evo_attn_fwd: strides must be multiples of 8 elements");
  EVO_REQUIRE(p->q_pos0 + p->Lq <= p->Lk, "evo_attn_fwd: queries extend past the keys (q_pos0 %lld + Lq %lld > Lk %lld)",
              (long long)p->q_pos0, (long long)p->Lq, (long long)p->Lk);
  EVO_REQUIRE(variant >= 0 && variant <= 3, "evo_attn_fwd: unknown variant %d", variant);
  EVO_REQUIRE(p->n_out_peers == 0 || variant == 2 || variant == 3, "evo_attn_fwd: peer-scattered output is implemented by variants 2 and 3 only");
  if (p->n_out_peers != 0) {
    EVO_REQUIRE(p->n_out_peers > 0 && p->n_out_peers <= 8 && p->out_peers != nullptr && p->B == 1 && p->out_rows_per_peer > 0 &&
                p->out_rows_per_peer * p->n_out_peers >= p->Lq && p->out_row_stride % 8 == 0 && p->out_col0 % 8 == 0,
                "evo_attn_fwd: peer-scattered output needs B == 1, 1..8 peers covering Lq rows, 16-byte aligned strides");
  }
  if (p->Lq == 0 || p->B == 0) return 0;
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  if ((rc = make_head_map(&tmQ, p->q, p->H, p->Lq, p->B, p->q_tok_stride, p->q_batch_stride, BQ))) return rc;
  if ((rc = make_head_map(&tmK, p->k, p->H, p->Lk, p->B, p->kv_tok_stride, p->kv_batch_stride, BKV))) return rc;
  if ((rc = make_head_map(&tmV, p->v, p->H, p->Lk, p->B, p->kv_tok_stride, p->kv_batch_stride, BKV))) return rc;
  AttArgs a;
  a.out = (bf16*)p->out; a.B = p->B; a.H = p->H; a.Lq = p->Lq; a.Lk = p->Lk; a.q_pos0 = p->q_pos0;
  a.scale_log2 = p->softmax_scale * 1.4426950408889634f;
  a.n_out_peers = p->n_out_peers; a.out_rows_per_peer = p->out_rows_per_peer; a.out_row_stride = p->out_row_stride; a.out_col0 = p->out_col0;
  for (int i = 0; i < 8; ++i) a.out_peer[i] = i < p->n_out_peers ? (bf16*)p->out_peers[i] : nullptr;
  return launch_attn<false, false>(tmQ, tmK, tmV, a, (cudaStream_t)stream, "evo_attn_fwd");
}

extern "C" int evo_attn_fwd_varlen(const evo_attn_varlen_params* p, void* stream) {
  EVO_REQUIRE(p->hd == HD, "evo_attn_fwd_varlen: head_dim %d unsupported (kernel is specialised for 128)", p->hd);
  EVO_REQUIRE(p->q_tok_stride % 8 == 0 && p->kv_tok_stride % 8 == 0, "evo_attn_fwd_varlen: strides must be multiples of 8 elements");
  EVO_REQUIRE(p->n_seq > 0 && p->n_seq <= 65535 && p->H > 0 && p->H <= 65535, "evo_attn_fwd_varlen: bad sequence count %d or head count %d", p->n_seq, p->H);
  int rc;
  if ((rc = check_packed("evo_attn_fwd_varlen", p->cu_seqlens, p->T, p->max_seqlen))) return rc;
  CUtensorMap tmQ, tmK, tmV;
  if ((rc = make_head_map(&tmQ, p->q, p->H, p->T, 1, p->q_tok_stride, p->T * p->q_tok_stride, BQ))) return rc;
  if ((rc = make_head_map(&tmK, p->k, p->H, p->T, 1, p->kv_tok_stride, p->T * p->kv_tok_stride, BKV))) return rc;
  if ((rc = make_head_map(&tmV, p->v, p->H, p->T, 1, p->kv_tok_stride, p->T * p->kv_tok_stride, BKV))) return rc;
  AttArgsV a = {};
  a.out = (bf16*)p->out; a.B = p->n_seq; a.H = p->H; a.Lq = a.Lk = p->max_seqlen; a.q_pos0 = 0;
  a.scale_log2 = p->softmax_scale * 1.4426950408889634f;
  a.cu_seqlens = (const long long*)p->cu_seqlens; a.T = p->T;
  return launch_attn<true, false>(tmQ, tmK, tmV, a, (cudaStream_t)stream, "evo_attn_fwd_varlen");
}

extern "C" int evo_attn_fwd_varlen_prefix(const evo_attn_varlen_prefix_params* p, void* stream) {
  EVO_REQUIRE(p->hd == HD, "evo_attn_fwd_varlen_prefix: head_dim %d unsupported (kernel is specialised for 128)", p->hd);
  EVO_REQUIRE(p->n_seq > 0 && p->n_seq <= 65535 && p->H > 0 && 3 * p->H <= 65535, "evo_attn_fwd_varlen_prefix: bad sequence count %d or head count %d", p->n_seq, p->H);
  int rc;
  if ((rc = check_packed("evo_attn_fwd_varlen_prefix", p->cu_seqlens, p->T, p->max_seqlen))) return rc;
  EVO_REQUIRE(p->cache != nullptr && p->n_cache > 0 && p->cache_len > 0 && p->cache_len < (1LL << 31) && p->prefix_seq != nullptr && p->prefix_len != nullptr,
              "evo_attn_fwd_varlen_prefix: needs a cache of n_cache > 0 rows of 0 < cache_len < 2^31 keys, prefix_seq and prefix_len");
  // q, k, v of the packed rows are heads h, H + h, 2H + h of one map; k, v of the cache are heads h, H + h of the other
  CUtensorMap tmQKV, tmC;
  const long long row = 3LL * p->H * HD, cache_row = 2LL * p->H * HD;
  if ((rc = make_head_map(&tmQKV, p->qkv, 3LL * p->H, p->T, 1, row, p->T * row, BQ))) return rc;
  if ((rc = make_head_map(&tmC, p->cache, 2LL * p->H, p->cache_len, p->n_cache, cache_row, p->cache_len * cache_row, BKV))) return rc;
  AttArgsP a = {};
  a.out = (bf16*)p->out; a.B = p->n_seq; a.H = p->H; a.Lq = a.Lk = p->max_seqlen; a.q_pos0 = 0;
  a.scale_log2 = p->softmax_scale * 1.4426950408889634f;
  a.cu_seqlens = (const long long*)p->cu_seqlens; a.T = p->T;
  a.prefix_seq = (const long long*)p->prefix_seq; a.prefix_len = (const long long*)p->prefix_len; a.cache_len = p->cache_len; a.n_cache = p->n_cache;
  return launch_attn<true, true>(tmQKV, tmC, tmC, a, (cudaStream_t)stream, "evo_attn_fwd_varlen_prefix");
}
