// Shared device helpers for the evo_b200 sm_90a kernels: error plumbing, bf16
// rounding helpers, and thin inline-PTX wrappers for mbarrier / TMA / wgmma.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

namespace evo {

// ---- error plumbing (C ABI: 0 = ok, negative = error, message via evo_last_error) ----
void set_error(const char* fmt, ...);
int  check_launch(const char* what);   // cudaGetLastError -> -3 + message

#define EVO_REQUIRE(cond, ...)                                   \
  do { if (!(cond)) { ::evo::set_error(__VA_ARGS__); return -1; } } while (0)
#define EVO_CUDA(call)                                                              \
  do { cudaError_t e_ = (call); if (e_ != cudaSuccess) {                            \
    ::evo::set_error("%s failed: %s", #call, cudaGetErrorString(e_)); return -2; } } while (0)

typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 bf162;

// ---- bf16 helpers: "round to bf16 and come back" marks a rounding point of the reference ----
__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ float bf_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  bf162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ uint32_t ld_pair(const bf16* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); }

// The reference's rounding chains (include/evo_b200.h states them per entry point), written once for every kernel that
// applies them.  A "word" is a bf16 pair (columns n, n + 1) packed as pack_bf16 packs it; arguments named for a bf16 tensor
// of the reference hold bf16 values.  Where a chain has a scalar and a word form, each keeps the order of operations its
// callers compile best with; both round at the same points.

// F.gelu (erf form).  erff stays IEEE: the library is built without --use_fast_math.
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// ParallelGatedMLP, act(l1 x) * l2 x: bf16(gelu(l1)) * l2 of the bf16 linear outputs l1, l2; rounded on store.
// gelu_gate_acc takes the fp32 sums a, b of the two linear layers instead: l1 = bf16(a), l2 = bf16(b).
__device__ __forceinline__ float gelu_gate(float l1, float l2) { return rbf(gelu_erf(l1)) * l2; }
__device__ __forceinline__ float gelu_gate_acc(float a, float b) { return rbf(gelu_erf(rbf(a))) * rbf(b); }

// nn.Linear, then the residual add: C = bf16(bf16(acc + bias) + r).  Without a residual the rounding of acc + bias is the
// store's; with one, acc + bias is rounded here and the sum is rounded on store.  linear_word reads the residual word through
// load_resid() after the bias add; it is not called without RESID.
template <bool BIAS, bool RESID>
__device__ __forceinline__ float linear_out(float acc, float bias, float r) {
  if constexpr (BIAS) acc += bias;
  if constexpr (RESID) acc = rbf(acc) + r;
  return acc;
}
template <bool BIAS, bool RESID, typename LoadResid>
__device__ __forceinline__ uint32_t linear_word(float acc0, float acc1, uint32_t bias, LoadResid load_resid) {
  if constexpr (BIAS) { acc0 += bf_lo(bias); acc1 += bf_hi(bias); }
  if constexpr (RESID) { const uint32_t r = load_resid(); acc0 = rbf(acc0) + bf_lo(r); acc1 = rbf(acc1) + bf_hi(r); }
  return pack_bf16(acc0, acc1);
}
// the residual add of linear_out on a word y that already holds bf16(acc + bias)
__device__ __forceinline__ uint32_t resid_word(uint32_t y, uint32_t r) { return pack_bf16(bf_lo(y) + bf_lo(r), bf_hi(y) + bf_hi(r)); }

// NeoX rotary (flash_attn apply_rotary) of head column c against c + 64, x and y their bf16 inputs, c and s the cos/sin table
// entries of the token's position: fp32 arithmetic, one rounding (xr to column c, yr to c + 64).
__device__ __forceinline__ void rope_rotate(float x, float y, float c, float s, bf16& xr, bf16& yr) {
  xr = __float2bfloat16_rn(x * c - y * s);
  yr = __float2bfloat16_rn(x * s + y * c);
}
// the same for columns (c, c + 1) against (c + 64, c + 65), cos/sin given as table words
__device__ __forceinline__ void rope_words(float x0, float x1, float y0, float y1, uint32_t cw, uint32_t sw, uint32_t& o1, uint32_t& o2) {
  const float cl = bf_lo(cw), ch = bf_hi(cw), sl = bf_lo(sw), sh = bf_hi(sw);
  o1 = pack_bf16(x0 * cl - y0 * sl, x1 * ch - y1 * sh);
  o2 = pack_bf16(x0 * sl + y0 * cl, x1 * sh + y1 * ch);
}
// the Wqkv projection with rotary (EVO_EPI_BIAS_ROPE): x = bf16(acc + bias), the reference's qkv tensor, for columns
// (col, col + 1) and y for (col + 64, col + 65); then, when `rotate` (q and k heads), the rotation of head columns (c, c + 1)
// with row l of the (positions, 64) cos/sin tables; else x and y as they are.
__device__ __forceinline__ void bias_rope_words(float ax0, float ax1, float ay0, float ay1, const bf16* bias, int col, bool rotate,
                                                const bf16* cos, const bf16* sin, long long l, int c, uint32_t& o1, uint32_t& o2) {
  const uint32_t b1 = ld_pair(bias + col), b2 = ld_pair(bias + col + 64);
  const float x0 = rbf(ax0 + bf_lo(b1)), x1 = rbf(ax1 + bf_hi(b1));
  const float y0 = rbf(ay0 + bf_lo(b2)), y1 = rbf(ay1 + bf_hi(b2));
  if (rotate) {
    rope_words(x0, x1, y0, y1, ld_pair(cos + l * 64 + c), ld_pair(sin + l * 64 + c), o1, o2);
  } else {
    o1 = pack_bf16(x0, x1); o2 = pack_bf16(y0, y1);
  }
}

// RMSNorm (layers.RMSNorm.forward, bf16 tensor ops): n = bf16(||x||), n = bf16(n * D^-1/2), n = bf16(n + eps), y = bf16(x / n),
// out = bf16(scale * y).  rms_rinv takes the row's fp32 sum of squares and returns 1/n: the quotient is x * rcp(n) (one
// reciprocal per row instead of an IEEE division per element, which made the kernels instruction-bound at ~50 % of HBM speed).
// That is exact after the bf16 rounding: x and n have 8-bit significands, so x/n is either exactly representable or at least
// 2^-17 (relative) away from every bf16 rounding midpoint (a 9-bit significand m with x = n*m would need x to have >= 9
// significant bits), while x * rcp_rn(n) is within 2^-23 of x/n: both round to the same bf16.
__device__ __forceinline__ float rms_rinv(float sumsq, float inv_sqrt_d, float eps) {
  float n = rbf(sqrtf(sumsq));
  n = rbf(n * inv_sqrt_d);
  n = rbf(n + eps);
  return __frcp_rn(n);
}
__device__ __forceinline__ uint32_t rms_word(uint32_t x, uint32_t scale, float rinv) {
  const float y0 = rbf(bf_lo(x) * rinv), y1 = rbf(bf_hi(x) * rinv);
  return pack_bf16(bf_lo(scale) * y0, bf_hi(scale) * y1);
}

// two-lane fp32 arithmetic with one IEEE round-to-nearest per lane (never contracted into an FMA)
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}

// ---- TMA (cp.async.bulk.tensor) ----
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// 1-D bulk copy of `bytes` (a multiple of 16, both addresses 16-byte aligned) into shared memory, completing on `bar`
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads/writes across an outstanding wgmma
template <int N> __device__ __forceinline__ void wgmma_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor for a 128-byte swizzled operand tile (what a TMA box {64 bf16, rows} with SWIZZLE_128B
// writes: rows of 128 B, 8-row groups 1024 B apart).  K-major: sbo = 1024 (the next 8 rows), +32 B per k16 step.
// MN-major (V of the PV product): lbo = byte distance between 64-wide MN halves, sbo = 1024 (the next 8 rows of K).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);        // [0,14)  start address >> 4
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;   // [16,30) leading byte offset
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;   // [32,46) stride byte offset
  d |= (uint64_t)1 << 62;                             // [62,64) layout = SWIZZLE_128B
  return d;
}
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) { return wgmma_desc_sw128(smem_addr, 16, 1024); }

// register budget hand-off between the producer and the consumer warpgroups of a warp-specialised kernel
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// host: TMA descriptor encode through the driver entry point (no link-time libcuda)
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer,
                      uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle128);

int make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                      const uint32_t* box, bool swizzle128);

// host: the packed-sequence geometry every varlen entry point needs (cu_seqlens given, 0 < max_seqlen <= T < 2^31); on failure
// returns -1 with the reason under `what`, the entry point's name.  Touches no device state.
int check_packed(const char* what, const int64_t* cu_seqlens, int64_t T, int64_t max_seqlen);

int device_sm_count();     // of the CURRENT device (cached per device ordinal)

int current_device();      // cudaGetDevice, -1 on error

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE attribute: `mask` keeps one "done" bit per device
// ordinal, so a process that drives a second GPU (model moved to cuda:1) raises the limit there too.
template <typename K>
inline int ensure_dyn_smem(K kern, int bytes, unsigned long long& mask) {
  const int dev = current_device();
  if (dev < 0 || dev >= 64 || !((mask >> dev) & 1ull)) {
    EVO_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    if (dev >= 0 && dev < 64) mask |= 1ull << dev;
  }
  return 0;
}
int pdl_level();         // evo_set_pdl(): 0 off, 1 all decode-step kernels, 2 weight-streaming GEMM only, 3 + the row-norm kernel, 4 + hyena_step

// Programmatic dependent launch: every kernel that may be launched with the attribute calls pdl_wait() before it
// first reads data written by (or writes data read by) the previous kernel; both are no-ops in a normal launch.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// host: kernel launch that adds the programmatic-serialization attribute when evo_set_pdl(1) is active (or, for a kernel launched
// through launch_pdl_light, at level 3 as well)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_at(int min_level_extra, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  if (pdl_level() == 1 || (min_level_extra > 0 && pdl_level() >= min_level_extra)) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
  }
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_light(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  return launch_pdl_at(3, kern, grid, block, smem, st, args...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  if (pdl_level() == 1) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
  }
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

}  // namespace evo
