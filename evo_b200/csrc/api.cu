// C-ABI plumbing: error string, launch counter, TMA descriptor encode, packed-geometry check, device query.
#include "common.cuh"
#include "../../include/evo_b200.h"
#include <stdarg.h>
#include <string.h>
#include <atomic>

namespace evo {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};
static std::atomic<int> g_pdl{0};
int pdl_level() { return g_pdl.load(std::memory_order_relaxed); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return -3;
  }
  return 0;
}

typedef CUresult (*encode_fn_t)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_fn_t get_encode_fn() {
  static encode_fn_t fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || !p) return nullptr;
    fn = (encode_fn_t)p;
  }
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer,
                      uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle128) {
  encode_fn_t fn = get_encode_fn();
  EVO_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  EVO_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d): inner=%llu outer=%llu stride=%llu box=%ux%u base=%p",
              (int)r, (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)row_stride_bytes,
              box_inner, box_outer, base);
  return 0;
}

int make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                      const uint32_t* box, bool swizzle128) {
  encode_fn_t fn = get_encode_fn();
  EVO_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t d[5]; cuuint64_t st[4]; cuuint32_t bx[5]; cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; bx[i] = box[i]; es[i] = 1; if (i + 1 < rank) st[i] = strides_bytes[i]; }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), d, st, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  EVO_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(rank %d) failed (%d): dims0=%llu dims1=%llu box0=%u box1=%u base=%p",
              rank, (int)r, (unsigned long long)d[0], (unsigned long long)d[1], bx[0], bx[1], base);
  return 0;
}

int check_packed(const char* what, const int64_t* cu_seqlens, int64_t T, int64_t max_seqlen) {
  EVO_REQUIRE(cu_seqlens != nullptr && max_seqlen > 0 && max_seqlen <= T && T < (1LL << 31),
              "%s: needs cu_seqlens and 0 < max_seqlen <= T < 2^31 (max_seqlen %lld, T %lld)", what, (long long)max_seqlen, (long long)T);
  return 0;
}

int current_device() {
  int dev = 0;
  return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}

int device_sm_count() {
  static int cache[64] = {0};
  const int dev = current_device();
  if (dev < 0) return 132;
  if (dev < 64 && cache[dev]) return cache[dev];
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  if (dev < 64) cache[dev] = n;
  return n;
}

}  // namespace evo

extern "C" {
const char* evo_last_error(void) { return evo::g_err; }
int evo_abi_version(void) { return 2; }
int64_t evo_launch_count(void) { return evo::g_launches.load(); }
void evo_reset_launch_count(void) { evo::g_launches.store(0); }
void evo_note_graph_replay(int64_t launches) { evo::g_launches.fetch_add(launches); }
int evo_set_pdl(int level) { return evo::g_pdl.exchange(level < 0 ? 0 : (level > 4 ? 4 : level)); }
}
