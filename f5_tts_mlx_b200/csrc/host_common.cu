#include "host_common.h"

#include <atomic>
#include <mutex>
#include <vector>

namespace f5 {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int sm_count() {
  static int cache[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev >= 0 && dev < 64 && cache[dev] > 0) return cache[dev];
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  if (dev >= 0 && dev < 64) cache[dev] = sms;
  return sms;
}

int device_check() {
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return set_error(F5_ERR_NO_DEVICE,
                     "no CUDA device (%s); libf5b200 has no CPU fallback", cudaGetErrorString(e));
  }
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9)
    return set_error(F5_ERR_NO_DEVICE,
                     "device %d is sm_%d%d; libf5b200 is built for sm_90a only", dev, major,
                     minor);
  return 0;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

static int make_tmap_any(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapDataType dt,
                         CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B);
int make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap_any(map, base, rank, dims, strides_bytes, box, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
}
int make_tmap_u8(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap_any(map, base, rank, dims, strides_bytes, box, CU_TENSOR_MAP_DATA_TYPE_UINT8);
}
int make_tmap_u8_sw64(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap_any(map, base, rank, dims, strides_bytes, box, CU_TENSOR_MAP_DATA_TYPE_UINT8,
                       CU_TENSOR_MAP_SWIZZLE_64B);
}
static int make_tmap_any(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapDataType dt,
                         CUtensorMapSwizzle swz) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(F5_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return set_error(F5_ERR_INVALID, "TMA base pointer %p not 16-byte aligned", base);
  for (int i = 0; i + 1 < rank; ++i)
    if (gstr[i] % 16 != 0)
      return set_error(F5_ERR_INVALID, "TMA stride %d = %llu bytes not a multiple of 16", i,
                       (unsigned long long)gstr[i]);
  CUresult r = enc(map, dt, (cuuint32_t)rank, const_cast<void*>(base),
                   gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(F5_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

int make_tmap_out(CUtensorMap* map, const void* base, int elem_bytes, uint64_t cols, uint64_t rows, uint64_t batches,
                  uint64_t ld_elems) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(F5_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return set_error(F5_ERR_INVALID, "TMA store base pointer %p not 16-byte aligned", base);
  if ((ld_elems * elem_bytes) % 16 != 0)
    return set_error(F5_ERR_INVALID, "TMA store row pitch %llu bytes not a multiple of 16",
                     (unsigned long long)(ld_elems * elem_bytes));
  cuuint64_t gdim[3] = {cols, rows, batches};
  cuuint64_t gstr[2] = {ld_elems * elem_bytes, ld_elems * elem_bytes * rows};
  cuuint32_t bx[3] = {32, 128, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapDataType odt = elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                  : (elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8);
  const CUtensorMapSwizzle osw = elem_bytes == 4 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : (elem_bytes == 2 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  CUresult r = enc(map, odt, 3,
                   const_cast<void*>(base), gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   osw,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(F5_ERR_CUDA, "cuTensorMapEncodeTiled (output map) failed with CUresult %d", (int)r);
  return 0;
}

// ---------------------------------------------------------------------------------------------
// launch accounting / in-graph timing
// ---------------------------------------------------------------------------------------------
static std::mutex g_prof_mu;
static std::atomic<long long> g_launches{0};
struct GraphSlotMeta { int kind; double flops, bytes; };
static unsigned long long* g_gslots = nullptr;
static int g_gslots_cap = 0;
static std::vector<GraphSlotMeta> g_gmeta;

ProfScope::ProfScope(int kind, double flops, double bytes) : slot(nullptr) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (g_gslots != nullptr) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    if ((int)g_gmeta.size() < g_gslots_cap) {
      slot = g_gslots + 2 * g_gmeta.size();
      g_gmeta.push_back({kind, flops, bytes});
    }
  }
}

}  // namespace f5

extern "C" {
long long f5_launch_count(void) { return f5::g_launches.load(); }
// In-graph timing: install a device buffer of `max_slots` x 2 uint64 (the caller fills [*,0] with UINT64_MAX and
// [*,1] with 0 before each run); slot i belongs to the i-th ProfScope opened from now on.  NULL uninstalls.
int f5_prof_graph_begin(void* slots, int32_t max_slots) {
  std::lock_guard<std::mutex> lk(f5::g_prof_mu);
  f5::g_gslots = reinterpret_cast<unsigned long long*>(slots);
  f5::g_gslots_cap = slots ? max_slots : 0;
  if (slots) f5::g_gmeta.clear();
  return 0;
}
// kind (PROF_* : 0 gemm, 1 attention, 2 ln_modulate, 3 other) and algorithmic flops / bytes of every slot handed out
// since the last f5_prof_graph_begin; returns the slot count
int f5_prof_graph_meta(int32_t* kinds, double* flops, double* bytes, int32_t cap) {
  std::lock_guard<std::mutex> lk(f5::g_prof_mu);
  const int n = (int)f5::g_gmeta.size();
  for (int i = 0; i < n && i < cap; ++i) {
    if (kinds) kinds[i] = f5::g_gmeta[i].kind;
    if (flops) flops[i] = f5::g_gmeta[i].flops;
    if (bytes) bytes[i] = f5::g_gmeta[i].bytes;
  }
  return n;
}
// sizeof() of every struct of the ABI, so a binding can verify its own layout at load time
int f5_struct_sizes(int32_t* out, int32_t n) {
  const int32_t v[10] = {(int32_t)sizeof(f5_gemm_args),          (int32_t)sizeof(f5_convnext_weights),
                         (int32_t)sizeof(f5_dit_block_weights),  (int32_t)sizeof(f5_dit_weights),
                         (int32_t)sizeof(f5_dit_buffers),        (int32_t)sizeof(f5_vocos_block_weights),
                         (int32_t)sizeof(f5_vocos_weights),      (int32_t)sizeof(f5_vocos_buffers),
                         (int32_t)sizeof(f5_duration_weights),   (int32_t)sizeof(f5_duration_buffers)};
  for (int i = 0; i < n && i < 10; ++i) out[i] = v[i];
  return 10;
}
const char* f5_last_error(void) { return f5::g_err; }
int f5_abi_version(void) { return 2007; }
int f5_device_check(void) { return f5::device_check(); }
}
