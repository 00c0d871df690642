// Host-side helpers shared by the C-ABI translation units: error reporting, device check,
// TMA tensor-map encoding through the driver entry point (no link-time libcuda dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/f5_b200.h"

namespace f5 {

int set_error(int code, const char* fmt, ...);

#define F5_CHECK_CUDA(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess)                                                               \
      return f5::set_error(F5_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,                  \
                           cudaGetErrorString(_e), __FILE__, __LINE__);                  \
  } while (0)

#define F5_REQUIRE(cond, ...)                                        \
  do {                                                               \
    if (!(cond)) return f5::set_error(F5_ERR_INVALID, __VA_ARGS__);  \
  } while (0)

// 0 if an sm_90 device is current, else F5_ERR_NO_DEVICE (message set)
int device_check();

// bf16 tensor map with 128-byte swizzle and zero OOB fill.  dims/strides innermost first;
// strides in BYTES for dims 1.. (rank-1 entries).  Returns 0 or error.
int make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box);
// the same for 1-byte elements (e4m3 operands of the FP8 mode): 128-byte swizzle, box[0] = 128 elements
int make_tmap_u8(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box);
// Tensor map of an OUTPUT matrix for the GEMM epilogue's TMA stores: elem_bytes 4 (fp32, 32-column boxes = 128 B rows,
// 128-byte swizzle), 2 (bf16, 32-column boxes = 64 B rows, 64-byte swizzle) or 1 (e4m3, 32 B rows, 32-byte swizzle);
// dims (cols, rows per utterance, utterances).
int make_tmap_out(CUtensorMap* map, const void* base, int elem_bytes, uint64_t cols, uint64_t rows, uint64_t batches,
                  uint64_t ld_elems);

inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// SM count of the CURRENT device (cached per device: one process may drive several GPUs)
int sm_count();

// Launch with the programmatic-dependent-launch attribute (see ptx.cuh); F5_PDL=0 disables it.
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                 cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per DEVICE: remember it per (kernel instantiation,
// device) so that one process driving several GPUs does not launch with the default 48 KB limit on the second.
struct SmemAttrOnce {
  unsigned long long done = 0;   // bit d: set on device d
};
template <typename K>
inline cudaError_t ensure_dyn_smem(SmemAttrOnce& once, K kern, int bytes) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 64 && ((once.done >> dev) & 1ull)) return cudaSuccess;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && dev < 64) once.done |= 1ull << dev;
  return e;
}

// ---- launch accounting + optional per-kernel-family device timing (bench.py roofline) ----
// Every launcher opens a ProfScope around its kernel launch.  The launch counter is always on;
// when profiling is enabled (f5_prof_enable) a CUDA event pair brackets the launch on its stream
// and f5_prof_summary returns the summed device time / algorithmic FLOPs / bytes per family.
enum ProfKind { PROF_GEMM = 0, PROF_ATTN = 1, PROF_LN = 2, PROF_OTHER = 3, PROF_NKINDS = 4 };
// In-graph timing (f5_prof_graph_begin): while a slot buffer is installed every ProfScope also hands its kernel one
// slot of two uint64 — [0] atomicMin(globaltimer) when a CTA has passed its dependency wait, [1] atomicMax at CTA
// exit — whose address is baked into a captured CUDA graph, so one replay yields every kernel's in-situ duration.
struct ProfScope {
  ProfScope(int kind, double flops, double bytes, cudaStream_t st);
  ~ProfScope();
  int idx_;
  cudaStream_t st_;
  unsigned long long* slot;   // device pointer or nullptr
};

}  // namespace f5
