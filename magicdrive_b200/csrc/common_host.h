// Host-side helpers shared by the C-ABI translation units.
#pragma once
#include <stdarg.h>
#include <stdio.h>

namespace mdb {
char* error_buffer();  // thread-local, 512 bytes (defined in capi_misc.cu)
inline int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(error_buffer(), 512, fmt, ap);
  va_end(ap);
  return code;
}
}  // namespace mdb

#ifdef MDB_NEED_TENSORMAP
#include <cuda.h>
#include <cuda_runtime.h>

#include <mutex>
namespace mdb {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);
// cuTensorMapEncodeIm2col, obtained the same way
inline EncodeIm2colFn get_encode_im2col() {
  static EncodeIm2colFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeIm2colFn>(p);
  });
  return fn;
}
}  // namespace mdb
#endif

#ifdef __CUDACC__
#include <cuda_runtime.h>
#include <stdlib.h>
namespace mdb {
// Programmatic dependent launch: the kernel may start while its stream predecessor drains; every kernel launched
// this way executes griddepcontrol.wait before touching global memory (see pdl_wait() in ptx.cuh / kernels).
// Who decides: MDB_PDL=0 | 1 in the environment forces it off / on for every launch; otherwise the caller switches it per
// region with mdb_set_pdl() (off by default).  It pays only where ONE stream is busy: with two concurrent branches the
// early-scheduled dependents park on SMs the other branch would have filled (measured: whole step 3 % slower).
inline int& pdl_region_flag() {
  static int v = 0;
  return v;
}
inline bool pdl_enabled() {
  static int forced = -2;
  if (forced == -2) {
    const char* e = getenv("MDB_PDL");
    forced = e ? ((e[0] == '1') ? 1 : 0) : -1;
  }
  return forced >= 0 ? forced == 1 : pdl_region_flag() == 1;
}
// append the PDL attribute to a launch that already carries `n_attrs` attributes (attrs must have room for one more)
inline void add_pdl_attr(cudaLaunchConfig_t& cfg, cudaLaunchAttribute* attrs, unsigned n_attrs) {
  if (pdl_enabled()) {
    attrs[n_attrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[n_attrs].val.programmaticStreamSerializationAllowed = 1;
    ++n_attrs;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = n_attrs;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
}  // namespace mdb
#endif

#define MDB_CHECK_LAUNCH(name)                                                                   \
  do {                                                                                           \
    cudaError_t e__ = cudaGetLastError();                                                        \
    if (e__ != cudaSuccess) return mdb::set_error(MDB_ERR_CUDA, name ": %s", cudaGetErrorString(e__)); \
  } while (0)
