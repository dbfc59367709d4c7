// Host-side helpers shared by the C-ABI translation units: error channel, driver entry points, tensor maps.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/b200mix.h"

namespace b200 {

void set_error(const char* fmt, ...);
int ensure_device();  // 0 if an sm_90 device is current, else negative status (with message)
int num_sms();
// K split of the weight-streaming GEMMs (gemm.cu skinny_linear_kernel, linear_w8.cu): ctas_n CTAs along N, kcap = the K
// elements one CTA stages in one pass, slots = CTAs resident on the machine. Returns the cluster size (<= 8) and the K
// elements per cluster rank (a multiple of 256). b200mix_debug_skinny_splits forces the split of both.
void skinny_split(int ctas_n, int K, int kcap, int slots, int* splits, int* kpart);

#define B200_CHECK_ARG(cond, ...)                 \
  do {                                            \
    if (!(cond)) {                                \
      ::b200::set_error(__VA_ARGS__);             \
      return B200MIX_ERR_INVALID;                 \
    }                                             \
  } while (0)

#define B200_CUDA(call)                                                                              \
  do {                                                                                               \
    cudaError_t _e = (call);                                                                         \
    if (_e != cudaSuccess) {                                                                         \
      ::b200::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return B200MIX_ERR_CUDA;                                                                       \
    }                                                                                                \
  } while (0)

#define B200_LAUNCH_CHECK()                                                                       \
  do {                                                                                            \
    cudaError_t _e = cudaGetLastError();                                                          \
    if (_e != cudaSuccess) {                                                                      \
      ::b200::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return B200MIX_ERR_CUDA;                                                                    \
    }                                                                                             \
  } while (0)

bool pdl_enabled();  // false when B200MIX_NO_PDL is set

// Launch with the programmatic-dependent-launch attribute (and optionally a cluster of `cluster_x` CTAs). Every kernel
// launched through this helper calls pdl_wait() before its first global-memory access.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Encode a bf16 tiled tensor map with 128-byte swizzle and zero OOB fill.
// dims/box have `rank` entries (innermost first); strides_bytes has rank-1 entries (for dims 1..rank-1).
int encode_tmap_bf16_sw128(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                           const uint64_t* strides_bytes, const uint32_t* box);

}  // namespace b200
