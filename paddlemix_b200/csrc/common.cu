// Error channel, device checks and tensor-map encoding for libb200mix.
#include "common.cuh"

#include <cstdlib>
#include <cstring>
#include <mutex>

namespace b200 {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int g_sms = 0;

int ensure_device() {
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_error("no CUDA device: %s (b200mix has no CPU fallback)", cudaGetErrorString(e));
    return B200MIX_ERR_NO_DEVICE;
  }
  static thread_local int checked_dev = -1;
  if (checked_dev == dev) return 0;
  int major = 0, minor = 0, sms = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (major != 9 || minor != 0) {
    set_error("device %d is sm_%d%d; b200mix kernels are sm_90a only", dev, major, minor);
    return B200MIX_ERR_NO_DEVICE;
  }
  g_sms = sms;
  checked_dev = dev;
  return 0;
}

int num_sms() { return g_sms > 0 ? g_sms : 132; }

bool pdl_enabled() {
  static const bool on = (getenv("B200MIX_NO_PDL") == nullptr);
  return on;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
  });
  return fn;
}

int encode_tmap_bf16_sw128(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                           const uint64_t* strides_bytes, const uint32_t* box) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled not available from the driver");
    return B200MIX_ERR_CUDA;
  }
  cuuint64_t gdims[5];
  cuuint64_t gstr[4];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  if ((reinterpret_cast<uintptr_t>(gptr) & 15) != 0) {
    set_error("tensor map base pointer must be 16-byte aligned");
    return B200MIX_ERR_INVALID;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (gstr[i] % 16 != 0) {
      set_error("tensor map stride %d (= %llu bytes) must be a multiple of 16 bytes", i,
                (unsigned long long)gstr[i]);
      return B200MIX_ERR_INVALID;
    }
  }
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(gptr), gdims, gstr, gbox,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu,.. box %u,%u,..)", (int)r, rank,
              (unsigned long long)gdims[0], (unsigned long long)(rank > 1 ? gdims[1] : 0), gbox[0],
              rank > 1 ? gbox[1] : 0);
    return B200MIX_ERR_CUDA;
  }
  return 0;
}

}  // namespace b200

extern "C" {

const char* b200mix_last_error(void) { return b200::g_err; }
const char* b200mix_version(void) { return "b200mix 0.1 (sm_90a)"; }

int b200mix_init(int device) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    cudaGetLastError();
    b200::set_error("cudaSetDevice(%d) failed: %s (b200mix has no CPU fallback)", device, cudaGetErrorString(e));
    return B200MIX_ERR_NO_DEVICE;
  }
  return b200::ensure_device();
}

/* Zero `bytes` bytes on the caller's stream (a memset node under stream capture): the folded-LayerNorm statistics tables
 * (b200mix_epilogue.stats_out) must be zero before the producing GEMM runs. */
int b200mix_zero_bytes(void* ptr, int64_t bytes, void* stream) {
  if (int rc = b200::ensure_device()) return rc;
  B200_CHECK_ARG(ptr && bytes >= 0, "zero_bytes: bad arguments");
  B200_CUDA(cudaMemsetAsync(ptr, 0, (size_t)bytes, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

int b200mix_num_sms(void) {
  if (b200::ensure_device() != 0) return B200MIX_ERR_NO_DEVICE;
  return b200::num_sms();
}

}  // extern "C"
