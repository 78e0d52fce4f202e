// Host-side setup shared by the wgmma kernels (conv_tc, conv_stem, tblock_tc, attn_tc): the tensor-map format of their
// operands and the per-device state their launches need.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>
#include <string>

namespace vt {

// Per-device tables below hold this many devices; a higher device index is rejected as cudaErrorInvalidDevice.
constexpr int kMaxDevices = 64;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// The driver's cuTensorMapEncodeTiled, looked up once; null when the driver does not provide it.
inline EncodeTiledFn tmap_encoder() {
  static const EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
                    q == cudaDriverEntryPointSuccess;
    return ok ? (EncodeTiledFn)f : nullptr;
  }();
  return fn;
}

// Tiled tensor map of 16-bit elements (bf16, or one fp16 plane of the split mode) in the layout every wgmma operand is
// loaded in: 128-byte swizzle, which the shared-memory descriptors (tcx::desc_lo / desc_hi in tc_ptx.cuh) assume, and
// zero fill out of bounds.  dims[0] is the contiguous dimension; strides[i] is the byte stride of dimension i + 1.  On
// failure writes "cuTensorMapEncodeTiled(<what>) failed: <code>" to err.
inline bool encode_tmap_16b(CUtensorMap* map, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides,
                            const cuuint32_t* box, const char* what, std::string& err) {
  const EncodeTiledFn enc = tmap_encoder();
  if (!enc) { err = "cuTensorMapEncodeTiled unavailable"; return false; }
  const cuuint32_t elem_strides[5] = {1, 1, 1, 1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box,
                         elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { err = std::string("cuTensorMapEncodeTiled(") + what + ") failed: " + std::to_string((int)r); return false; }
  return true;
}

// The calling thread's current device, 0 <= dev < kMaxDevices.
inline cudaError_t current_device(int& dev) {
  const cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  return dev >= 0 && dev < kMaxDevices ? cudaSuccess : cudaErrorInvalidDevice;
}

// SM count of device `dev` (from current_device), queried once per device.
inline int device_sms(int dev) {
  static std::atomic<int> sms[kMaxDevices];   // 0: not queried yet
  int n = sms[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
    sms[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// Raises the dynamic shared-memory limit of a fixed set of kernels, once per device: the attribute applies to the current
// device only.  One static instance per kernel set.  Threads that race on a device both set it, which is harmless.
class SmemLimitOnce {
 public:
  template <class... Kernels>
  cudaError_t ensure(int dev, int bytes, Kernels... kernels) {
    if (done_[dev].load(std::memory_order_acquire)) return cudaSuccess;
    cudaError_t e = cudaSuccess;
    for (const void* k : {(const void*)kernels...}) {
      const cudaError_t x = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
      if (x != cudaSuccess) e = x;
    }
    if (e == cudaSuccess) done_[dev].store(true, std::memory_order_release);
    return e;
  }

 private:
  std::atomic<bool> done_[kMaxDevices] = {};
};

}  // namespace vt
