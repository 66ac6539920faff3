// Library-wide host runtime: the thread-local error message, the device check every entry point makes first, the
// tensor-map encoder of the TMA kernels, the per-kernel launch setup, and the exported version / error / device / option
// calls.
#include "omt_common.cuh"
#include <mutex>
#include <string.h>

namespace omt {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int g_pdl = 0;   // programmatic dependent launch is opt-in (dependent CTAs hold SM resources during the tail)

static std::atomic<int> g_sms[MAX_DEVICES];   // 0 not checked yet, -1 not sm_90, else the device's SM count
static thread_local int t_dev = -1;            // the launch device: the one check_device() last accepted on this thread

int check_device() {
  int dev = 0;
  OMT_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= MAX_DEVICES) { set_error("device ordinal %d out of range", dev); return OMT_E_ARG; }
  int sms = g_sms[dev].load(std::memory_order_relaxed);
  if (sms == 0) {
    cudaDeviceProp p;
    OMT_CUDA(cudaGetDeviceProperties(&p, dev));
    sms = (p.major == 9 && p.minor == 0) ? p.multiProcessorCount : -1;
    g_sms[dev].store(sms, std::memory_order_relaxed);
  }
  if (sms < 0) {
    set_error("omnitok_b200 kernels are built for sm_90a (H100) only (no fallback path)");
    return OMT_E_ARCH;
  }
  t_dev = dev;
  return OMT_OK;
}

int sm_count() { return g_sms[t_dev].load(std::memory_order_relaxed); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_tiled(CUtensorMap* m, CUtensorMapDataType dt, const void* base, int rank, const cuuint64_t* dims,
                 const cuuint64_t* strides, const cuuint32_t* box) {
  static const EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    const bool found = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
                       qres == cudaDriverEntryPointSuccess;
    return found ? reinterpret_cast<EncodeTiledFn>(p) : nullptr;
  }();
  if (fn == nullptr) { set_error("cuTensorMapEncodeTiled entry point not found"); return OMT_E_CUDA; }
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, dt, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return OMT_E_CUDA; }
  return OMT_OK;
}

// Serialises the first-time setup and the growth of every KernelSetup; the fast paths only load.
static std::mutex g_setup_lock;

int KernelSetup::grow(const void* kernel, int dev, size_t bytes) {
  if ((size_t)smem_[dev].load(std::memory_order_relaxed) >= bytes) return OMT_OK;   // another thread got here first
  OMT_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  smem_[dev].store((int)bytes, std::memory_order_release);
  return OMT_OK;
}

int KernelSetup::smem_impl(const void* kernel, size_t bytes) {
  const int dev = t_dev;
  if ((size_t)smem_[dev].load(std::memory_order_acquire) >= bytes) return OMT_OK;
  std::lock_guard<std::mutex> lock(g_setup_lock);
  return grow(kernel, dev, bytes);
}

int KernelSetup::resident_impl(const void* kernel, int threads, size_t bytes, int* ctas) {
  const int dev = t_dev;
  int n = ctas_[dev].load(std::memory_order_acquire);
  if (n == 0) {
    std::lock_guard<std::mutex> lock(g_setup_lock);
    n = ctas_[dev].load(std::memory_order_relaxed);
    if (n == 0) {
      const int rc = grow(kernel, dev, bytes);
      if (rc != OMT_OK) return rc;
      int per_sm = 0;
      OMT_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, bytes));
      OMT_REQUIRE(per_sm > 0, "no CTA of %d threads and %zu bytes of shared memory fits on an SM of device %d", threads,
                  bytes, dev);
      n = per_sm * sm_count();
      ctas_[dev].store(n, std::memory_order_release);
    }
  }
  *ctas = n;
  return OMT_OK;
}

extern int g_peg_kernel; extern int g_attn_kernel; extern int g_f16_bn; extern int g_attn_f16_ctas;

}  // namespace omt

extern "C" int omt_abi_version(void) { return OMT_ABI_VERSION; }
extern "C" const char* omt_last_error(void) { return omt::g_err; }

extern "C" int omt_device_info(int* sms, int* major, int* minor) {
  int dev = 0;
  OMT_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  OMT_CUDA(cudaGetDeviceProperties(&p, dev));
  if (sms) *sms = p.multiProcessorCount;
  if (major) *major = p.major;
  if (minor) *minor = p.minor;
  return OMT_OK;
}

extern "C" int omt_set_option(const char* name, int value) {
  if (name == nullptr) return OMT_E_ARG;
  if (strcmp(name, "pdl") == 0) { omt::g_pdl = value ? 1 : 0; return OMT_OK; }
  if (strcmp(name, "peg_kernel") == 0) {
    if (value != 3 && value != 4) { omt::set_error("peg_kernel must be 3 or 4"); return OMT_E_ARG; }
    omt::g_peg_kernel = value;
    return OMT_OK;
  }
  if (strcmp(name, "attn_kernel") == 0) {
    if (value != 1 && value != 3) { omt::set_error("attn_kernel must be 1 or 3"); return OMT_E_ARG; }
    omt::g_attn_kernel = value;
    return OMT_OK;
  }
  if (strcmp(name, "f16_bn") == 0) {
    if (value != 0 && value != 128 && value != 256) { omt::set_error("f16_bn must be 0, 128 or 256"); return OMT_E_ARG; }
    omt::g_f16_bn = value;
    return OMT_OK;
  }
  if (strcmp(name, "attn_f16_ctas") == 0) {
    if (value != 1 && value != 2) { omt::set_error("attn_f16_ctas must be 1 or 2"); return OMT_E_ARG; }
    omt::g_attn_f16_ctas = value;
    return OMT_OK;
  }
  omt::set_error("unknown option %s", name);
  return OMT_E_ARG;
}
