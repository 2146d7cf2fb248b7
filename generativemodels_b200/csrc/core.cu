// Error reporting, version and device checks for libb200gen.so.
#include "common.cuh"

namespace b200 {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
  return B200_ECUDA;
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace b200

extern "C" const char* b200_last_error_string(void) { return b200::g_err; }

extern "C" int b200_version(void) { return 200; }

#ifdef B200_H16_IS_BF16
extern "C" int b200_act_dtype(void) { return B200_H16_BF16; }
#else
extern "C" int b200_act_dtype(void) { return B200_H16_FP16; }
#endif

extern "C" int b200_sm_count(void) { return b200::sm_count(); }

extern "C" int b200_device_check(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return b200::cuda_fail(e, "cudaGetDevice");
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) {
    b200::set_error("libb200gen needs an sm_90 GPU (wgmma/TMA, built for sm_90a); device %d is sm_%d%d", dev, major,
                    minor);
    return B200_ENODEV;
  }
  return B200_OK;
}

extern "C" int b200_abi_sizeof(int which) {
  switch (which) {
    case 0: return (int)sizeof(b200_igemm_params);
    case 1: return (int)sizeof(b200_gn_stats_params);
    case 2: return (int)sizeof(b200_gn_apply_params);
    case 3: return (int)sizeof(b200_ddim_coef);
    case 4: return (int)sizeof(b200_ddpm_coef);
    case 5: return (int)sizeof(b200_pndm_coef);
    case 6: return (int)sizeof(b200_igemm_seg);
    case 7: return (int)sizeof(b200_flash_params);
    case 8: return (int)sizeof(b200_kl_coef);
    case 9: return (int)sizeof(b200_repack_block);
    default: return -1;
  }
}
