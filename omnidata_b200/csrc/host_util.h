// Host-side helpers shared by the C-ABI entry points: error reporting, launch accounting,
// device properties and the TMA tensor-map encoder (resolved from the driver at run time so that
// the library links against libcudart only).
#pragma once

#include <cmath>

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/omnidata_b200.h"

namespace odb {

int fail(int status, const char* msg);
int fail_cuda(cudaError_t e, const char* where);
int check_launch(const char* where);
void count_launch();
int num_sms();            // of the current device (cached per device)
constexpr int kMaxDevices = 64;
int current_device();     // cudaGetDevice, clamped to [0, kMaxDevices)

int encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, int rank, void* base,
                 const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box,
                 const cuuint32_t* elem_strides, CUtensorMapSwizzle swizzle);

bool pdl_enabled();

// argument checks of the entry points
inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }
// b images (a grid dimension) of h x w planes
inline bool planes_ok(int32_t b, int32_t h, int32_t w) {
  return b >= 1 && b <= 65535 && h >= 1 && h <= 65535 && w >= 1 && w <= 65535;
}
// mask argument of the metrics and the sparse alignment: NULL with ODB_MASK_NONE, else uint8 or (4-byte aligned) fp32
inline bool metric_mask_ok(const void* mask, int32_t kind) {
  if (kind == ODB_MASK_NONE) return mask == nullptr;
  if (kind == ODB_MASK_U8) return mask != nullptr;
  return kind == ODB_MASK_F32 && mask != nullptr && aligned(mask, 4);
}
// The per-pixel reductions (metrics.cu, ensemble.cu) cut every image into fixed slabs of kSlab pixels, so the partition
// depends on h x w only, never on the batch.
constexpr long long kSlab = 4096;
inline int slab_count(int32_t h, int32_t w) { return (int)(((long long)h * w + kSlab - 1) / kSlab); }
constexpr int kPartStride = 8;            // doubles per slab partial / image record of those reductions
// metrics.cu: out[i][q] (stride kPartStride) = the fixed-order reduction of part[i][slab][q] over the slabs of each of
// `images` images, q < nq: the sum, or the minimum / maximum where bit q of min_mask / max_mask is set.  One launch.
void launch_slab_reduce(const double* part, int images, int slabs, int nq, unsigned min_mask, unsigned max_mask,
                        double* out, cudaStream_t stream);

// a 4 x 4 row-major camera-to-world matrix: finite, last row 0 0 0 1, |R^T R - I| <= 1e-6 entrywise
inline bool pose_ok(const double* T, double out[12]) {
  for (int e = 0; e < 16; ++e)
    if (!std::isfinite(T[e])) return false;
  if (T[12] != 0.0 || T[13] != 0.0 || T[14] != 0.0 || T[15] != 1.0) return false;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      double s = 0.0;
      for (int r = 0; r < 3; ++r) s += T[4 * r + a] * T[4 * r + b];
      if (std::fabs(s - (a == b ? 1.0 : 0.0)) > 1e-6) return false;
    }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) out[3 * r + c] = T[4 * r + c];
    out[9 + r] = T[4 * r + 3];
  }
  return true;
}

// fp32 correctness mode of odb_conv_gemm (fp32_path.cu)


// diagnostics (odb_debug_conv_trace): device buffer of kTraceSlots uint64 per CTA, or nullptr
constexpr int kTraceSlots = 128;
unsigned long long* debug_trace();

// Launch with programmatic dependent launch allowed (the kernel must call grid_dep_wait()).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace odb
