// Host plumbing of the tensor-core kernels (gemm_sk.cu, gemm_ns.cu, dep_fused.cu, mimi_tc.cu): the driver's tensor-map
// encoder, the device's SM count, the 2-D activation map and one kernel launch helper.  Definitions in common.cu.
#pragma once

#include <cuda.h>

#include <utility>

#include "common.cuh"

namespace b200 {

// cuTensorMapEncodeTiled (resolved once through the runtime) with SWIZZLE_128B, 256-byte L2 promotion and no OOB fill;
// B200_ERR_CUDA naming `what` if the driver refuses the map
int encode_tiled(CUtensorMap* m, CUtensorMapDataType type, cuuint32_t rank, const void* base, const cuuint64_t* dims,
                 const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr, const char* what);

// 2-D map of row-major activations [rows][cols] (row stride ld elements) with a [box_rows x 128 bytes] box;
// elem_bytes = 2 (bf16) or 1 (int8 / uint8)
int act_map(CUtensorMap* m, const void* base, long long ld, int rows, int cols, int box_rows, int elem_bytes);

// multiprocessors of the device current at the first call (0 if it cannot be read)
int num_sms();

struct LaunchOpts {
  int pdl = 0;              // programmatic stream serialization (the kernel waits on its predecessor itself)
  int cluster = 0;          // > 0: cluster dimension attribute of that many CTAs
  bool cooperative = false;
};

// cudaLaunchKernelEx with the attributes of `o`, counted in g_launches and checked
template <typename... KArgs, typename... Args>
int launch(const char* what, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, LaunchOpts o,
           Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[3];
  int n = 0;
  if (o.cluster > 0) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = o.cluster; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (o.pdl) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (o.cooperative) {
    attr[n].id = cudaLaunchAttributeCooperative;
    attr[n].val.cooperative = 1;
    ++n;
  }
  cfg.attrs = attr; cfg.numAttrs = n;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (e != cudaSuccess) B200_FAIL(B200_ERR_CUDA, "%s launch failed: %s", what, cudaGetErrorString(e));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_launch(what);
}

}  // namespace b200
