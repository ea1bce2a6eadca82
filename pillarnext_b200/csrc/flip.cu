// flip.cu -- point expansion of double-flip test-time augmentation, sm_90a.
//
// Frame b of a batch becomes frames 4b + k: k = 0 as is, k = 1 mirrored in y (y -> -y, the reference's
// box_np_ops.flip(axis='x')), k = 2 mirrored in x (x -> -x, flip(axis='y')), k = 3 both.  Copy k of point i is written to
// row k*N + i, so the output is NOT grouped by frame: the global-bitmap voxelizer (pnx_voxelize) accepts any order, and
// inside each frame the points keep their input order.  Negation and 4b + k are exact in fp32.
#include "pnx_common.cuh"

namespace {

__global__ void __launch_bounds__(256) flip4_points_kernel(const float* __restrict__ pts, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = pts + (size_t)i * 6;
  const float b = p[0], x = p[1], y = p[2], z = p[3], in = p[4], t = p[5];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float* o = out + ((size_t)k * n + i) * 6;
    o[0] = 4.0f * b + (float)k;
    o[1] = (k & 2) ? -x : x;
    o[2] = (k & 1) ? -y : y;
    o[3] = z; o[4] = in; o[5] = t;
  }
}

}  // namespace

// Contract: include/pnx.h.  points [n, 6] (batch_idx, x, y, z, intensity, time) fp32 -> out [4n, 6] fp32 (device).
extern "C" int pnx_flip4_points(const float* points, int n, float* out, cudaStream_t stream) {
  PNX_CHECK_ARG(n >= 0, "n");
  if (n == 0) return PNX_OK;
  PNX_CHECK_ARG(points && out && points != out, "points / out");
  flip4_points_kernel<<<pnx_cdiv(n, 256), 256, 0, stream>>>(points, n, out);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}
