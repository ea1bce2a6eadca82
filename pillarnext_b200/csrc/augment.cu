// augment.cu -- global training augmentation (rotation, scaling, translation, flip) of points and raw boxes, sm_90a.
//
// The data-loader workers draw the parameters exactly as the reference does (det3d/datasets/pipelines/augmentation.py of
// this repo) and ship aug [B, 4, 4] fp64: per frame up to four records (code, p0, p1, p2), applied in slot order.  One
// launch transforms the points ([n, 6], frame index in column 0) and the raw boxes ([B, M, 9] x y z dx dy dz vx vy yaw)
// into new tensors, before label assignment.  Point order is kept.
//
// The arithmetic is numpy's, to the bit (pinned by tests/golden/ref_aug.npz):
//   rotation    : xyz (and vx, vy, 0) @ rot_mat_T in fp64, rounded once to fp32.  The BLAS kernel behind numpy's `@`
//                 accumulates each output as fma(v2, R2j, fma(v1, R1j, v0 * R0j)); so does rotate().  yaw += fp32(theta).
//   scaling     : fp32 multiply by fp32(s): point xyz, box columns 0-7.
//   translation : x, y, z + t in fp64 (t is a float64 array in numpy), rounded to fp32.
//   flip        : x flip negates point y and box y, vy, yaw; y flip negates point x and box x, vx and sets
//                 yaw = -yaw + fp32(pi).  After each flip yaw > fp32(pi) -> yaw - fp32(2 pi), then yaw < -fp32(pi) ->
//                 yaw + fp32(2 pi) (numpy compares and subtracts the Python floats at fp32).
//   NaN         : every op reads a NaN box element as 0 and writes NaN (0x7fc00000, numpy's np.nan in fp32) back.
// Every fp32 / fp64 operation is rounded on its own (the _rn intrinsics on the device, plain operators in the host
// twin, whose compiler has no FMA to contract into), except the fma()s that reproduce the BLAS accumulation.
#include <math.h>

#include "pnx_common.cuh"

namespace {

enum { AUG_EMPTY = 0, AUG_ROTATION = 1, AUG_SCALING = 2, AUG_TRANSLATION = 3, AUG_FLIP = 4 };

__host__ __device__ inline double mul_d(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline double add_d(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ inline float mul_f(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline float add_f(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ inline float to_f(double a) {
#ifdef __CUDA_ARCH__
  return __double2float_rn(a);
#else
  return (float)a;
#endif
}
__host__ __device__ inline float nan_f() {
#ifdef __CUDA_ARCH__
  return __int_as_float(0x7fc00000);
#else
  return __builtin_nanf("");
#endif
}

// fp32(pi) and fp32(2 pi): numpy's np.pi and 2 * np.pi met by a float32 array
#define AUG_PI_F 3.14159274101257324f
#define AUG_TWO_PI_F 6.28318548202514648f

// (x, y, z) @ [[c, s, 0], [-s, c, 0], [0, 0, 1]] in fp64, each output rounded once to fp32
__host__ __device__ inline void rotate(double c, double s, float& x, float& y, float& z) {
  const double X = x, Y = y, Z = z;
  const double nx = fma(Z, 0.0, fma(Y, -s, mul_d(X, c)));
  const double ny = fma(Z, 0.0, fma(Y, c, mul_d(X, s)));
  const double nz = fma(Z, 1.0, fma(Y, 0.0, mul_d(X, 0.0)));
  x = to_f(nx);
  y = to_f(ny);
  z = to_f(nz);
}

__host__ __device__ inline float wrap_yaw(float yaw) {
  if (yaw > AUG_PI_F) yaw = add_f(yaw, -AUG_TWO_PI_F);
  if (yaw < -AUG_PI_F) yaw = add_f(yaw, AUG_TWO_PI_F);
  return yaw;
}

// one frame's records (aug + 16 * frame) applied to one point's x, y, z
__host__ __device__ inline void aug_point(const double* a, float& x, float& y, float& z) {
  for (int k = 0; k < 4; ++k) {
    const int code = (int)a[4 * k];
    const double p0 = a[4 * k + 1], p1 = a[4 * k + 2], p2 = a[4 * k + 3];
    if (code == AUG_ROTATION) {
      rotate(p1, p2, x, y, z);
    } else if (code == AUG_SCALING) {
      const float s = to_f(p0);
      x = mul_f(x, s);
      y = mul_f(y, s);
      z = mul_f(z, s);
    } else if (code == AUG_TRANSLATION) {
      x = to_f(add_d(x, p0));
      y = to_f(add_d(y, p0));
      z = to_f(add_d(z, p0));
    } else if (code == AUG_FLIP) {
      if (p0 != 0.0) y = -y;
      if (p1 != 0.0) x = -x;
    }
  }
}

// ... and to one raw box (x, y, z, dx, dy, dz, vx, vy, yaw)
__host__ __device__ inline void aug_box(const double* a, float* b) {
  for (int k = 0; k < 4; ++k) {
    const int code = (int)a[4 * k];
    if (code < AUG_ROTATION || code > AUG_FLIP) continue;
    const double p0 = a[4 * k + 1], p1 = a[4 * k + 2], p2 = a[4 * k + 3];
    unsigned nan_mask = 0;
    for (int j = 0; j < 9; ++j)
      if (b[j] != b[j]) {
        nan_mask |= 1u << j;
        b[j] = 0.0f;
      }
    if (code == AUG_ROTATION) {
      rotate(p1, p2, b[0], b[1], b[2]);
      float vz = 0.0f;
      rotate(p1, p2, b[6], b[7], vz);
      b[8] = add_f(b[8], to_f(p0));
    } else if (code == AUG_SCALING) {
      const float s = to_f(p0);
      for (int j = 0; j < 8; ++j) b[j] = mul_f(b[j], s);
    } else if (code == AUG_TRANSLATION) {
      for (int j = 0; j < 3; ++j) b[j] = to_f(add_d(b[j], p0));
    } else {
      if (p0 != 0.0) {
        b[1] = -b[1];
        b[7] = -b[7];
        b[8] = wrap_yaw(-b[8]);
      }
      if (p1 != 0.0) {
        b[0] = -b[0];
        b[6] = -b[6];
        b[8] = wrap_yaw(add_f(-b[8], AUG_PI_F));
      }
    }
    for (int j = 0; j < 9; ++j)
      if (nan_mask & (1u << j)) b[j] = nan_f();
  }
}

// Point i, or box i - n.  A point whose frame index is not an integer in [0, B) is copied unchanged.
__host__ __device__ inline void aug_row(const float* __restrict__ pts, int n, const float* __restrict__ boxes, int B, int M,
                                        const double* __restrict__ aug, float* __restrict__ pts_out,
                                        float* __restrict__ boxes_out, long long i) {
  if (i < n) {
    const float* p = pts + i * 6;
    float v[6];
    for (int j = 0; j < 6; ++j) v[j] = p[j];
    const float f = v[0];
    if (f >= 0.0f && f < (float)B && f == floorf(f)) aug_point(aug + 16 * (long long)f, v[1], v[2], v[3]);
    float* o = pts_out + i * 6;
    for (int j = 0; j < 6; ++j) o[j] = v[j];
  } else {
    const long long r = i - n;
    if (r >= (long long)B * M) return;
    float v[9];
    for (int j = 0; j < 9; ++j) v[j] = boxes[r * 9 + j];
    aug_box(aug + 16 * (r / M), v);
    for (int j = 0; j < 9; ++j) boxes_out[r * 9 + j] = v[j];
  }
}

__global__ void __launch_bounds__(256) global_aug_kernel(const float* __restrict__ pts, int n, const float* __restrict__ boxes,
                                                         int B, int M, const double* __restrict__ aug,
                                                         float* __restrict__ pts_out, float* __restrict__ boxes_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n + (long long)B * M) return;
  aug_row(pts, n, boxes, B, M, aug, pts_out, boxes_out, i);
}

int check_args(const float* points, int n, const float* boxes, int B, int M, const double* aug, const float* points_out,
               const float* boxes_out) {
  PNX_CHECK_ARG(n >= 0 && B >= 0 && M >= 0, "n / B / M");
  PNX_CHECK_ARG(n == 0 || (points && points_out && points != points_out), "points / points_out");
  PNX_CHECK_ARG((long long)B * M == 0 || (boxes && boxes_out && boxes != boxes_out), "boxes / boxes_out");
  PNX_CHECK_ARG(B == 0 || aug, "aug");
  return PNX_OK;
}

}  // namespace

// Contract: include/pnx.h.  All pointers are device memory; one launch over n + B*M threads.
extern "C" int pnx_global_aug(const float* points, int n, const float* boxes, int B, int M, const double* aug,
                              float* points_out, float* boxes_out, cudaStream_t stream) {
  const int rc = check_args(points, n, boxes, B, M, aug, points_out, boxes_out);
  if (rc) return rc;
  const long long total = n + (long long)B * M;
  if (total == 0) return PNX_OK;
  global_aug_kernel<<<pnx_cdiv(total, 256), 256, 0, stream>>>(points, n, boxes, B, M, aug, points_out, boxes_out);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

// Host twin: the same per-row math on HOST memory (the CPU tests pin it to the goldens).
extern "C" int pnx_global_aug_host(const float* points, int n, const float* boxes, int B, int M, const double* aug,
                                   float* points_out, float* boxes_out) {
  const int rc = check_args(points, n, boxes, B, M, aug, points_out, boxes_out);
  if (rc) return rc;
  const long long total = n + (long long)B * M;
  for (long long i = 0; i < total; ++i) aug_row(points, n, boxes, B, M, aug, points_out, boxes_out, i);
  return PNX_OK;
}
