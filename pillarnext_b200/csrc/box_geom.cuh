// box_geom.cuh -- box geometry shared by postproc.cu (rotated NMS, `iou` head target), gt_sample.cu (point test) and
// det_eval.cu (Waymo-style evaluation).  Every routine is `__host__ __device__`, so each file's host twins run the same
// source as its kernels.  Internal linkage: each translation unit compiles its own copy with its own flags.
//
// Rotated BEV overlap (iou3d_cpu.cpp:62-237 algorithm: edge crossings + contained corners, sorted by angle about their
// centroid, shoelace area).  It deliberately follows the ARITHMETIC of the reference's own device code,
// det3d/core/iou3d_nms/src/iou3d_nms_kernel.cu:39-235 (and its host twin iou3d_cpu.cpp), statement by statement -- same
// operation order, same 1e-2 margin, same angular ordering of the polygon vertices: the keep / suppress decision of every
// box pair must come out bit-identical to the reference's NMS, and any algebraically equivalent rewrite flips decisions for
// IoUs near the threshold.  det_box_overlap_t takes each box's trigonometry from a HeadingTrig (cosf / sinf, as the
// reference's kernel computes it: det_box_overlap) or a GivenTrig (values the caller supplies).
//
// Point test (points_in_boxes_jit): |z - bz| <= dz / 2 first, then |lx| <= dx / 2 and |ly| <= dy / 2 with
// lx = fl(fl(sx * c) + fl(sy * s)), ly = fl(fl(-sx * s) + fl(sy * c)); the halves compared in fp64, as numba promotes
// `x / 2.0`.  Every fp32 operation is rounded on its own (the _rn intrinsics on the device, plain operators on the host,
// whose compiler has no FMA to contract into).
#pragma once
#include <math.h>

namespace {

// ------------------------------------------------------------------ separately rounded fp32 operations
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
__host__ __device__ inline float sub_f(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ inline float min_f(float a, float b) { return b < a ? b : a; }
__host__ __device__ inline float max_f(float a, float b) { return b > a ? b : a; }

// points_in_boxes_jit for one (point, box) pair; box is 9-column (yaw last), (c, s) = libm cosf / sinf of the yaw
__host__ __device__ inline bool point_in_box(float x, float y, float z, const float* box, float c, float s) {
  if (!((double)fabsf(sub_f(z, box[2])) <= (double)box[5] / 2.0)) return false;
  const float sx = sub_f(x, box[0]), sy = sub_f(y, box[1]);
  const float lx = add_f(mul_f(sx, c), mul_f(sy, s));
  const float ly = add_f(mul_f(-sx, s), mul_f(sy, c));
  return (double)fabsf(lx) <= (double)box[3] / 2.0 && (double)fabsf(ly) <= (double)box[4] / 2.0;
}

// frame index of a point row: an integer in [0, B), else -1 (the row is dropped)
__host__ __device__ inline int frame_of(float f, int B) {
  return (f >= 0.0f && f < (float)B && f == floorf(f)) ? (int)f : -1;
}

// ------------------------------------------------------------------ rotated BEV overlap, aligned 3-D IoU
struct P2 { float x, y; };

__host__ __device__ inline float cross3(const P2& p1, const P2& p2, const P2& p0) {
  return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}

__host__ __device__ inline bool rect_cross(const P2& p1, const P2& p2, const P2& q1, const P2& q2) {
  return fminf(p1.x, p2.x) <= fmaxf(q1.x, q2.x) && fminf(q1.x, q2.x) <= fmaxf(p1.x, p2.x) &&
         fminf(p1.y, p2.y) <= fmaxf(q1.y, q2.y) && fminf(q1.y, q2.y) <= fmaxf(p1.y, p2.y);
}

// Trigonometry of a box's heading h, as det_box_overlap_t reads it: HeadingTrig computes it with cosf / sinf where the
// reference's kernel does; GivenTrig reads t = (cos h, sin h, cos -h, sin -h) supplied by the caller.
struct HeadingTrig {
  const float* box;
  __host__ __device__ float cos_h() const { return cosf(box[6]); }
  __host__ __device__ float sin_h() const { return sinf(box[6]); }
  __host__ __device__ float cos_neg() const { return cosf(-box[6]); }
  __host__ __device__ float sin_neg() const { return sinf(-box[6]); }
};
struct GivenTrig {
  const float* t;
  __host__ __device__ float cos_h() const { return t[0]; }
  __host__ __device__ float sin_h() const { return t[1]; }
  __host__ __device__ float cos_neg() const { return t[2]; }
  __host__ __device__ float sin_neg() const { return t[3]; }
};

// box7 = (x, y, z, dx, dy, dz, heading)
template <class T>
__host__ __device__ inline bool in_box2d(const float* box, const T& tr, const P2& p) {
  const float kMargin = 1e-2f;
  const float c = tr.cos_neg(), s = tr.sin_neg();
  const float rx = (p.x - box[0]) * c + (p.y - box[1]) * (-s);
  const float ry = (p.x - box[0]) * s + (p.y - box[1]) * c;
  return fabsf(rx) < box[3] / 2 + kMargin && fabsf(ry) < box[4] / 2 + kMargin;
}

__host__ __device__ inline bool seg_intersection(const P2& p1, const P2& p0, const P2& q1, const P2& q0, P2* ans) {
  const float kEps = 1e-8f;
  if (!rect_cross(p0, p1, q0, q1)) return false;
  const float s1 = cross3(q0, p1, p0), s2 = cross3(p1, q1, p0), s3 = cross3(p0, q1, q0), s4 = cross3(q1, p1, q0);
  if (!(s1 * s2 > 0 && s3 * s4 > 0)) return false;
  const float s5 = cross3(q1, p1, p0);
  if (fabsf(s5 - s1) > kEps) {
    ans->x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
    ans->y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
  } else {
    const float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
    const float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
    const float D = a0 * b1 - a1 * b0;
    ans->x = (b0 * c1 - b1 * c0) / D;
    ans->y = (a1 * c0 - a0 * c1) / D;
  }
  return true;
}

// The axis-aligned corners x1 = x - dx / 2, ... are rounded first and rotated about the centre as (x1 - x), ...: the
// reference's form.  (x1 - x) is not -dx / 2 in fp32, so writing the offsets as +-dx / 2 directly moves corners by an
// ulp of the centre and flips decisions near the threshold.
template <class T>
__host__ __device__ inline void box_corners(const float* box, const T& tr, P2* c5) {
  const float hx = box[3] / 2, hy = box[4] / 2;
  const float x1 = box[0] - hx, y1 = box[1] - hy, x2 = box[0] + hx, y2 = box[1] + hy;
  const float ca = tr.cos_h(), sa = tr.sin_h();
  const float px[4] = {x1 - box[0], x2 - box[0], x2 - box[0], x1 - box[0]};
  const float py[4] = {y1 - box[1], y1 - box[1], y2 - box[1], y2 - box[1]};
  for (int k = 0; k < 4; ++k) {
    c5[k].x = px[k] * ca + py[k] * (-sa) + box[0];
    c5[k].y = px[k] * sa + py[k] * ca + box[1];
  }
  c5[4] = c5[0];
}

template <class T>
__host__ __device__ inline float det_box_overlap_t(const float* a, const float* b, const T& ta, const T& tb) {
  P2 ca[5], cb[5], pts[16];
  box_corners(a, ta, ca);
  box_corners(b, tb, cb);
  int cnt = 0;
  float sx = 0.f, sy = 0.f;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      P2 q;
      if (cnt < 16 && seg_intersection(ca[i + 1], ca[i], cb[j + 1], cb[j], &q)) {
        sx += q.x; sy += q.y;
        pts[cnt++] = q;
      }
    }
  for (int k = 0; k < 4; ++k) {
    if (cnt < 16 && in_box2d(a, ta, cb[k])) { sx += cb[k].x; sy += cb[k].y; pts[cnt++] = cb[k]; }
    if (cnt < 16 && in_box2d(b, tb, ca[k])) { sx += ca[k].x; sy += ca[k].y; pts[cnt++] = ca[k]; }
  }
  if (cnt == 0) return 0.f;
  const float cx = sx / cnt, cy = sy / cnt;
  float ang[16];
  for (int k = 0; k < cnt; ++k) ang[k] = atan2f(pts[k].y - cy, pts[k].x - cx);
  for (int j = 0; j < cnt - 1; ++j)
    for (int i = 0; i < cnt - j - 1; ++i)
      if (ang[i] > ang[i + 1]) {
        const P2 t = pts[i]; pts[i] = pts[i + 1]; pts[i + 1] = t;
        const float ta = ang[i]; ang[i] = ang[i + 1]; ang[i + 1] = ta;
      }
  float area = 0.f;
  for (int k = 0; k < cnt - 1; ++k) {
    const float ax = pts[k].x - pts[0].x, ay = pts[k].y - pts[0].y;
    const float bx = pts[k + 1].x - pts[0].x, by = pts[k + 1].y - pts[0].y;
    area += ax * by - ay * bx;
  }
  return fabsf(area) / 2.0f;
}

__host__ __device__ inline float det_box_overlap(const float* a, const float* b) {
  return det_box_overlap_t(a, b, HeadingTrig{a}, HeadingTrig{b});
}

__host__ __device__ inline float det_iou_bev(const float* a, const float* b) {
  const float sa = a[3] * a[4], sb = b[3] * b[4];
  const float so = det_box_overlap(a, b);
  return so / fmaxf(sa + sb - so, 1e-8f);
}

// aligned 3-D IoU of two (x, y, z, dx, dy, dz, heading) boxes: BEV overlap x height overlap over the union volume
// (reference det3d/core/iou3d_nms/iou3d_nms_utils.py:11-87, boxes_iou3d_gpu / boxes_aligned_iou3d_gpu; the training
// target of the `iou` head)
template <class T>
__host__ __device__ inline float det_aligned_iou3d_t(const float* a, const float* b, const T& ta, const T& tb) {
  const float a_max = a[2] + a[5] / 2, a_min = a[2] - a[5] / 2;
  const float b_max = b[2] + b[5] / 2, b_min = b[2] - b[5] / 2;
  const float oh = fmaxf(fminf(a_max, b_max) - fmaxf(a_min, b_min), 0.f);
  const float o3 = det_box_overlap_t(a, b, ta, tb) * oh;
  const float va = a[3] * a[4] * a[5], vb = b[3] * b[4] * b[5];
  return o3 / fmaxf(va + vb - o3, 1e-6f);
}

__host__ __device__ inline float det_aligned_iou3d(const float* a, const float* b) {
  return det_aligned_iou3d_t(a, b, HeadingTrig{a}, HeadingTrig{b});
}

}  // namespace
