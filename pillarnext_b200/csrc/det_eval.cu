// det_eval.cu -- detection evaluation on sm_90a: the per-pair workloads of the Waymo-style metric
// (pillarnext_b200/evaluate_waymo.py) and of the nuScenes detection score (pillarnext_b200/evaluate_nuscenes.py).
//   pnx_eval_count_points  one thread per point, looping over its frame's ground-truth boxes with the reference's
//                          points_in_boxes_jit test (box_geom.cuh point_in_box); integer atomics, so the counts are exact
//                          and do not depend on the schedule.  The counts decide each box's difficulty level (Waymo) or
//                          drop the boxes without points (nuScenes).
//   pnx_points_in_boxes    the same test for every (point, box) pair of one frame: the [n, m] mask the gt-database tool
//                          cuts objects with (the device twin of gt_sample.cu's pnx_points_in_boxes_host).
//   pnx_eval_match         one warp per (frame, class) segment of detections, pre-sorted by the 64-bit key
//                          (segment << 32 | descending score, as postproc.cu's keys): the greedy score-ordered match.
//                          For each detection in order the lanes compute its IoUs against the segment's still unmatched
//                          ground-truth boxes (a lane per box), then a shuffle arg-max picks the highest IoU, ties to the
//                          lower box index.  The class's boxes, their trigonometry and the matched flags live in shared
//                          memory, so the match needs memory in proportion to the detections plus the boxes only.
//   pnx_eval_match_center  the nuScenes centre-distance match, laid out like pnx_eval_match: one warp per segment, the
//                          class's box centres in shared memory with one matched-flag array per distance threshold.  Each
//                          lane computes the fp64 centre distance of the detection to its boxes once, and one shuffle
//                          arg-min per threshold picks the nearest unmatched box, ties to the lower box index; the match
//                          holds if that distance is strictly below the threshold.
// The IoU is the reference's boxes_iou3d_gpu arithmetic (box_geom.cuh det_aligned_iou3d_t) with
// each box's (cos, sin) of the yaw supplied by the caller, so the kernels, their host twins and the CPU oracle see the
// same trigonometry.  This file is compiled with -fmad=false (pillarnext_b200/build.py): no multiply-add is
// contracted, so the device results equal the host twins' to the bit.  No host synchronisation inside.
#include <math.h>

#include "box_geom.cuh"
#include "pnx_common.cuh"

namespace {

constexpr int kMaxBoxesPerFrame = 4096;
constexpr int kSlot = 12;          // shared-memory record per ground-truth box: box7, trig4, half-diagonal
constexpr float kSkipPad = 0.05f;  // > in_box2d's 1e-2 margin on both axes (1e-2 * sqrt(2)) plus fp32 slack
constexpr float kSkipRel = 1e-5f;  // rounding of corners far from the origin: ~80 ulp of the largest coordinate
constexpr int kMaxThresholds = 8;  // distance thresholds of one centre-distance match (nuScenes uses 4)
constexpr int kNone = 0x7fffffff;  // arg-min / arg-max sentinel: no box

// (x, y, z, dx, dy, dz, vx, vy, yaw) + (cos yaw, sin yaw) -> box7 + t = (cos yaw, sin yaw, cos -yaw, sin -yaw)
__host__ __device__ inline void eval_box(const float* b9, const float* cs, float* rec) {
  for (int k = 0; k < 6; ++k) rec[k] = b9[k];
  rec[6] = b9[8];
  rec[7] = cs[0]; rec[8] = cs[1]; rec[9] = cs[0]; rec[10] = -cs[1];
  rec[11] = 0.5f * sqrtf(b9[3] * b9[3] + b9[4] * b9[4]);
}

// aligned 3-D IoU of detection d and box g (records of eval_box).  A pair whose centres are farther apart than the two
// half-diagonals plus the pad cannot share a point of the margin-widened boxes in_box2d tests, nor cross an edge, so the
// full routine returns exactly 0 for it: skipped.
__host__ __device__ inline float eval_pair_iou(const float* d, const float* g) {
  const float ex = d[0] - g[0], ey = d[1] - g[1];
  const float reach = d[11] + g[11] + kSkipPad + kSkipRel * (fabsf(d[0]) + fabsf(d[1]) + fabsf(g[0]) + fabsf(g[1]) + d[11] + g[11]);
  if (ex * ex + ey * ey > reach * reach) return 0.0f;
  return det_aligned_iou3d_t(d, g, GivenTrig{d + 7}, GivenTrig{g + 7});
}

// 1 - min(|d|, 2 pi - |d|) / pi with d the yaw difference wrapped to [-pi, pi]
__host__ __device__ inline float heading_accuracy(float a, float b) {
  const float kPi = 3.14159265358979323846f, kTwoPi = 6.28318530717958647692f;
  const float d = fmodf(fabsf(a - b), kTwoPi);
  return 1.0f - fminf(d, kTwoPi - d) / kPi;
}

// The indices of one frame's boxes of class c (row = that frame's gt_classes), in index order, into idx[0 .. G); returns G.
// One warp, every lane gets G.
__device__ inline int warp_class_boxes(const int* row, int M, int c, int lane, int* idx) {
  int G = 0;
  for (int j0 = 0; j0 < M; j0 += 32) {
    const int j = j0 + lane;
    const bool mine = j < M && row[j] == c;
    const unsigned bal = __ballot_sync(0xffffffffu, mine);
    if (mine) idx[G + __popc(bal & ((1u << lane) - 1u))] = j;
    G += __popc(bal);
  }
  return G;
}

inline int host_class_boxes(const int* row, int M, int c, int* idx) {
  int G = 0;
  for (int j = 0; j < M; ++j)
    if (row[j] == c) idx[G++] = j;
  return G;
}

struct MatchArgs {
  const float* det_boxes;     // [D, 9]
  const float* det_trig;      // [D, 2]
  const long long* order;     // [D] detection indices, sorted by segment then descending score
  const int* seg_start;       // [B C]
  const int* seg_count;       // [B C]
  const float* gt_boxes;      // [B, M, 9]
  const int* gt_classes;      // [B, M], -1 = padding
  const float* gt_trig;       // [B, M, 2]
  int B, M, C;
  const float* thresholds;    // [C]
  int* match;                 // [D] box index within the frame, -1 = none
  float* iou;                 // [D]
  float* heading;             // [D]
};

__global__ void __launch_bounds__(256) eval_count_kernel(const float* __restrict__ points, long long n, int stride,
                                                         const float* __restrict__ boxes, const int* __restrict__ classes,
                                                         const float* __restrict__ trig, int B, int M,
                                                         int* __restrict__ counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = points + i * stride;
  const int f = frame_of(p[0], B);
  if (f < 0) return;
  const float x = p[1], y = p[2], z = p[3];
  for (int j = 0; j < M; ++j) {
    const long long k = (long long)f * M + j;
    if (classes[k] >= 0 && point_in_box(x, y, z, boxes + k * 9, trig[2 * k], trig[2 * k + 1])) atomicAdd(&counts[k], 1);
  }
}

// inside[i m + j] = point i inside box j: one thread per (point, box) pair, so consecutive threads write consecutive bytes
__global__ void __launch_bounds__(256) points_in_boxes_kernel(const float* __restrict__ points, long long n, int stride,
                                                              const float* __restrict__ boxes,
                                                              const float* __restrict__ trig, int m,
                                                              unsigned char* __restrict__ inside) {
  const long long total = n * m;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / m;
    const int j = (int)(e - i * m);
    const float* p = points + i * stride;
    inside[e] = point_in_box(p[0], p[1], p[2], boxes + (long long)j * 9, trig[2 * j], trig[2 * j + 1]);
  }
}

__global__ void __launch_bounds__(32) eval_match_kernel(MatchArgs a) {
  extern __shared__ float smem[];
  const int s = blockIdx.x, lane = threadIdx.x;
  const int f = s / a.C, c = s - f * a.C;
  float* rec = smem;                                          // [M, kSlot]
  int* idx = (int*)(rec + (size_t)a.M * kSlot);               // [M] box index within the frame
  unsigned char* used = (unsigned char*)(idx + a.M);          // [M] matched flags
  // the frame's boxes of class c, in index order
  const int G = warp_class_boxes(a.gt_classes + (long long)f * a.M, a.M, c, lane, idx);
  __syncwarp();
  for (int q = lane; q < G; q += 32) {
    const long long k = (long long)f * a.M + idx[q];
    eval_box(a.gt_boxes + k * 9, a.gt_trig + 2 * k, rec + (size_t)q * kSlot);
    used[q] = 0;
  }
  __syncwarp();
  const float thr = a.thresholds[c];
  const int n = a.seg_count[s], base = a.seg_start[s];
  for (int t = 0; t < n; ++t) {
    const long long di = a.order[base + t];
    float d[kSlot];
    eval_box(a.det_boxes + di * 9, a.det_trig + 2 * di, d);
    float best = -1.0f;
    int bk = kNone;
    for (int q = lane; q < G; q += 32) {
      if (used[q]) continue;
      const float v = eval_pair_iou(d, rec + (size_t)q * kSlot);
      if (v > best) { best = v; bk = q; }                     // ascending q: the first maximum of the lane
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, off);
      const int ok = __shfl_xor_sync(0xffffffffu, bk, off);
      if (ob > best || (ob == best && ok < bk)) { best = ob; bk = ok; }
    }
    if (lane == 0) {
      const bool hit = bk != kNone && best >= thr;
      if (hit) used[bk] = 1;
      a.match[di] = hit ? idx[bk] : -1;
      a.iou[di] = bk != kNone ? best : 0.0f;
      a.heading[di] = hit ? heading_accuracy(d[6], rec[(size_t)bk * kSlot + 6]) : 0.0f;
    }
    __syncwarp();
  }
}

size_t match_smem(int M) { return (size_t)M * (kSlot * sizeof(float) + sizeof(int) + 1); }

int check_match_args(const MatchArgs& a, int n_det) {
  PNX_CHECK_ARG(a.B >= 0 && a.C >= 1 && n_det >= 0, "B / C / number of detections");
  PNX_CHECK_ARG(a.M >= 0 && a.M <= kMaxBoxesPerFrame, "at most 4096 boxes per frame");
  PNX_CHECK_ARG((long long)a.B * a.C < (1LL << 31), "too many segments");
  PNX_CHECK_ARG(n_det == 0 || (a.det_boxes && a.det_trig && a.order), "detection pointers");
  PNX_CHECK_ARG((long long)a.B * a.M == 0 || (a.gt_boxes && a.gt_classes && a.gt_trig), "ground-truth pointers");
  PNX_CHECK_ARG(a.B == 0 || (a.seg_start && a.seg_count && a.thresholds), "segment / threshold pointers");
  PNX_CHECK_ARG(n_det == 0 || (a.match && a.iou && a.heading), "output pointers");
  return PNX_OK;
}

struct CenterArgs {
  const float* det_boxes;     // [D, 9]
  const long long* order;     // [D] detection indices, sorted by segment, then in visit order
  const int* seg_start;       // [B C]
  const int* seg_count;       // [B C]
  const float* gt_boxes;      // [B, M, 9]
  const int* gt_classes;      // [B, M], -1 = padding or filtered out
  int B, M, C;
  const double* dist_ths;     // [T] metres
  int T;
  long long D;
  int* match;                 // [T, D] box index within the frame, -1 = none
};

// centre distance in the ground plane: fp64 differences of the fp32 coordinates (the devkit's center_distance)
__host__ __device__ inline double center_distance(const float* d, const float* g) {
  const double dx = (double)d[0] - (double)g[0], dy = (double)d[1] - (double)g[1];
  return sqrt(dx * dx + dy * dy);
}

__global__ void __launch_bounds__(32) eval_match_center_kernel(CenterArgs a) {
  extern __shared__ float smem[];
  const int s = blockIdx.x, lane = threadIdx.x;
  const int f = s / a.C, c = s - f * a.C;
  float* xy = smem;                                           // [M, 2] box centres
  int* idx = (int*)(xy + 2 * (size_t)a.M);                    // [M] box index within the frame
  unsigned char* used = (unsigned char*)(idx + a.M);          // [T, G] matched flags, one array per threshold
  const int G = warp_class_boxes(a.gt_classes + (long long)f * a.M, a.M, c, lane, idx);
  __syncwarp();
  for (int q = lane; q < G; q += 32) {
    const float* g = a.gt_boxes + ((long long)f * a.M + idx[q]) * 9;
    xy[2 * q] = g[0];
    xy[2 * q + 1] = g[1];
    for (int t = 0; t < a.T; ++t) used[t * G + q] = 0;
  }
  __syncwarp();
  double ths[kMaxThresholds];
#pragma unroll
  for (int t = 0; t < kMaxThresholds; ++t) ths[t] = t < a.T ? a.dist_ths[t] : 0.0;
  const int n = a.seg_count[s], base = a.seg_start[s];
  for (int k = 0; k < n; ++k) {
    const long long di = a.order[base + k];
    const float* d = a.det_boxes + di * 9;
    double best[kMaxThresholds];
    int bk[kMaxThresholds];
#pragma unroll
    for (int t = 0; t < kMaxThresholds; ++t) { best[t] = INFINITY; bk[t] = kNone; }
    for (int q = lane; q < G; q += 32) {
      const double v = center_distance(d, xy + 2 * q);
#pragma unroll
      for (int t = 0; t < kMaxThresholds; ++t)                // ascending q: the first minimum of the lane
        if (t < a.T && !used[t * G + q] && v < best[t]) { best[t] = v; bk[t] = q; }
    }
#pragma unroll
    for (int t = 0; t < kMaxThresholds; ++t) {
      if (t >= a.T) break;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best[t], off);
        const int ok = __shfl_xor_sync(0xffffffffu, bk[t], off);
        if (ob < best[t] || (ob == best[t] && ok < bk[t])) { best[t] = ob; bk[t] = ok; }
      }
      if (lane == 0) {
        const bool hit = bk[t] != kNone && best[t] < ths[t];
        if (hit) used[t * G + bk[t]] = 1;
        a.match[t * a.D + di] = hit ? idx[bk[t]] : -1;
      }
    }
    __syncwarp();
  }
}

size_t match_center_smem(int M, int T) { return (size_t)M * (2 * sizeof(float) + sizeof(int) + T); }

int check_center_args(const CenterArgs& a) {
  PNX_CHECK_ARG(a.D >= 0 && a.D < (1LL << 31), "number of detections");
  PNX_CHECK_ARG(a.B >= 0 && a.C >= 1, "B / C");
  PNX_CHECK_ARG(a.T >= 1 && a.T <= kMaxThresholds, "1 to 8 distance thresholds");
  PNX_CHECK_ARG(a.M >= 0 && a.M <= kMaxBoxesPerFrame, "at most 4096 boxes per frame");
  PNX_CHECK_ARG((long long)a.B * a.C < (1LL << 31), "too many segments");
  PNX_CHECK_ARG(a.D == 0 || (a.det_boxes && a.order && a.match), "detection pointers");
  PNX_CHECK_ARG((long long)a.B * a.M == 0 || (a.gt_boxes && a.gt_classes), "ground-truth pointers");
  PNX_CHECK_ARG(a.B == 0 || (a.seg_start && a.seg_count && a.dist_ths), "segment / threshold pointers");
  return PNX_OK;
}


}  // namespace

// Contract: include/pnx.h.
extern "C" int pnx_eval_count_points(const float* points, long long n, int stride, const float* boxes, const int* classes,
                                     const float* trig, int B, int M, int* counts, cudaStream_t stream) {
  PNX_CHECK_ARG(n >= 0 && B >= 0 && M >= 0 && stride >= 4, "n / B / M / stride");
  PNX_CHECK_ARG((long long)B * M == 0 || (boxes && classes && trig && counts), "box pointers");
  PNX_CHECK_ARG(n == 0 || points, "points");
  if ((long long)B * M == 0) return PNX_OK;
  PNX_CUDA(cudaMemsetAsync(counts, 0, (size_t)B * M * sizeof(int), stream));
  if (n == 0) return PNX_OK;
  eval_count_kernel<<<pnx_cdiv(n, 256), 256, 0, stream>>>(points, n, stride, boxes, classes, trig, B, M, counts);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_points_in_boxes(const float* points, int n, int stride, const float* boxes, const float* trig, int m,
                                   unsigned char* inside, cudaStream_t stream) {
  PNX_CHECK_ARG(n >= 0 && m >= 0 && stride >= 3, "n / m / stride");
  PNX_CHECK_ARG((long long)n * m == 0 || (points && boxes && trig && inside), "pointers");
  if ((long long)n * m == 0) return PNX_OK;
  const long long blocks = ((long long)n * m + 255) / 256;
  points_in_boxes_kernel<<<(int)(blocks < 65536 ? blocks : 65536), 256, 0, stream>>>(points, n, stride, boxes, trig, m,
                                                                                     inside);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_eval_match(const float* det_boxes, const float* det_trig, long long n_det, const long long* order,
                              const int* seg_start, const int* seg_count, const float* gt_boxes, const int* gt_classes,
                              const float* gt_trig, int B, int M, int C, const float* thresholds, int* match, float* iou,
                              float* heading, cudaStream_t stream) {
  const MatchArgs a{det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, B, M, C, thresholds,
                    match, iou, heading};
  PNX_CHECK_ARG(n_det >= 0 && n_det < (1LL << 31), "number of detections");
  int rc = check_match_args(a, (int)n_det);
  if (rc) return rc;
  if (B == 0) return PNX_OK;
  const size_t smem = match_smem(M);
  if (smem > 48 * 1024) PNX_CUDA(cudaFuncSetAttribute(eval_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  eval_match_kernel<<<B * C, 32, smem, stream>>>(a);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

// Host twins: the same per-point and per-pair routines on HOST memory, sequentially.
extern "C" int pnx_eval_count_points_host(const float* points, long long n, int stride, const float* boxes,
                                          const int* classes, const float* trig, int B, int M, int* counts) {
  PNX_CHECK_ARG(n >= 0 && B >= 0 && M >= 0 && stride >= 4, "n / B / M / stride");
  PNX_CHECK_ARG((long long)B * M == 0 || (boxes && classes && trig && counts), "box pointers");
  PNX_CHECK_ARG(n == 0 || points, "points");
  for (long long k = 0; k < (long long)B * M; ++k) counts[k] = 0;
  if ((long long)B * M == 0) return PNX_OK;
  for (long long i = 0; i < n; ++i) {
    const float* p = points + i * stride;
    const int f = frame_of(p[0], B);
    if (f < 0) continue;
    for (int j = 0; j < M; ++j) {
      const long long k = (long long)f * M + j;
      if (classes[k] >= 0 && point_in_box(p[1], p[2], p[3], boxes + k * 9, trig[2 * k], trig[2 * k + 1])) ++counts[k];
    }
  }
  return PNX_OK;
}

extern "C" int pnx_eval_match_host(const float* det_boxes, const float* det_trig, long long n_det, const long long* order,
                                   const int* seg_start, const int* seg_count, const float* gt_boxes, const int* gt_classes,
                                   const float* gt_trig, int B, int M, int C, const float* thresholds, int* match, float* iou,
                                   float* heading) {
  const MatchArgs a{det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, B, M, C, thresholds,
                    match, iou, heading};
  PNX_CHECK_ARG(n_det >= 0 && n_det < (1LL << 31), "number of detections");
  int rc = check_match_args(a, (int)n_det);
  if (rc) return rc;
  float* rec = new float[(size_t)(M > 0 ? M : 1) * kSlot];
  int* idx = new int[M > 0 ? M : 1];
  unsigned char* used = new unsigned char[M > 0 ? M : 1];
  for (long long s = 0; s < (long long)B * C; ++s) {
    const int f = (int)(s / C), c = (int)(s % C);
    const int G = host_class_boxes(gt_classes + (long long)f * M, M, c, idx);
    for (int q = 0; q < G; ++q) {
      const long long k = (long long)f * M + idx[q];
      eval_box(gt_boxes + k * 9, gt_trig + 2 * k, rec + (size_t)q * kSlot);
      used[q] = 0;
    }
    for (int t = 0; t < seg_count[s]; ++t) {
      const long long di = order[seg_start[s] + t];
      float d[kSlot];
      eval_box(det_boxes + di * 9, det_trig + 2 * di, d);
      float best = -1.0f;
      int bk = -1;
      for (int q = 0; q < G; ++q) {
        if (used[q]) continue;
        const float v = eval_pair_iou(d, rec + (size_t)q * kSlot);
        if (v > best) { best = v; bk = q; }
      }
      const bool hit = bk >= 0 && best >= thresholds[c];
      if (hit) used[bk] = 1;
      match[di] = hit ? idx[bk] : -1;
      iou[di] = bk >= 0 ? best : 0.0f;
      heading[di] = hit ? heading_accuracy(d[6], rec[(size_t)bk * kSlot + 6]) : 0.0f;
    }
  }
  delete[] rec;
  delete[] idx;
  delete[] used;
  return PNX_OK;
}

extern "C" int pnx_eval_match_center(const float* det_boxes, long long n_det, const long long* order, const int* seg_start,
                                     const int* seg_count, const float* gt_boxes, const int* gt_classes, int B, int M, int C,
                                     const double* dist_ths, int T, int* match, cudaStream_t stream) {
  const CenterArgs a{det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, B, M, C, dist_ths, T, n_det, match};
  int rc = check_center_args(a);
  if (rc) return rc;
  if (B == 0) return PNX_OK;
  const size_t smem = match_center_smem(M, T);
  if (smem > 48 * 1024)
    PNX_CUDA(cudaFuncSetAttribute(eval_match_center_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  eval_match_center_kernel<<<B * C, 32, smem, stream>>>(a);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_eval_match_center_host(const float* det_boxes, long long n_det, const long long* order,
                                          const int* seg_start, const int* seg_count, const float* gt_boxes,
                                          const int* gt_classes, int B, int M, int C, const double* dist_ths, int T,
                                          int* match) {
  const CenterArgs a{det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, B, M, C, dist_ths, T, n_det, match};
  int rc = check_center_args(a);
  if (rc) return rc;
  int* idx = new int[M > 0 ? M : 1];
  unsigned char* used = new unsigned char[M > 0 ? M : 1];
  for (long long s = 0; s < (long long)B * C; ++s) {
    const int f = (int)(s / C), c = (int)(s % C);
    const int G = host_class_boxes(gt_classes + (long long)f * M, M, c, idx);
    for (int t = 0; t < T; ++t) {
      for (int q = 0; q < G; ++q) used[q] = 0;
      for (int k = 0; k < seg_count[s]; ++k) {
        const long long di = order[seg_start[s] + k];
        double best = INFINITY;
        int bk = -1;
        for (int q = 0; q < G; ++q) {
          if (used[q]) continue;
          const double v = center_distance(det_boxes + di * 9, gt_boxes + ((long long)f * M + idx[q]) * 9);
          if (v < best) { best = v; bk = q; }
        }
        const bool hit = bk >= 0 && best < dist_ths[t];
        if (hit) used[bk] = 1;
        match[t * n_det + di] = hit ? idx[bk] : -1;
      }
    }
  }
  delete[] idx;
  delete[] used;
  return PNX_OK;
}
