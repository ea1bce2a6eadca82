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
//   pnx_eval_pairs         the Hungarian mode's first pass, laid out like pnx_eval_match: one warp per segment writes
//                          every pair with IoU >= threshold, a ballot compacting each detection's boxes in index order
//                          (a count pass, then a write pass at the prefix-summed offsets).
//   pnx_eval_components    one warp per segment; lane 0 joins the pairs sharing a detection or a box (union-find, the
//                          first pair of a component is its root) and lays each component's pairs out contiguously.
//   pnx_eval_assign        the exact maximum-IoU assignment of each component per (breakdown, score cutoff): the
//                          O(N^3) shortest-augmenting-path Hungarian method on the square problem with an "unmatched"
//                          column per detection and row per box, in 40-bit fixed-point integers, then the tie rule by
//                          re-solving with the earlier choices fixed wherever the duals leave an option open.  One warp
//                          and shared memory per (component, breakdown, cutoff) up to kSmallEdges pairs; one CTA and a
//                          global workspace per larger component.  The same template runs the host twin.
//   pnx_eval_mot           the CLEAR-MOT frame matching of evaluate_waymo_tracking.py: one warp per (sequence, class,
//                          score cutoff) walks the sequence's frames; per frame the leader keeps the pairs that carry
//                          each object's previous id, then every component is solved by the same tie-ruled assignment
//                          over the pairs left active, its state in the row's slice of a global workspace, and the
//                          leader counts matches, mismatches and sum(1 - IoU) per level.  The host twin runs the same
//                          template one row at a time.
//   pnx_eval_pairs_center  nuScenes tracking's pairs (evaluate_nuscenes_tracking.py), laid out like pnx_eval_pairs: every
//                          pair with the fp64 centre distance of pnx_eval_match_center < max_dist, written as fp32.
//   pnx_eval_mot_center    the same frame walk as pnx_eval_mot (mot_row, one warp per (scene, class, cutoff)) with
//                          another counting rule: the assignment takes the most pairs, then the smallest distance sum,
//                          and the leader counts matches, identity switches, fragmentations and the distance sum, and
//                          optionally flags each matched detection.
// The IoU is the reference's boxes_iou3d_gpu arithmetic (box_geom.cuh det_aligned_iou3d_t) with
// each box's (cos, sin) of the yaw supplied by the caller, so the kernels, their host twins and the CPU oracle see the
// same trigonometry.  This file is compiled with -fmad=false (pillarnext_b200/build.py): no multiply-add is
// contracted, so the device results equal the host twins' to the bit.  No host synchronisation inside.
#include <limits.h>
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

// ---------------------------------------------------------------- maximum-IoU assignment (the Hungarian mode)
constexpr int kSmallEdges = 32;              // components with at most this many feasible pairs: one warp, shared memory
constexpr int kLargeThreads = 256;           // larger components: one CTA, global workspace
constexpr long long kInf = LLONG_MAX;        // "no finite reduced cost yet"
constexpr double kFix = 1099511627776.0;     // 2^40: an fp32 IoU >= 2^-17 is an exact multiple of 2^-40

struct PairArgs {
  MatchArgs m;                // inputs as for the greedy match; match / iou / heading unused
  const int* edge_start;      // [B C] or null: count only
  int* edge_count;            // [B C]
  int* e_det;                 // [E] detection index
  int* e_box;                 // [E] f M + j
  float* e_iou;               // [E]
  float* e_head;              // [E] heading accuracy of the pair (heading_accuracy, as the greedy match)
};

// One warp per (frame, class) segment: the detection's IoU against each of the class's boxes (the greedy match's pair
// routine), and every pair with IoU >= threshold in (detection in visit order, ascending box index) order.
__global__ void __launch_bounds__(32) eval_pairs_kernel(PairArgs p) {
  extern __shared__ float smem[];
  const MatchArgs& a = p.m;
  const int s = blockIdx.x, lane = threadIdx.x;
  const int f = s / a.C, c = s - f * a.C;
  float* rec = smem;
  int* idx = (int*)(rec + (size_t)a.M * kSlot);
  const int G = warp_class_boxes(a.gt_classes + (long long)f * a.M, a.M, c, lane, idx);
  __syncwarp();
  for (int q = lane; q < G; q += 32) {
    const long long k = (long long)f * a.M + idx[q];
    eval_box(a.gt_boxes + k * 9, a.gt_trig + 2 * k, rec + (size_t)q * kSlot);
  }
  __syncwarp();
  const float thr = a.thresholds[c];
  const int n = a.seg_count[s], base = a.seg_start[s];
  int cursor = p.edge_start ? p.edge_start[s] : 0;
  for (int t = 0; t < n; ++t) {
    const long long di = a.order[base + t];
    float d[kSlot];
    eval_box(a.det_boxes + di * 9, a.det_trig + 2 * di, d);
    for (int q0 = 0; q0 < G; q0 += 32) {
      const int q = q0 + lane;
      const float v = q < G ? eval_pair_iou(d, rec + (size_t)q * kSlot) : 0.0f;
      const bool hit = q < G && v >= thr;
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      if (hit && p.edge_start) {
        const int e = cursor + __popc(bal & ((1u << lane) - 1u));
        p.e_det[e] = (int)di;
        p.e_box[e] = f * a.M + idx[q];
        p.e_iou[e] = v;
        p.e_head[e] = heading_accuracy(d[6], rec[(size_t)q * kSlot + 6]);
      }
      cursor += __popc(bal);
    }
  }
  if (lane == 0 && !p.edge_start) p.edge_count[s] = cursor;
}

inline void host_pairs(const PairArgs& p) {
  const MatchArgs& a = p.m;
  float* rec = new float[(size_t)(a.M > 0 ? a.M : 1) * kSlot];
  int* idx = new int[a.M > 0 ? a.M : 1];
  for (long long s = 0; s < (long long)a.B * a.C; ++s) {
    const int f = (int)(s / a.C), c = (int)(s % a.C);
    const int G = host_class_boxes(a.gt_classes + (long long)f * a.M, a.M, c, idx);
    for (int q = 0; q < G; ++q) {
      const long long k = (long long)f * a.M + idx[q];
      eval_box(a.gt_boxes + k * 9, a.gt_trig + 2 * k, rec + (size_t)q * kSlot);
    }
    int cursor = p.edge_start ? p.edge_start[s] : 0;
    for (int t = 0; t < a.seg_count[s]; ++t) {
      const long long di = a.order[a.seg_start[s] + t];
      float d[kSlot];
      eval_box(a.det_boxes + di * 9, a.det_trig + 2 * di, d);
      for (int q = 0; q < G; ++q) {
        const float v = eval_pair_iou(d, rec + (size_t)q * kSlot);
        if (!(v >= a.thresholds[c])) continue;
        if (p.edge_start) {
          p.e_det[cursor] = (int)di;
          p.e_box[cursor] = f * a.M + idx[q];
          p.e_iou[cursor] = v;
          p.e_head[cursor] = heading_accuracy(d[6], rec[(size_t)q * kSlot + 6]);
        }
        ++cursor;
      }
    }
    if (!p.edge_start) p.edge_count[s] = cursor;
  }
  delete[] rec;
  delete[] idx;
}

// Union-find over edge ids with the smaller root winning, so each component's root is its first edge.
__host__ __device__ inline int uf_find(int* parent, int e) {
  while (parent[e] != e) {
    parent[e] = parent[parent[e]];
    e = parent[e];
  }
  return e;
}

__host__ __device__ inline void uf_union(int* parent, int a, int b) {
  a = uf_find(parent, a);
  b = uf_find(parent, b);
  if (a < b) parent[b] = a;
  else if (b < a) parent[a] = b;
}

// The connected components of one segment's feasible graph, edges [e0, e1): two edges are joined when they share a
// detection (consecutive edges, as the pair pass writes them) or a box (last[] = the latest edge of each box, -1 on
// entry and on exit).  root[e] = the component's first edge; for a root, comp_start = where its edges begin in grouped
// and comp_nedge = how many there are (components in root order, each one's edges in edge order); otherwise -1 and 0.
__host__ __device__ inline void segment_components(int e0, int e1, int M, const int* e_det, const int* e_box, int* last,
                                                   int* root, int* comp_start, int* comp_nedge, int* grouped) {
  for (int e = e0; e < e1; ++e) {
    root[e] = e;
    comp_start[e] = -1;
    comp_nedge[e] = 0;
  }
  for (int e = e0; e < e1; ++e) {
    if (e > e0 && e_det[e] == e_det[e - 1]) uf_union(root, e, e - 1);
    const int j = e_box[e] % M;
    if (last[j] >= 0) uf_union(root, e, last[j]);
    last[j] = e;
  }
  for (int e = e0; e < e1; ++e) {
    root[e] = uf_find(root, e);
    ++comp_nedge[root[e]];
  }
  int pos = e0;
  for (int e = e0; e < e1; ++e)
    if (root[e] == e) { comp_start[e] = pos; pos += comp_nedge[e]; }
  for (int e = e0; e < e1; ++e) grouped[comp_start[root[e]]++] = e;
  for (int e = e0; e < e1; ++e) {
    if (root[e] == e) comp_start[e] -= comp_nedge[e];
    last[e_box[e] % M] = -1;
  }
}

struct CompArgs {
  const int* edge_start;      // [B C]
  const int* edge_count;      // [B C]
  int B, M, C;
  const int* e_det;
  const int* e_box;
  int* root;                  // [E]
  int* comp_start;            // [E]
  int* comp_nedge;            // [E]
  int* grouped;               // [E]
};

// One warp per segment: the lanes clear the box table, lane 0 walks the segment's edges (a handful per segment).
__global__ void __launch_bounds__(32) eval_components_kernel(CompArgs a) {
  extern __shared__ int last[];                               // [M]
  const int s = blockIdx.x;
  for (int j = threadIdx.x; j < a.M; j += 32) last[j] = -1;
  __syncwarp();
  if (threadIdx.x == 0 && a.edge_count[s] > 0)
    segment_components(a.edge_start[s], a.edge_start[s] + a.edge_count[s], a.M, a.e_det, a.e_box, last, a.root,
                       a.comp_start, a.comp_nedge, a.grouped);
}

struct AssignArgs {
  const int* grouped;         // [E]
  const int* comp_start;      // [E]
  const int* comp_nedge;      // [E]
  const int* e_det;           // [E]
  const int* e_box;           // [E]
  const float* e_iou;         // [E]
  const float* e_head;        // [E]
  const int* small_roots;     // [n_small] roots of the components of at most kSmallEdges pairs
  const int* large_roots;     // [n_large] roots of the larger ones
  const long long* large_off; // [n_large] exclusive prefix sum of the larger components' pair counts
  int n_small, n_large;
  long long E, D, L;          // L = pairs in the larger components
  const int* det_pass;        // [D] number of score cutoffs the detection passes
  const int* det_range;       // [D]
  const int* gt_range;        // [B M]
  int M, K;
  int* match;                 // [2, K, D]
  float* heading;             // [2, K, D]
  void* workspace;
};

// One component's state.  Edge arrays hold n_e entries; node arrays (square problem of N = n_d + n_g rows and columns,
// 1-based as in the textbook O(N^3) Hungarian method) hold N + 1 <= n_e + 2.
struct CompMem {
  int *col, *row_start, *row_det, *col_box, *fixed, *p, *way, *pb;
  long long *w, *u, *v, *minv, *ub, *vb;
  unsigned char *act, *used;
  int* scal;                  // [2] n_d, n_g
};

struct HostGroup {
  __host__ __device__ int tid() const { return 0; }
  __host__ __device__ int size() const { return 1; }
  __host__ __device__ bool leader() const { return true; }
  __host__ __device__ void sync() const {}
  __host__ __device__ void argmin(long long&, int&) const {}
};

template <int T>
struct DevGroup {
  long long* sv;              // [T / 32] shared scratch of the arg-min
  int* sj;
  __device__ int tid() const { return threadIdx.x; }
  __device__ int size() const { return T; }
  __device__ bool leader() const { return threadIdx.x == 0; }
  __device__ void sync() const { __syncthreads(); }
  // every thread gets the minimum value and, among equal values, the lowest index
  __device__ void argmin(long long& v, int& j) const {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const long long ov = __shfl_xor_sync(0xffffffffu, v, off);
      const int oj = __shfl_xor_sync(0xffffffffu, j, off);
      if (ov < v || (ov == v && oj < j)) { v = ov; j = oj; }
    }
    if (T > 32) {
      if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = v; sj[threadIdx.x >> 5] = j; }
      __syncthreads();
      for (int k = 0; k < T / 32; ++k)
        if (sv[k] < v || (sv[k] == v && sj[k] < j)) { v = sv[k]; j = sj[k]; }
      __syncthreads();
    }
  }
};

// Cost of square entry (i, j), false if forbidden.  Rows 1..n_d are the detections (visit order), rows n_d+1..N stand
// for "box j unmatched"; columns 1..n_g are the boxes (ascending index), columns n_g+1..N stand for "detection i
// unmatched".  A detection row costs -w on its active edges and 0 on its own unmatched column; a box row costs 0 on its
// own box and on every detection's unmatched column.  fixed[i] != 0 restricts row i to that column.
__host__ __device__ inline bool lap_cost(const CompMem& m, int n_d, int n_g, int i, int j, long long* c) {
  if (i <= n_d) {
    const int f = m.fixed[i];
    if (f && f != j) return false;
    if (j > n_g) {
      *c = 0;
      return j - n_g == i;
    }
    for (int l = m.row_start[i - 1]; l < m.row_start[i] && m.col[l] <= j - 1; ++l)
      if (m.col[l] == j - 1) {
        *c = -m.w[l];
        return m.act[l] != 0;
      }
    return false;
  }
  *c = 0;
  return j > n_g || i - n_d == j;
}

// Minimum-cost perfect assignment of the square problem (successive shortest paths with potentials u, v): p[j] = the
// row of column j.  Returns the total weight of the detection-box pairs (the maximum total IoU, fixed point), or -1 if
// the constraints leave no assignment.  Integer arithmetic: the result is the same on every thread count.
template <class G>
__host__ __device__ long long lap_solve(const G& g, const CompMem& m, int n_d, int n_g) {
  const int N = n_d + n_g;
  for (int j = g.tid(); j <= N; j += g.size()) { m.u[j] = 0; m.v[j] = 0; m.p[j] = 0; m.way[j] = 0; }
  g.sync();
  for (int i = 1; i <= N; ++i) {
    if (g.leader()) m.p[0] = i;
    for (int j = g.tid(); j <= N; j += g.size()) { m.minv[j] = kInf; m.used[j] = 0; }
    g.sync();
    int j0 = 0;
    for (;;) {
      if (g.leader()) m.used[j0] = 1;
      g.sync();
      const int i0 = m.p[j0];
      long long best = kInf;
      int bj = kNone;
      for (int j = 1 + g.tid(); j <= N; j += g.size()) {
        if (m.used[j]) continue;
        long long c;
        if (lap_cost(m, n_d, n_g, i0, j, &c)) {
          const long long cur = c - m.u[i0] - m.v[j];
          if (cur < m.minv[j]) { m.minv[j] = cur; m.way[j] = j0; }
        }
        if (m.minv[j] < best) { best = m.minv[j]; bj = j; }
      }
      g.argmin(best, bj);
      g.sync();
      if (bj == kNone || best == kInf) return -1;
      // read before the barrier: the update loop does not write p, the leader's augmentation after the break does
      const bool free_col = m.p[bj] == 0;
      for (int j = g.tid(); j <= N; j += g.size()) {
        if (m.used[j]) { m.u[m.p[j]] += best; m.v[j] -= best; }
        else if (m.minv[j] != kInf) m.minv[j] -= best;
      }
      g.sync();
      j0 = bj;
      if (free_col) break;
    }
    if (g.leader()) {
      do {
        const int j1 = m.way[j0];
        m.p[j0] = m.p[j1];
        j0 = j1;
      } while (j0);
    }
    g.sync();
  }
  long long total = 0;
  for (int j = 1; j <= n_g; ++j) {
    long long c;
    if (m.p[j] <= n_d && lap_cost(m, n_d, n_g, m.p[j], j, &c)) total -= c;
  }
  g.sync();
  return total;
}

// The tie rule: of all maximum-IoU assignments, the one chosen detection by detection in visit order, each taking the
// first still possible of its active boxes in ascending index, then "unmatched".  An option is possible when some
// optimal assignment agrees with every earlier choice and with it; an option off the current duals' tight set is not,
// the current assignment's own is, and any other is decided by solving again with it fixed.
template <class G>
__host__ __device__ void lex_assign(const G& g, const CompMem& m, int n_d, int n_g) {
  const int N = n_d + n_g;
  for (int i = g.tid(); i <= n_d; i += g.size()) m.fixed[i] = 0;
  g.sync();
  const long long V = lap_solve(g, m, n_d, n_g);
  for (int i = 1; i <= n_d; ++i) {
    int cc = 0;
    for (int j = 1; j <= N; ++j)
      if (m.p[j] == i) cc = j;
    int l = m.row_start[i - 1];
    const int l1 = m.row_start[i];
    for (;;) {
      while (l < l1 && !m.act[l]) ++l;
      const int o = l < l1 ? m.col[l++] + 1 : n_g + i;
      if (o == cc) break;
      if (o <= n_g && m.p[o] >= 1 && m.p[o] < i) continue;        // held by an earlier, fixed detection
      long long c;
      lap_cost(m, n_d, n_g, i, o, &c);
      if (c - m.u[i] - m.v[o] == 0) {
        for (int j = g.tid(); j <= N; j += g.size()) { m.ub[j] = m.u[j]; m.vb[j] = m.v[j]; m.pb[j] = m.p[j]; }
        if (g.leader()) m.fixed[i] = o;
        g.sync();
        if (lap_solve(g, m, n_d, n_g) == V) { cc = o; break; }
        for (int j = g.tid(); j <= N; j += g.size()) { m.u[j] = m.ub[j]; m.v[j] = m.vb[j]; m.p[j] = m.pb[j]; }
        if (g.leader()) m.fixed[i] = 0;
        g.sync();
      }
      if (o > n_g) break;                                         // unreachable: the current column is an option
    }
    if (g.leader()) m.fixed[i] = cc;
    g.sync();
  }
}

// Loads the component of pairs ge[0 .. n_e): rows (its detections in visit order), columns (its boxes in ascending
// index), edge weights (weight(e), fixed point, maximised) and which edges are active (active(e, det, box)).  Returns
// (n_d, n_g) through m.scal.
template <class G, class Weight, class Active>
__host__ __device__ void load_edges(const G& g, const int* ge, int n_e, const int* e_det, const int* e_box,
                                    const Weight& weight, const CompMem& m, const Active& active) {
  for (int l = g.tid(); l < n_e; l += g.size()) {
    const int k = e_box[ge[l]];
    bool first = true;
    for (int q = 0; q < l && first; ++q) first = e_box[ge[q]] != k;
    m.used[l] = first;
  }
  g.sync();
  for (int l = g.tid(); l < n_e; l += g.size()) {
    const int e = ge[l], k = e_box[e], det = e_det[e];
    int c = 0;
    for (int q = 0; q < n_e; ++q) c += m.used[q] && e_box[ge[q]] < k;
    m.col[l] = c;
    if (m.used[l]) m.col_box[c] = k;
    m.w[l] = weight(e);
    m.act[l] = active(e, det, k);
  }
  if (g.leader()) {
    int n_d = 0, n_g = 0;
    for (int l = 0; l < n_e; ++l) {
      n_g += m.used[l];
      if (l == 0 || e_det[ge[l]] != e_det[ge[l - 1]]) { m.row_det[n_d] = e_det[ge[l]]; m.row_start[n_d++] = l; }
    }
    m.row_start[n_d] = n_e;
    m.scal[0] = n_d;
    m.scal[1] = n_g;
  }
  g.sync();
}

// The IoU of pair e in 40-bit fixed point: exact for every fp32 IoU >= 2^-17, so the sums compare as the IoU sums do.
struct IouWeight {
  const float* e_iou;
  __host__ __device__ long long operator()(int e) const { return (long long)((double)e_iou[e] * kFix); }
};

// The detection-metric rule: the detection passes cutoff kc and, in mode 1, lies in the box's range.
struct CutoffRange {
  const AssignArgs& a;
  int mode, kc;
  __host__ __device__ bool operator()(int, int det, int k) const {
    return kc < a.det_pass[det] && (mode == 0 || a.det_range[det] == a.gt_range[k]);
  }
};

// Loads component `root` for (mode, cutoff kc).
template <class G>
__host__ __device__ void load_component(const G& g, const AssignArgs& a, int root, const CompMem& m, int mode, int kc) {
  load_edges(g, a.grouped + a.comp_start[root], a.comp_nedge[root], a.e_det, a.e_box, IouWeight{a.e_iou}, m,
             CutoffRange{a, mode, kc});
}

template <class G>
__host__ __device__ void assign_component(const G& g, const AssignArgs& a, int root, const CompMem& m, int mode,
                                          int kc) {
  load_component(g, a, root, m, mode, kc);
  const int n_d = m.scal[0], n_g = m.scal[1];
  lex_assign(g, m, n_d, n_g);
  const long long at = ((long long)mode * a.K + kc) * a.D;
  const int* ge = a.grouped + a.comp_start[root];
  for (int i = 1 + g.tid(); i <= n_d; i += g.size()) {
    const int f = m.fixed[i], det = m.row_det[i - 1];
    float h = 0.0f;
    for (int l = m.row_start[i - 1]; l < m.row_start[i]; ++l)
      if (m.col[l] == f - 1) h = a.e_head[ge[l]];
    a.match[at + det] = f <= n_g ? m.col_box[f - 1] % a.M : -1;
    a.heading[at + det] = h;
  }
  g.sync();
}

// Components of at most kSmallEdges pairs, one warp per (component, breakdown, cutoff), all state in shared memory.
__global__ void __launch_bounds__(32) eval_assign_small_kernel(AssignArgs a) {
  constexpr int kE = kSmallEdges, kN = kSmallEdges + 2;
  __shared__ int col[kE], row_start[kE + 1], row_det[kE], col_box[kE], fixed[kE + 1], p[kN], way[kN], pb[kN], scal[2];
  __shared__ long long w[kE], u[kN], v[kN], minv[kN], ub[kN], vb[kN];
  __shared__ unsigned char act[kE], used[kN];
  const int root = a.small_roots[blockIdx.x];
  const CompMem m{col, row_start, row_det, col_box, fixed, p, way, pb, w, u, v, minv, ub, vb, act, used, scal};
  assign_component(DevGroup<32>{nullptr, nullptr}, a, root, m, blockIdx.y / a.K, blockIdx.y % a.K);
}

// Offsets of one component's state in the global workspace: every array is 2L long (L = the pairs of all the larger
// components), the component's at twice its large_off (n_e > kSmallEdges >= 2 pairs, so 2 n_e >= n_e + 2 covers the node
// arrays).
__host__ __device__ inline CompMem workspace_mem(void* ws, long long E, long long at, int* scal) {
  long long* L = (long long*)ws;
  int* I = (int*)(L + 6 * 2 * E);
  unsigned char* U = (unsigned char*)(I + 8 * 2 * E);
  const long long n = 2 * E;
  return CompMem{I + at, I + n + at, I + 2 * n + at, I + 3 * n + at, I + 4 * n + at, I + 5 * n + at, I + 6 * n + at,
                 I + 7 * n + at, L + at, L + n + at, L + 2 * n + at, L + 3 * n + at, L + 4 * n + at, L + 5 * n + at,
                 U + at, U + n + at, scal};
}

__host__ __device__ inline long long assign_workspace_bytes(long long E) { return 2 * E * (6 * 8 + 8 * 4 + 2); }

// Components of more than kSmallEdges pairs: one CTA each, every breakdown and cutoff in turn, state in the workspace.
__global__ void __launch_bounds__(kLargeThreads) eval_assign_large_kernel(AssignArgs a) {
  __shared__ long long sv[kLargeThreads / 32];
  __shared__ int sj[kLargeThreads / 32], scal[2];
  const int root = a.large_roots[blockIdx.x];
  const CompMem m = workspace_mem(a.workspace, a.L, 2 * a.large_off[blockIdx.x], scal);
  for (int y = 0; y < 2 * a.K; ++y) assign_component(DevGroup<kLargeThreads>{sv, sj}, a, root, m, y / a.K, y % a.K);
}

int check_assign_args(const AssignArgs& a) {
  PNX_CHECK_ARG(a.E >= 0 && a.E < (1LL << 30) && a.D >= 0 && a.D < (1LL << 31), "number of pairs / detections");
  PNX_CHECK_ARG(a.K >= 1 && a.K <= 1024 && a.M >= 1, "1 to 1024 score cutoffs, M >= 1");
  PNX_CHECK_ARG(a.E == 0 || (a.grouped && a.comp_start && a.comp_nedge && a.e_det && a.e_box && a.e_iou && a.e_head &&
                              a.gt_range), "pair pointers");
  PNX_CHECK_ARG(a.n_small >= 0 && a.n_large >= 0 && (long long)a.n_small + a.n_large <= a.E && a.L >= 0 && a.L <= a.E,
                "component lists");
  PNX_CHECK_ARG(a.n_small == 0 || a.small_roots, "small_roots");
  PNX_CHECK_ARG(a.n_large == 0 || (a.large_roots && a.large_off), "large_roots / large_off");
  PNX_CHECK_ARG(a.D == 0 || (a.det_pass && a.det_range && a.match && a.heading), "detection pointers");
  return PNX_OK;
}

// ---------------------------------------------------------------- CLEAR-MOT frame matching (evaluate_waymo_tracking.py)
// The inputs of the frame walk both tracking metrics share.
struct MotWalk {
  const int* edge_start;      // [B C] first pair of each segment (pnx_eval_pairs / pnx_eval_pairs_center)
  const int* edge_count;      // [B C]
  const int* grouped;         // [E] components of pnx_eval_components
  const int* comp_start;      // [E]
  const int* comp_nedge;      // [E]
  const int* e_det;           // [E]
  const int* e_box;           // [E] f M + j
  const int* det_pass;        // [D] number of score cutoffs the detection passes
  const int* det_id;          // [D] tracking id >= 0
  const int* gt_obj;          // [B M] object index in [0, n_obj), -1 = none
  const int* seq_start;       // [S + 1] the frames of sequence s are [seq_start[s], seq_start[s + 1])
  int S, B, M, C, K, n_obj, cap;
  long long E, D;
  int* last_id;               // [K, n_obj] the tracking id of each object's last match, -1 = none yet
  void* workspace;            // [S C K] x mot_row_bytes(M, cap)
};

struct MotArgs {
  MotWalk w;
  const float* e_iou;         // [E]
  const int* gt_points;       // [B M] point count (difficulty level)
  long long* counts;          // [S, C, K, 5] matches; L1 matches, L1 mismatches; L2 matches, L2 mismatches
  double* dist;               // [S, C, K, 2] sum of 1 - IoU over the L1 / L2 matches
};

constexpr int kMotCounts = 5;

// one row's workspace: the assignment state of a component of up to cap pairs, then the frame's kept-box table [M]
__host__ __device__ inline long long mot_comp_bytes(int cap) { return (assign_workspace_bytes(cap) + 15) / 16 * 16; }
__host__ __device__ inline long long mot_row_bytes(int M, int cap) {
  return mot_comp_bytes(cap) + ((long long)M * sizeof(int) + 15) / 16 * 16;
}

// Pairs the assignment may use at cutoff kc: the detection passes it, and neither the detection nor the box was kept
// by the carry-over (kept[j] = the detection holding box j, -1 = none; a detection's pairs are consecutive in [e0, e1)).
struct MotActive {
  const MotWalk& a;
  const int* kept;
  int kc, e0, e1;
  __host__ __device__ bool operator()(int e, int det, int k) const {
    if (kc >= a.det_pass[det] || kept[k % a.M] >= 0) return false;
    for (int q = e; q >= e0 && a.e_det[q] == det; --q)
      if (kept[a.e_box[q] % a.M] == det) return false;
    for (int q = e + 1; q < e1 && a.e_det[q] == det; ++q)
      if (kept[a.e_box[q] % a.M] == det) return false;
    return true;
  }
};

// The Waymo rule (Rule of mot_row): the maximum-IoU assignment, and per match of (detection det, box kb, pair e) the
// counts of the levels the box belongs to and sum(1 - IoU).
struct LevelCounts {
  const MotArgs& a;
  IouWeight weight;
  long long n[kMotCounts] = {0, 0, 0, 0, 0};
  double d[2] = {0.0, 0.0};
  __host__ __device__ explicit LevelCounts(const MotArgs& args) : a(args), weight{args.e_iou} {}
  __host__ __device__ void match(int, int, int, int kb, int e, int, bool mism) {
    const int pts = a.gt_points[kb];
    const double miss_iou = 1.0 - (double)a.e_iou[e];
    ++n[0];
    if (pts > 5) { ++n[1]; n[2] += mism; d[0] += miss_iou; }
    if (pts >= 1) { ++n[3]; n[4] += mism; d[1] += miss_iou; }
  }
  __host__ __device__ void finish(int row) const {
    for (int q = 0; q < kMotCounts; ++q) a.counts[(long long)row * kMotCounts + q] = n[q];
    a.dist[2 * (long long)row] = d[0];
    a.dist[2 * (long long)row + 1] = d[1];
  }
};

// One match: a mismatch when the object's previous match carried another id, the rule's counts, the object's last id.
template <class Rule>
__host__ __device__ inline void mot_match(const MotWalk& a, int* last, Rule& r, int kc, int f, int det, int kb, int e) {
  const int o = a.gt_obj[kb], id = a.det_id[det];
  const bool mism = o >= 0 && last[o] >= 0 && last[o] != id;
  r.match(kc, f, det, kb, e, o, mism);
  if (o >= 0) last[o] = id;
}

// One (sequence, class, cutoff) row, frames in order: the carry-over (leader, pairs in order), then every component of
// the frame's pairs solved by the tie-ruled assignment maximising r.weight over the pairs left active.  The rule counts
// the matches on the leader and writes the row in r.finish.
template <class G, class Rule>
__host__ __device__ void mot_row(const G& g, const MotWalk& a, int row, const CompMem& m, int* kept, Rule& r) {
  const int s = row / (a.C * a.K), c = (row / a.K) % a.C, kc = row % a.K;
  int* last = a.last_id + (long long)kc * a.n_obj;
  for (int f = a.seq_start[s]; f < a.seq_start[s + 1]; ++f) {
    const int seg = f * a.C + c;
    const int e0 = a.edge_start[seg], e1 = e0 + a.edge_count[seg];
    for (int e = e0 + g.tid(); e < e1; e += g.size()) kept[a.e_box[e] % a.M] = -1;
    g.sync();
    if (g.leader()) {
      bool det_kept = false;
      for (int e = e0; e < e1; ++e) {
        const int det = a.e_det[e], kb = a.e_box[e], j = kb % a.M;
        if (e > e0 && det != a.e_det[e - 1]) det_kept = false;
        if (det_kept || kc >= a.det_pass[det] || kept[j] >= 0) continue;
        const int o = a.gt_obj[kb];
        if (o < 0 || last[o] != a.det_id[det]) continue;
        kept[j] = det;
        det_kept = true;
        mot_match(a, last, r, kc, f, det, kb, e);
      }
    }
    g.sync();
    for (int q = e0; q < e1; ++q) {
      if (a.comp_start[q] < 0) continue;                       // not a component's first pair
      const int* ge = a.grouped + a.comp_start[q];
      load_edges(g, ge, a.comp_nedge[q], a.e_det, a.e_box, r.weight, m, MotActive{a, kept, kc, e0, e1});
      bool any = false;
      for (int l = 0; l < a.comp_nedge[q]; ++l) any |= m.act[l] != 0;
      if (!any) continue;
      const int n_d = m.scal[0], n_g = m.scal[1];
      lex_assign(g, m, n_d, n_g);
      if (g.leader())
        for (int i = 1; i <= n_d; ++i) {
          const int fx = m.fixed[i];
          if (fx > n_g) continue;
          for (int l = m.row_start[i - 1]; l < m.row_start[i]; ++l)
            if (m.col[l] == fx - 1) { mot_match(a, last, r, kc, f, m.row_det[i - 1], a.e_box[ge[l]], ge[l]); break; }
        }
      g.sync();
    }
  }
  if (g.leader()) r.finish(row);
}

// One warp per (sequence, class, cutoff) row, its state in its slice of the workspace.
template <class Args, class Rule>
__global__ void __launch_bounds__(32) eval_mot_kernel(Args a) {
  __shared__ int scal[2];
  const MotWalk& w = a.w;
  char* base = (char*)w.workspace + (long long)blockIdx.x * mot_row_bytes(w.M, w.cap);
  const CompMem m = workspace_mem(base, w.cap, 0, scal);
  Rule r(a);
  mot_row(DevGroup<32>{nullptr, nullptr}, w, blockIdx.x, m, (int*)(base + mot_comp_bytes(w.cap)), r);
}

// The host twin of eval_mot_kernel: every row in turn through one row's workspace.
template <class Args, class Rule>
void host_mot(const Args& a) {
  const MotWalk& w = a.w;
  for (long long i = 0; i < (long long)w.K * w.n_obj; ++i) w.last_id[i] = -1;
  char* ws = new char[mot_row_bytes(w.M, w.cap)];
  int scal[2];
  const CompMem m = workspace_mem(ws, w.cap, 0, scal);
  for (long long row = 0; row < (long long)w.S * w.C * w.K; ++row) {
    Rule r(a);
    mot_row(HostGroup{}, w, (int)row, m, (int*)(ws + mot_comp_bytes(w.cap)), r);
  }
  delete[] ws;
}

int check_mot_walk(const MotWalk& a) {
  PNX_CHECK_ARG(a.S >= 0 && a.B >= 0 && a.C >= 1 && a.K >= 1 && a.n_obj >= 0, "S / B / C / K / n_obj");
  PNX_CHECK_ARG(a.M >= 1 && a.M <= kMaxBoxesPerFrame, "1 to 4096 boxes per frame");
  PNX_CHECK_ARG((long long)a.S * a.C * a.K < (1LL << 31) && (long long)a.B * a.C < (1LL << 31), "too many rows");
  PNX_CHECK_ARG(a.cap >= kSmallEdges + 2, "cap >= pnx_eval_assign_warp_pairs() + 2");
  PNX_CHECK_ARG(a.E >= 0 && a.E < (1LL << 30) && a.D >= 0 && a.D < (1LL << 31), "number of pairs / detections");
  PNX_CHECK_ARG(a.seq_start && (a.B == 0 || (a.edge_start && a.edge_count)), "segment pointers");
  PNX_CHECK_ARG(a.E == 0 || (a.grouped && a.comp_start && a.comp_nedge && a.e_det && a.e_box && a.det_pass &&
                              a.det_id && a.gt_obj), "pair pointers");
  PNX_CHECK_ARG(a.S == 0 || a.last_id, "last_id");
  return PNX_OK;
}

int check_mot_args(const MotArgs& a) {
  int rc = check_mot_walk(a.w);
  if (rc) return rc;
  PNX_CHECK_ARG(a.w.E == 0 || (a.e_iou && a.gt_points), "pair pointers");
  PNX_CHECK_ARG(a.w.S == 0 || (a.counts && a.dist), "output pointers");
  return PNX_OK;
}

// ---------------------------------------------------------------- nuScenes tracking (evaluate_nuscenes_tracking.py)
// Cardinality first, then the smallest distance sum, in one maximised integer weight per pair: 2^40 - dq with dq =
// round(d 2^26) of the fp32 distance d <= 2^1 (so dq <= 2^27).  A component's matches are at most its boxes, M <= 2^12,
// so the dq of any assignment sum to at most 2^39 < 2^40: one more match always outweighs every distance difference.
constexpr long long kMatchUnit = 1LL << 40;
constexpr double kDistFix = 67108864.0;      // 2^26: d 2^26 is exact in fp64, + 0.5 rounds half up
constexpr int kCenterCounts = 3;

struct CenterWeight {
  const float* e_dist;
  __host__ __device__ long long operator()(int e) const {
    return kMatchUnit - (long long)((double)e_dist[e] * kDistFix + 0.5);
  }
};

struct CenterMotArgs {
  MotWalk w;
  const float* e_dist;        // [E] fp32 centre distance
  const int* gt_prev;         // [B M] the frame of the object's previous box, -1 = none (first box, or no object)
  int* last_frame;            // [K, n_obj] the frame of each object's last match, -1 = none yet
  long long* counts;          // [S, C, K, 3] matches, identity switches, fragmentations
  double* dist;               // [S, C, K] sum of the matches' fp32 distances
  unsigned char* matched;     // [D] or null: 1 for each matched detection (K = 1 only)
};

// The nuScenes rule (Rule of mot_row): the cardinality-first minimum-distance assignment; per match the count, the
// identity switch, a fragmentation when the object was matched before and has a box after that match, and sum(d).
struct CenterCounts {
  const CenterMotArgs& a;
  CenterWeight weight;
  long long n[kCenterCounts] = {0, 0, 0};
  double d = 0.0;
  __host__ __device__ explicit CenterCounts(const CenterMotArgs& args) : a(args), weight{args.e_dist} {}
  __host__ __device__ void match(int kc, int f, int det, int kb, int e, int o, bool mism) {
    ++n[0];
    n[1] += mism;
    if (o >= 0) {
      int* lf = a.last_frame + (long long)kc * a.w.n_obj + o;
      n[2] += *lf >= 0 && a.gt_prev[kb] > *lf;
      *lf = f;
    }
    d += (double)a.e_dist[e];
    if (a.matched) a.matched[det] = 1;
  }
  __host__ __device__ void finish(int row) const {
    for (int q = 0; q < kCenterCounts; ++q) a.counts[(long long)row * kCenterCounts + q] = n[q];
    a.dist[row] = d;
  }
};

int check_center_mot_args(const CenterMotArgs& a) {
  int rc = check_mot_walk(a.w);
  if (rc) return rc;
  PNX_CHECK_ARG(a.w.E == 0 || (a.e_dist && a.gt_prev), "pair pointers");
  PNX_CHECK_ARG(a.w.S == 0 || (a.last_frame && a.counts && a.dist), "output pointers");
  PNX_CHECK_ARG(!a.matched || a.w.K == 1, "matched flags need K = 1");
  return PNX_OK;
}

struct CenterPairArgs {
  const float* det_boxes;     // [D, 9]
  const long long* order;     // [D] detection indices, sorted by segment, then in visit order
  const int* seg_start;       // [B C]
  const int* seg_count;       // [B C]
  const float* gt_boxes;      // [B, M, 9]
  const int* gt_classes;      // [B, M], -1 = padding or filtered out
  int B, M, C;
  double max_dist;            // a pair needs centre distance < max_dist
  long long D;
  const int* edge_start;      // [B C] or null: count only
  int* edge_count;            // [B C]
  int* e_det;                 // [E] detection index
  int* e_box;                 // [E] f M + j
  float* e_dist;              // [E] the fp64 distance rounded to fp32
};

// One warp per (frame, class) segment: every pair with centre distance < max_dist, laid out as eval_pairs_kernel's.
__global__ void __launch_bounds__(32) eval_pairs_center_kernel(CenterPairArgs p) {
  extern __shared__ float smem[];
  const int s = blockIdx.x, lane = threadIdx.x;
  const int f = s / p.C, c = s - f * p.C;
  float* xy = smem;                                           // [M, 2] box centres
  int* idx = (int*)(xy + 2 * (size_t)p.M);                    // [M] box index within the frame
  const int G = warp_class_boxes(p.gt_classes + (long long)f * p.M, p.M, c, lane, idx);
  __syncwarp();
  for (int q = lane; q < G; q += 32) {
    const float* g = p.gt_boxes + ((long long)f * p.M + idx[q]) * 9;
    xy[2 * q] = g[0];
    xy[2 * q + 1] = g[1];
  }
  __syncwarp();
  const int n = p.seg_count[s], base = p.seg_start[s];
  int cursor = p.edge_start ? p.edge_start[s] : 0;
  for (int t = 0; t < n; ++t) {
    const long long di = p.order[base + t];
    const float* d = p.det_boxes + di * 9;
    for (int q0 = 0; q0 < G; q0 += 32) {
      const int q = q0 + lane;
      const double v = q < G ? center_distance(d, xy + 2 * q) : INFINITY;
      const bool hit = v < p.max_dist;
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      if (hit && p.edge_start) {
        const int e = cursor + __popc(bal & ((1u << lane) - 1u));
        p.e_det[e] = (int)di;
        p.e_box[e] = f * p.M + idx[q];
        p.e_dist[e] = (float)v;
      }
      cursor += __popc(bal);
    }
  }
  if (lane == 0 && !p.edge_start) p.edge_count[s] = cursor;
}

void host_pairs_center(const CenterPairArgs& p) {
  int* idx = new int[p.M > 0 ? p.M : 1];
  for (long long s = 0; s < (long long)p.B * p.C; ++s) {
    const int f = (int)(s / p.C), c = (int)(s % p.C);
    const int G = host_class_boxes(p.gt_classes + (long long)f * p.M, p.M, c, idx);
    int cursor = p.edge_start ? p.edge_start[s] : 0;
    for (int t = 0; t < p.seg_count[s]; ++t) {
      const long long di = p.order[p.seg_start[s] + t];
      for (int q = 0; q < G; ++q) {
        const double v = center_distance(p.det_boxes + di * 9, p.gt_boxes + ((long long)f * p.M + idx[q]) * 9);
        if (!(v < p.max_dist)) continue;
        if (p.edge_start) {
          p.e_det[cursor] = (int)di;
          p.e_box[cursor] = f * p.M + idx[q];
          p.e_dist[cursor] = (float)v;
        }
        ++cursor;
      }
    }
    if (!p.edge_start) p.edge_count[s] = cursor;
  }
  delete[] idx;
}

int check_pairs_center_args(const CenterPairArgs& p) {
  PNX_CHECK_ARG(p.D >= 0 && p.D < (1LL << 31), "number of detections");
  PNX_CHECK_ARG(p.B >= 0 && p.C >= 1 && p.M >= 0 && p.M <= kMaxBoxesPerFrame, "B / C / at most 4096 boxes per frame");
  PNX_CHECK_ARG((long long)p.B * p.C < (1LL << 31), "too many segments");
  PNX_CHECK_ARG(p.max_dist > 0.0 && p.max_dist <= 2.0, "max_dist in (0, 2] metres");
  PNX_CHECK_ARG(p.D == 0 || (p.det_boxes && p.order), "detection pointers");
  PNX_CHECK_ARG((long long)p.B * p.M == 0 || (p.gt_boxes && p.gt_classes), "ground-truth pointers");
  PNX_CHECK_ARG(p.B == 0 || (p.seg_start && p.seg_count), "segment pointers");
  PNX_CHECK_ARG(p.B == 0 || (p.edge_start ? (p.e_det && p.e_box && p.e_dist) : p.edge_count != nullptr), "pair outputs");
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

extern "C" int pnx_eval_pairs(const float* det_boxes, const float* det_trig, long long n_det, const long long* order,
                              const int* seg_start, const int* seg_count, const float* gt_boxes, const int* gt_classes,
                              const float* gt_trig, int B, int M, int C, const float* thresholds, const int* edge_start,
                              int* edge_count, int* e_det, int* e_box, float* e_iou, float* e_head, cudaStream_t stream) {
  const PairArgs p{{det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, B, M, C, thresholds,
                    nullptr, nullptr, nullptr},
                   edge_start, edge_count, e_det, e_box, e_iou, e_head};
  PNX_CHECK_ARG(n_det >= 0 && n_det < (1LL << 31), "number of detections");
  PNX_CHECK_ARG(B == 0 || (edge_start ? (e_det && e_box && e_iou && e_head) : edge_count != nullptr), "pair outputs");
  const MatchArgs& a = p.m;
  const int nd = (int)n_det;
  PNX_CHECK_ARG(a.B >= 0 && a.C >= 1 && a.M >= 0 && a.M <= kMaxBoxesPerFrame, "B / C / at most 4096 boxes per frame");
  PNX_CHECK_ARG((long long)a.B * a.C < (1LL << 31), "too many segments");
  PNX_CHECK_ARG(nd == 0 || (a.det_boxes && a.det_trig && a.order), "detection pointers");
  PNX_CHECK_ARG((long long)a.B * a.M == 0 || (a.gt_boxes && a.gt_classes && a.gt_trig), "ground-truth pointers");
  PNX_CHECK_ARG(a.B == 0 || (a.seg_start && a.seg_count && a.thresholds), "segment / threshold pointers");
  if (B == 0) return PNX_OK;
  const size_t smem = (size_t)M * (kSlot * sizeof(float) + sizeof(int));
  if (smem > 48 * 1024) PNX_CUDA(cudaFuncSetAttribute(eval_pairs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  eval_pairs_kernel<<<B * C, 32, smem, stream>>>(p);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_eval_pairs_host(const float* det_boxes, const float* det_trig, long long n_det, const long long* order,
                                   const int* seg_start, const int* seg_count, const float* gt_boxes, const int* gt_classes,
                                   const float* gt_trig, int B, int M, int C, const float* thresholds,
                                   const int* edge_start, int* edge_count, int* e_det, int* e_box, float* e_iou, float* e_head) {
  const PairArgs p{{det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, B, M, C, thresholds,
                    nullptr, nullptr, nullptr},
                   edge_start, edge_count, e_det, e_box, e_iou, e_head};
  PNX_CHECK_ARG(n_det >= 0 && n_det < (1LL << 31), "number of detections");
  PNX_CHECK_ARG(B == 0 || (edge_start ? (e_det && e_box && e_iou && e_head) : edge_count != nullptr), "pair outputs");
  const MatchArgs& a = p.m;
  PNX_CHECK_ARG(a.B >= 0 && a.C >= 1 && a.M >= 0 && a.M <= kMaxBoxesPerFrame, "B / C / at most 4096 boxes per frame");
  PNX_CHECK_ARG((long long)a.B * a.C < (1LL << 31), "too many segments");
  PNX_CHECK_ARG(n_det == 0 || (a.det_boxes && a.det_trig && a.order), "detection pointers");
  PNX_CHECK_ARG((long long)a.B * a.M == 0 || (a.gt_boxes && a.gt_classes && a.gt_trig), "ground-truth pointers");
  PNX_CHECK_ARG(a.B == 0 || (a.seg_start && a.seg_count && a.thresholds), "segment / threshold pointers");
  host_pairs(p);
  return PNX_OK;
}

static int check_comp_args(const CompArgs& a, long long n_edges) {
  PNX_CHECK_ARG(a.B >= 0 && a.C >= 1 && a.M >= 0 && a.M <= kMaxBoxesPerFrame, "B / C / at most 4096 boxes per frame");
  PNX_CHECK_ARG((long long)a.B * a.C < (1LL << 31) && n_edges >= 0 && n_edges < (1LL << 30), "segments / pairs");
  PNX_CHECK_ARG(a.B == 0 || (a.edge_start && a.edge_count), "segment pointers");
  PNX_CHECK_ARG(n_edges == 0 || (a.e_det && a.e_box && a.root && a.comp_start && a.comp_nedge && a.grouped),
                "pair pointers");
  return PNX_OK;
}

extern "C" int pnx_eval_components(const int* edge_start, const int* edge_count, int B, int M, int C, long long n_edges,
                                   const int* e_det, const int* e_box, int* root, int* comp_start, int* comp_nedge,
                                   int* grouped, cudaStream_t stream) {
  const CompArgs a{edge_start, edge_count, B, M, C, e_det, e_box, root, comp_start, comp_nedge, grouped};
  int rc = check_comp_args(a, n_edges);
  if (rc) return rc;
  if (n_edges == 0) return PNX_OK;
  eval_components_kernel<<<B * C, 32, (size_t)M * sizeof(int), stream>>>(a);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_eval_components_host(const int* edge_start, const int* edge_count, int B, int M, int C,
                                        long long n_edges, const int* e_det, const int* e_box, int* root,
                                        int* comp_start, int* comp_nedge, int* grouped) {
  const CompArgs a{edge_start, edge_count, B, M, C, e_det, e_box, root, comp_start, comp_nedge, grouped};
  int rc = check_comp_args(a, n_edges);
  if (rc) return rc;
  if (n_edges == 0) return PNX_OK;
  int* last = new int[M];
  for (int j = 0; j < M; ++j) last[j] = -1;
  for (long long s = 0; s < (long long)B * C; ++s)
    if (edge_count[s] > 0)
      segment_components(edge_start[s], edge_start[s] + edge_count[s], M, e_det, e_box, last, root, comp_start,
                         comp_nedge, grouped);
  delete[] last;
  return PNX_OK;
}

extern "C" long long pnx_eval_assign_workspace(long long large_pairs) { return assign_workspace_bytes(large_pairs); }

extern "C" int pnx_eval_assign_warp_pairs(void) { return kSmallEdges; }

extern "C" int pnx_eval_assign(long long n_edges, const int* grouped, const int* comp_start, const int* comp_nedge,
                               const int* e_det, const int* e_box, const float* e_iou, const float* e_head,
                               const int* small_roots, int n_small, const int* large_roots, const long long* large_off,
                               int n_large, long long large_pairs, long long n_det, const int* det_pass,
                               const int* det_range, const int* gt_range, int M, int K, int* match, float* heading,
                               void* workspace, cudaStream_t stream) {
  const AssignArgs a{grouped, comp_start, comp_nedge, e_det, e_box, e_iou, e_head, small_roots, large_roots, large_off,
                     n_small, n_large, n_edges, n_det, large_pairs, det_pass, det_range, gt_range, M, K, match, heading,
                     workspace};
  int rc = check_assign_args(a);
  if (rc) return rc;
  PNX_CHECK_ARG(n_large == 0 || workspace, "workspace");
  PNX_CHECK_ARG(2 * K <= 65535, "at most 32767 score cutoffs on the device");
  if (n_det > 0) {
    PNX_CUDA(cudaMemsetAsync(match, 0xff, (size_t)2 * K * n_det * sizeof(int), stream));
    PNX_CUDA(cudaMemsetAsync(heading, 0, (size_t)2 * K * n_det * sizeof(float), stream));
  }
  if (n_small > 0) {
    eval_assign_small_kernel<<<dim3((unsigned)n_small, 2 * K), 32, 0, stream>>>(a);
    PNX_CHECK_LAUNCH();
  }
  if (n_large > 0) {
    eval_assign_large_kernel<<<(unsigned)n_large, kLargeThreads, 0, stream>>>(a);
    PNX_CHECK_LAUNCH();
  }
  return PNX_OK;
}

extern "C" int pnx_eval_assign_host(long long n_edges, const int* grouped, const int* comp_start, const int* comp_nedge,
                                    const int* e_det, const int* e_box, const float* e_iou, const float* e_head,
                                    const int* small_roots, int n_small, const int* large_roots,
                                    const long long* large_off, int n_large, long long large_pairs, long long n_det,
                                    const int* det_pass, const int* det_range, const int* gt_range, int M, int K,
                                    int* match, float* heading) {
  const AssignArgs a{grouped, comp_start, comp_nedge, e_det, e_box, e_iou, e_head, small_roots, large_roots, large_off,
                     n_small, n_large, n_edges, n_det, large_pairs, det_pass, det_range, gt_range, M, K, match, heading,
                     nullptr};
  int rc = check_assign_args(a);
  if (rc) return rc;
  for (long long i = 0; i < 2 * K * n_det; ++i) { match[i] = -1; heading[i] = 0.0f; }
  // every component through the same state layout, one at a time: one region sized for kSmallEdges + 2 or the largest
  long long cap = kSmallEdges + 2;
  for (int r = 0; r < n_large; ++r) cap = comp_nedge[large_roots[r]] > cap ? comp_nedge[large_roots[r]] : cap;
  void* ws = new char[assign_workspace_bytes(cap)];
  int scal[2];
  for (int r = 0; r < n_small + n_large; ++r) {
    const int root = r < n_small ? small_roots[r] : large_roots[r - n_small];
    const CompMem m = workspace_mem(ws, cap, 0, scal);
    for (int y = 0; y < 2 * K; ++y) assign_component(HostGroup{}, a, root, m, y / K, y % K);
  }
  delete[] (char*)ws;
  return PNX_OK;
}

extern "C" long long pnx_eval_mot_workspace(int rows, int M, int cap) { return (long long)rows * mot_row_bytes(M, cap); }

extern "C" int pnx_eval_mot(const int* edge_start, const int* edge_count, long long n_edges, const int* grouped,
                            const int* comp_start, const int* comp_nedge, const int* e_det, const int* e_box,
                            const float* e_iou, long long n_det, const int* det_pass, const int* det_id,
                            const int* gt_obj, const int* gt_points, const int* seq_start, int S, int B, int M, int C,
                            int K, int n_obj, int cap, int* last_id, long long* counts, double* dist, void* workspace,
                            cudaStream_t stream) {
  const MotArgs a{{edge_start, edge_count, grouped, comp_start, comp_nedge, e_det, e_box, det_pass, det_id, gt_obj,
                   seq_start, S, B, M, C, K, n_obj, cap, n_edges, n_det, last_id, workspace},
                  e_iou, gt_points, counts, dist};
  int rc = check_mot_args(a);
  if (rc) return rc;
  const long long rows = (long long)S * C * K;
  if (rows == 0) return PNX_OK;
  PNX_CHECK_ARG(workspace, "workspace");
  if (n_obj > 0) PNX_CUDA(cudaMemsetAsync(last_id, 0xff, (size_t)K * n_obj * sizeof(int), stream));
  eval_mot_kernel<MotArgs, LevelCounts><<<(unsigned)rows, 32, 0, stream>>>(a);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_eval_mot_host(const int* edge_start, const int* edge_count, long long n_edges, const int* grouped,
                                 const int* comp_start, const int* comp_nedge, const int* e_det, const int* e_box,
                                 const float* e_iou, long long n_det, const int* det_pass, const int* det_id,
                                 const int* gt_obj, const int* gt_points, const int* seq_start, int S, int B, int M,
                                 int C, int K, int n_obj, int cap, int* last_id, long long* counts, double* dist) {
  const MotArgs a{{edge_start, edge_count, grouped, comp_start, comp_nedge, e_det, e_box, det_pass, det_id, gt_obj,
                   seq_start, S, B, M, C, K, n_obj, cap, n_edges, n_det, last_id, nullptr},
                  e_iou, gt_points, counts, dist};
  int rc = check_mot_args(a);
  if (rc) return rc;
  host_mot<MotArgs, LevelCounts>(a);
  return PNX_OK;
}

extern "C" int pnx_eval_pairs_center(const float* det_boxes, long long n_det, const long long* order,
                                     const int* seg_start, const int* seg_count, const float* gt_boxes,
                                     const int* gt_classes, int B, int M, int C, double max_dist, const int* edge_start,
                                     int* edge_count, int* e_det, int* e_box, float* e_dist, cudaStream_t stream) {
  const CenterPairArgs p{det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, B, M, C, max_dist, n_det,
                         edge_start, edge_count, e_det, e_box, e_dist};
  int rc = check_pairs_center_args(p);
  if (rc) return rc;
  if (B == 0) return PNX_OK;
  const size_t smem = (size_t)M * (2 * sizeof(float) + sizeof(int));
  eval_pairs_center_kernel<<<B * C, 32, smem, stream>>>(p);    // at most 48 KB: M <= 4096
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_eval_pairs_center_host(const float* det_boxes, long long n_det, const long long* order,
                                          const int* seg_start, const int* seg_count, const float* gt_boxes,
                                          const int* gt_classes, int B, int M, int C, double max_dist,
                                          const int* edge_start, int* edge_count, int* e_det, int* e_box,
                                          float* e_dist) {
  const CenterPairArgs p{det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, B, M, C, max_dist, n_det,
                         edge_start, edge_count, e_det, e_box, e_dist};
  int rc = check_pairs_center_args(p);
  if (rc) return rc;
  host_pairs_center(p);
  return PNX_OK;
}

extern "C" int pnx_eval_mot_center(const int* edge_start, const int* edge_count, long long n_edges, const int* grouped,
                                   const int* comp_start, const int* comp_nedge, const int* e_det, const int* e_box,
                                   const float* e_dist, long long n_det, const int* det_pass, const int* det_id,
                                   const int* gt_obj, const int* gt_prev, const int* seq_start, int S, int B, int M,
                                   int C, int K, int n_obj, int cap, int* last_id, int* last_frame, long long* counts,
                                   double* dist, unsigned char* matched, void* workspace, cudaStream_t stream) {
  const CenterMotArgs a{{edge_start, edge_count, grouped, comp_start, comp_nedge, e_det, e_box, det_pass, det_id,
                         gt_obj, seq_start, S, B, M, C, K, n_obj, cap, n_edges, n_det, last_id, workspace},
                        e_dist, gt_prev, last_frame, counts, dist, matched};
  int rc = check_center_mot_args(a);
  if (rc) return rc;
  if (matched && n_det > 0) PNX_CUDA(cudaMemsetAsync(matched, 0, (size_t)n_det, stream));
  const long long rows = (long long)S * C * K;
  if (rows == 0) return PNX_OK;
  PNX_CHECK_ARG(workspace, "workspace");
  if (n_obj > 0) {
    PNX_CUDA(cudaMemsetAsync(last_id, 0xff, (size_t)K * n_obj * sizeof(int), stream));
    PNX_CUDA(cudaMemsetAsync(last_frame, 0xff, (size_t)K * n_obj * sizeof(int), stream));
  }
  eval_mot_kernel<CenterMotArgs, CenterCounts><<<(unsigned)rows, 32, 0, stream>>>(a);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_eval_mot_center_host(const int* edge_start, const int* edge_count, long long n_edges,
                                        const int* grouped, const int* comp_start, const int* comp_nedge,
                                        const int* e_det, const int* e_box, const float* e_dist, long long n_det,
                                        const int* det_pass, const int* det_id, const int* gt_obj, const int* gt_prev,
                                        const int* seq_start, int S, int B, int M, int C, int K, int n_obj, int cap,
                                        int* last_id, int* last_frame, long long* counts, double* dist,
                                        unsigned char* matched) {
  const CenterMotArgs a{{edge_start, edge_count, grouped, comp_start, comp_nedge, e_det, e_box, det_pass, det_id,
                         gt_obj, seq_start, S, B, M, C, K, n_obj, cap, n_edges, n_det, last_id, nullptr},
                        e_dist, gt_prev, last_frame, counts, dist, matched};
  int rc = check_center_mot_args(a);
  if (rc) return rc;
  if (matched)
    for (long long i = 0; i < n_det; ++i) matched[i] = 0;
  for (long long i = 0; i < (long long)K * n_obj; ++i) last_frame[i] = -1;
  host_mot<CenterMotArgs, CenterCounts>(a);
  return PNX_OK;
}
