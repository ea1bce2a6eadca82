// sweeps.cu -- multi-sweep accumulation: past LiDAR sweeps taken into the key frame and merged behind it, sm_90a.
//
// What the reference's data-loader workers do per frame in numpy, for a collated batch:
//   nuScenes  NuScenesDataset.load_pointcloud / read_sweep / remove_close (det3d/datasets/nuscenes/nusc.py): each sweep's
//             xyz goes through its 4x4 transform_matrix in fp64 and is written back into the sweep's fp32 array; then the
//             sweep loses the points with |x| < min_distance and |y| < min_distance (strict, AND, on the rounded fp32
//             coordinates; min_distance = 1.0).  A sweep whose transform_matrix is None keeps its coordinates.  The key
//             frame is never filtered.  The time column is float32(time_lag).
//   Waymo     WaymoDataset.load_pointcloud (det3d/datasets/waymo/waymo.py): the transform is rel_pose = inv(pose) @
//             sweep_pose (fp64, computed by the caller), no close-point removal (min_distance = 0), time float32(timestamp).
// Output per frame: the key frame's points, then sweep 1, 2, ... in order, each sweep's points in file order; frames in
// batch order, so frame-sorted input stays frame-sorted.
//
// Arithmetic: each output coordinate is computed in fp64 in one fixed, FMA-free order, ((m0 x + m1 y) + m2 z) + m3 with
// x, y, z the fp32 inputs widened exactly, and rounded once to fp32 (the _rn intrinsics on the device; plain operators in
// the host twin, whose compiler has no FMA to contract into).  A sweep without transform (its matrix's [3][3] entry is
// NaN) is copied, not multiplied by the identity: -0.0 * 1 + 0.0 = +0.0 would change the bits.  numpy evaluates the
// reference's dot / @ through BLAS, whose FMA use and summation order are not fixed, so its result can differ from this
// one by one fp32 ulp -- only where the exact value lies next to the midpoint between two fp32 neighbours.
//
// Three launches on the stream, no host sync:
//   mark   (only with min_distance > 0) one thread per sweep point: transform, close-point test; one keep bit per point
//          (a ballot word per warp) and a kept count per block.
//   scan   one CTA: exclusive scan of the block counts; for every frame f the kept sweep points of frames < f; the count.
//   write  one thread per sweep point (transform again, rank from the keep bits, write; the tail row n + p when it lies
//          past the count) and one thread per key-frame point (copy to its shifted slot).
// A sweep row is read twice when min_distance > 0 (the second read mostly from L2) and once otherwise.
#include <math.h>

#include "pnx_common.cuh"

namespace {

constexpr int kThreads = 512;  // mark / write block size: both kernels must partition the sweep points alike
constexpr int kWarps = kThreads / 32;

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
__host__ __device__ inline float to_f(double a) {
#ifdef __CUDA_ARCH__
  return __double2float_rn(a);
#else
  return (float)a;
#endif
}

// xyz of one sweep row taken through the row-major 4x4 matrix m (copied when m[15] is NaN: no transform)
__host__ __device__ inline void transform_xyz(const double* m, const float* p, float* o) {
  if (m[15] != m[15]) {
    o[0] = p[0], o[1] = p[1], o[2] = p[2];
    return;
  }
  const double x = p[0], y = p[1], z = p[2];
  for (int r = 0; r < 3; ++r)
    o[r] = to_f(add_d(add_d(add_d(mul_d(m[4 * r], x), mul_d(m[4 * r + 1], y)), mul_d(m[4 * r + 2], z)), m[4 * r + 3]));
}

__host__ __device__ inline bool keep_point(const float* o, float md) {
  return !(md > 0.0f && fabsf(o[0]) < md && fabsf(o[1]) < md);
}

// last i in [0, m) with off[i] <= v (off non-decreasing, off[0] <= v < off[m])
__host__ __device__ inline int segment_of(const int* off, int m, long long v) {
  int lo = 0, hi = m;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= v) lo = mid; else hi = mid;
  }
  return lo;
}

struct Args {
  const float* points;
  int n;
  const int* point_off;
  int B;
  const float* sweeps;
  int S;
  const int* sweep_off;
  int K;
  const double* transforms;
  float md;
  float* out;
  int* count;
};

// workspace: offsets (in 4-byte words) of its parts
struct Work {
  long long blockcnt, blockoff, bits, frame_base, total;
};

__host__ __device__ inline Work work_layout(int S, int B) {
  Work w;
  const long long nblk = (S + kThreads - 1) / kThreads;
  w.blockcnt = 0;
  w.blockoff = nblk;
  w.bits = 2 * nblk;
  w.frame_base = w.bits + nblk * kWarps;
  w.total = w.frame_base + B + 1;
  return w;
}

// ---------------------------------------------------------------- mark: keep bits + per-block kept counts
__global__ void __launch_bounds__(kThreads) sweeps_mark_kernel(Args a, int* __restrict__ ws) {
  __shared__ int warp_cnt[kWarps];
  const Work wl = work_layout(a.S, a.B);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const long long p = (long long)blockIdx.x * kThreads + t;
  bool keep = false;
  if (p < a.S) {
    const int seg = segment_of(a.sweep_off, a.B * a.K, p);
    float o[3];
    transform_xyz(a.transforms + (size_t)seg * 16, a.sweeps + p * 5, o);
    keep = keep_point(o, a.md);
  }
  const unsigned bits = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) {
    ws[wl.bits + (long long)blockIdx.x * kWarps + warp] = (int)bits;
    warp_cnt[warp] = __popc(bits);
  }
  __syncthreads();
  if (t == 0) {
    int c = 0;
    for (int w = 0; w < kWarps; ++w) c += warp_cnt[w];
    ws[wl.blockcnt + blockIdx.x] = c;
  }
}

// kept sweep points before sweep point q (q <= S), after the scan
__device__ inline int kept_before(const Args& a, const int* ws, const Work& wl, long long q, int total) {
  if (!(a.md > 0.0f)) return (int)q;
  if (q >= a.S) return total;
  const long long blk = q / kThreads, w = q >> 5;
  int r = ws[wl.blockoff + blk];
  for (long long k = blk * kWarps; k < w; ++k) r += __popc((unsigned)ws[wl.bits + k]);
  return r + __popc((unsigned)ws[wl.bits + w] & ((1u << (q & 31)) - 1u));
}

// ---------------------------------------------------------------- scan: block offsets, frame bases, count
__global__ void __launch_bounds__(1024) sweeps_scan_kernel(Args a, int* __restrict__ ws) {
  __shared__ int warp_sum[32];
  __shared__ int s_total;
  const Work wl = work_layout(a.S, a.B);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int nblk = (a.S + kThreads - 1) / kThreads;
  int running = 0;
  if (a.md > 0.0f) {
    for (int c0 = 0; c0 < nblk; c0 += 1024) {
      const int b = c0 + t;
      const int v = b < nblk ? ws[wl.blockcnt + b] : 0;
      int x = v;
      for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
      }
      if (lane == 31) warp_sum[warp] = x;
      __syncthreads();
      if (warp == 0) {
        int s = warp_sum[lane];
        for (int d = 1; d < 32; d <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, s, d);
          if (lane >= d) s += y;
        }
        warp_sum[lane] = s;
      }
      __syncthreads();
      if (b < nblk) ws[wl.blockoff + b] = running + x - v + (warp > 0 ? warp_sum[warp - 1] : 0);
      running += warp_sum[31];
      __syncthreads();
    }
  } else {
    running = a.S;
  }
  if (t == 0) {
    s_total = running;
    *a.count = a.n + running;
  }
  __syncthreads();
  for (int f = t; f <= a.B; f += blockDim.x)
    ws[wl.frame_base + f] = kept_before(a, ws, wl, a.sweep_off[(long long)f * a.K], s_total);
}

// ---------------------------------------------------------------- write: sweep points, tail rows, key-frame points
__global__ void __launch_bounds__(kThreads) sweeps_write_kernel(Args a, const int* __restrict__ ws, int nblk_s) {
  __shared__ int warp_base[kWarps];
  const Work wl = work_layout(a.S, a.B);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if ((int)blockIdx.x < nblk_s) {
    const long long p = (long long)blockIdx.x * kThreads + t;
    const bool filter = a.md > 0.0f;
    if (filter && t == 0) {
      int r = ws[wl.blockoff + blockIdx.x];
      for (int w = 0; w < kWarps; ++w) {
        warp_base[w] = r;
        r += __popc((unsigned)ws[wl.bits + (long long)blockIdx.x * kWarps + w]);
      }
    }
    __syncthreads();
    if (p >= a.S) return;
    int rank = (int)p;
    bool keep = true;
    if (filter) {
      const unsigned bits = (unsigned)ws[wl.bits + (long long)blockIdx.x * kWarps + warp];
      keep = (bits >> lane) & 1u;
      rank = warp_base[warp] + __popc(bits & ((1u << lane) - 1u));
    }
    if (keep) {
      const int seg = segment_of(a.sweep_off, a.B * a.K, p);
      const int f = seg / a.K;
      const float* q = a.sweeps + p * 5;
      float o[3];
      transform_xyz(a.transforms + (size_t)seg * 16, q, o);
      float* d = a.out + ((long long)a.point_off[f + 1] + rank) * 6;
      d[0] = (float)f, d[1] = o[0], d[2] = o[1], d[3] = o[2], d[4] = q[3], d[5] = q[4];
    }
    const long long tail = (long long)a.n + p;
    if (tail >= *a.count) {
      float* d = a.out + tail * 6;
      d[0] = (float)a.B;
      for (int j = 1; j < 6; ++j) d[j] = 0.0f;
    }
  } else {
    const long long i = (long long)(blockIdx.x - nblk_s) * kThreads + t;
    if (i >= a.n) return;
    const int f = segment_of(a.point_off, a.B, i);
    const float* s = a.points + i * 6;      // scalar copies: the caller's points need only 4-byte alignment
    float* d = a.out + (i + ws[wl.frame_base + f]) * 6;
    for (int j = 0; j < 6; ++j) d[j] = s[j];
  }
}

int check_args(const Args& a) {
  PNX_CHECK_ARG(a.n >= 0 && a.B >= 0 && a.S >= 0 && a.K >= 0, "n / B / S / K");
  PNX_CHECK_ARG((long long)a.n + a.S < 2147483647LL, "n + S must fit in int32");
  PNX_CHECK_ARG(a.B > 0 || (a.n == 0 && a.S == 0), "points without frames");
  PNX_CHECK_ARG(a.K > 0 || a.S == 0, "sweep points without sweep slots (K = 0)");
  PNX_CHECK_ARG(a.md >= 0.0f && a.md < INFINITY, "min_distance must be finite and >= 0");
  PNX_CHECK_ARG(a.count && a.sweep_off && (a.B == 0 || a.point_off), "count / sweep_off / point_off");
  PNX_CHECK_ARG(a.n == 0 || (a.points && a.out && a.points != a.out), "points / points_out");
  PNX_CHECK_ARG(a.S == 0 || (a.sweeps && a.transforms && a.out), "sweep_points / transforms / points_out");
  return PNX_OK;
}

}  // namespace

// Contract: include/pnx.h.
extern "C" long long pnx_accumulate_sweeps_workspace(int S, int B) {
  return work_layout(S, B).total * 4;
}

extern "C" int pnx_accumulate_sweeps(const float* points, int n, const int* point_off, int B, const float* sweep_points,
                                     int S, const int* sweep_off, int K, const double* transforms, float min_distance,
                                     float* points_out, int* count, void* workspace, cudaStream_t stream) {
  const Args a{points, n, point_off, B, sweep_points, S, sweep_off, K, transforms, min_distance, points_out, count};
  const int rc = check_args(a);
  if (rc) return rc;
  PNX_CHECK_ARG(workspace, "workspace");
  int* ws = static_cast<int*>(workspace);
  const int nblk_s = pnx_cdiv(S, kThreads), nblk_k = pnx_cdiv(n, kThreads);
  if (nblk_s > 0 && min_distance > 0.0f) {
    sweeps_mark_kernel<<<nblk_s, kThreads, 0, stream>>>(a, ws);
    PNX_CHECK_LAUNCH();
  }
  sweeps_scan_kernel<<<1, 1024, 0, stream>>>(a, ws);
  PNX_CHECK_LAUNCH();
  if (nblk_s + nblk_k > 0) {
    sweeps_write_kernel<<<nblk_s + nblk_k, kThreads, 0, stream>>>(a, ws, nblk_s);
    PNX_CHECK_LAUNCH();
  }
  return PNX_OK;
}

// Host twin: the same arithmetic on HOST memory, frame by frame (the CPU tests pin it to the goldens and the oracle).
extern "C" int pnx_accumulate_sweeps_host(const float* points, int n, const int* point_off, int B, const float* sweep_points,
                                          int S, const int* sweep_off, int K, const double* transforms, float min_distance,
                                          float* points_out, int* count) {
  const Args a{points, n, point_off, B, sweep_points, S, sweep_off, K, transforms, min_distance, points_out, count};
  const int rc = check_args(a);
  if (rc) return rc;
  PNX_CHECK_ARG(B == 0 || (point_off[0] == 0 && point_off[B] == n), "point_off must run from 0 to n");
  PNX_CHECK_ARG(sweep_off[0] == 0 && sweep_off[(long long)B * K] == S, "sweep_off must run from 0 to S");
  long long w = 0;
  for (int f = 0; f < B; ++f) {
    for (long long i = point_off[f]; i < point_off[f + 1]; ++i, ++w)
      for (int j = 0; j < 6; ++j) points_out[w * 6 + j] = points[i * 6 + j];
    for (int k = 0; k < K; ++k) {
      const long long seg = (long long)f * K + k;
      for (long long p = sweep_off[seg]; p < sweep_off[seg + 1]; ++p) {
        const float* q = sweep_points + p * 5;
        float o[3];
        transform_xyz(transforms + seg * 16, q, o);
        if (!keep_point(o, min_distance)) continue;
        float* d = points_out + w * 6;
        d[0] = (float)f, d[1] = o[0], d[2] = o[1], d[3] = o[2], d[4] = q[3], d[5] = q[4];
        ++w;
      }
    }
  }
  *count = (int)w;
  for (long long i = w; i < (long long)n + S; ++i) {
    points_out[i * 6] = (float)B;
    for (int j = 1; j < 6; ++j) points_out[i * 6 + j] = 0.0f;
  }
  return PNX_OK;
}
