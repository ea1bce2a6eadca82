// gt_sample.cu -- ground-truth database sampling: collision test, scene-point removal and paste, sm_90a.
//
// The data-loader workers draw the candidates exactly as the reference does (DataBaseSamplerV2 in
// det3d/datasets/pipelines/sample_ops.py of this repo) and ship every drawn object: its box, class, stored points and
// two (cos, sin) pairs of its yaw -- numpy's vectorised fp32 pair, which the reference's corner path uses, and libm's
// cosf / sinf, which its numba point test uses.  Neither is recomputed here.  Per batch, four launches, no host sync:
//   select  one CTA per frame: BEV corners + standup boxes of the scene boxes and candidates in shared memory, the
//           collision test parallel over box pairs, the greedy pass sequential within each class call (a run of equal
//           class ids); writes the output boxes and the frame's accepted-box list.
//   mark    one thread per scene point: inside any accepted box of its frame?  Per-block, per-frame kept counts.
//   scan    one CTA: per-frame exclusive scan of the block counts, then the frame bases and the valid row count.
//   write   one thread per output row: kept scene points and accepted objects' points to their slots (order kept),
//           unused tail rows get frame index B.
//
// The arithmetic is the reference's, to the bit (pinned by tests/golden/ref_gts.npz):
//   corners   box_np_ops.center_to_corner_box2d in fp32: (dx, dy) * (+-0.5), then
//             x' = fl(fl(px * c) + fl(py * -s)) + cx, y' = fl(fl(px * s) + fl(py * c)) + cy, no FMA.
//   collision box_collision_test(total, total)[i, j] with the candidate i as the first argument (the matrix is not
//             symmetric in fp32): standup overlap (iw > 0, ih > 0), then any strict segment crossing, then either box's
//             four corners strictly inside the other.
//   greedy    sample_class_v2: candidate i is rejected if it collides with a scene box, a candidate accepted by an
//             earlier class call, an accepted earlier candidate of its call, or ANY later candidate of its call
//             (accepted or not: row i still holds them).  A rejected candidate's column is cleared.
//   points    points_in_boxes_jit: |z - bz| <= dz / 2 first, then |lx| <= dx / 2 and |ly| <= dy / 2 with
//             lx = fl(fl(sx * c) + fl(sy * s)), ly = fl(fl(-sx * s) + fl(sy * c)); the halves compared in fp64, as numba
//             promotes `x / 2.0`.  Pasted points get xyz + box[:3] in fp32.
// Every fp32 operation is rounded on its own (the _rn intrinsics on the device, plain operators in the host twin, whose
// compiler has no FMA to contract into).
#include <math.h>

#include <vector>

#include "box_geom.cuh"
#include "pnx_common.cuh"

namespace {

constexpr int kTrig = 4;        // cand_trig per candidate: numpy cos, numpy sin, cosf, sinf
constexpr int kAcc = 11;        // accepted-box record: box[9], cosf, sinf
constexpr int kGeo = 12;        // BEV geometry: x0 y0 .. x3 y3, standup min x, min y, max x, max y
constexpr int kPtThreads = 512;  // mark / write block size (both kernels must partition the points alike)
constexpr int kPtWarps = kPtThreads / 32;
constexpr int kSelThreads = 256;

// center_to_corner_box2d of box (x, y, dx, dy from a 9-column box) with numpy's (c, s), + corner_to_standup_nd
__host__ __device__ inline void bev_geometry(const float* box, float c, float s, float* g) {
  const float nx[4] = {-0.5f, -0.5f, 0.5f, 0.5f}, ny[4] = {-0.5f, 0.5f, 0.5f, -0.5f};
  for (int k = 0; k < 4; ++k) {
    const float px = mul_f(box[3], nx[k]), py = mul_f(box[4], ny[k]);
    g[2 * k] = add_f(add_f(mul_f(px, c), mul_f(py, -s)), box[0]);
    g[2 * k + 1] = add_f(add_f(mul_f(px, s), mul_f(py, c)), box[1]);
  }
  g[8] = min_f(min_f(min_f(g[0], g[2]), g[4]), g[6]);
  g[9] = min_f(min_f(min_f(g[1], g[3]), g[5]), g[7]);
  g[10] = max_f(max_f(max_f(g[0], g[2]), g[4]), g[6]);
  g[11] = max_f(max_f(max_f(g[1], g[3]), g[5]), g[7]);
}

// every corner of q strictly inside b (box_collision_test's containment loops, clockwise = True)
__host__ __device__ inline bool corners_inside(const float* b, const float* q) {
  for (int l = 0; l < 4; ++l)
    for (int k = 0; k < 4; ++k) {
      const int k1 = (k + 1) & 3;
      const float v0 = -sub_f(b[2 * k], b[2 * k1]), v1 = -sub_f(b[2 * k + 1], b[2 * k1 + 1]);
      float cross = mul_f(v1, sub_f(b[2 * k], q[2 * l]));
      cross = sub_f(cross, mul_f(v0, sub_f(b[2 * k + 1], q[2 * l + 1])));
      if (cross >= 0.0f) return false;
    }
  return true;
}

// box_collision_test(boxes, qboxes)[i, j] for one pair: b = boxes[i], q = qboxes[j]
__host__ __device__ inline bool collide(const float* b, const float* q) {
  const float iw = sub_f(min_f(b[10], q[10]), max_f(b[8], q[8]));
  if (!(iw > 0.0f)) return false;
  const float ih = sub_f(min_f(b[11], q[11]), max_f(b[9], q[9]));
  if (!(ih > 0.0f)) return false;
  for (int k = 0; k < 4; ++k) {
    const float A0 = b[2 * k], A1 = b[2 * k + 1], B0 = b[2 * ((k + 1) & 3)], B1 = b[2 * ((k + 1) & 3) + 1];
    for (int l = 0; l < 4; ++l) {
      const float C0 = q[2 * l], C1 = q[2 * l + 1], D0 = q[2 * ((l + 1) & 3)], D1 = q[2 * ((l + 1) & 3) + 1];
      const bool acd = mul_f(sub_f(D1, A1), sub_f(C0, A0)) > mul_f(sub_f(C1, A1), sub_f(D0, A0));
      const bool bcd = mul_f(sub_f(D1, B1), sub_f(C0, B0)) > mul_f(sub_f(C1, B1), sub_f(D0, B0));
      if (acd != bcd) {
        const bool abc = mul_f(sub_f(C1, A1), sub_f(B0, A0)) > mul_f(sub_f(B1, A1), sub_f(C0, A0));
        const bool abd = mul_f(sub_f(D1, A1), sub_f(B0, A0)) > mul_f(sub_f(B1, A1), sub_f(D0, A0));
        if (abc != abd) return true;
      }
    }
  }
  return corners_inside(b, q) || corners_inside(q, b);
}

struct Args {
  const float* points;
  int n;
  const float* boxes;
  const int* classes;
  const float* box_trig;
  int B, M;
  const float* cand_boxes;
  const int* cand_classes;
  const float* cand_trig;
  int S;
  const float* cand_points;
  const int* cand_off;
  int P;
  float* points_out;
  float* boxes_out;
  int* classes_out;
  int* accepted;
  int* count;
};

// workspace: offsets (in 4-byte words) of its parts
struct Work {
  long long acc_box, acc_off, n_acc, acc_pts, frame_base, blockcnt, blockoff, keep, total;
};

__host__ __device__ inline Work work_layout(int n, int B, int S) {
  Work w;
  const long long nblk = (n + kPtThreads - 1) / kPtThreads;
  w.acc_box = 0;
  w.acc_off = w.acc_box + (long long)B * S * kAcc;
  w.n_acc = w.acc_off + (long long)B * S;
  w.acc_pts = w.n_acc + B;
  w.frame_base = w.acc_pts + B;
  w.blockcnt = w.frame_base + B;
  w.blockoff = w.blockcnt + nblk * B;
  w.keep = w.blockoff + nblk * B;
  w.total = w.keep + (n + 3) / 4;  // one byte per point
  return w;
}

inline size_t select_smem(int M, int S) {
  const int W = (S + 31) / 32;
  return (size_t)(M + S) * kGeo * 4 + (size_t)(M + S) * 4 + (size_t)S * 4 * 2 + (size_t)S * W * 4 + (size_t)W * 4;
}

// ---------------------------------------------------------------- select: one CTA per frame
__global__ void __launch_bounds__(kSelThreads) gts_select_kernel(Args a, int* __restrict__ ws) {
  extern __shared__ float smem[];
  const int f = blockIdx.x, M = a.M, S = a.S, W = (S + 31) / 32, t = threadIdx.x;
  float* geo = smem;                                          // [M + S][kGeo]: scene rows by scene slot, candidates at M + s
  int* avoid = reinterpret_cast<int*>(geo + (size_t)(M + S) * kGeo);  // geometry rows the candidates must avoid
  int* ext = avoid + M + S;                                   // [S] collides with an avoid box
  int* acc = ext + S;                                         // [S] accepted
  uint32_t* rows = reinterpret_cast<uint32_t*>(acc + S);      // [S][W] collisions within the call
  uint32_t* valid = rows + (size_t)S * W;                     // [W] columns not cleared
  __shared__ int n_avoid;
  const Work wl = work_layout(a.n, a.B, S);
  float* acc_box = reinterpret_cast<float*>(ws + wl.acc_box) + (size_t)f * S * kAcc;
  int* acc_off = ws + wl.acc_off + (size_t)f * S;

  for (int i = t; i < M + S; i += blockDim.x) {
    const bool scene = i < M;
    const long long r = scene ? (long long)f * M + i : (long long)f * S + (i - M);
    const float* box = (scene ? a.boxes : a.cand_boxes) + r * 9;
    const float c = scene ? a.box_trig[r * 2] : a.cand_trig[r * kTrig];
    const float s = scene ? a.box_trig[r * 2 + 1] : a.cand_trig[r * kTrig + 1];
    const int cls = scene ? a.classes[r] : a.cand_classes[r];
    if (cls >= 0) bev_geometry(box, c, s, geo + (size_t)i * kGeo);
    if (!scene) acc[i - M] = 0;
  }
  if (t == 0) {
    int k = 0;
    for (int i = 0; i < M; ++i)
      if (a.classes[(long long)f * M + i] >= 0) avoid[k++] = i;
    n_avoid = k;
  }
  __syncthreads();

  const int* ccls = a.cand_classes + (long long)f * S;
  for (int c0 = 0; c0 < S;) {
    if (ccls[c0] < 0) {
      ++c0;
      continue;
    }
    int c1 = c0 + 1;
    while (c1 < S && ccls[c1] == ccls[c0]) ++c1;
    const int L = c1 - c0, na = n_avoid;
    for (int i = t; i < L; i += blockDim.x) ext[i] = 0;
    for (int i = t; i < L * W; i += blockDim.x) rows[i] = 0;
    __syncthreads();
    for (int p = t; p < L * (na + L); p += blockDim.x) {
      const int i = p / (na + L), j = p % (na + L);
      if (j < na) {
        if (collide(geo + (size_t)(M + c0 + i) * kGeo, geo + (size_t)avoid[j] * kGeo)) ext[i] = 1;
      } else if (j - na != i) {
        if (collide(geo + (size_t)(M + c0 + i) * kGeo, geo + (size_t)(M + c0 + j - na) * kGeo))
          atomicOr(&rows[i * W + (j - na) / 32], 1u << ((j - na) & 31));
      }
    }
    __syncthreads();
    if (t == 0) {
      for (int w = 0; w < W; ++w) valid[w] = w * 32 + 32 <= L ? 0xffffffffu : (w * 32 < L ? (1u << (L - w * 32)) - 1 : 0u);
      for (int i = 0; i < L; ++i) {
        bool hit = ext[i] != 0;
        for (int w = 0; w < W && !hit; ++w) hit = (rows[i * W + w] & valid[w]) != 0;
        if (hit) {
          valid[i / 32] &= ~(1u << (i & 31));
        } else {
          acc[c0 + i] = 1;
          avoid[n_avoid++] = M + c0 + i;
        }
      }
    }
    __syncthreads();
    c0 = c1;
  }

  // accepted-box list, point offsets within the frame, output boxes
  __shared__ int s_nacc, s_nreal;
  if (t == 0) {
    int k = 0, pts = 0, nreal = 0;
    for (int i = 0; i < M; ++i) nreal += a.classes[(long long)f * M + i] >= 0;
    for (int s = 0; s < S; ++s) {
      const long long r = (long long)f * S + s;
      if (acc[s]) {
        acc_off[s] = pts;
        pts += a.cand_off[r + 1] - a.cand_off[r];
        float* o = acc_box + (size_t)k * kAcc;
        for (int j = 0; j < 9; ++j) o[j] = a.cand_boxes[r * 9 + j];
        o[9] = a.cand_trig[r * kTrig + 2];
        o[10] = a.cand_trig[r * kTrig + 3];
        ++k;
      } else {
        acc_off[s] = -1;
      }
      if (a.accepted) a.accepted[r] = acc[s];
    }
    ws[wl.n_acc + f] = k;
    ws[wl.acc_pts + f] = pts;
    s_nacc = k;
    s_nreal = nreal;
  }
  __syncthreads();
  const int MS = M + S, nreal = s_nreal, nacc = s_nacc;
  for (int r = t; r < MS; r += blockDim.x) {
    float* o = a.boxes_out + ((long long)f * MS + r) * 9;
    int cls = -1;
    if (r < nreal) {
      int i = avoid[r];                       // avoid[0, nreal) = the real scene boxes in order
      for (int j = 0; j < 9; ++j) o[j] = a.boxes[((long long)f * M + i) * 9 + j];
      cls = a.classes[(long long)f * M + i];
    } else if (r < nreal + nacc) {
      int s = avoid[r] - M;                   // then the accepted candidates in acceptance order
      for (int j = 0; j < 9; ++j) o[j] = a.cand_boxes[((long long)f * S + s) * 9 + j];
      cls = ccls[s];
    } else {
      for (int j = 0; j < 9; ++j) o[j] = (j >= 3 && j < 6) ? 1.0f : 0.0f;
    }
    a.classes_out[(long long)f * MS + r] = cls;
  }
}

// ---------------------------------------------------------------- mark: keep flags + per-block, per-frame counts
__global__ void __launch_bounds__(kPtThreads) gts_mark_kernel(Args a, int* __restrict__ ws) {
  extern __shared__ int cnt[];  // [B]
  const Work wl = work_layout(a.n, a.B, a.S);
  const int t = threadIdx.x, B = a.B;
  for (int f = t; f < B; f += blockDim.x) cnt[f] = 0;
  __syncthreads();
  const long long i = (long long)blockIdx.x * kPtThreads + t;
  int key = -1;
  if (i < a.n) {
    const float* p = a.points + i * 6;
    const int f = frame_of(p[0], B);
    bool keep = f >= 0;
    if (keep) {
      const float* acc = reinterpret_cast<const float*>(ws + wl.acc_box) + (size_t)f * a.S * kAcc;
      const int na = ws[wl.n_acc + f];
      const float x = p[1], y = p[2], z = p[3];
      for (int k = 0; k < na && keep; ++k) {
        const float* b = acc + (size_t)k * kAcc;
        keep = !point_in_box(x, y, z, b, b[9], b[10]);
      }
    }
    reinterpret_cast<uint8_t*>(ws + wl.keep)[i] = keep;
    key = keep ? f : -1;
  }
  const unsigned peers = __match_any_sync(0xffffffffu, key);
  if (key >= 0 && (t & 31) == 31 - __clz(peers)) atomicAdd(&cnt[key], __popc(peers));
  __syncthreads();
  for (int f = t; f < B; f += blockDim.x) ws[wl.blockcnt + (long long)blockIdx.x * B + f] = cnt[f];
}

// ---------------------------------------------------------------- scan: block offsets per frame, frame bases, count
__global__ void __launch_bounds__(1024) gts_scan_kernel(Args a, int* __restrict__ ws) {
  __shared__ int warp_sum[32];
  const Work wl = work_layout(a.n, a.B, a.S);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, B = a.B;
  const int nblk = (a.n + kPtThreads - 1) / kPtThreads;
  for (int f = 0; f < B; ++f) {
    int running = 0;
    for (int c0 = 0; c0 < nblk; c0 += 1024) {
      const int b = c0 + t;
      const int v = b < nblk ? ws[wl.blockcnt + (long long)b * B + f] : 0;
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
      const int excl = x - v + (warp > 0 ? warp_sum[warp - 1] : 0);
      if (b < nblk) ws[wl.blockoff + (long long)b * B + f] = running + excl;
      running += warp_sum[31];
      __syncthreads();
    }
    if (t == 0) ws[wl.frame_base + f] = running;           // kept count; turned into the base below
  }
  __syncthreads();
  if (t == 0) {
    int base = 0;
    for (int f = 0; f < B; ++f) {
      const int k = ws[wl.frame_base + f];
      ws[wl.frame_base + f] = base;
      base += ws[wl.acc_pts + f] + k;
    }
    *a.count = base;
  }
}

// ---------------------------------------------------------------- write: one thread per output row
__global__ void __launch_bounds__(kPtThreads) gts_write_kernel(Args a, const int* __restrict__ ws) {
  extern __shared__ int wcnt[];  // [kPtWarps][B]
  const Work wl = work_layout(a.n, a.B, a.S);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, B = a.B, S = a.S;
  for (int k = t; k < kPtWarps * B; k += blockDim.x) wcnt[k] = 0;
  __syncthreads();
  const long long i = (long long)blockIdx.x * kPtThreads + t;
  int key = -1;
  if (i < a.n && reinterpret_cast<const uint8_t*>(ws + wl.keep)[i]) key = (int)a.points[i * 6];
  const unsigned peers = __match_any_sync(0xffffffffu, key);
  if (key >= 0 && lane == 31 - __clz(peers)) wcnt[warp * B + key] = __popc(peers);
  __syncthreads();
  const long long total = (long long)a.n + a.P;
  if (key >= 0) {
    int rank = __popc(peers & ((1u << lane) - 1));
    for (int w = 0; w < warp; ++w) rank += wcnt[w * B + key];
    const long long dst = (long long)ws[wl.frame_base + key] + ws[wl.acc_pts + key] +
                          ws[wl.blockoff + (long long)blockIdx.x * B + key] + rank;
    const float* p = a.points + i * 6;
    float* o = a.points_out + dst * 6;
    for (int j = 0; j < 6; ++j) o[j] = p[j];
  } else if (i >= a.n && i < total) {
    const int p = (int)(i - a.n);
    int lo = 0, hi = B * S;  // candidate c with cand_off[c] <= p < cand_off[c + 1]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (a.cand_off[mid] <= p) lo = mid; else hi = mid;
    }
    const int off = ws[wl.acc_off + lo];
    if (off >= 0) {
      const int f = lo / S;
      const long long dst = (long long)ws[wl.frame_base + f] + off + (p - a.cand_off[lo]);
      const float* q = a.cand_points + (long long)p * 5;
      const float* box = a.cand_boxes + (long long)lo * 9;
      float* o = a.points_out + dst * 6;
      o[0] = (float)f;
      for (int j = 0; j < 3; ++j) o[1 + j] = add_f(q[j], box[j]);
      o[4] = q[3];
      o[5] = q[4];
    }
  }
  if (i < total && i >= *a.count) {
    float* o = a.points_out + i * 6;
    o[0] = (float)B;
    for (int j = 1; j < 6; ++j) o[j] = 0.0f;
  }
}

int check_args(const Args& a) {
  PNX_CHECK_ARG(a.n >= 0 && a.B >= 0 && a.M >= 0 && a.S >= 0 && a.P >= 0, "n / B / M / S / P");
  PNX_CHECK_ARG((long long)a.n + a.P < 2147483647LL, "n + P must fit in int32");
  PNX_CHECK_ARG(a.B <= 512, "at most 512 frames");
  PNX_CHECK_ARG(a.n == 0 || (a.points && a.points_out && a.points != a.points_out), "points / points_out");
  PNX_CHECK_ARG(a.P == 0 || (a.cand_points && a.points_out), "cand_points");
  PNX_CHECK_ARG((long long)a.B * a.M == 0 || (a.boxes && a.classes && a.box_trig), "boxes / classes / box_trig");
  PNX_CHECK_ARG((long long)a.B * a.S == 0 || (a.cand_boxes && a.cand_classes && a.cand_trig), "cand_boxes / classes / trig");
  PNX_CHECK_ARG(a.B == 0 || (a.cand_off && a.boxes_out && a.classes_out && a.count), "cand_off / boxes_out / classes_out / count");
  PNX_CHECK_ARG(a.B == 0 || a.M + a.S > 0, "M + S must be > 0");
  return PNX_OK;
}

}  // namespace

// Contract: include/pnx.h.
extern "C" long long pnx_gt_sample_workspace(int n, int B, int S) {
  return work_layout(n, B, S).total * 4;
}

extern "C" int pnx_gt_sample(const float* points, int n, const float* boxes, const int* classes, const float* box_trig,
                             int B, int M, const float* cand_boxes, const int* cand_classes, const float* cand_trig, int S,
                             const float* cand_points, const int* cand_off, int P, float* points_out, float* boxes_out,
                             int* classes_out, int* accepted, int* count, void* workspace, cudaStream_t stream) {
  const Args a{points, n, boxes, classes, box_trig, B, M, cand_boxes, cand_classes, cand_trig, S, cand_points, cand_off, P,
               points_out, boxes_out, classes_out, accepted, count};
  const int rc = check_args(a);
  if (rc) return rc;
  PNX_CHECK_ARG(B == 0 || workspace, "workspace");
  if (B == 0) return PNX_OK;
  int* ws = static_cast<int*>(workspace);
  const size_t sel = select_smem(M, S);
  PNX_CHECK_ARG(sel <= 200 * 1024, "too many boxes per frame (M + S) for the select kernel's shared memory");
  if (sel > 48 * 1024) PNX_CUDA(cudaFuncSetAttribute(gts_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel));
  gts_select_kernel<<<B, kSelThreads, sel, stream>>>(a, ws);
  PNX_CHECK_LAUNCH();
  const int nblk = pnx_cdiv(n, kPtThreads);
  if (nblk > 0) {
    gts_mark_kernel<<<nblk, kPtThreads, (size_t)B * 4, stream>>>(a, ws);
    PNX_CHECK_LAUNCH();
  }
  gts_scan_kernel<<<1, 1024, 0, stream>>>(a, ws);
  PNX_CHECK_LAUNCH();
  const int wblk = pnx_cdiv((long long)n + P, kPtThreads);
  if (wblk > 0) {
    gts_write_kernel<<<wblk, kPtThreads, (size_t)kPtWarps * B * 4, stream>>>(a, ws);
    PNX_CHECK_LAUNCH();
  }
  return PNX_OK;
}

// Host twin: the same selection and point math on HOST memory, sequentially (the CPU tests pin it to the goldens).
extern "C" int pnx_gt_sample_host(const float* points, int n, const float* boxes, const int* classes, const float* box_trig,
                                  int B, int M, const float* cand_boxes, const int* cand_classes, const float* cand_trig,
                                  int S, const float* cand_points, const int* cand_off, int P, float* points_out,
                                  float* boxes_out, int* classes_out, int* accepted, int* count) {
  const Args a{points, n, boxes, classes, box_trig, B, M, cand_boxes, cand_classes, cand_trig, S, cand_points, cand_off, P,
               points_out, boxes_out, classes_out, accepted, count};
  const int rc = check_args(a);
  if (rc) return rc;
  if (B == 0) return PNX_OK;
  const int MS = M + S;
  std::vector<float> geo((size_t)MS * kGeo);
  std::vector<std::vector<int>> order(B);        // per frame: real scene slots, then accepted candidate slots (M + s)
  std::vector<std::vector<char>> acc(B, std::vector<char>(S, 0));
  for (int f = 0; f < B; ++f) {
    std::vector<int>& avoid = order[f];
    for (int i = 0; i < MS; ++i) {
      const bool scene = i < M;
      const long long r = scene ? (long long)f * M + i : (long long)f * S + (i - M);
      const int cls = scene ? classes[r] : cand_classes[r];
      if (cls < 0) continue;
      if (scene) {
        bev_geometry(boxes + r * 9, box_trig[r * 2], box_trig[r * 2 + 1], &geo[(size_t)i * kGeo]);
        avoid.push_back(i);
      } else {
        bev_geometry(cand_boxes + r * 9, cand_trig[r * kTrig], cand_trig[r * kTrig + 1], &geo[(size_t)i * kGeo]);
      }
    }
    const int* ccls = cand_classes + (long long)f * S;
    for (int c0 = 0; c0 < S;) {
      if (ccls[c0] < 0) {
        ++c0;
        continue;
      }
      int c1 = c0 + 1;
      while (c1 < S && ccls[c1] == ccls[c0]) ++c1;
      const int L = c1 - c0;
      const size_t na = avoid.size();
      std::vector<char> cleared(L, 0);
      for (int i = 0; i < L; ++i) {
        const float* gi = &geo[(size_t)(M + c0 + i) * kGeo];
        bool hit = false;
        for (size_t j = 0; j < na && !hit; ++j) hit = collide(gi, &geo[(size_t)avoid[j] * kGeo]);
        for (int j = 0; j < L && !hit; ++j)
          if (j != i && !cleared[j]) hit = collide(gi, &geo[(size_t)(M + c0 + j) * kGeo]);
        if (hit) {
          cleared[i] = 1;
        } else {
          acc[f][c0 + i] = 1;
          avoid.push_back(M + c0 + i);
        }
      }
      c0 = c1;
    }
    for (int s = 0; s < S; ++s)
      if (accepted) accepted[(long long)f * S + s] = acc[f][s];
    int nreal = 0;
    for (int i = 0; i < M; ++i) nreal += classes[(long long)f * M + i] >= 0;
    for (int r = 0; r < MS; ++r) {
      float* o = boxes_out + ((long long)f * MS + r) * 9;
      int cls = -1;
      if (r < (int)avoid.size()) {
        const int i = avoid[r];
        const long long src = i < M ? (long long)f * M + i : (long long)f * S + (i - M);
        for (int j = 0; j < 9; ++j) o[j] = (i < M ? boxes : cand_boxes)[src * 9 + j];
        cls = i < M ? classes[src] : cand_classes[src];
      } else {
        for (int j = 0; j < 9; ++j) o[j] = (j >= 3 && j < 6) ? 1.0f : 0.0f;
      }
      classes_out[(long long)f * MS + r] = cls;
    }
  }
  // points, frame by frame: accepted objects' points, then the kept scene points in their original order
  long long w = 0;
  for (int f = 0; f < B; ++f) {
    for (int s = 0; s < S; ++s) {
      if (!acc[f][s]) continue;
      const long long r = (long long)f * S + s;
      for (int p = cand_off[r]; p < cand_off[r + 1]; ++p, ++w) {
        float* o = points_out + w * 6;
        o[0] = (float)f;
        for (int j = 0; j < 3; ++j) o[1 + j] = add_f(cand_points[(long long)p * 5 + j], cand_boxes[r * 9 + j]);
        o[4] = cand_points[(long long)p * 5 + 3];
        o[5] = cand_points[(long long)p * 5 + 4];
      }
    }
    const std::vector<int>& ord = order[f];
    for (long long i = 0; i < n; ++i) {
      const float* p = points + i * 6;
      if (frame_of(p[0], B) != f) continue;
      bool keep = true;
      for (size_t k = 0; k < ord.size() && keep; ++k) {
        if (ord[k] < M) continue;
        const long long r = (long long)f * S + (ord[k] - M);
        keep = !point_in_box(p[1], p[2], p[3], cand_boxes + r * 9, cand_trig[r * kTrig + 2], cand_trig[r * kTrig + 3]);
      }
      if (!keep) continue;
      for (int j = 0; j < 6; ++j) points_out[w * 6 + j] = p[j];
      ++w;
    }
  }
  *count = (int)w;
  for (long long i = w; i < (long long)n + P; ++i) {
    points_out[i * 6] = (float)B;
    for (int j = 1; j < 6; ++j) points_out[i * 6 + j] = 0.0f;
  }
  return PNX_OK;
}

// points_in_rbbox on HOST memory: inside[i * m + j] = point i (x, y, z at columns 0-2 of a `stride`-float row) inside
// 9-column box j, with (cosf, sinf) of its yaw in trig[2 j], trig[2 j + 1].  The gt-database tool cuts objects with it.
extern "C" int pnx_points_in_boxes_host(const float* points, int n, int stride, const float* boxes, const float* trig,
                                        int m, unsigned char* inside) {
  PNX_CHECK_ARG(n >= 0 && m >= 0 && stride >= 3, "n / m / stride");
  PNX_CHECK_ARG((long long)n * m == 0 || (points && boxes && trig && inside), "pointers");
  for (long long i = 0; i < n; ++i) {
    const float* p = points + i * stride;
    for (int j = 0; j < m; ++j)
      inside[i * m + j] = point_in_box(p[0], p[1], p[2], boxes + (long long)j * 9, trig[2 * j], trig[2 * j + 1]);
  }
  return PNX_OK;
}
