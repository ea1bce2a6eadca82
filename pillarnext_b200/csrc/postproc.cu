// postproc.cu -- detection decode + rotated NMS of the CenterPoint head (row F1 of SURVEY.md section 8f), sm_90a.
//
// Replaces CenterHead.predict / post_processing (reference det3d/models/heads/centerhead.py:231-384),
// rotate_nms_pcdet (det3d/core/bbox/box_torch_ops.py:5-31) and the native NMS it calls
// (det3d/core/iou3d_nms/src/iou3d_nms_kernel.cu:280-324 mask kernel, iou3d_nms.cpp:113-159 host sweep), for one task:
//   1. pnx_det_keys   : one pass over the head's channels-last output matrix [B*H*W, ld] (fp32): sigmoid/max over the
//                       heat-map channels, score + range filter, IoU rectification, and a 64-bit sort key per pixel
//                       (segment = frame*C + class in the high word, descending score in the low word); per-segment counts.
//   (the keys are sorted by the caller -- one device radix sort per task)
//   2. pnx_det_nms    : per segment, the top pre_max candidates: suppression bit-mask (rotated BEV IoU > thresh, boxes
//                       decoded on the fly from the head output) and the greedy sweep ON the GPU (one warp per segment;
//                       the reference copies the mask to the host and sweeps there).
//   3. pnx_det_gather : decode the kept candidates into [segments, post_max, 9] boxes / scores / labels.
// No host synchronisation inside; the caller reads the per-segment counts once.
// Provenance note: the rotated-rectangle overlap routines below (cross3, rect_cross, in_box2d, seg_intersection,
// det_box_overlap, det_iou_bev) deliberately follow the ARITHMETIC of the reference's own device code,
// det3d/core/iou3d_nms/src/iou3d_nms_kernel.cu:39-235 (and its host twin iou3d_cpu.cpp), statement by statement -- same
// operation order, same 1e-2 margin, same angular ordering of the polygon vertices: the keep / suppress decision of every
// box pair must come out bit-identical to the reference's NMS, and any algebraically equivalent rewrite flips decisions for
// IoUs near the threshold.  Everything around them (fused decode, 64-bit sort keys, batched per-(frame, class) mask, the
// on-GPU sweep with up to 4 slots of 2048 candidates, `__host__ __device__` for the CPU parity leg) is this repository's.
// Hot loop character: HBM-bound single pass (1) and a few hundred thousand polygon clips (2) -- no tensor-core work.
#include <math.h>

#include "pnx_common.cuh"

namespace {

struct DetParams {
  const float* out;      // [B*H*W, ld] fp32, channels-last head output of one task
  long long ld;
  int B, H, W, C;
  int o_reg, o_height, o_dim, o_rot, o_vel, o_hm, o_iou;  // column offsets (o_iou < 0: no iou head -> iou = 1)
  float osf, vs_x, vs_y, pc_x, pc_y;                       // xs = (x + reg0) * osf * vs_x + pc_x  (centerhead.py:293-296)
  float score_thr;
  float range[6];        // post_center_limit_range
  float rect[8];         // rectifier per class (centerhead.py:352-354)
  float nms_thr[8];      // nms_iou_threshold per class
};

constexpr int kMaxClasses = 8;

// ------------------------------------------------------------------ decode of one pixel (centerhead.py:247-304,336-354)
// Returns false when the pixel is filtered out.  box = (x, y, z, dx, dy, dz, vx, vy, yaw).
__host__ __device__ inline bool det_decode_pixel(const DetParams& p, long long m, float* box, float* score, int* label) {
  const float* row = p.out + m * p.ld;
  const int hw = p.H * p.W;
  const int rem = (int)(m % hw);
  const int y = rem / p.W, x = rem - y * p.W;
  // heat map: sigmoid is monotonic, so the arg-max over logits is the arg-max over scores (first maximum, as torch.max)
  int best = 0;
  float bl = row[p.o_hm];
  for (int c = 1; c < p.C; ++c) {
    const float v = row[p.o_hm + c];
    if (v > bl) { bl = v; best = c; }
  }
  float s = 1.0f / (1.0f + expf(-bl));
  if (!(s > p.score_thr)) return false;
  // xs = xs * out_size_factor * voxel_size + pc_range: three separately rounded fp32 operations, like the reference
  float xs = (float)x + row[p.o_reg], ys = (float)y + row[p.o_reg + 1];
#ifdef __CUDA_ARCH__
  xs = __fadd_rn(__fmul_rn(__fmul_rn(xs, p.osf), p.vs_x), p.pc_x);
  ys = __fadd_rn(__fmul_rn(__fmul_rn(ys, p.osf), p.vs_y), p.pc_y);
#else
  { volatile float t = xs * p.osf; t = t * p.vs_x; xs = t + p.pc_x; }
  { volatile float t = ys * p.osf; t = t * p.vs_y; ys = t + p.pc_y; }
#endif
  const float z = row[p.o_height];
  if (!(xs >= p.range[0] && ys >= p.range[1] && z >= p.range[2] && xs <= p.range[3] && ys <= p.range[4] && z <= p.range[5]))
    return false;
  float iou = 1.0f;
  if (p.o_iou >= 0) iou = fminf(fmaxf((row[p.o_iou] + 1.0f) * 0.5f, 0.0f), 1.0f);
  const float r = p.rect[best];
  if (r != 0.0f) s = powf(s, 1.0f - r) * powf(iou, r);     // r == 0: pow(s, 1) * pow(iou, 0) == s exactly
  box[0] = xs; box[1] = ys; box[2] = z;
  box[3] = expf(row[p.o_dim]); box[4] = expf(row[p.o_dim + 1]); box[5] = expf(row[p.o_dim + 2]);
  box[6] = row[p.o_vel]; box[7] = row[p.o_vel + 1];
  box[8] = atan2f(row[p.o_rot], row[p.o_rot + 1]);
  *score = s;
  *label = best;
  return true;
}

// ------------------------------------------------------------------ rotated BEV IoU (iou3d_cpu.cpp:62-237 algorithm:
// edge crossings + contained corners, sorted by angle about their centroid, shoelace area)
struct P2 { float x, y; };

__host__ __device__ inline float cross3(const P2& p1, const P2& p2, const P2& p0) {
  return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}

__host__ __device__ inline bool rect_cross(const P2& p1, const P2& p2, const P2& q1, const P2& q2) {
  return fminf(p1.x, p2.x) <= fmaxf(q1.x, q2.x) && fminf(q1.x, q2.x) <= fmaxf(p1.x, p2.x) &&
         fminf(p1.y, p2.y) <= fmaxf(q1.y, q2.y) && fminf(q1.y, q2.y) <= fmaxf(p1.y, p2.y);
}

// box7 = (x, y, z, dx, dy, dz, heading)
__host__ __device__ inline bool in_box2d(const float* box, const P2& p) {
  const float kMargin = 1e-2f;
  const float c = cosf(-box[6]), s = sinf(-box[6]);
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

__host__ __device__ inline void box_corners(const float* box, P2* c5) {
  const float hx = box[3] / 2, hy = box[4] / 2;
  const float ca = cosf(box[6]), sa = sinf(box[6]);
  const float px[4] = {-hx, hx, hx, -hx}, py[4] = {-hy, -hy, hy, hy};
  for (int k = 0; k < 4; ++k) {
    c5[k].x = px[k] * ca + py[k] * (-sa) + box[0];
    c5[k].y = px[k] * sa + py[k] * ca + box[1];
  }
  c5[4] = c5[0];
}

__host__ __device__ inline float det_box_overlap(const float* a, const float* b) {
  P2 ca[5], cb[5], pts[16];
  box_corners(a, ca);
  box_corners(b, cb);
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
    if (cnt < 16 && in_box2d(a, cb[k])) { sx += cb[k].x; sy += cb[k].y; pts[cnt++] = cb[k]; }
    if (cnt < 16 && in_box2d(b, ca[k])) { sx += ca[k].x; sy += ca[k].y; pts[cnt++] = ca[k]; }
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

__host__ __device__ inline float det_iou_bev(const float* a, const float* b) {
  const float sa = a[3] * a[4], sb = b[3] * b[4];
  const float so = det_box_overlap(a, b);
  return so / fmaxf(sa + sb - so, 1e-8f);
}

// aligned 3-D IoU of two (x, y, z, dx, dy, dz, heading) boxes: BEV overlap x height overlap over the union volume
// (reference det3d/core/iou3d_nms/iou3d_nms_utils.py:45-87 boxes_aligned_iou3d_gpu; training target of the `iou` head)
__host__ __device__ inline float det_aligned_iou3d(const float* a, const float* b) {
  const float a_max = a[2] + a[5] / 2, a_min = a[2] - a[5] / 2;
  const float b_max = b[2] + b[5] / 2, b_min = b[2] - b[5] / 2;
  const float oh = fmaxf(fminf(a_max, b_max) - fmaxf(a_min, b_min), 0.f);
  const float o3 = det_box_overlap(a, b) * oh;
  const float va = a[3] * a[4] * a[5], vb = b[3] * b[4] * b[5];
  return o3 / fmaxf(va + vb - o3, 1e-6f);
}

// (x, y, z, dx, dy, dz, vx, vy, yaw) -> (x, y, z, dx, dy, dz, yaw): boxes_for_nms = box[:, [0,1,2,3,4,5,-1]]
__host__ __device__ inline void box9_to_box7(const float* b9, float* b7) {
  for (int k = 0; k < 6; ++k) b7[k] = b9[k];
  b7[6] = b9[8];
}

// ------------------------------------------------------------------ kernels
constexpr unsigned long long kInvalidKey = 0x7fffffffffffffffULL;

__global__ void __launch_bounds__(256) det_keys_kernel(DetParams p, long long M, long long* __restrict__ keys,
                                                       int* __restrict__ seg_count) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float box[9], score;
  int label;
  unsigned long long key = kInvalidKey;
  if (det_decode_pixel(p, m, box, &score, &label)) {
    const int b = (int)(m / ((long long)p.H * p.W));
    const unsigned int seg = (unsigned int)(b * p.C + label);
    key = ((unsigned long long)seg << 32) | (unsigned long long)(0xffffffffu - __float_as_uint(score));  // score > 0
    atomicAdd(&seg_count[seg], 1);
  }
  keys[m] = (long long)key;
}

// suppression mask: row block rb (64 candidates) x all later column blocks of one segment
__global__ void __launch_bounds__(64) det_mask_kernel(DetParams p, const long long* __restrict__ order,
                                                      const int* __restrict__ seg_start, const int* __restrict__ seg_count,
                                                      int pre_max, int col_blocks, unsigned long long* __restrict__ mask) {
  const int s = blockIdx.y, rb = blockIdx.x;
  const int n = min(seg_count[s], pre_max);
  if (rb * 64 >= n) return;
  const float thr = p.nms_thr[s % p.C];
  const long long base = seg_start[s];
  __shared__ float cbox[64 * 7];
  const int i = rb * 64 + threadIdx.x;
  float rbox[7];
  if (i < n) {
    float b9[9], sc; int lb;
    det_decode_pixel(p, order[base + i], b9, &sc, &lb);
    box9_to_box7(b9, rbox);
  }
  for (int cb = rb; cb * 64 < n; ++cb) {
    const int j = cb * 64 + threadIdx.x;
    __syncthreads();
    if (j < n) {
      float b9[9], sc; int lb;
      det_decode_pixel(p, order[base + j], b9, &sc, &lb);
      box9_to_box7(b9, cbox + threadIdx.x * 7);
    }
    __syncthreads();
    if (i < n) {
      const int ncol = min(64, n - cb * 64);
      unsigned long long t = 0;
      for (int k = (cb == rb ? threadIdx.x + 1 : 0); k < ncol; ++k)
        if (det_iou_bev(rbox, cbox + k * 7) > thr) t |= 1ULL << k;
      mask[((size_t)s * pre_max + i) * col_blocks + cb] = t;
    }
  }
}

// greedy sweep of one segment by one warp: word w of the removed-set lives in lane w % 32, slot w / 32
// (col_blocks <= 32 * kSweepSlots, i.e. pre_max <= 8192: the reference's Waymo configs use nms_pre_max_size 4096)
constexpr int kSweepSlots = 4;
__global__ void __launch_bounds__(32) det_sweep_kernel(const int* __restrict__ seg_count, int pre_max, int post_max,
                                                       int col_blocks, const unsigned long long* __restrict__ mask,
                                                       int* __restrict__ keep, int* __restrict__ keep_count) {
  const int s = blockIdx.x, lane = threadIdx.x;
  const int n = min(seg_count[s], pre_max);
  unsigned long long remv[kSweepSlots];
#pragma unroll
  for (int q = 0; q < kSweepSlots; ++q) remv[q] = 0;
  int kept = 0;
  for (int i = 0; i < n && kept < post_max; ++i) {
    const int wi = i >> 6, slot = wi >> 5;
    unsigned long long mine = remv[0];
#pragma unroll
    for (int q = 1; q < kSweepSlots; ++q) mine = slot == q ? remv[q] : mine;
    const unsigned long long w = __shfl_sync(0xffffffffu, mine, wi & 31);
    if (!((w >> (i & 63)) & 1ULL)) {
      if (lane == 0) keep[s * post_max + kept] = i;
      ++kept;
      const unsigned long long* row = mask + ((size_t)s * pre_max + i) * col_blocks;
#pragma unroll
      for (int q = 0; q < kSweepSlots; ++q) {
        const int word = q * 32 + lane;
        if (word < col_blocks && word * 64 < n && word >= wi) remv[q] |= row[word];
      }
    }
  }
  if (lane == 0) keep_count[s] = kept;
}

__global__ void __launch_bounds__(128) det_gather_kernel(DetParams p, const long long* __restrict__ order,
                                                         const int* __restrict__ seg_start, const int* __restrict__ keep,
                                                         const int* __restrict__ keep_count, int post_max, int label_offset,
                                                         float* __restrict__ det_box, float* __restrict__ det_score,
                                                         long long* __restrict__ det_label) {
  const int s = blockIdx.x;
  const int n = keep_count[s];
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    float b9[9], sc; int lb;
    det_decode_pixel(p, order[seg_start[s] + keep[s * post_max + k]], b9, &sc, &lb);
    const size_t o = (size_t)s * post_max + k;
#pragma unroll
    for (int q = 0; q < 9; ++q) det_box[o * 9 + q] = b9[q];
    det_score[o] = sc;
    det_label[o] = lb + label_offset;
  }
}

__global__ void __launch_bounds__(128) aligned_iou3d_kernel(const float* __restrict__ a, const float* __restrict__ b, int n,
                                                            float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float ba[7], bb[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) { ba[k] = a[(size_t)i * 7 + k]; bb[k] = b[(size_t)i * 7 + k]; }
  out[i] = det_aligned_iou3d(ba, bb);
}

int fill_params(DetParams* p, const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6, const float* rect,
                const float* nms_thr) {
  PNX_CHECK_ARG(out && B > 0 && H > 0 && W > 0, "shape");
  PNX_CHECK_ARG(C >= 1 && C <= kMaxClasses, "1..8 classes per task");
  PNX_CHECK_ARG(offs && range6 && rect, "offs/range/rectifier");
  p->out = out; p->ld = ld; p->B = B; p->H = H; p->W = W; p->C = C;
  p->o_reg = offs[0]; p->o_height = offs[1]; p->o_dim = offs[2]; p->o_rot = offs[3]; p->o_vel = offs[4];
  p->o_hm = offs[5]; p->o_iou = offs[6];
  p->osf = osf; p->vs_x = vs_x; p->vs_y = vs_y; p->pc_x = pc_x; p->pc_y = pc_y; p->score_thr = score_thr;
  for (int k = 0; k < 6; ++k) p->range[k] = range6[k];
  for (int k = 0; k < kMaxClasses; ++k) {
    p->rect[k] = k < C ? rect[k] : 0.f;
    p->nms_thr[k] = (nms_thr && k < C) ? nms_thr[k] : 1.f;
  }
  return PNX_OK;
}

}  // namespace

// Contract: include/pnx.h.  offs = column offsets {reg, height, dim, rot, vel, hm, iou (-1: none)} (host ints);
// range6 / rect / nms_thr are HOST float arrays (6 / C / C values).
extern "C" int pnx_det_keys(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                            float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                            const float* rect, long long* keys, int* seg_count, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr);
  if (rc) return rc;
  const long long M = (long long)B * H * W;
  PNX_CUDA(cudaMemsetAsync(seg_count, 0, (size_t)B * C * sizeof(int), stream));
  det_keys_kernel<<<pnx_cdiv(M, 256), 256, 0, stream>>>(p, M, keys, seg_count);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

// order = argsort of the keys (ascending); seg_start = exclusive prefix sum of seg_count; mask scratch
// [B*C, pre_max, pre_max/64] u64; keep [B*C, post_max] int32 (positions inside the segment's sorted run), keep_count [B*C].
extern "C" int pnx_det_nms(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                           float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                           const float* rect, const float* nms_thr, const long long* order, const int* seg_start,
                           const int* seg_count, int pre_max, int post_max, unsigned long long* mask, int* keep,
                           int* keep_count, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nms_thr);
  if (rc) return rc;
  PNX_CHECK_ARG(nms_thr, "nms thresholds");
  PNX_CHECK_ARG(pre_max >= 1 && pre_max <= 64 * 32 * kSweepSlots, "pre_max in [1, 8192]");
  PNX_CHECK_ARG(post_max >= 1 && post_max <= pre_max, "post_max");
  const int col_blocks = (pre_max + 63) / 64;
  const int n_seg = B * C;
  det_mask_kernel<<<dim3(col_blocks, n_seg), 64, 0, stream>>>(p, order, seg_start, seg_count, pre_max, col_blocks, mask);
  PNX_CHECK_LAUNCH();
  det_sweep_kernel<<<n_seg, 32, 0, stream>>>(seg_count, pre_max, post_max, col_blocks, mask, keep, keep_count);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_det_gather(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                              float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                              const float* rect, const long long* order, const int* seg_start, const int* keep,
                              const int* keep_count, int post_max, int label_offset, float* det_box, float* det_score,
                              long long* det_label, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr);
  if (rc) return rc;
  det_gather_kernel<<<B * C, 128, 0, stream>>>(p, order, seg_start, keep, keep_count, post_max, label_offset, det_box,
                                               det_score, det_label);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

// F2 helper: out[i] = aligned 3-D IoU of boxes a[i], b[i] ([n, 7] fp32 each), the target of the Waymo `iou` head loss.
extern "C" int pnx_aligned_iou3d(const float* a, const float* b, int n, float* out, cudaStream_t stream) {
  PNX_CHECK_ARG(n >= 0, "n");
  if (n == 0) return PNX_OK;
  PNX_CHECK_ARG(a && b && out, "null pointer");
  aligned_iou3d_kernel<<<pnx_cdiv(n, 128), 128, 0, stream>>>(a, b, n, out);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" float pnx_aligned_iou3d_host(const float* box7_a, const float* box7_b) { return det_aligned_iou3d(box7_a, box7_b); }

// Host-side evaluation of the same inline math (no GPU): lets the CPU test-suite pin the decode and the rotated IoU
// against the oracle.  `out` is HOST memory here.
extern "C" float pnx_det_iou_bev_host(const float* box7_a, const float* box7_b) { return det_iou_bev(box7_a, box7_b); }

extern "C" int pnx_det_decode_host(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                                   float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                                   const float* rect, long long m, float* box9, float* score, int* label) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr);
  if (rc) return rc;
  PNX_CHECK_ARG(m >= 0 && m < (long long)B * H * W, "pixel index");
  return det_decode_pixel(p, m, box9, score, label) ? 1 : 0;
}
