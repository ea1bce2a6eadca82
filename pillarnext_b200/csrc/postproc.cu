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
// Double-flip testing (pnx_det_*_flip4): the same three passes over the 4B-frame head output of a flip4_points batch
// (flip.cu); the decode reads the four copies of each pixel at their mirrored positions and merges them
// (det_decode_pixel_flip4), so no flipped or averaged copy of any head map is ever written.
// Provenance note: the rotated-rectangle overlap routines (box_geom.cuh: cross3, rect_cross, in_box2d, seg_intersection,
// det_box_overlap, det_iou_bev) deliberately follow the ARITHMETIC of the reference's own device code,
// det3d/core/iou3d_nms/src/iou3d_nms_kernel.cu:39-235 (and its host twin iou3d_cpu.cpp), statement by statement -- same
// operation order (corners rounded as x - dx / 2 and rotated as (x1 - x)), same 1e-2 margin, same angular ordering of
// the polygon vertices: any algebraically equivalent rewrite flips decisions for IoUs near the threshold.  Which builds
// this matches: this file as compiled by build.py (nvcc -O3, fp32 contraction on) against the reference's nms_gpu
// compiled for sm_90a with nvcc's defaults (contraction on; oracle/build_ref_nms.py): equal keep lists at the bench's
// configurations and on segments built to sit on the threshold (tests/test_production_postproc_gpu.py); the host twin
// (no FMA) against iou3d_cpu.cpp built by g++ without FMA: bit-identical IoUs (tests/test_predict_cpu.py).  A device
// build with different contraction is not covered by either.  Everything around them (fused decode, 64-bit sort keys, batched per-(frame, class) mask, the
// on-GPU sweep with up to 4 slots of 2048 candidates, `__host__ __device__` for the CPU parity leg) is this repository's.
// Hot loop character: HBM-bound single pass (1) and a few hundred thousand polygon clips (2) -- no tensor-core work.
#include <math.h>

#include "box_geom.cuh"
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
  int flip4;             // double-flip merge: `out` holds 4B frames, frame 4b + k = copy k of merged frame b
};

constexpr int kMaxClasses = 8;

// ------------------------------------------------------------------ decode of one pixel (centerhead.py:247-304,336-354)
// Shared tail of both decodes: grid position (gx, gy) = pixel + reg offset -> metric centre, range filter, IoU
// rectification.  iou_raw is the raw `iou` head value (ignored without an iou head).  Writes box[0..2], score, label.
__host__ __device__ inline bool det_finish(const DetParams& p, float xs, float ys, float z, float s, int best, float iou_raw,
                                           float* box, float* score, int* label) {
  // xs = xs * out_size_factor * voxel_size + pc_range: three separately rounded fp32 operations, like the reference
#ifdef __CUDA_ARCH__
  xs = __fadd_rn(__fmul_rn(__fmul_rn(xs, p.osf), p.vs_x), p.pc_x);
  ys = __fadd_rn(__fmul_rn(__fmul_rn(ys, p.osf), p.vs_y), p.pc_y);
#else
  { volatile float t = xs * p.osf; t = t * p.vs_x; xs = t + p.pc_x; }
  { volatile float t = ys * p.osf; t = t * p.vs_y; ys = t + p.pc_y; }
#endif
  if (!(xs >= p.range[0] && ys >= p.range[1] && z >= p.range[2] && xs <= p.range[3] && ys <= p.range[4] && z <= p.range[5]))
    return false;
  float iou = 1.0f;
  if (p.o_iou >= 0) iou = fminf(fmaxf((iou_raw + 1.0f) * 0.5f, 0.0f), 1.0f);
  const float r = p.rect[best];
  if (r != 0.0f) s = powf(s, 1.0f - r) * powf(iou, r);     // r == 0: pow(s, 1) * pow(iou, 0) == s exactly
  box[0] = xs; box[1] = ys; box[2] = z;
  *score = s;
  *label = best;
  return true;
}

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
  const float s = 1.0f / (1.0f + expf(-bl));
  if (!(s > p.score_thr)) return false;
  if (!det_finish(p, (float)x + row[p.o_reg], (float)y + row[p.o_reg + 1], row[p.o_height], s, best,
                  p.o_iou >= 0 ? row[p.o_iou] : 0.0f, box, score, label))
    return false;
  box[3] = expf(row[p.o_dim]); box[4] = expf(row[p.o_dim + 1]); box[5] = expf(row[p.o_dim + 2]);
  box[6] = row[p.o_vel]; box[7] = row[p.o_vel + 1];
  box[8] = atan2f(row[p.o_rot], row[p.o_rot + 1]);
  return true;
}

// Mean of the four copies, in the one order that makes the merged maps bit-identically equivariant under both mirrors
// (a y mirror swaps copies 0<->1 and 2<->3, an x mirror 0<->2 and 1<->3; fp32 addition is commutative).
__host__ __device__ inline float det_merge4(const float* v) { return ((v[0] + v[1]) + (v[2] + v[3])) * 0.25f; }

// Double-flip decode of merged pixel m = (b, y, x): reads copy k of frame b at its mirrored pixel -- copy 1 at
// (H-1-y, x), copy 2 at (y, W-1-x), copy 3 at (H-1-y, W-1-x) -- undoes the mirror and merges.  Undo of a y mirror
// (copies 1, 3): reg_y -> 1 - reg_y, sin -> -sin, vy -> -vy; of an x mirror (copies 2, 3): reg_x -> 1 - reg_x,
// cos -> -cos, vx -> -vx (the reference's box_np_ops.flip with the rot = (sin, cos) encoding of assign.py).
// hm: sigmoid per copy, merge per class, first maximum; dim: exp per copy, then merge; height and iou: raw merge.
__host__ __device__ inline bool det_decode_pixel_flip4(const DetParams& p, long long m, float* box, float* score, int* label) {
  const long long hw = (long long)p.H * p.W;
  const long long b = m / hw;
  const int rem = (int)(m - b * hw);
  const int y = rem / p.W, x = rem - y * p.W;
  const int ym = p.H - 1 - y, xm = p.W - 1 - x;
  const float* row[4] = {p.out + ((4 * b + 0) * hw + (long long)y * p.W + x) * p.ld,
                         p.out + ((4 * b + 1) * hw + (long long)ym * p.W + x) * p.ld,
                         p.out + ((4 * b + 2) * hw + (long long)y * p.W + xm) * p.ld,
                         p.out + ((4 * b + 3) * hw + (long long)ym * p.W + xm) * p.ld};
  float v[4];
  int best = 0;
  float s = 0.0f;
  for (int c = 0; c < p.C; ++c) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = 1.0f / (1.0f + expf(-row[k][p.o_hm + c]));
    const float sc = det_merge4(v);
    if (c == 0 || sc > s) { s = sc; best = c; }
  }
  if (!(s > p.score_thr)) return false;
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (k & 2) ? 1.0f - row[k][p.o_reg] : row[k][p.o_reg];
  const float rx = det_merge4(v);
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (k & 1) ? 1.0f - row[k][p.o_reg + 1] : row[k][p.o_reg + 1];
  const float ry = det_merge4(v);
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = row[k][p.o_height];
  const float z = det_merge4(v);
  float iou_raw = 0.0f;
  if (p.o_iou >= 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = row[k][p.o_iou];
    iou_raw = det_merge4(v);
  }
  if (!det_finish(p, (float)x + rx, (float)y + ry, z, s, best, iou_raw, box, score, label)) return false;
  for (int d = 0; d < 3; ++d) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = expf(row[k][p.o_dim + d]);
    box[3 + d] = det_merge4(v);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (k & 2) ? -row[k][p.o_vel] : row[k][p.o_vel];
  box[6] = det_merge4(v);
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (k & 1) ? -row[k][p.o_vel + 1] : row[k][p.o_vel + 1];
  box[7] = det_merge4(v);
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (k & 1) ? -row[k][p.o_rot] : row[k][p.o_rot];
  const float sn = det_merge4(v);
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (k & 2) ? -row[k][p.o_rot + 1] : row[k][p.o_rot + 1];
  box[8] = atan2f(sn, det_merge4(v));
  return true;
}

// The one decode every kernel (keys, NMS mask, gather) and the host twins go through, so keys, masks and gathered
// boxes always agree.
__host__ __device__ inline bool det_decode(const DetParams& p, long long m, float* box, float* score, int* label) {
  return p.flip4 ? det_decode_pixel_flip4(p, m, box, score, label) : det_decode_pixel(p, m, box, score, label);
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
  if (det_decode(p, m, box, &score, &label)) {
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
    det_decode(p, order[base + i], b9, &sc, &lb);
    box9_to_box7(b9, rbox);
  }
  for (int cb = rb; cb * 64 < n; ++cb) {
    const int j = cb * 64 + threadIdx.x;
    __syncthreads();
    if (j < n) {
      float b9[9], sc; int lb;
      det_decode(p, order[base + j], b9, &sc, &lb);
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
    det_decode(p, order[seg_start[s] + keep[s * post_max + k]], b9, &sc, &lb);
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
                const float* nms_thr, int flip4) {
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
  p->flip4 = flip4;
  return PNX_OK;
}

// The launches behind the plain and the double-flip entry points (they differ only in DetParams::flip4).  B is the
// number of output frames either way: the keys, segments, masks and results are those of the merged frames.
int det_keys(const DetParams& p, long long* keys, int* seg_count, cudaStream_t stream) {
  const long long M = (long long)p.B * p.H * p.W;
  PNX_CUDA(cudaMemsetAsync(seg_count, 0, (size_t)p.B * p.C * sizeof(int), stream));
  det_keys_kernel<<<pnx_cdiv(M, 256), 256, 0, stream>>>(p, M, keys, seg_count);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

int det_nms(const DetParams& p, const long long* order, const int* seg_start, const int* seg_count, int pre_max,
            int post_max, unsigned long long* mask, int* keep, int* keep_count, cudaStream_t stream) {
  PNX_CHECK_ARG(pre_max >= 1 && pre_max <= 64 * 32 * kSweepSlots, "pre_max in [1, 8192]");
  PNX_CHECK_ARG(post_max >= 1 && post_max <= pre_max, "post_max");
  const int col_blocks = (pre_max + 63) / 64;
  const int n_seg = p.B * p.C;
  det_mask_kernel<<<dim3(col_blocks, n_seg), 64, 0, stream>>>(p, order, seg_start, seg_count, pre_max, col_blocks, mask);
  PNX_CHECK_LAUNCH();
  det_sweep_kernel<<<n_seg, 32, 0, stream>>>(seg_count, pre_max, post_max, col_blocks, mask, keep, keep_count);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

int det_gather(const DetParams& p, const long long* order, const int* seg_start, const int* keep, const int* keep_count,
               int post_max, int label_offset, float* det_box, float* det_score, long long* det_label, cudaStream_t stream) {
  det_gather_kernel<<<p.B * p.C, 128, 0, stream>>>(p, order, seg_start, keep, keep_count, post_max, label_offset, det_box,
                                                   det_score, det_label);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

}  // namespace

// Contract: include/pnx.h.  offs = column offsets {reg, height, dim, rot, vel, hm, iou (-1: none)} (host ints);
// range6 / rect / nms_thr are HOST float arrays (6 / C / C values).
extern "C" int pnx_det_keys(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                            float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                            const float* rect, long long* keys, int* seg_count, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr, 0);
  return rc ? rc : det_keys(p, keys, seg_count, stream);
}

// order = argsort of the keys (ascending); seg_start = exclusive prefix sum of seg_count; mask scratch
// [B*C, pre_max, pre_max/64] u64; keep [B*C, post_max] int32 (positions inside the segment's sorted run), keep_count [B*C].
extern "C" int pnx_det_nms(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                           float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                           const float* rect, const float* nms_thr, const long long* order, const int* seg_start,
                           const int* seg_count, int pre_max, int post_max, unsigned long long* mask, int* keep,
                           int* keep_count, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nms_thr, 0);
  if (rc) return rc;
  PNX_CHECK_ARG(nms_thr, "nms thresholds");
  return det_nms(p, order, seg_start, seg_count, pre_max, post_max, mask, keep, keep_count, stream);
}

extern "C" int pnx_det_gather(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                              float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                              const float* rect, const long long* order, const int* seg_start, const int* keep,
                              const int* keep_count, int post_max, int label_offset, float* det_box, float* det_score,
                              long long* det_label, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr, 0);
  return rc ? rc : det_gather(p, order, seg_start, keep, keep_count, post_max, label_offset, det_box, det_score, det_label,
                              stream);
}

// Double-flip twins of the three entry points: same arguments, but `out` holds the 4B frames of the flipped batch
// ([4B*H*W, ld], frame 4b + k = copy k of frame b, see det_decode_pixel_flip4) and B counts the merged frames.
extern "C" int pnx_det_keys_flip4(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                                  float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                                  const float* rect, long long* keys, int* seg_count, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr, 1);
  return rc ? rc : det_keys(p, keys, seg_count, stream);
}

extern "C" int pnx_det_nms_flip4(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                                 float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                                 const float* rect, const float* nms_thr, const long long* order, const int* seg_start,
                                 const int* seg_count, int pre_max, int post_max, unsigned long long* mask, int* keep,
                                 int* keep_count, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nms_thr, 1);
  if (rc) return rc;
  PNX_CHECK_ARG(nms_thr, "nms thresholds");
  return det_nms(p, order, seg_start, seg_count, pre_max, post_max, mask, keep, keep_count, stream);
}

extern "C" int pnx_det_gather_flip4(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                                    float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                                    const float* rect, const long long* order, const int* seg_start, const int* keep,
                                    const int* keep_count, int post_max, int label_offset, float* det_box,
                                    float* det_score, long long* det_label, cudaStream_t stream) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr, 1);
  return rc ? rc : det_gather(p, order, seg_start, keep, keep_count, post_max, label_offset, det_box, det_score, det_label,
                              stream);
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
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr, 0);
  if (rc) return rc;
  PNX_CHECK_ARG(m >= 0 && m < (long long)B * H * W, "pixel index");
  return det_decode(p, m, box9, score, label) ? 1 : 0;
}

// Double-flip host twin: `out` holds 4B frames (HOST memory), m indexes the B*H*W merged pixels.
extern "C" int pnx_det_decode_flip4_host(const float* out, long long ld, int B, int H, int W, int C, const int* offs,
                                         float osf, float vs_x, float vs_y, float pc_x, float pc_y, float score_thr,
                                         const float* range6, const float* rect, long long m, float* box9, float* score,
                                         int* label) {
  DetParams p;
  int rc = fill_params(&p, out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect, nullptr, 1);
  if (rc) return rc;
  PNX_CHECK_ARG(m >= 0 && m < (long long)B * H * W, "pixel index");
  return det_decode(p, m, box9, score, label) ? 1 : 0;
}
