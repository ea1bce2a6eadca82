// assign.cu -- CenterPoint label assignment on the GPU (row F3 of SURVEY.md section 8f).
//
// Replaces, for one task, reference det3d/datasets/pipelines/assign.py:23-116 (AssignLabel.__call__) together with
// center_utils.py:12-60 (gaussian_radius / gaussian2D / draw_gaussian) and the batching of loader/collate.py:23-33:
// from the raw ground-truth boxes of a batch it writes the training targets the loss consumes --
//   hm [B, C, H, W] gaussian heat-map splat (max over objects), anno_box [B, M, 10], ind [B, M], mask [B, M],
//   cat [B, M], gt_boxes [B, M, 7]
// so the per-step host->device traffic is the boxes (36 B/object) instead of the dense heat-maps (5.5 MB/frame for
// the six nuScenes tasks).  The reference does this in numpy on the data-loader workers: float64 for the radius, the
// centre coordinate and the gaussian, float32 storage -- the same mix is used here (the work is a few thousand cells).
// Kernel 1, one CTA per frame: objects are compacted in their original order (slot = number of accepted objects of the
// task before it), exactly like the reference's running `task_nums`.  Kernel 2, one CTA per (object, frame): the splat.
#include "pnx_common.cuh"

namespace {

constexpr int kAssignThreads = 512;

struct AssignParams {
  const float* boxes;     // [B, N, 9] (x, y, z, dx, dy, dz, vx, vy, yaw)
  const int* cls;         // [B, N] global class index, < 0 = ignore
  int B, N;
  const int* cls_task;    // [n_classes] task of a class
  const int* cls_id;      // [n_classes] index of the class inside its task
  int n_classes, task;
  double vs_x, vs_y, pc_x, pc_y, osf, overlap;
  int min_radius, M, C, H, W;
  float* hm;
  float* anno;
  long long* ind;
  unsigned char* mask;
  long long* cat;
  float* gtb;
  int* obj;               // [B, N, 4] scratch: (cx, cy, radius, class id) of every object, cx = -1: not drawn
};

// center_utils.py:12-34, float64
__device__ double gaussian_radius(double height, double width, double min_overlap) {
  const double b1 = height + width;
  const double c1 = width * height * (1 - min_overlap) / (1 + min_overlap);
  const double r1 = (b1 + sqrt(b1 * b1 - 4 * c1)) / 2;
  const double b2 = 2 * (height + width);
  const double c2 = (1 - min_overlap) * width * height;
  const double r2 = (b2 + sqrt(b2 * b2 - 16 * c2)) / 2;
  const double a3 = 4 * min_overlap;
  const double b3 = -2 * min_overlap * (height + width);
  const double c3 = (min_overlap - 1) * width * height;
  const double r3 = (b3 + sqrt(b3 * b3 - 4 * a3 * c3)) / 2;
  return fmin(r1, fmin(r2, r3));
}

__global__ void __launch_bounds__(kAssignThreads) assign_kernel(AssignParams p) {
  __shared__ int s_scan[kAssignThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // running slot base of the chunk: every thread keeps it in a register and adds all of s_scan once the barrier has
  // published it, so no thread writes shared state that another warp of the same barrier interval still reads
  int base = 0;
  for (int k0 = 0; k0 < p.N; k0 += kAssignThreads) {
    const int k = k0 + tid;
    bool ok = false;
    int cid = 0, radius = 0, cxi = 0, cyi = 0;
    float ctx = 0.f, cty = 0.f;
    const float* bx = p.boxes + ((size_t)b * p.N + (k < p.N ? k : 0)) * 9;
    if (k < p.N) {
      const int c = p.cls[(size_t)b * p.N + k];
      if (c >= 0 && c < p.n_classes && p.cls_task[c] == p.task) {
        // assign.py:66-70 -- float32 box value / float64 voxel size / integer factor
        const double sx = (double)bx[3] / p.vs_x / p.osf, sy = (double)bx[4] / p.vs_y / p.osf;
        if (sx > 0 && sy > 0) {
          cid = p.cls_id[c];
          radius = max(p.min_radius, (int)gaussian_radius(sy, sx, p.overlap));              // :74-76
          ctx = (float)(((double)bx[0] - p.pc_x) / p.vs_x / p.osf);                           // :79-83 (float32 ct)
          cty = (float)(((double)bx[1] - p.pc_y) / p.vs_y / p.osf);
          cxi = (int)ctx;                                                                     // astype(int32): truncation
          cyi = (int)cty;
          ok = cxi >= 0 && cxi < p.W && cyi >= 0 && cyi < p.H;                                 // :86-88
        }
      }
    }
    // slot = accepted objects of this task before k (reference task_nums, :92)
    const unsigned int bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_scan[warp] = __popc(bal);
    __syncthreads();
    int before = base + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) before += s_scan[w];
    for (int w = 0; w < kAssignThreads / 32; ++w) base += s_scan[w];
    if (ok && before < p.M) {
      const size_t o = (size_t)b * p.M + before;
      p.cat[o] = cid;
      p.ind[o] = (long long)cyi * p.W + cxi;
      p.mask[o] = 1;
      float* a = p.anno + o * 10;
      a[0] = ctx - (float)cxi;                                                                // :100-103
      a[1] = cty - (float)cyi;
      a[2] = bx[2];
      a[3] = logf(bx[3]); a[4] = logf(bx[4]); a[5] = logf(bx[5]);
      a[6] = bx[6]; a[7] = bx[7];
      a[8] = sinf(bx[8]); a[9] = cosf(bx[8]);
      float* g = p.gtb + o * 7;                                                               // :104-107
      for (int q = 0; q < 6; ++q) g[q] = bx[q];
      g[6] = bx[8];
    }
    // hand the accepted objects to the splat kernel (one CTA per object)
    if (k < p.N) {
      int4 o = make_int4(ok ? cxi : -1, cyi, radius, cid);
      reinterpret_cast<int4*>(p.obj)[(size_t)b * p.N + k] = o;
    }
    __syncthreads();  // s_scan is rewritten by the next chunk
  }
}

// gaussian splat, one CTA per (object, frame): draw_gaussian = max with exp(-(dx^2+dy^2)/(2 sigma^2)), sigma = (2r+1)/6,
// entries below eps dropped; float64 like numpy, stored float32; atomicMax on the bit pattern (values >= 0)
__global__ void __launch_bounds__(128) assign_splat_kernel(AssignParams p) {
  const int k = blockIdx.x, b = blockIdx.y;
  const int4 o = reinterpret_cast<const int4*>(p.obj)[(size_t)b * p.N + k];
  const int ox = o.x, oy = o.y, r = o.z, oc = o.w;
  if (ox < 0) return;
  const int d = 2 * r + 1;
  const double sigma = (double)d / 6.0;
  float* plane = p.hm + ((size_t)b * p.C + oc) * p.H * p.W;
  for (int q = threadIdx.x; q < d * d; q += blockDim.x) {
    const int gy = q / d - r, gx = q - (q / d) * d - r;
    const int yy = oy + gy, xx = ox + gx;
    if (yy < 0 || yy >= p.H || xx < 0 || xx >= p.W) continue;
    const double v = exp(-(double)(gx * gx + gy * gy) / (2 * sigma * sigma));
    if (v < 2.220446049250313e-16) continue;                                                   // np.finfo(float64).eps * max (= 1)
    atomicMax(reinterpret_cast<int*>(plane + (size_t)yy * p.W + xx), __float_as_int((float)v));
  }
}

}  // namespace

// Contract: include/pnx.h (pnx_assign_labels).  hm / anno / ind / mask / cat / gtb must be zeroed by the caller.
extern "C" int pnx_assign_labels(const float* boxes, const int* cls, int B, int N, const int* cls_task, const int* cls_id,
                                 int n_classes, int task, double vs_x, double vs_y, double pc_x, double pc_y, int osf,
                                 double gaussian_overlap, int min_radius, int max_objs, int C, int H, int W, float* hm,
                                 float* anno_box, long long* ind, unsigned char* mask, long long* cat, float* gt_boxes,
                                 int* obj_scratch, cudaStream_t stream) {
  PNX_CHECK_ARG(B > 0 && N >= 0 && n_classes > 0 && C > 0 && H > 0 && W > 0 && max_objs > 0 && osf > 0, "shapes");
  if (N == 0) return PNX_OK;
  AssignParams p;
  p.boxes = boxes; p.cls = cls; p.B = B; p.N = N; p.cls_task = cls_task; p.cls_id = cls_id; p.n_classes = n_classes;
  p.task = task; p.vs_x = vs_x; p.vs_y = vs_y; p.pc_x = pc_x; p.pc_y = pc_y; p.osf = (double)osf; p.overlap = gaussian_overlap;
  p.min_radius = min_radius; p.M = max_objs; p.C = C; p.H = H; p.W = W;
  p.hm = hm; p.anno = anno_box; p.ind = ind; p.mask = mask; p.cat = cat; p.gtb = gt_boxes; p.obj = obj_scratch;
  PNX_CHECK_ARG(obj_scratch && (reinterpret_cast<uintptr_t>(obj_scratch) & 15) == 0, "obj_scratch [B, N, 4] int32, 16-byte aligned");
  assign_kernel<<<B, kAssignThreads, 0, stream>>>(p);
  PNX_CHECK_LAUNCH();
  assign_splat_kernel<<<dim3(N, B), 128, 0, stream>>>(p);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}
