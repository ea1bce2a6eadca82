// pfn_bwd.cu -- backward of the PillarFeatureNet encoder (rows P1-P3), fp32, sm_90a.
// The reference gets this from autograd through torch_scatter.scatter_max / BatchNorm1d / Linear
// (det3d/models/readers/pillar_encoder.py:35-50,174-182; trainer/trainer/trainer.py:94-108).
// Same bucketed layout as the forward (pfn.cu): per-pillar work is an in-order loop, no atomics on any
// per-pillar reduction; only the per-channel BatchNorm sums and the weight gradients use (fp64/fp32)
// atomics across blocks.
//   B1 pfn_bwd_max1 : route dfeat through the last max (first arg-max point, ReLU) + BN1 reductions
//   B2 pfn_bwd_lin1 : dy1 = BN1 backward; d_in1 = dy1 . W1 ; dW1 += dy1^T . in1
//   B3 pfn_bwd_max0 : sum the x0max half of d_in1 over each pillar, route through max0/ReLU, BN0 reductions
//   B4 pfn_bwd_lin0 : dy0 = BN0 backward; dW0 += dy0^T . features
#include "pnx_common.cuh"

namespace {

struct PfnGeom {
  float min_x, min_y, vs_x, vs_y;
};

constexpr int kLd = 257;  // padded row stride of the [channel][point] shared-memory tiles

__global__ void pfn_bwd_max1_kernel(const float* __restrict__ y1, const float* __restrict__ feat,
                                    const float* __restrict__ dfeat, const int* __restrict__ bucket_off,
                                    const int* __restrict__ counts, int cap_p, const float* __restrict__ scale1,
                                    const float* __restrict__ shift1, const float* __restrict__ mean1,
                                    const float* __restrict__ invstd1, int* __restrict__ argq1,
                                    double* __restrict__ red1) {
  const int lane = pnx::lane_id();
  const int n_p = min(counts[0], cap_p);
  const float2 sc = reinterpret_cast<const float2*>(scale1)[lane], sh = reinterpret_cast<const float2*>(shift1)[lane];
  const float2 mu = reinterpret_cast<const float2*>(mean1)[lane], is = reinterpret_cast<const float2*>(invstd1)[lane];
  double sg0 = 0, sg1 = 0, sx0 = 0, sx1 = 0;
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_p; p += (gridDim.x * blockDim.x) >> 5) {
    const int lo = bucket_off[p], hi = bucket_off[p + 1];
    const float2 f = reinterpret_cast<const float2*>(feat + (size_t)p * 64)[lane];
    int a0 = -1, a1 = -1;
    float v0 = 0.f, v1 = 0.f;
    for (int q = lo; q < hi; ++q) {
      const float2 v = reinterpret_cast<const float2*>(y1 + (size_t)q * 64)[lane];
      const float x0 = fmaxf(fmaf(v.x, sc.x, sh.x), 0.f), x1 = fmaxf(fmaf(v.y, sc.y, sh.y), 0.f);
      if (a0 < 0 && f.x > 0.f && x0 == f.x) { a0 = q; v0 = v.x; }
      if (a1 < 0 && f.y > 0.f && x1 == f.y) { a1 = q; v1 = v.y; }
    }
    const float2 g = reinterpret_cast<const float2*>(dfeat + (size_t)p * 64)[lane];
    if (a0 >= 0) { sg0 += g.x; sx0 += (double)g.x * (double)((v0 - mu.x) * is.x); }
    if (a1 >= 0) { sg1 += g.y; sx1 += (double)g.y * (double)((v1 - mu.y) * is.y); }
    reinterpret_cast<int2*>(argq1 + (size_t)p * 64)[lane] = make_int2(a0, a1);
  }
  atomicAdd(&red1[2 * lane], sg0);
  atomicAdd(&red1[2 * lane + 1], sg1);
  atomicAdd(&red1[64 + 2 * lane], sx0);
  atomicAdd(&red1[64 + 2 * lane + 1], sx1);
}

__global__ void __launch_bounds__(256)
    pfn_bwd_lin1_kernel(const float* __restrict__ y0, const float* __restrict__ y1, const float* __restrict__ x0max,
                        const float* __restrict__ dfeat, const int* __restrict__ argq1,
                        const int* __restrict__ bucket_pts, const int* __restrict__ pillar_of_point,
                        const int* __restrict__ counts, int cap_n, const float* __restrict__ scale0,
                        const float* __restrict__ shift0, const float* __restrict__ mean1,
                        const float* __restrict__ invstd1, const float* __restrict__ gamma1,
                        const double* __restrict__ red1, const float* __restrict__ w1, float* __restrict__ d_x0,
                        float* __restrict__ dxm_part, double* __restrict__ dW1, const int* __restrict__ bn_count) {
  extern __shared__ float smem[];
  float* sdy = smem;                  // [64][kLd]
  float* sin_ = smem + 64 * kLd;      // [64][kLd]
  float* sw = sin_ + 64 * kLd;        // [64 o][64 k]
  float* sc0 = sw + 4096;             // scale0[32], shift0[32]
  float* sbn = sc0 + 64;              // a[64] = gamma*invstd, b[64] = sum_g/n, c[64] = sum_gx/n, mean[64], invstd[64]
  const int nv = min(counts[1], cap_n);
  const float inv_n = 1.f / (float)max(bn_count ? *bn_count : nv, 1);   // SyncBatchNorm: population of all ranks
  for (int k = threadIdx.x; k < 4096; k += 256) sw[k] = w1[k];
  if (threadIdx.x < 32) {
    sc0[threadIdx.x] = scale0[threadIdx.x];
    sc0[32 + threadIdx.x] = shift0[threadIdx.x];
  }
  if (threadIdx.x < 64) {
    const int c = threadIdx.x;
    sbn[c] = gamma1[c] * invstd1[c];
    sbn[64 + c] = (float)red1[c] * inv_n;
    sbn[128 + c] = (float)red1[64 + c] * inv_n;
    sbn[192 + c] = mean1[c];
    sbn[256 + c] = invstd1[c];
  }
  __syncthreads();
  const int q = blockIdx.x * 256 + threadIdx.x;
  const bool active = q < nv;
  int p = 0;
  if (active) p = pillar_of_point[bucket_pts[q]];
  float din[64];
#pragma unroll
  for (int k = 0; k < 64; ++k) din[k] = 0.f;
  // in1 -> smem (column layout), dy1 -> smem + registers-free accumulation of d_in1
#pragma unroll 4
  for (int k = 0; k < 32; ++k) {
    float a = 0.f, b = 0.f;
    if (active) {
      a = fmaxf(fmaf(y0[(size_t)q * 32 + k], sc0[k], sc0[32 + k]), 0.f);
      b = x0max[(size_t)p * 32 + k];
    }
    sin_[k * kLd + threadIdx.x] = a;
    sin_[(32 + k) * kLd + threadIdx.x] = b;
  }
  for (int o = 0; o < 64; ++o) {
    float dy = 0.f;
    if (active) {
      const float g = (argq1[(size_t)p * 64 + o] == q) ? dfeat[(size_t)p * 64 + o] : 0.f;
      const float xh = (y1[(size_t)q * 64 + o] - sbn[192 + o]) * sbn[256 + o];
      dy = sbn[o] * (g - sbn[64 + o] - xh * sbn[128 + o]);
    }
    sdy[o * kLd + threadIdx.x] = dy;
    const float4* wr = reinterpret_cast<const float4*>(sw + o * 64);
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 w = wr[k];
      din[4 * k + 0] = fmaf(dy, w.x, din[4 * k + 0]);
      din[4 * k + 1] = fmaf(dy, w.y, din[4 * k + 1]);
      din[4 * k + 2] = fmaf(dy, w.z, din[4 * k + 2]);
      din[4 * k + 3] = fmaf(dy, w.w, din[4 * k + 3]);
    }
  }
  if (active) {
    float4* d0 = reinterpret_cast<float4*>(d_x0 + (size_t)q * 32);
    float4* d1 = reinterpret_cast<float4*>(dxm_part + (size_t)q * 32);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      d0[k] = make_float4(din[4 * k], din[4 * k + 1], din[4 * k + 2], din[4 * k + 3]);
      d1[k] = make_float4(din[32 + 4 * k], din[32 + 4 * k + 1], din[32 + 4 * k + 2], din[32 + 4 * k + 3]);
    }
  }
  __syncthreads();
  // dW1[o][k] partial over this block's 256 points: thread -> k = t%64, o in [16*(t/64), +16)
  {
    const int k = threadIdx.x & 63, og = (threadIdx.x >> 6) * 16;
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    const float* ik = sin_ + k * kLd;
    for (int qq = 0; qq < 256; ++qq) {
      const float v = ik[qq];
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = fmaf(sdy[(og + i) * kLd + qq], v, acc[i]);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) atomicAdd(&dW1[(og + i) * 64 + k], (double)acc[i]);  // fp64: order-insensitive across CTAs
  }
}

__global__ void pfn_bwd_max0_kernel(const float* __restrict__ y0, const float* __restrict__ x0max,
                                    const float* __restrict__ dxm_part, const int* __restrict__ bucket_off,
                                    const int* __restrict__ counts, int cap_p, const float* __restrict__ scale0,
                                    const float* __restrict__ shift0, const float* __restrict__ mean0,
                                    const float* __restrict__ invstd0, float* __restrict__ d_x0,
                                    double* __restrict__ red0) {
  const int lane = pnx::lane_id();
  const int n_p = min(counts[0], cap_p);
  const float sc = scale0[lane], sh = shift0[lane], mu = mean0[lane], is = invstd0[lane];
  double sg = 0, sx = 0;
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_p; p += (gridDim.x * blockDim.x) >> 5) {
    const int lo = bucket_off[p], hi = bucket_off[p + 1];
    const float m = x0max[(size_t)p * 32 + lane];
    float dsum = 0.f;
    int arg = -1;
    for (int q = lo; q < hi; ++q) {
      dsum += dxm_part[(size_t)q * 32 + lane];
      const float x = fmaxf(fmaf(y0[(size_t)q * 32 + lane], sc, sh), 0.f);
      if (arg < 0 && m > 0.f && x == m) arg = q;
    }
    for (int q = lo; q < hi; ++q) {
      const float v = y0[(size_t)q * 32 + lane];
      const float x = fmaxf(fmaf(v, sc, sh), 0.f);
      float g = d_x0[(size_t)q * 32 + lane] + (q == arg ? dsum : 0.f);
      g = x > 0.f ? g : 0.f;
      d_x0[(size_t)q * 32 + lane] = g;  // now holds g0 = grad w.r.t. bn0 output (post ReLU mask)
      sg += g;
      sx += (double)g * (double)((v - mu) * is);
    }
  }
  atomicAdd(&red0[lane], sg);
  atomicAdd(&red0[32 + lane], sx);
}

__global__ void __launch_bounds__(320)
    pfn_bwd_lin0_kernel(const float* __restrict__ points, const int* __restrict__ bucket_pts,
                        const int* __restrict__ pillar_of_point, const int* __restrict__ coords,
                        const float* __restrict__ pmean, const float* __restrict__ y0, const float* __restrict__ g0,
                        const int* __restrict__ counts, int cap_n, PfnGeom geo, const float* __restrict__ mean0,
                        const float* __restrict__ invstd0, const float* __restrict__ gamma0,
                        const double* __restrict__ red0, double* __restrict__ dW0, const int* __restrict__ bn_count) {
  __shared__ float sdy[32 * kLd];
  __shared__ float sf[10 * kLd];
  __shared__ float sbn[5 * 32];
  const int nv = min(counts[1], cap_n);
  const float inv_n = 1.f / (float)max(bn_count ? *bn_count : nv, 1);
  if (threadIdx.x < 32) {
    const int c = threadIdx.x;
    sbn[c] = gamma0[c] * invstd0[c];
    sbn[32 + c] = (float)red0[c] * inv_n;
    sbn[64 + c] = (float)red0[32 + c] * inv_n;
    sbn[96 + c] = mean0[c];
    sbn[128 + c] = invstd0[c];
  }
  __syncthreads();
  if (threadIdx.x < 256) {
    const int q = blockIdx.x * 256 + threadIdx.x;
    const bool active = q < nv;
    float f[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) f[k] = 0.f;
    if (active) {
      const int i = bucket_pts[q];
      const int p = pillar_of_point[i];
      const float2* pt = reinterpret_cast<const float2*>(points + (size_t)i * 6);
      const float2 a = __ldg(pt), b = __ldg(pt + 1), c = __ldg(pt + 2);
      f[0] = a.y; f[1] = b.x; f[2] = b.y; f[3] = c.x; f[4] = c.y;
      f[5] = __fsub_rn(a.y, pmean[p * 3 + 0]);
      f[6] = __fsub_rn(b.x, pmean[p * 3 + 1]);
      f[7] = __fsub_rn(b.y, pmean[p * 3 + 2]);
      const float xi = (float)coords[p * 3 + 2], yi = (float)coords[p * 3 + 1];
      f[8] = __fsub_rn(a.y, __fadd_rn(__fadd_rn(__fmul_rn(xi, geo.vs_x), __fdiv_rn(geo.vs_x, 2.f)), geo.min_x));
      f[9] = __fsub_rn(b.x, __fadd_rn(__fadd_rn(__fmul_rn(yi, geo.vs_y), __fdiv_rn(geo.vs_y, 2.f)), geo.min_y));
    }
#pragma unroll
    for (int k = 0; k < 10; ++k) sf[k * kLd + threadIdx.x] = f[k];
    for (int o = 0; o < 32; ++o) {
      float dy = 0.f;
      if (active) {
        const float g = g0[(size_t)q * 32 + o];
        const float xh = (y0[(size_t)q * 32 + o] - sbn[96 + o]) * sbn[128 + o];
        dy = sbn[o] * (g - sbn[32 + o] - xh * sbn[64 + o]);
      }
      sdy[o * kLd + threadIdx.x] = dy;
    }
  }
  __syncthreads();
  {
    const int o = threadIdx.x / 10, k = threadIdx.x - o * 10;
    float acc = 0.f;
    for (int qq = 0; qq < 256; ++qq) acc = fmaf(sdy[o * kLd + qq], sf[k * kLd + qq], acc);
    atomicAdd(&dW0[o * 10 + k], (double)acc);
  }
}

}  // namespace

// Contract: include/pnx.h (pnx_pfn_backward).  red [2*32 + 2*64] fp64 and dW0 [32,10] / dW1 [64,64] fp64 must be zeroed
// (fp64 accumulators: the per-CTA partials are summed by global atomics, whose order then does not matter at fp32 level).
extern "C" int pnx_pfn_backward(const float* points, const int* bucket_off, const int* bucket_pts,
                                const int* pillar_of_point, const int* coords, const int* counts, int cap_points,
                                int cap_pillars, float min_x, float min_y, float vs_x, float vs_y, const float* pmean,
                                const float* y0, const float* y1, const float* x0max, const float* feat,
                                const float* dfeat, const float* w1, const float* scale0, const float* shift0,
                                const float* mean0, const float* invstd0, const float* gamma0, const float* scale1,
                                const float* shift1, const float* mean1, const float* invstd1, const float* gamma1,
                                int* argq1, float* d_x0, float* dxm_part, double* red, double* dW0, double* dW1,
                                int phases, const int* bn_count, cudaStream_t stream) {
  if (cap_points == 0 || cap_pillars == 0) return PNX_OK;
  static bool attr_set = false;
  const size_t smem_lin1 = (size_t)(2 * 64 * kLd + 4096 + 64 + 5 * 64) * sizeof(float);
  if (!attr_set) {
    PNX_CUDA(cudaFuncSetAttribute(pfn_bwd_lin1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_lin1));
    attr_set = true;
  }
  double* red0 = red;        // [64]: sum g0, sum g0*xhat0
  double* red1 = red + 64;   // [128]
  PfnGeom g{min_x, min_y, vs_x, vs_y};
  const int pblocks = min(pnx_cdiv((long long)cap_pillars * 32, 256), 148 * 8);
  // phases (bit mask; 0 = all four): 1 max1 | 2 lin1 | 4 max0 | 8 lin0.  SyncBatchNorm callers run {1}, all-reduce red1,
  // {2,4}, all-reduce red0, {8}, and pass bn_count = device int holding the population of all ranks.
  if (phases == 0) phases = 15;
  if (phases & 1) {
    pfn_bwd_max1_kernel<<<pblocks, 256, 0, stream>>>(y1, feat, dfeat, bucket_off, counts, cap_pillars, scale1, shift1,
                                                     mean1, invstd1, argq1, red1);
    PNX_CHECK_LAUNCH();
  }
  if (phases & 2) {
    pfn_bwd_lin1_kernel<<<pnx_cdiv(cap_points, 256), 256, smem_lin1, stream>>>(
        y0, y1, x0max, dfeat, argq1, bucket_pts, pillar_of_point, counts, cap_points, scale0, shift0, mean1, invstd1,
        gamma1, red1, w1, d_x0, dxm_part, dW1, bn_count);
    PNX_CHECK_LAUNCH();
  }
  if (phases & 4) {
    pfn_bwd_max0_kernel<<<pblocks, 256, 0, stream>>>(y0, x0max, dxm_part, bucket_off, counts, cap_pillars, scale0,
                                                     shift0, mean0, invstd0, d_x0, red0);
    PNX_CHECK_LAUNCH();
  }
  if (phases & 8) {
    pfn_bwd_lin0_kernel<<<pnx_cdiv(cap_points, 256), 320, 0, stream>>>(points, bucket_pts, pillar_of_point, coords,
                                                                       pmean, y0, d_x0, counts, cap_points, g, mean0,
                                                                       invstd0, gamma0, red0, dW0, bn_count);
    PNX_CHECK_LAUNCH();
  }
  return PNX_OK;
}
