// pfn.cu -- PillarFeatureNet encoder (rows V3, P1-P3 of SURVEY.md section 8a) for sm_90a, fp32.
//
// Replaces reference det3d/models/readers/pillar_encoder.py:113-123 (scatter_mean + decoration),
// :35-50 (PFNLayer: Linear(no bias) -> BatchNorm1d(eps 1e-3) -> ReLU -> scatter_max -> gather -> cat)
// twice and :180 (final scatter_max, idempotent on the last layer's output).
// Points arrive bucketed by pillar (voxelize.cu): every per-pillar reduction is an in-order loop over
// the bucket (mean: one thread per pillar, ascending point id == the reference CPU summation order;
// max: one warp per pillar, lane = channel) -- no atomics and no shuffles on the max reduction.
// Training-mode BatchNorm needs whole-batch statistics before the ReLU/max, hence three phases:
//   lin0+stats0 | bn0/relu/max0 -> lin1+stats1 | bn1/relu/max1.
#include "pnx_common.cuh"

namespace {

struct PfnGeom {
  float min_x, min_y, vs_x, vs_y;
};

// Butterfly transpose-reduce: returns sum over the warp's lanes of v[lane_id] (31 shuffles / 32 channels)
__device__ __forceinline__ float warp_colsum32(float (&v)[32]) {
  const uint32_t lane = pnx::lane_id();
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int k = 0; k < off; ++k) {
      float send = upper ? v[k] : v[k + off];
      float keep = upper ? v[k + off] : v[k];
      v[k] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  return v[0];
}

// accumulate per-channel sum / sumsq of a 32-channel slab held one row per thread into stats (fp64)
template <int kWarps>
__device__ __forceinline__ void block_stats32(float (&y)[32], bool active, double* __restrict__ stats_sum,
                                              double* __restrict__ stats_sq, float (*red)[2][32]) {
  float a[32], b[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    float t = active ? y[k] : 0.f;
    a[k] = t;
    b[k] = t * t;
  }
  float s = warp_colsum32(a);
  float q = warp_colsum32(b);
  const int w = threadIdx.x >> 5;
  red[w][0][pnx::lane_id()] = s;
  red[w][1][pnx::lane_id()] = q;
  __syncthreads();
  if (threadIdx.x < 64) {
    int which = threadIdx.x >> 5, c = threadIdx.x & 31;
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < kWarps; ++k) acc += (double)red[k][which][c];
    atomicAdd(which ? &stats_sq[c] : &stats_sum[c], acc);
  }
  __syncthreads();
}

// V3: per-pillar mean of xyz (scatter_mean, pillar_encoder.py:113-114). One thread per pillar,
// sequential ascending-point-id sum, then a true fp32 division by the count.
__global__ void pfn_mean_kernel(const float* __restrict__ points, const int* __restrict__ bucket_off,
                                const int* __restrict__ bucket_pts, const int* __restrict__ counts, int cap,
                                float* __restrict__ mean) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= min(counts[0], cap)) return;
  int lo = bucket_off[p], hi = bucket_off[p + 1];
  float sx = 0.f, sy = 0.f, sz = 0.f;
  for (int q = lo; q < hi; ++q) {
    const float* pt = points + (size_t)bucket_pts[q] * 6;
    sx = __fadd_rn(sx, pt[1]);
    sy = __fadd_rn(sy, pt[2]);
    sz = __fadd_rn(sz, pt[3]);
  }
  float n = (float)max(hi - lo, 1);
  mean[p * 3 + 0] = __fdiv_rn(sx, n);
  mean[p * 3 + 1] = __fdiv_rn(sy, n);
  mean[p * 3 + 2] = __fdiv_rn(sz, n);
}

// P1 (layer 0): decorate (pillar_encoder.py:116-123) + Linear(10->32) (:37) + BN statistics.
__global__ void __launch_bounds__(256)
    pfn_lin0_kernel(const float* __restrict__ points, const int* __restrict__ bucket_pts,
                    const int* __restrict__ pillar_of_point, const int* __restrict__ coords,
                    const float* __restrict__ mean, const int* __restrict__ counts, int cap_n, PfnGeom g,
                    const float* __restrict__ w0, float* __restrict__ y0, double* __restrict__ stats, int training) {
  __shared__ float sw[32 * 10];
  __shared__ float red[8][2][32];
  for (int k = threadIdx.x; k < 320; k += 256) sw[k] = w0[k];
  __syncthreads();
  const int nv = min(counts[1], cap_n);
  const int q = blockIdx.x * 256 + threadIdx.x;
  const bool active = q < nv;
  float y[32];
#pragma unroll
  for (int o = 0; o < 32; ++o) y[o] = 0.f;
  if (active) {
    const int i = bucket_pts[q];
    const int p = pillar_of_point[i];
    const float2* pt = reinterpret_cast<const float2*>(points + (size_t)i * 6);
    const float2 a = __ldg(pt), b = __ldg(pt + 1), c = __ldg(pt + 2);  // (b,x) (y,z) (i,t)
    float f[10];
    f[0] = a.y; f[1] = b.x; f[2] = b.y; f[3] = c.x; f[4] = c.y;
    f[5] = __fsub_rn(a.y, mean[p * 3 + 0]);
    f[6] = __fsub_rn(b.x, mean[p * 3 + 1]);
    f[7] = __fsub_rn(b.y, mean[p * 3 + 2]);
    const float xi = (float)coords[p * 3 + 2], yi = (float)coords[p * 3 + 1];
    // :119-120  (idx*vs + vs/2) + pc_min, separate fp32 mul/add
    f[8] = __fsub_rn(a.y, __fadd_rn(__fadd_rn(__fmul_rn(xi, g.vs_x), __fdiv_rn(g.vs_x, 2.f)), g.min_x));
    f[9] = __fsub_rn(b.x, __fadd_rn(__fadd_rn(__fmul_rn(yi, g.vs_y), __fdiv_rn(g.vs_y, 2.f)), g.min_y));
#pragma unroll
    for (int o = 0; o < 32; ++o) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 10; ++k) acc = fmaf(f[k], sw[o * 10 + k], acc);
      y[o] = acc;
    }
    float4* dst = reinterpret_cast<float4*>(y0 + (size_t)q * 32);
#pragma unroll
    for (int k = 0; k < 8; ++k) dst[k] = make_float4(y[4 * k], y[4 * k + 1], y[4 * k + 2], y[4 * k + 3]);
  }
  if (training) block_stats32<8>(y, active, stats, stats + 32, red);
}

// P3 (layer 0): x0max[p][c] = max over the pillar's points of relu(bn0(y0)) (pillar_encoder.py:39,43)
__global__ void pfn_max0_kernel(const float* __restrict__ y0, const int* __restrict__ bucket_off,
                                const int* __restrict__ counts, int cap_p, const float* __restrict__ scale,
                                const float* __restrict__ shift, float* __restrict__ x0max) {
  const int lane = pnx::lane_id();
  const int n_p = min(counts[0], cap_p);
  const float sc = scale[lane], sh = shift[lane];
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_p; p += (gridDim.x * blockDim.x) >> 5) {
    int lo = bucket_off[p], hi = bucket_off[p + 1];
    float m = 0.f;  // relu output >= 0 and every pillar has >= 1 point
    for (int q = lo; q < hi; ++q) m = fmaxf(m, fmaf(y0[(size_t)q * 32 + lane], sc, sh));
    x0max[(size_t)p * 32 + lane] = m;
  }
}

// P1 (layer 1): cat[relu(bn0(y0)), x0max[pillar]] (:46-50) -> Linear(64->64) (:37) + BN statistics.
__global__ void __launch_bounds__(256)
    pfn_lin1_kernel(const float* __restrict__ y0, const float* __restrict__ x0max,
                    const int* __restrict__ bucket_pts, const int* __restrict__ pillar_of_point,
                    const int* __restrict__ counts, int cap_n, const float* __restrict__ scale0,
                    const float* __restrict__ shift0, const float* __restrict__ w1, float* __restrict__ y1,
                    double* __restrict__ stats, int training) {
  __shared__ float4 sw[64 * 16];  // w1 [64 out][64 in]
  __shared__ float red[8][2][32];
  __shared__ float ssc[32], ssh[32];
  for (int k = threadIdx.x; k < 1024; k += 256) sw[k] = reinterpret_cast<const float4*>(w1)[k];
  if (threadIdx.x < 32) {
    ssc[threadIdx.x] = scale0[threadIdx.x];
    ssh[threadIdx.x] = shift0[threadIdx.x];
  }
  __syncthreads();
  const int nv = min(counts[1], cap_n);
  const int q = blockIdx.x * 256 + threadIdx.x;
  const bool active = q < nv;
  float in[64];
  if (active) {
    const int p = pillar_of_point[bucket_pts[q]];
    const float4* a = reinterpret_cast<const float4*>(y0 + (size_t)q * 32);
    const float4* b = reinterpret_cast<const float4*>(x0max + (size_t)p * 32);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float4 v = a[k];
      in[4 * k + 0] = fmaxf(fmaf(v.x, ssc[4 * k + 0], ssh[4 * k + 0]), 0.f);
      in[4 * k + 1] = fmaxf(fmaf(v.y, ssc[4 * k + 1], ssh[4 * k + 1]), 0.f);
      in[4 * k + 2] = fmaxf(fmaf(v.z, ssc[4 * k + 2], ssh[4 * k + 2]), 0.f);
      in[4 * k + 3] = fmaxf(fmaf(v.w, ssc[4 * k + 3], ssh[4 * k + 3]), 0.f);
      float4 m = b[k];
      in[32 + 4 * k + 0] = m.x; in[32 + 4 * k + 1] = m.y; in[32 + 4 * k + 2] = m.z; in[32 + 4 * k + 3] = m.w;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 64; ++k) in[k] = 0.f;
  }
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    float y[32];
#pragma unroll
    for (int o = 0; o < 32; ++o) {
      float acc = 0.f;
      const float4* wr = sw + (half * 32 + o) * 16;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        float4 w = wr[k];
        acc = fmaf(in[4 * k + 0], w.x, acc);
        acc = fmaf(in[4 * k + 1], w.y, acc);
        acc = fmaf(in[4 * k + 2], w.z, acc);
        acc = fmaf(in[4 * k + 3], w.w, acc);
      }
      y[o] = acc;
    }
    if (active) {
      float4* dst = reinterpret_cast<float4*>(y1 + (size_t)q * 64 + half * 32);
#pragma unroll
      for (int k = 0; k < 8; ++k) dst[k] = make_float4(y[4 * k], y[4 * k + 1], y[4 * k + 2], y[4 * k + 3]);
    }
    if (training) block_stats32<8>(y, active, stats + half * 32, stats + 64 + half * 32, red);
  }
}

// P3 (layer 1 + final scatter_max :180): feat[p][c] = max over bucket of relu(bn1(y1)); fp32 + bf16 copies
__global__ void pfn_max1_kernel(const float* __restrict__ y1, const int* __restrict__ bucket_off,
                                const int* __restrict__ counts, int cap_p, const float* __restrict__ scale,
                                const float* __restrict__ shift, float* __restrict__ feat_f32,
                                __nv_bfloat16* __restrict__ feat_bf16) {
  const int lane = pnx::lane_id();
  const int n_p = min(counts[0], cap_p);
  const float2 sc = reinterpret_cast<const float2*>(scale)[lane], sh = reinterpret_cast<const float2*>(shift)[lane];
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_p; p += (gridDim.x * blockDim.x) >> 5) {
    int lo = bucket_off[p], hi = bucket_off[p + 1];
    float m0 = 0.f, m1 = 0.f;
    for (int q = lo; q < hi; ++q) {
      float2 v = reinterpret_cast<const float2*>(y1 + (size_t)q * 64)[lane];
      m0 = fmaxf(m0, fmaf(v.x, sc.x, sh.x));
      m1 = fmaxf(m1, fmaf(v.y, sc.y, sh.y));
    }
    if (feat_f32) reinterpret_cast<float2*>(feat_f32 + (size_t)p * 64)[lane] = make_float2(m0, m1);
    if (feat_bf16)
      reinterpret_cast<__nv_bfloat162*>(feat_bf16 + (size_t)p * 64)[lane] = __floats2bfloat162_rn(m0, m1);
  }
}

}  // namespace

extern "C" int pnx_pfn_mean(const float* points, const int* bucket_off, const int* bucket_pts, const int* counts,
                            int cap_pillars, float* mean, cudaStream_t stream) {
  if (cap_pillars == 0) return PNX_OK;
  pfn_mean_kernel<<<pnx_cdiv(cap_pillars, 128), 128, 0, stream>>>(points, bucket_off, bucket_pts, counts,
                                                                 cap_pillars, mean);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_pfn_lin0(const float* points, const int* bucket_pts, const int* pillar_of_point,
                            const int* coords, const float* mean, const int* counts, int cap_points, float min_x,
                            float min_y, float vs_x, float vs_y, const float* w0, float* y0, double* stats,
                            int training, cudaStream_t stream) {
  if (cap_points == 0) return PNX_OK;
  PfnGeom g{min_x, min_y, vs_x, vs_y};
  pfn_lin0_kernel<<<pnx_cdiv(cap_points, 256), 256, 0, stream>>>(points, bucket_pts, pillar_of_point, coords, mean,
                                                                 counts, cap_points, g, w0, y0, stats, training);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_pfn_max0(const float* y0, const int* bucket_off, const int* counts, int cap_pillars,
                            const float* scale, const float* shift, float* x0max, cudaStream_t stream) {
  if (cap_pillars == 0) return PNX_OK;
  int blocks = min(pnx_cdiv((long long)cap_pillars * 32, 256), 148 * 8);
  pfn_max0_kernel<<<blocks, 256, 0, stream>>>(y0, bucket_off, counts, cap_pillars, scale, shift, x0max);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_pfn_lin1(const float* y0, const float* x0max, const int* bucket_pts, const int* pillar_of_point,
                            const int* counts, int cap_points, const float* scale0, const float* shift0,
                            const float* w1, float* y1, double* stats, int training, cudaStream_t stream) {
  if (cap_points == 0) return PNX_OK;
  pfn_lin1_kernel<<<pnx_cdiv(cap_points, 256), 256, 0, stream>>>(y0, x0max, bucket_pts, pillar_of_point, counts,
                                                                 cap_points, scale0, shift0, w1, y1, stats, training);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_pfn_max1(const float* y1, const int* bucket_off, const int* counts, int cap_pillars,
                            const float* scale, const float* shift, float* feat_f32, void* feat_bf16,
                            cudaStream_t stream) {
  if (cap_pillars == 0) return PNX_OK;
  int blocks = min(pnx_cdiv((long long)cap_pillars * 32, 256), 148 * 8);
  pfn_max1_kernel<<<blocks, 256, 0, stream>>>(y1, bucket_off, counts, cap_pillars, scale, shift, feat_f32,
                                              (__nv_bfloat16*)feat_bf16);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}
