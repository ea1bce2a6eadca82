// split.cu -- row-wise kernels of the fp32-grade ("split") precision mode.
//
// The reference computes the whole path in fp32 (no autocast anywhere: det3d/models/necks/aspp.py:19-32,
// heads/centerhead.py:128-136, utils/sparse_conv.py:31-39).  The production path stores activations as bf16; this
// mode stores every activation row as a PAIR of bf16 values (hi = bf16(v), lo = bf16(v - hi), ~16 mantissa bits,
// hi at column c and lo at column lo_off + c of the same row matrix) and runs the same wgmma kernels over the
// hi/lo segments (igemm.cu nseg, three wgrad launches), with raw convolution outputs, BatchNorm arithmetic and
// gradient accumulation in fp32.  It exists to show that the kernels reproduce the reference's numbers to the
// north-star tolerance (1e-3 abs on heat-maps / boxes); the kernels here are the row-wise glue of that mode:
//   fp32 rows <-> split rows, BatchNorm apply / backward (sparse_conv.py:33-39,55-63; conv.py:29-34,44-51),
//   add+ReLU and its backward.  The reductions are two-stage with a fixed order (bit-reproducible).
// One thread = 8 consecutive channels of one row.
#include "pnx_common.cuh"

namespace {

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float2 t = __bfloat1622float2(h[k]);
    f[2 * k] = t.x;
    f[2 * k + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pnx::pack_bf16x2(f[0], f[1]), pnx::pack_bf16x2(f[2], f[3]), pnx::pack_bf16x2(f[4], f[5]),
                    pnx::pack_bf16x2(f[6], f[7]));
}

struct Rows {  // a split row matrix: piece q of channel c at p[m*ld + q*lo + c], value = sum of the pieces
  __nv_bfloat16* p;
  long long ld, lo;
  int pieces;
};

__device__ __forceinline__ void load_split8(const Rows& r, long long m, int c0, float (&f)[8]) {
  // smallest piece first: the partial sums are exact in fp32 (pieces are non-overlapping 8-bit windows of one fp32)
  unpack8(*reinterpret_cast<const uint4*>(r.p + m * r.ld + (r.pieces - 1) * r.lo + c0), f);
  for (int q = r.pieces - 2; q >= 0; --q) {
    float g[8];
    unpack8(*reinterpret_cast<const uint4*>(r.p + m * r.ld + q * r.lo + c0), g);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] += g[k];
  }
}
__device__ __forceinline__ void store_split8(const Rows& r, long long m, int c0, const float (&f)[8]) {
  float rem[8], pc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) rem[k] = f[k];
  for (int q = 0; q < r.pieces; ++q) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      pc[k] = pnx::bf16_round(rem[k]);
      rem[k] -= pc[k];            // exact: the residual of a bf16 rounding is representable in fp32
    }
    *reinterpret_cast<uint4*>(r.p + m * r.ld + q * r.lo + c0) = pack8(pc);
  }
}
__device__ __forceinline__ void load_f32x8(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void store_f32x8(float* p, const float (&f)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}

#define PNX_ROW_LOOP(M, C)                                                              \
  const int cg = (C) >> 3;                                                              \
  const long long total = (long long)(M) * cg;                                          \
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;       \
       t += (long long)gridDim.x * blockDim.x)

__global__ void rows_split_kernel(const float* __restrict__ x, long long ldx, long long M, int C, Rows y) {
  PNX_ROW_LOOP(M, C) {
    const long long m = t / cg;
    const int c0 = (int)(t - m * cg) << 3;
    float f[8];
    load_f32x8(x + m * ldx + c0, f);
    store_split8(y, m, c0, f);
  }
}

__global__ void rows_merge_kernel(Rows x, long long M, int C, float* __restrict__ y, long long ldy, int accumulate) {
  PNX_ROW_LOOP(M, C) {
    const long long m = t / cg;
    const int c0 = (int)(t - m * cg) << 3;
    float f[8];
    load_split8(x, m, c0, f);
    if (accumulate) {
      float a[8];
      load_f32x8(y + m * ldy + c0, a);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] += a[k];
    }
    store_f32x8(y + m * ldy + c0, f);
  }
}

// y = relu?(x*scale + shift (+ res)); x fp32 raw conv output, res / y split rows
__global__ void bn_apply_split_kernel(const float* __restrict__ x, long long ldx, long long M, int C,
                                      const float* __restrict__ scale, const float* __restrict__ shift, Rows res,
                                      int relu, Rows y) {
  PNX_ROW_LOOP(M, C) {
    const long long m = t / cg;
    const int c0 = (int)(t - m * cg) << 3;
    float v[8], r[8];
    load_f32x8(x + m * ldx + c0, v);
    if (res.p) load_split8(res, m, c0, r);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float o = fmaf(v[k], scale[c0 + k], shift[c0 + k]);
      if (res.p) o += r[k];
      if (relu) o = fmaxf(o, 0.f);
      v[k] = o;
    }
    store_split8(y, m, c0, v);
  }
}

// BatchNorm backward, stage 1: per-block partial sums of g and g*xhat (g = dy masked by the ReLU gate).  The gate
// comes from y (residual layers) or is recomputed from x with the forward affine -- the same fmaf as the forward.
constexpr int kRedThreads = 256;
__global__ void __launch_bounds__(kRedThreads)
    bn_bwd_reduce_split_kernel(Rows dy, Rows y, const float* __restrict__ x, long long ldx, long long M, int C,
                               const float* __restrict__ mean, const float* __restrict__ invstd, int relu,
                               const float* __restrict__ fscale, const float* __restrict__ fshift,
                               double* __restrict__ part) {
  extern __shared__ float sred[];  // [kRedThreads][16]
  const int cg = C >> 3;
  const int my_cg = threadIdx.x % cg, my_row = threadIdx.x / cg;
  const int rpb = kRedThreads / cg;
  const int c0 = my_cg << 3;
  float sg[8], sgx[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) sg[k] = sgx[k] = 0.f;
  if (my_row < rpb) {
    for (long long m = (long long)blockIdx.x * rpb + my_row; m < M; m += (long long)gridDim.x * rpb) {
      float g[8], xx[8], yy[8];
      load_split8(dy, m, c0, g);
      load_f32x8(x + m * ldx + c0, xx);
      if (relu) {
        if (y.p) load_split8(y, m, c0, yy);
        else {
#pragma unroll
          for (int k = 0; k < 8; ++k) yy[k] = fmaf(xx[k], fscale[c0 + k], fshift[c0 + k]);
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float gg = (relu && !(yy[k] > 0.f)) ? 0.f : g[k];
        sg[k] += gg;
        sgx[k] += gg * (xx[k] - mean[c0 + k]) * invstd[c0 + k];
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    sred[threadIdx.x * 16 + k] = sg[k];
    sred[threadIdx.x * 16 + 8 + k] = sgx[k];
  }
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * C; j += kRedThreads) {
    const int which = j / C, c = j - which * C;
    const int g_ = c >> 3, k = c & 7;
    double acc = 0.0;
    for (int r = 0; r < rpb; ++r) acc += (double)sred[(r * cg + g_) * 16 + which * 8 + k];
    part[(size_t)blockIdx.x * 2 * C + j] = acc;
  }
}
// stage 2: fixed-order sum over the blocks
__global__ void reduce_parts_kernel(const double* __restrict__ part, int n_parts, int n, double* __restrict__ red) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  double acc = 0.0;
  for (int b = 0; b < n_parts; ++b) acc += part[(size_t)b * n + j];
  red[j] = acc;
}

// dx = gamma*invstd*(g - sum_g/n - xhat*sum_gx/n); optional dres = g (residual branch)
__global__ void bn_bwd_apply_split_kernel(Rows dy, Rows y, const float* __restrict__ x, long long ldx, long long M,
                                          int C, const float* __restrict__ mean, const float* __restrict__ invstd,
                                          const float* __restrict__ gamma, const double* __restrict__ red,
                                          double inv_n, int relu, const float* __restrict__ fscale,
                                          const float* __restrict__ fshift, Rows dx, Rows dres) {
  PNX_ROW_LOOP(M, C) {
    const long long m = t / cg;
    const int c0 = (int)(t - m * cg) << 3;
    float g[8], xx[8], yy[8], o[8];
    load_split8(dy, m, c0, g);
    load_f32x8(x + m * ldx + c0, xx);
    if (relu) {
      if (y.p) load_split8(y, m, c0, yy);
      else {
#pragma unroll
        for (int k = 0; k < 8; ++k) yy[k] = fmaf(xx[k], fscale[c0 + k], fshift[c0 + k]);
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = c0 + k;
      const float gg = (relu && !(yy[k] > 0.f)) ? 0.f : g[k];
      g[k] = gg;
      const float is = invstd[c];
      const float xh = (xx[k] - mean[c]) * is;
      o[k] = gamma[c] * is * (gg - (float)(red[c] * inv_n) - xh * (float)(red[C + c] * inv_n));
    }
    store_split8(dx, m, c0, o);
    if (dres.p) store_split8(dres, m, c0, g);
  }
}

__global__ void add_relu_split_kernel(Rows a, Rows b, long long M, int C, Rows y) {
  PNX_ROW_LOOP(M, C) {
    const long long m = t / cg;
    const int c0 = (int)(t - m * cg) << 3;
    float x[8], z[8];
    load_split8(a, m, c0, x);
    load_split8(b, m, c0, z);
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = fmaxf(x[k] + z[k], 0.f);
    store_split8(y, m, c0, x);
  }
}

// g = dy * (y > 0); dy fp32 rows, y / g split rows
__global__ void relu_bwd_split_kernel(const float* __restrict__ dy, long long lddy, Rows y, long long M, int C, Rows g) {
  PNX_ROW_LOOP(M, C) {
    const long long m = t / cg;
    const int c0 = (int)(t - m * cg) << 3;
    float d[8], yy[8];
    load_f32x8(dy + m * lddy + c0, d);
    load_split8(y, m, c0, yy);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = yy[k] > 0.f ? d[k] : 0.f;
    store_split8(g, m, c0, d);
  }
}

inline int ew_blocks(long long total) {
  long long b = (total + 255) / 256;
  const long long cap = 148LL * 16;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}
int g_pieces = 2;  // pieces per value of every split row matrix handled by this library instance (pnx_split_set_pieces)
inline Rows rows(const void* p, long long ld, long long lo) { return Rows{(__nv_bfloat16*)p, ld, lo, g_pieces}; }
inline bool rows_ok(const void* p, long long ld, long long lo, int C) {
  return !p || (ld % 8 == 0 && lo % 8 == 0 && lo >= C && (g_pieces - 1) * lo + C <= ld && (reinterpret_cast<uintptr_t>(p) & 15) == 0);
}
constexpr int kRedBlocks = 296;

}  // namespace

// Pieces per value (2 = hi+lo, 16 mantissa bits; 3 = hi+mid+lo, 24 bits) of the split row matrices handled by the
// pnx_*_split entry points and pnx_tap_scatter.  Process-wide setting of the parity mode; returns the previous value.
extern "C" int pnx_split_set_pieces(int pieces) {
  const int prev = g_pieces;
  if (pieces == 2 || pieces == 3) g_pieces = pieces;
  return prev;
}
extern "C" int pnx_split_get_pieces(void) { return g_pieces; }

extern "C" int pnx_rows_split(const float* x, long long ldx, long long M, int C, void* y, long long ldy, long long lo_y,
                              cudaStream_t stream) {
  PNX_CHECK_ARG(C % 8 == 0 && ldx % 4 == 0 && rows_ok(y, ldy, lo_y, C), "C % 8, ldx % 4, split rows layout");
  if (M == 0) return PNX_OK;
  rows_split_kernel<<<ew_blocks(M * (C / 8)), 256, 0, stream>>>(x, ldx, M, C, rows(y, ldy, lo_y));
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_rows_merge(const void* x, long long ldx, long long lo_x, long long M, int C, float* y, long long ldy,
                              int accumulate, cudaStream_t stream) {
  PNX_CHECK_ARG(C % 8 == 0 && ldy % 4 == 0 && rows_ok(x, ldx, lo_x, C), "C % 8, ldy % 4, split rows layout");
  if (M == 0) return PNX_OK;
  rows_merge_kernel<<<ew_blocks(M * (C / 8)), 256, 0, stream>>>(rows(x, ldx, lo_x), M, C, y, ldy, accumulate);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_bn_apply_split(const float* x, long long ldx, long long M, int C, const float* scale,
                                  const float* shift, const void* res, long long ldr, long long lo_r, int relu, void* y,
                                  long long ldy, long long lo_y, cudaStream_t stream) {
  PNX_CHECK_ARG(C % 8 == 0 && ldx % 4 == 0 && rows_ok(res, ldr, lo_r, C) && rows_ok(y, ldy, lo_y, C), "layout");
  if (M == 0) return PNX_OK;
  bn_apply_split_kernel<<<ew_blocks(M * (C / 8)), 256, 0, stream>>>(x, ldx, M, C, scale, shift, rows(res, ldr, lo_r), relu,
                                                                   rows(y, ldy, lo_y));
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

// number of doubles of the `part` scratch of pnx_bn_bwd_reduce_split
extern "C" long long pnx_bn_bwd_reduce_split_scratch(int C) { return (long long)kRedBlocks * 2 * C; }

extern "C" int pnx_bn_bwd_reduce_split(const void* dy, long long lddy, long long lo_dy, const void* y, long long ldy,
                                       long long lo_y, const float* x, long long ldx, long long M, int C,
                                       const float* mean, const float* invstd, int relu, const float* fscale,
                                       const float* fshift, double* part, double* red, cudaStream_t stream) {
  PNX_CHECK_ARG(!relu || y || (fscale && fshift), "relu backward needs y or the forward affine (scale, shift)");
  PNX_CHECK_ARG(C % 8 == 0 && C <= 2048 && ldx % 4 == 0 && rows_ok(dy, lddy, lo_dy, C) && rows_ok(y, ldy, lo_y, C), "layout");
  int nb = kRedBlocks;
  const int rpb = kRedThreads / (C / 8);
  if ((long long)nb * rpb > M) nb = (int)((M + rpb - 1) / rpb);
  if (nb < 1) nb = 1;
  bn_bwd_reduce_split_kernel<<<nb, kRedThreads, kRedThreads * 16 * sizeof(float), stream>>>(
      rows(dy, lddy, lo_dy), rows(y, ldy, lo_y), x, ldx, M, C, mean, invstd, relu, fscale, fshift, part);
  PNX_CHECK_LAUNCH();
  reduce_parts_kernel<<<pnx_cdiv(2 * C, 128), 128, 0, stream>>>(part, nb, 2 * C, red);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_bn_bwd_apply_split(const void* dy, long long lddy, long long lo_dy, const void* y, long long ldy,
                                      long long lo_y, const float* x, long long ldx, long long M, int C,
                                      const float* mean, const float* invstd, const float* gamma, const double* red,
                                      double count, int relu, const float* fscale, const float* fshift, void* dx,
                                      long long lddx, long long lo_dx, void* dres, long long lddres, long long lo_dres,
                                      cudaStream_t stream) {
  PNX_CHECK_ARG(!relu || y || (fscale && fshift), "relu backward needs y or the forward affine (scale, shift)");
  PNX_CHECK_ARG(C % 8 == 0 && ldx % 4 == 0 && rows_ok(dy, lddy, lo_dy, C) && rows_ok(y, ldy, lo_y, C) &&
                    rows_ok(dx, lddx, lo_dx, C) && rows_ok(dres, lddres, lo_dres, C), "layout");
  if (M == 0) return PNX_OK;
  bn_bwd_apply_split_kernel<<<ew_blocks(M * (C / 8)), 256, 0, stream>>>(
      rows(dy, lddy, lo_dy), rows(y, ldy, lo_y), x, ldx, M, C, mean, invstd, gamma, red, 1.0 / count, relu, fscale, fshift,
      rows(dx, lddx, lo_dx), rows(dres, lddres, lo_dres));
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_add_relu_split(const void* a, long long lda, long long lo_a, const void* b, long long ldb,
                                  long long lo_b, long long M, int C, void* y, long long ldy, long long lo_y,
                                  cudaStream_t stream) {
  PNX_CHECK_ARG(C % 8 == 0 && rows_ok(a, lda, lo_a, C) && rows_ok(b, ldb, lo_b, C) && rows_ok(y, ldy, lo_y, C), "layout");
  if (M == 0) return PNX_OK;
  add_relu_split_kernel<<<ew_blocks(M * (C / 8)), 256, 0, stream>>>(rows(a, lda, lo_a), rows(b, ldb, lo_b), M, C,
                                                                   rows(y, ldy, lo_y));
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" int pnx_relu_bwd_split(const float* dy, long long lddy, const void* y, long long ldy, long long lo_y,
                                  long long M, int C, void* g, long long ldg, long long lo_g, cudaStream_t stream) {
  PNX_CHECK_ARG(C % 8 == 0 && lddy % 4 == 0 && rows_ok(y, ldy, lo_y, C) && rows_ok(g, ldg, lo_g, C), "layout");
  if (M == 0) return PNX_OK;
  relu_bwd_split_kernel<<<ew_blocks(M * (C / 8)), 256, 0, stream>>>(dy, lddy, rows(y, ldy, lo_y), M, C, rows(g, ldg, lo_g));
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}
