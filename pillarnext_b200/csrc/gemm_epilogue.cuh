// gemm_epilogue.cuh -- epilogue of igemm.cu / igemm_win.cu on the wgmma accumulator fragment: bias, addend, ReLU, bf16 or
// fp32 store (pixel-shuffled for ConvTranspose2d k2s2), BatchNorm statistics of the stored values.  F: 0 bf16 output,
// 1 + fused BatchNorm-backward reduce (dy of y = relu(bn(raw)): stores g = dy * gate, sums g and g * xhat), 2 fp32 paths.
#pragma once
#include "pnx_common.cuh"

namespace pnx {

struct EpiParams {
  void* out;
  long long ldc;
  int has_bias, relu;
  const __nv_bfloat16* addend;  // optional, added before the store
  const float* addend_f32;      // F = 2
  long long ld_add;
  double* stats;                // [2 * stats_C] sums / sums of squares, channel = column % stats_mod
  int stats_C, stats_mod;
  int stats_direct;             // deterministic mode: per-warp partials straight into fp64
  int shuffle, Hout, Wout;      // ConvTranspose2d k2s2: column q * 64 + c -> pixel (2y + q/2, 2x + q%2), channel c
  const __nv_bfloat16* bnr_raw; // F = 1
  long long bnr_ld;
};

// consumer warps per CTA; each keeps its own shared-memory sums (fp32 shared atomics are CAS loops that serialise)
constexpr int kEpiWarps = 8;

// acc: rows [64 * half, +64) of the tile; tile row r < nvalid is output row row_base + r.  s_stat: [kEpiWarps][2 * BN],
// s_bnc (F = 1): scale, shift, mean, invstd of the CTA's BN columns.
template <int BN, int F>
__device__ __forceinline__ void gemm_epilogue(const float (&acc)[BN / 2], const EpiParams& e, long long row_base, int nvalid,
                                              int half, int n0, const float* s_bias, float* s_stat, const float* s_bnc) {
  const int lane = threadIdx.x & 31;
  const int lr0 = half * 64 + 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2);
  float* s_mine = s_stat + (half * 4 + ((threadIdx.x >> 5) & 3)) * 2 * BN;  // this warp's slice: lanes 0-3 own distinct columns
  bool act[2];
  long long mrow[2], sh_base[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int lr = lr0 + 8 * h;
    act[h] = lr < nvalid;
    mrow[h] = row_base + lr;
    sh_base[h] = 0;
    if (e.shuffle && act[h]) {
      const int hw = e.Hout * e.Wout;
      const int b = (int)(mrow[h] / hw), rem = (int)(mrow[h] - (long long)b * hw);
      const int y = rem / e.Wout, x = rem - y * e.Wout;
      sh_base[h] = ((long long)(b * 2 * e.Hout + 2 * y)) * (2 * e.Wout) + 2 * x;
    }
  }
  const bool want_stats = F == 1 || e.stats != nullptr;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = 8 * j + 2 * (lane & 3);  // this thread's column pair (c, c + 1) inside the CTA's column block
    const int gc = n0 + c;
    float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (e.has_bias) { v0 += s_bias[c]; v1 += s_bias[c + 1]; }
      if (act[h]) {
        if (e.addend) {
          const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(e.addend + mrow[h] * e.ld_add + gc));
          v0 += a.x; v1 += a.y;
        }
        if (F == 2 && e.addend_f32) {
          const float2 a = *reinterpret_cast<const float2*>(e.addend_f32 + mrow[h] * e.ld_add + gc);
          v0 += a.x; v1 += a.y;
        }
      }
      if (e.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      long long orow = mrow[h];
      int ocol = gc;
      if (e.shuffle) {
        const int q = gc >> 6;
        orow = sh_base[h] + (long long)(q >> 1) * (2 * e.Wout) + (q & 1);
        ocol = gc & 63;
      }
      if (F == 2) {
        if (act[h]) {
          *reinterpret_cast<float2*>(reinterpret_cast<float*>(e.out) + orow * e.ldc + ocol) = make_float2(v0, v1);
          s0 += v0; s1 += v1;
          q0 = fmaf(v0, v0, q0); q1 = fmaf(v1, v1, q1);
        }
      } else {
        const __nv_bfloat162 pk = __floats2bfloat162_rn(v0, v1);
        float2 r = __bfloat1622float2(pk);  // the stored values: the statistics are of these
        if (F == 1) {
          if (act[h]) {
            const float2 raw = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(e.bnr_raw + mrow[h] * e.bnr_ld + gc));
            const float g0 = fmaf(raw.x, s_bnc[c], s_bnc[BN + c]) > 0.f ? r.x : 0.f;
            const float g1 = fmaf(raw.y, s_bnc[c + 1], s_bnc[BN + c + 1]) > 0.f ? r.y : 0.f;
            *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(e.out) + orow * e.ldc + ocol) =
                __floats2bfloat162_rn(g0, g1);
            s0 += g0; s1 += g1;
            q0 = fmaf(g0, (raw.x - s_bnc[2 * BN + c]) * s_bnc[3 * BN + c], q0);
            q1 = fmaf(g1, (raw.y - s_bnc[2 * BN + c + 1]) * s_bnc[3 * BN + c + 1], q1);
          }
        } else if (act[h]) {
          *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(e.out) + orow * e.ldc + ocol) = pk;
          s0 += r.x; s1 += r.y;
          q0 = fmaf(r.x, r.x, q0); q1 = fmaf(r.y, r.y, q1);
        }
      }
    }
    if (want_stats) {
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, off);
        s1 += __shfl_xor_sync(0xffffffffu, s1, off);
        q0 += __shfl_xor_sync(0xffffffffu, q0, off);
        q1 += __shfl_xor_sync(0xffffffffu, q1, off);
      }
      if (lane < 4) {
        if (F != 1 && (F == 2 || e.stats_direct)) {  // order-insensitive fp64 accumulation (see pnx_set_deterministic)
          const int ch0 = gc % e.stats_mod, ch1 = (gc + 1) % e.stats_mod;
          atomicAdd(&e.stats[ch0], (double)s0); atomicAdd(&e.stats[ch1], (double)s1);
          atomicAdd(&e.stats[e.stats_C + ch0], (double)q0); atomicAdd(&e.stats[e.stats_C + ch1], (double)q1);
        } else {
          s_mine[c] += s0; s_mine[c + 1] += s1;
          s_mine[BN + c] += q0; s_mine[BN + c + 1] += q1;
        }
      }
    }
  }
}

// after the last tile and a barrier of the consumer threads: per-warp sums, added in warp order, into the fp64 accumulators
template <int BN, int F>
__device__ __forceinline__ void gemm_epilogue_flush(const EpiParams& e, int n0, const float* s_stat, double* bnr_red, int bnr_C,
                                                    int tid, int nthreads) {
  const bool smem_sums = F == 1 || (F == 0 && e.stats && !e.stats_direct);
  if (!smem_sums) return;
  double* dst = F == 1 ? bnr_red : e.stats;
  const int dst_C = F == 1 ? bnr_C : e.stats_C;
  for (int c = tid; c < 2 * BN; c += nthreads) {
    const int col = c < BN ? c : c - BN;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kEpiWarps; ++w) v += s_stat[w * 2 * BN + c];
    const int ch = F == 1 ? n0 + col : (n0 + col) % e.stats_mod;
    atomicAdd(&dst[(c < BN ? 0 : dst_C) + ch], (double)v);
  }
}

}  // namespace pnx
