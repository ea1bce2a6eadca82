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

// ------------------------------------------------------------------ staged epilogue
// The consumer warpgroups only write the tile (bf16, or fp32 for F = 2) into a shared staging buffer and go straight back
// to their MMAs; store warps drain it while the next tile's mainloop runs: the BatchNorm statistics (or, F = 1, the
// BN-backward gate and its sums) and coalesced 16-byte row stores.  A tile is staged in P passes of BN / P columns when
// one buffer for the whole tile would leave too few pipeline stages.  igemm's fp32 output at BN = 192 and 256 (the split
// mode) keeps the in-register epilogue above.
template <int BN, int P, int kElem = 2>  // kElem: bytes per staged value (2 bf16, 4 fp32)
struct Staging {
  static_assert(BN % P == 0 && (BN / P) % 8 == 0, "staging pass width");
  static constexpr int kCols = BN / P;
  static constexpr int kPitch = kElem * kCols + 16;  // bytes per staged row; the pad keeps the fragment stores conflict-free
  static constexpr int kBytes = 128 * kPitch;
};
template <int BN, int P, int F>
using StagingF = Staging<BN, P, F == 2 ? 4 : 2>;

// consumer half: rows [64 * half, +64) of the tile, relu(acc + bias + addend) into the staging buffer (bf16; F = 2: fp32,
// the same sum as the in-register epilogue's), pass by pass.  `staged` counts the 256 consumer threads; `sfree` is released
// by the store warps; spass counts passes over all tiles.
template <int BN, int P, int F = 0>
__device__ __forceinline__ void gemm_epilogue_stage(const float (&acc)[BN / 2], const EpiParams& e, long long row_base, int nvalid,
                                                    int half, int n0, const float* s_bias, uint8_t* stg, uint64_t* staged,
                                                    uint64_t* sfree, uint32_t& spass) {
  using S = StagingF<BN, P, F>;
  const int lane = threadIdx.x & 31;
  const int lr0 = half * 64 + 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2);
#pragma unroll
  for (int pp = 0; pp < P; ++pp) {
    mbar_wait(sfree, (spass & 1) ^ 1);
#pragma unroll
    for (int jj = 0; jj < S::kCols / 8; ++jj) {
      const int j = pp * (S::kCols / 8) + jj;
      const int c = 8 * j + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int lr = lr0 + 8 * h;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (e.has_bias) { v0 += s_bias[c]; v1 += s_bias[c + 1]; }
        if (e.addend && lr < nvalid) {
          const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(e.addend + (row_base + lr) * e.ld_add + n0 + c));
          v0 += a.x; v1 += a.y;
        }
        if (F == 2 && e.addend_f32 && lr < nvalid) {
          const float2 a = *reinterpret_cast<const float2*>(e.addend_f32 + (row_base + lr) * e.ld_add + n0 + c);
          v0 += a.x; v1 += a.y;
        }
        if (e.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        if constexpr (F == 2)
          *reinterpret_cast<float2*>(stg + lr * S::kPitch + (c - pp * S::kCols) * 4) = make_float2(v0, v1);
        else
          *reinterpret_cast<__nv_bfloat162*>(stg + lr * S::kPitch + (c - pp * S::kCols) * 2) = __floats2bfloat162_rn(v0, v1);
      }
    }
    mbar_arrive(staged);
    ++spass;
  }
}

// store half, run by `nthreads` threads (a multiple of 32, named barrier `bar_id`) for every tile the consumers stage.
// The statistics of warp slot w (rows 16w .. 16w + 15) are summed exactly as the in-register epilogue sums them: the pair
// of rows (g, g + 8), then ((t0 + t1) + (t2 + t3)) + ((t4 + t5) + (t6 + t7)) over the 8 row groups g, then into
// s_stat[w] in tile order -- so the statistics are bit-identical to it.  kRegStats (one pass, nthreads = BN / 2): thread
// tid always owns column pair tid, so its 8 slots live in r_stat[w] instead of shared memory, with the same additions.
// F = 2 adds each slot's sums straight into the fp64 statistics, as the in-register epilogue does.
template <int BN, int F, int P, bool kRegStats = false>
__device__ __forceinline__ void gemm_epilogue_drain(const EpiParams& e, long long row_base, int nvalid, int n0, uint8_t* stg,
                                                    float* s_stat, const float* s_bnc, uint64_t* staged, uint64_t* sfree,
                                                    uint32_t& spass, int tid, int nthreads, int bar_id, float4* r_stat = nullptr) {
  using S = StagingF<BN, P, F>;
  constexpr int kElem = F == 2 ? 4 : 2;
  constexpr int kPairs = S::kCols / 2, kChunks = S::kCols * kElem / 16;
  static_assert(!kRegStats || (P == 1 && F != 2), "register statistics: one pass, bf16 output");
  const bool want_stats = F == 1 || e.stats != nullptr;
  if constexpr (F == 1) {  // raw does not depend on the MMAs: pull the tile's rows into L2 while the consumers still compute it
    constexpr int kLines = BN / 64;  // 128-byte lines per row
    for (int i = tid; i < nvalid * kLines; i += nthreads) {
      const int r = i / kLines, l = i - r * kLines;
      asm volatile("prefetch.global.L2 [%0];" ::"l"(e.bnr_raw + (row_base + r) * e.bnr_ld + n0 + 64 * l));
    }
  }
  for (int pp = 0; pp < P; ++pp) {
    mbar_wait(staged, spass & 1);
    if (want_stats) {
      auto item = [&](int w, int pr) {
        const int c = pp * S::kCols + 2 * pr;  // column pair (c, c + 1) inside the CTA's column block
        const int gc = n0 + c;
        // F = 1: the raw pairs of row groups [g0, g0 + 4), both halves, loaded together ahead of their use
        uint32_t raw2[8];
        auto load_raw = [&](int g0) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int lr = 16 * w + g0 + (i & 3) + 8 * (i >> 2);
            raw2[i] = lr < nvalid ? __ldg(reinterpret_cast<const unsigned int*>(e.bnr_raw + (row_base + lr) * e.bnr_ld + gc)) : 0u;
          }
        };
        // sums over the rows (16w + g, 16w + g + 8) of the column pair: s0, s1, q0, q1
        auto rows = [&](int g) {
          float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int lr = 16 * w + g + 8 * h;
            if (lr < nvalid) {
              uint8_t* sp = stg + lr * S::kPitch + 2 * kElem * pr;
              const float2 r = F == 2 ? *reinterpret_cast<const float2*>(sp) : __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(sp));
              if (F == 1) {
                const float2 raw = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw2[(g & 3) + 4 * h]));
                const float g0 = fmaf(raw.x, s_bnc[c], s_bnc[BN + c]) > 0.f ? r.x : 0.f;
                const float g1 = fmaf(raw.y, s_bnc[c + 1], s_bnc[BN + c + 1]) > 0.f ? r.y : 0.f;
                *reinterpret_cast<__nv_bfloat162*>(sp) = __floats2bfloat162_rn(g0, g1);
                t.x += g0; t.y += g1;
                t.z = fmaf(g0, (raw.x - s_bnc[2 * BN + c]) * s_bnc[3 * BN + c], t.z);
                t.w = fmaf(g1, (raw.y - s_bnc[2 * BN + c + 1]) * s_bnc[3 * BN + c + 1], t.w);
              } else {
                t.x += r.x; t.y += r.y;
                t.z = fmaf(r.x, r.x, t.z); t.w = fmaf(r.y, r.y, t.w);
              }
            }
          }
          return t;
        };
        auto add = [](float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); };
        if (F == 1) load_raw(0);
        float4 lo = add(rows(0), rows(1));
        lo = add(lo, add(rows(2), rows(3)));
        if (F == 1) load_raw(4);
        float4 hi = add(rows(4), rows(5));
        hi = add(hi, add(rows(6), rows(7)));
        const float4 s = add(lo, hi);
        if (F == 2 || (F == 0 && e.stats_direct)) {  // order-insensitive fp64 accumulation (see pnx_set_deterministic)
          const int ch0 = gc % e.stats_mod, ch1 = (gc + 1) % e.stats_mod;
          atomicAdd(&e.stats[ch0], (double)s.x); atomicAdd(&e.stats[ch1], (double)s.y);
          atomicAdd(&e.stats[e.stats_C + ch0], (double)s.z); atomicAdd(&e.stats[e.stats_C + ch1], (double)s.w);
        } else if constexpr (kRegStats) {
          r_stat[w] = add(r_stat[w], s);
        } else {
          float* s_mine = s_stat + w * 2 * BN;
          s_mine[c] += s.x; s_mine[c + 1] += s.y;
          s_mine[BN + c] += s.z; s_mine[BN + c + 1] += s.w;
        }
      };
      if constexpr (kRegStats) {
#pragma unroll
        for (int w = 0; w < kEpiWarps; ++w) item(w, tid);
      } else {
        for (int it = tid; it < 8 * kPairs; it += nthreads) {
          const int w = it / kPairs;
          item(w, it - w * kPairs);
        }
      }
      if (F == 1) asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(nthreads) : "memory");  // the gated values are staged
    }
    for (int idx = tid; idx < 128 * kChunks; idx += nthreads) {
      const int r = idx / kChunks, ch = idx - r * kChunks;
      if (r >= nvalid) break;
      const uint4 v = *reinterpret_cast<const uint4*>(stg + r * S::kPitch + ch * 16);
      const int gc = n0 + pp * S::kCols + ch * (16 / kElem);
      long long orow = row_base + r;
      int ocol = gc;
      if (e.shuffle) {
        const int hw = e.Hout * e.Wout;
        const int b = (int)(orow / hw), rem = (int)(orow - (long long)b * hw);
        const int y = rem / e.Wout, x = rem - y * e.Wout;
        const int q = gc >> 6;
        orow = ((long long)(b * 2 * e.Hout + 2 * y)) * (2 * e.Wout) + 2 * x + (long long)(q >> 1) * (2 * e.Wout) + (q & 1);
        ocol = gc & 63;
      }
      *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(e.out) + (orow * e.ldc + ocol) * kElem) = v;
    }
    mbar_arrive(sfree);
    ++spass;
  }
}

// after the last tile and a barrier of the threads that own s_stat: per-warp sums, added in warp order, into the fp64
// accumulators
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

// the same for a kRegStats drain, after its last tile: thread tid adds its slots of column pair tid in warp order
template <int BN, int F>
__device__ __forceinline__ void gemm_epilogue_flush_regs(const EpiParams& e, int n0, const float4* r_stat, double* bnr_red,
                                                         int bnr_C, int tid) {
  const bool slot_sums = F == 1 || (F == 0 && e.stats && !e.stats_direct);
  if (!slot_sums) return;
  double* dst = F == 1 ? bnr_red : e.stats;
  const int dst_C = F == 1 ? bnr_C : e.stats_C;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int w = 0; w < kEpiWarps; ++w) {
    v.x += r_stat[w].x; v.y += r_stat[w].y; v.z += r_stat[w].z; v.w += r_stat[w].w;
  }
  const int c = n0 + 2 * tid;
  const int ch0 = F == 1 ? c : c % e.stats_mod, ch1 = F == 1 ? c + 1 : (c + 1) % e.stats_mod;
  atomicAdd(&dst[ch0], (double)v.x); atomicAdd(&dst[ch1], (double)v.y);
  atomicAdd(&dst[dst_C + ch0], (double)v.z); atomicAdd(&dst[dst_C + ch1], (double)v.w);
}

}  // namespace pnx
