// wgrad.cu -- weight-gradient of every convolution on the path as a wgmma GEMM over rows (sm_90a).
//
//   dW[t, x, y] += sum_m  X[m, x] * Y[g(m,t), y]          fp32, accumulated with red.global.add
// X is the DIRECT operand (read at row m), Y the GATHERED one (read through the neighbour table / the dense
// geometry at tap t).  For a convolution X = output gradient, Y = layer input; for ConvTranspose2d k2s2 the
// roles swap (X = input, Y = output gradient at the pixel-shuffled position).
// Both operands are MN-major for the MMA (the reduction index K = row m is the slow one in memory):
// tiles are staged as [64 rows x 128 B] blocks per 64-channel group with the 128-byte swizzle and
// described to wgmma as transposed operands (LBO = block stride, SBO = 8-row group stride).
// One CTA owns a 128-channel block of X, an NYC-channel chunk of Y and a GROUP of up to TG taps: the X tile of a
// 64-row chunk is staged ONCE and multiplied against the gathered Y tile of every tap of the group, so the direct
// operand is not re-read per tap (NYC * TG <= 256 register accumulator columns).
// Grid = (x blocks * y chunks, tap groups, K splits), two full waves of one CTA per SM.  Warpgroup 0: X by TMA, Y rows by
// cp.async through a (tap, row) table; warpgroups 1-2: wgmma, then red.global.add (or a split's slab) from registers.
// This is the backward of: spconv SparseConv2d/SubMConv2d (reference sparse_conv.py:25-29,50-51),
// nn.Conv2d/F.conv2d (aspp.py:19-32, conv.py:9-10, centerhead.py:35-46,108-114), nn.ConvTranspose2d
// (centerhead.py:26-27) -- autograd derives these in the reference (trainer.py:94-108 loss.backward()).
#include "pnx_common.cuh"

namespace {

struct WgradParams {
  const __nv_bfloat16* X;
  const __nv_bfloat16* Y;
  long long ldx, ldy;
  int M, T;
  const int* nbr;  // [M, T] or null
  int gathered;    // 0: Y read at row m (taps == 1)
  int Hout, Wout, Hin, Win, kw, mul, dil, pad;
  int shuffle;     // ConvTranspose k2s2: tap q selects pixel (2y+q/2, 2x+q%2) of the gathered operand
  float* dW;       // [T, X_total, Y_total]
  float* partials; // deterministic mode: [splits][T, X_total, Y_total], plain stores, reduced in split order afterwards
  int X_total, Y_total;
  int x_dup;       // X has only 64 channels: the second consumer warpgroup has no X channels
  int y_chunks;    // Y_total / NYC
  int taps_per_group;
  int rows_per_split;
};

constexpr int kThreads = 384;         // producer warpgroup + two consumer warpgroups
constexpr int kKS = 64;               // rows (K) per stage
constexpr uint32_t kBlk = kKS * 128;  // bytes of one [64 rows x 64 ch] block

// NYC = Y channels per CTA (64..256), TG = max taps per group (NYC * TG <= 256 accumulator columns)
template <int NYC, int TG>
struct WCfg {
  static constexpr int kYAtoms = NYC / 64;
  static constexpr uint32_t kStageBytes = (2 + TG * kYAtoms) * kBlk;
  static constexpr int kStagesRaw = (200 * 1024) / (int)kStageBytes;
  static constexpr int kStages = kStagesRaw > 6 ? 6 : kStagesRaw;
  static constexpr size_t kSmem = 1024 + (size_t)kStages * kStageBytes + 256 + (size_t)TG * kKS * 4;
  static_assert(NYC * TG <= 256, "register accumulator budget");
  static_assert(kStages >= 2, "need at least two stages");
  static_assert(kSmem <= 227 * 1024, "shared memory budget");
};

template <int NYC, int TG>
__global__ void __launch_bounds__(kThreads, 1) wgrad_kernel(const __grid_constant__ CUtensorMap xmap, WgradParams p) {
  using C = WCfg<NYC, TG>;
  constexpr int kStages = C::kStages, kYAtoms = C::kYAtoms;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)kStages * C::kStageBytes);
  uint64_t* empty = full + kStages;
  int* s_idx = reinterpret_cast<int*>(smem + (size_t)kStages * C::kStageBytes + 256);  // [TG][kKS] gathered row (-1 = absent)

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int xb = blockIdx.x / p.y_chunks, yc = blockIdx.x - xb * p.y_chunks;
  const int t0 = blockIdx.y * p.taps_per_group;
  const int ntaps = min(p.taps_per_group, p.T - t0);
  const int split = blockIdx.z;
  const int m_begin = split * p.rows_per_split;
  const int m_end = min(p.M, m_begin + p.rows_per_split);
  const int num_k = (m_end - m_begin + kKS - 1) / kKS;

  if (threadIdx.x == 0) {
    pnx::tma_prefetch_desc(&xmap);
    for (int s = 0; s < kStages; ++s) {
      pnx::mbar_init(&full[s], 1 + 128);  // X tiles (expect_tx) + the 128 gathering threads (cp.async arrive)
      pnx::mbar_init(&empty[s], 8);       // one arrival per consumer warp
    }
    pnx::fence_barrier_init();
  }
  __syncthreads();
  if (num_k <= 0) return;

  if (wg == 0) {
    // ---------------------------------------------------------------- producer
    pnx::regs_dealloc<56>();
    const int ptid = threadIdx.x;
    const int y_ch0 = yc * NYC;
    const int nchunks = ntaps * kYAtoms * kKS * 8;  // 16-byte copies of Y per stage
    const int nblk = p.x_dup ? 1 : 2;
    const int hw = p.Hout * p.Wout;
    int stage = 0;
    uint32_t phase = 0;
    for (int kc = 0; kc < num_k; ++kc) {
      const int mb = m_begin + kc * kKS;
      // gathered row of (tap j, row r) for e = j * 64 + r
      int val[(TG * kKS + 127) / 128];
#pragma unroll
      for (int n = 0; n < (TG * kKS + 127) / 128; ++n) {
        const int e = n * 128 + ptid, j = e >> 6, m = mb + (e & (kKS - 1));
        int g = -1;
        if (j < ntaps && m < m_end) {
          const int t = t0 + j;
          if (!p.gathered) {
            g = m;
          } else if (p.nbr) {
            g = p.nbr[(size_t)m * p.T + t];
          } else {
            const int b = m / hw, rem = m - b * hw, y = rem / p.Wout, x = rem - y * p.Wout;
            if (p.shuffle) {
              g = (b * 2 * p.Hout + 2 * y + (t >> 1)) * (2 * p.Wout) + 2 * x + (t & 1);
            } else {
              const int rr = t / p.kw, ss = t - rr * p.kw;
              const int yi = y * p.mul + rr * p.dil - p.pad, xi = x * p.mul + ss * p.dil - p.pad;
              g = (yi >= 0 && yi < p.Hin && xi >= 0 && xi < p.Win) ? (b * p.Hin + yi) * p.Win + xi : -1;
            }
          }
        }
        val[n] = g;
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");  // the previous chunk's table has been read
#pragma unroll
      for (int n = 0; n < (TG * kKS + 127) / 128; ++n)
        if (n * 128 + ptid < TG * kKS) s_idx[n * 128 + ptid] = val[n];
      asm volatile("bar.sync 1, 128;" ::: "memory");
      pnx::mbar_wait(&empty[stage], phase ^ 1);
      uint8_t* st = smem + (size_t)stage * C::kStageBytes;
      if (ptid == 0) {
        // X: plain 2-D TMA boxes of [64 rows x 64 channels] (rows past M are zero-filled by the tensor map bounds)
        pnx::mbar_arrive_expect_tx(&full[stage], (uint32_t)nblk * kBlk);
        for (int b2 = 0; b2 < nblk; ++b2) pnx::tma_load_2d(&xmap, &full[stage], st + b2 * kBlk, xb * 128 + b2 * 64, mb);
      }
      const uint32_t sy = pnx::smem_u32(st) + 2 * kBlk;
      for (int c = ptid; c < nchunks; c += 128) {  // a warp instruction copies 4 whole 128-byte rows
        const int sub = c & 7, row = (c >> 3) & (kKS - 1), blk = c >> 9;  // blk = tap * kYAtoms + atom
        const int tap = blk / kYAtoms, atom = blk - tap * kYAtoms;
        const int g = s_idx[tap * kKS + row];
        const __nv_bfloat16* src = p.Y + (long long)(g < 0 ? 0 : g) * p.ldy + y_ch0 + atom * 64 + sub * 8;
        pnx::cp_async_16(sy + blk * kBlk + pnx::sw128_offset(row, sub), src, g < 0 ? 0u : 16u);
      }
      pnx::cp_async_mbar_arrive(&full[stage]);
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
  } else {
    // ---------------------------------------------------------------- consumers: X channels [64 * half, +64) of the block
    pnx::regs_alloc<224>();
    const int half = wg - 1;
    const bool mine = !(p.x_dup && half == 1);
    float acc[TG][NYC / 2];
#pragma unroll
    for (int j = 0; j < TG; ++j)
#pragma unroll
      for (int i = 0; i < NYC / 2; ++i) acc[j][i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kc = 0; kc < num_k; ++kc) {
      pnx::mbar_wait(&full[stage], phase);
      pnx::fence_proxy_async_smem();  // the cp.async rows were written through the generic proxy; wgmma reads async
      if (mine) {
        pnx::wgmma_fence();
#pragma unroll
        for (int j = 0; j < TG; ++j) pnx::fence_acc(acc[j]);
        const uint32_t sx = pnx::smem_u32(smem + (size_t)stage * C::kStageBytes) + half * kBlk;
        const uint32_t sy = pnx::smem_u32(smem + (size_t)stage * C::kStageBytes) + 2 * kBlk;
#pragma unroll
        for (int k = 0; k < kKS / 16; ++k) {
          const uint64_t dx = pnx::make_smem_desc_sw128(sx + k * 2048, kBlk, 1024);
#pragma unroll
          for (int j = 0; j < TG; ++j)
            if (j < ntaps)
              pnx::Wgmma<NYC, 1, 1>::mma(acc[j], dx, pnx::make_smem_desc_sw128(sy + j * kYAtoms * kBlk + k * 2048, kBlk, 1024),
                                         (kc > 0 || k > 0) ? 1u : 0u);
        }
        pnx::wgmma_commit();
        pnx::wgmma_wait<1>();
      }
      if (kc > 0 && lane == 0) pnx::mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    if (!mine) return;
    pnx::wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < TG; ++j) pnx::fence_acc(acc[j]);
    // ---------------------------------------------------------------- epilogue: registers -> red.global.add
    float* out = p.partials ? p.partials + (size_t)blockIdx.z * ((size_t)p.T * p.X_total * p.Y_total) : p.dW;
#pragma unroll
    for (int j = 0; j < TG; ++j) {
      if (j >= ntaps) break;
#pragma unroll
      for (int i = 0; i < NYC / 2; i += 2) {
        const int xch = xb * 128 + half * 64 + pnx::acc_row(i);
        if (xch >= p.X_total) continue;
        float* dst = out + ((size_t)(t0 + j) * p.X_total + xch) * p.Y_total + yc * NYC + pnx::acc_col(i);
        if (p.partials) {  // every (tap, x, y) of a split's slab is written by exactly one CTA
          *reinterpret_cast<float2*>(dst) = make_float2(acc[j][i], acc[j][i + 1]);
        } else {
          atomicAdd(dst, acc[j][i]);
          atomicAdd(dst + 1, acc[j][i + 1]);
        }
      }
    }
  }
}

// dW[i] += sum over the splits, in split order (deterministic mode)
__global__ void wgrad_reduce_partials_kernel(const float* __restrict__ partials, int splits, long long n, float* __restrict__ dW) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int z = 0; z < splits; ++z) acc += partials[(size_t)z * n + i];
    dW[i] += acc;
  }
}

// grid plan shared by the launcher and pnx_wgrad_splits
struct WPlan { int taps_per_group, groups, rows_per_split, splits; };
inline WPlan wgrad_plan(int TG, int NYC, int x_blocks, int Y_total, int T, int M, int sm_count) {
  WPlan w;
  const int y_chunks = Y_total / NYC;
  w.taps_per_group = T < TG ? T : TG;
  w.groups = (T + w.taps_per_group - 1) / w.taps_per_group;
  w.taps_per_group = (T + w.groups - 1) / w.groups;  // balance the groups (e.g. 9 taps, TG = 8 -> 5 + 4)
  w.groups = (T + w.taps_per_group - 1) / w.taps_per_group;
  const int ctas_xy = x_blocks * y_chunks * w.groups;
  // two full waves of CTAs (one CTA per SM): round DOWN -- 2*132 + a few CTAs would run a third, nearly empty wave
  int splits = (2 * sm_count) / ctas_xy;
  const int max_splits = (M + 8 * kKS - 1) / (8 * kKS);  // at least 8 K-chunks per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  w.rows_per_split = ((M + splits - 1) / splits + kKS - 1) / kKS * kKS;
  w.splits = (M + w.rows_per_split - 1) / w.rows_per_split;
  return w;
}
// the (NYC, TG) variant pnx_wgrad picks for a shape: the largest Y chunk of 256/192/128/64 dividing y_channels, taps per
// group bounded by the 256 accumulator columns
inline void wgrad_variant(int y_channels, int* NYC, int* TG) {
  if (y_channels % 256 == 0) { *NYC = 256; *TG = 1; }
  else if (y_channels % 192 == 0) { *NYC = 192; *TG = 1; }
  else if (y_channels % 128 == 0) { *NYC = 128; *TG = 2; }
  else { *NYC = 64; *TG = 4; }
}

template <int NYC, int TG>
int launch_wgrad(const CUtensorMap& xmap, WgradParams p, int x_blocks, int sm_count, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    PNX_CUDA(cudaFuncSetAttribute(wgrad_kernel<NYC, TG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WCfg<NYC, TG>::kSmem));
    attr_set = true;
  }
  const WPlan w = wgrad_plan(TG, NYC, x_blocks, p.Y_total, p.T, p.M, sm_count);
  p.y_chunks = p.Y_total / NYC;
  p.taps_per_group = w.taps_per_group;
  p.rows_per_split = w.rows_per_split;
  const int groups = w.groups, splits = w.splits;
  dim3 grid(x_blocks * p.y_chunks, groups, splits);
  wgrad_kernel<NYC, TG><<<grid, kThreads, WCfg<NYC, TG>::kSmem, stream>>>(xmap, p);
  PNX_CHECK_LAUNCH();
  if (p.partials) {
    const long long n = (long long)p.T * p.X_total * p.Y_total;
    wgrad_reduce_partials_kernel<<<(int)((n + 255) / 256 < 592 ? (n + 255) / 256 : 592), 256, 0, stream>>>(p.partials, splits, n, p.dW);
    PNX_CHECK_LAUNCH();
  }
  return PNX_OK;
}

}  // namespace

// Number of K splits pnx_wgrad uses for a shape (deterministic mode: `partials` holds splits * taps * X * Y floats).
extern "C" int pnx_wgrad_splits(int x_channels, int y_channels, int taps, int M, int sm_count) {
  if (M <= 0 || x_channels <= 0 || y_channels <= 0 || taps <= 0) return 0;
  if (sm_count <= 0) sm_count = 132;
  int NYC, TG;
  wgrad_variant(y_channels, &NYC, &TG);
  return wgrad_plan(TG, NYC, x_channels == 64 ? 1 : x_channels / 128, y_channels, taps, M, sm_count).splits;
}

// Contract: include/pnx.h (pnx_wgrad).  dW must be zeroed (or hold the value to accumulate into).
extern "C" int pnx_wgrad(const void* X, long long ldx, int x_channels, const void* Y, long long ldy, long long y_rows,
                         int y_channels, int gathered, int M, int taps, const int* nbr, int Hout, int Wout, int Hin, int Win, int kw,
                         int mul, int dil, int pad, int shuffle, float* dW, float* partials, int sm_count, cudaStream_t stream) {
  PNX_CHECK_ARG(M >= 0, "M");
  if (M == 0) return PNX_OK;
  PNX_CHECK_ARG(taps >= 1 && taps <= 9, "taps");
  PNX_CHECK_ARG(x_channels % 64 == 0 && y_channels % 64 == 0, "channel counts must be multiples of 64");
  PNX_CHECK_ARG(x_channels == 64 || x_channels % 128 == 0, "x_channels must be 64 or a multiple of 128");
  PNX_CHECK_ARG(gathered || taps == 1, "taps > 1 needs a gathered operand");
  PNX_CHECK_ARG(!gathered || nbr || shuffle || (Hout > 0 && Wout > 0), "gather needs a table or geometry");
  PNX_CHECK_ARG(ldx % 8 == 0 && ldy % 8 == 0, "ldx/ldy % 8");
  if (sm_count <= 0) sm_count = 132;
  WgradParams p;
  p.X = (const __nv_bfloat16*)X; p.Y = (const __nv_bfloat16*)Y;
  p.ldx = ldx; p.ldy = ldy; p.M = M; p.T = taps;
  p.nbr = nbr; p.gathered = gathered;
  p.Hout = Hout > 0 ? Hout : 1; p.Wout = Wout > 0 ? Wout : 1; p.Hin = Hin; p.Win = Win;
  p.kw = kw > 0 ? kw : 1; p.mul = mul; p.dil = dil; p.pad = pad; p.shuffle = shuffle;
  p.dW = dW; p.partials = partials; p.X_total = x_channels; p.Y_total = y_channels;
  PNX_CHECK_ARG(!partials || (reinterpret_cast<uintptr_t>(partials) & 15) == 0, "partials 16-byte aligned");
  p.x_dup = x_channels == 64 ? 1 : 0;
  p.y_chunks = 1; p.taps_per_group = 1; p.rows_per_split = M;
  const int x_blocks = x_channels == 64 ? 1 : x_channels / 128;
  PNX_CHECK_ARG((reinterpret_cast<uintptr_t>(X) & 15) == 0 && (reinterpret_cast<uintptr_t>(Y) & 15) == 0, "X/Y 16-byte aligned");
  CUtensorMap xmap;
  int rc = pnx_encode_tmap_2d_bf16(&xmap, X, (uint64_t)M, (uint64_t)x_channels, (uint64_t)ldx * 2, kKS, 64);
  if (rc) return rc;
  PNX_CHECK_ARG(y_rows >= 1 && y_rows < 0x7fffffffLL, "y_rows = number of rows of Y");
  int NYC, TG;
  wgrad_variant(y_channels, &NYC, &TG);
  if (NYC == 256) return launch_wgrad<256, 1>(xmap, p, x_blocks, sm_count, stream);
  if (NYC == 192) return launch_wgrad<192, 1>(xmap, p, x_blocks, sm_count, stream);
  if (NYC == 128) return launch_wgrad<128, 2>(xmap, p, x_blocks, sm_count, stream);
  return launch_wgrad<64, 4>(xmap, p, x_blocks, sm_count, stream);
}
