// wgrad.cu -- weight-gradient of every convolution on the path as a wgmma GEMM over rows (sm_90a).
//
//   dW[t, x, y] += sum_m  X[m, x] * Y[g(m,t), y]          fp32, accumulated with red.global.add
// X is the DIRECT operand (read at row m), Y the GATHERED one (read through the neighbour table / the dense
// geometry at tap t).  For a convolution X = output gradient, Y = layer input; for ConvTranspose2d k2s2 the
// roles swap (X = input, Y = output gradient at the pixel-shuffled position).
// Both operands are MN-major for the MMA (the reduction index K = row m is the slow one in memory):
// tiles are staged as [64 rows x 128 B] blocks per 64-channel group with the 128-byte swizzle and
// described to wgmma as transposed operands (LBO = block stride, SBO = 8-row group stride).
// One CTA owns a 128-channel block of X, an NYC-channel chunk of Y and a GROUP of TG taps: the X tile of a 64-row chunk
// is staged ONCE, and the group's Y tiles sit side by side as TG * NYC / 64 consecutive 64-channel atoms, so one
// m64nNk16 wgmma with N = TG * NYC (<= 256 register accumulator columns) multiplies X against every tap of the group.
// A group past the last tap is padded with zero tiles (every CTA of a launch runs the same N, with no branch around
// the MMAs).  Accumulator column c is tap c / NYC, Y channel c % NYC.
// Grid = (x blocks * y chunks, tap groups, K splits), two full waves of one CTA per SM.  Warpgroup 0: X by TMA, Y rows by
// cp.async, each warp gathering the rows whose indices its lanes hold; warpgroups 1-2: wgmma, then a split's slab (or
// red.global.add) from registers.  With a 64-channel X both consumer warpgroups multiply the one X block, each over
// half of the group's columns.  Either way every dW element is one accumulator summing the split's rows in order.
// Window producer (WIN; dense 3 x 3, stride 1, dilation 1, 'same', image width a multiple of 16; see igemm_win.cu for the
// forward's version): a CTA's tap group is one kernel row r, and a K chunk is up to `chunk` consecutive pixels of one
// image row inside one split.  Per chunk one thread issues the X tiles and ONE 4-D TMA load of the (chunk + 2)-pixel
// window of Y at image row y + r - 1, zero-filled outside the image (the padding the gather path zero-fills per absent
// neighbour).  Tap s of the row is the window shifted by s
// pixels = s * 128 bytes, so the wgmma descriptor with LBO = 128 bytes reads the three taps as three side-by-side
// 64-channel column blocks of the one buffer (the 128B swizzle is applied on absolute shared-memory address bits, as
// igemm_win.cu relies on too): one window load feeds three taps, where the gather path copies each row once per tap.
// Both paths run the same split plan and the same k16 steps (16 consecutive rows; with W % 16 == 0 they never straddle
// an image row) in the same order; the X rows of a short chunk's unused k16 steps are zero-filled, so those steps add
// exact zeros.  The window path's dW is therefore bit-identical to the gather path's.
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
  int y_chunks;    // Y_total / NYC
  int taps_per_group;
  int rows_per_split;
  int chunk;       // window path: most pixels per K chunk (16 * WKS)
};

constexpr int kThreads = 384;         // producer warpgroup + two consumer warpgroups
constexpr int kKS = 64;               // rows (K) per stage
constexpr uint32_t kBlk = kKS * 128;  // bytes of one [64 rows x 64 ch] block
constexpr int kWinMaxChunk = 128;
constexpr uint32_t kWinXAtom = kWinMaxChunk * 128;  // one [chunk pixels x 64 ch] X tile of the window path
constexpr uint32_t kWinSlot = 17 * 1024;  // the (chunk + 2)-pixel window, plus the row a fourth shifted column block reads

// NYC = Y channels per CTA (64..256), TG = taps per group: one MMA per k16 step spans the N = NYC * TG columns of the
// group.  XD (X has 64 channels): both consumer warpgroups multiply the one X block, each over half of the columns.
// WKS > 0: the window path (WIN), chunks of up to 16 * WKS pixels.  NYC = 64 and the group is one kernel row; with XD the
// columns are four shifts of the window, two per warpgroup, and the fourth (shift 3) is computed and never stored, as the
// padding taps of the gather path are.
template <int NYC, int TG, bool XD, int WKS>
struct WCfg {
  static constexpr bool WIN = WKS > 0;
  static constexpr int kN = NYC * TG;
  static constexpr int kNW = XD ? kN / 2 : kN;  // accumulator columns of one consumer warpgroup
  static constexpr int kYAtoms = NYC / 64;
  static constexpr uint32_t kXBytes = WIN ? (XD ? 1 : 2) * kWinXAtom : 2 * kBlk;  // the X tiles of a stage come first
  static constexpr uint32_t kStageBytes = kXBytes + (WIN ? kWinSlot : TG * kYAtoms * kBlk);
  static constexpr int kStagesRaw = (200 * 1024) / (int)kStageBytes;
  static constexpr int kStages = kStagesRaw > 6 ? 6 : kStagesRaw;
  static constexpr size_t kSmem = 1024 + (size_t)kStages * kStageBytes + 256;
  static_assert(kN <= 256 && (kNW == 64 || kNW == 128 || kNW == 192 || kNW == 256), "one wgmma shape, <= 256 register accumulator columns");
  static_assert(!XD || kN % 128 == 0, "a warpgroup's half of the columns is whole 64-channel atoms");
  static_assert(kStages >= 2, "need at least two stages");
  static_assert(kSmem <= 227 * 1024, "shared memory budget");
  static_assert(!WIN || (NYC == 64 && TG == (XD ? 4 : 3)), "window: the three taps of one kernel row, 64 Y channels");
  static_assert((kWinMaxChunk + 2 + 1) * 128 <= kWinSlot, "window slot");
};

// window path: chunks of the split's rows [m_begin, m_end) -- image-row pieces, each cut into runs of at most `chunk`
__device__ __forceinline__ int win_chunks(int m_begin, int m_end, int W, int chunk) {
  int n = 0;
  for (int m = m_begin; m < m_end;) {
    const int e = min(m_end, (m / W + 1) * W);
    n += (e - m + chunk - 1) / chunk;
    m = e;
  }
  return n;
}

// xmap: X, 2-D [M, X_total] (gather path) or 4-D [X_total, W, H, B] (window path); ymap: Y, 4-D (window path only)
template <int NYC, int TG, bool XD, int WKS>
__global__ void __launch_bounds__(kThreads, 1) wgrad_kernel(const __grid_constant__ CUtensorMap xmap,
                                                            const __grid_constant__ CUtensorMap ymap, WgradParams p) {
  using C = WCfg<NYC, TG, XD, WKS>;
  constexpr bool WIN = C::WIN;
  constexpr int kStages = C::kStages, kYAtoms = C::kYAtoms, kNW = C::kNW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)kStages * C::kStageBytes);
  uint64_t* empty = full + kStages;

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int xb = blockIdx.x / p.y_chunks, yc = blockIdx.x - xb * p.y_chunks;
  const int t0 = blockIdx.y * p.taps_per_group;
  const int ntaps = WIN ? 3 : min(TG, p.T - t0);  // taps [ntaps, TG) of the group are zero tiles (window: never stored)
  const int split = blockIdx.z;
  const int m_begin = split * p.rows_per_split;
  const int m_end = min(p.M, m_begin + p.rows_per_split);
  const int num_k = WIN ? win_chunks(m_begin, m_end, p.Wout, p.chunk) : (m_end - m_begin + kKS - 1) / kKS;

  if (threadIdx.x == 0) {
    pnx::tma_prefetch_desc(&xmap);
    if (WIN) pnx::tma_prefetch_desc(&ymap);
    for (int s = 0; s < kStages; ++s) {
      pnx::mbar_init(&full[s], WIN ? 1 : 1 + 128);  // X tiles (expect_tx) + the 128 gathering threads (cp.async arrive)
      pnx::mbar_init(&empty[s], 8);                 // one arrival per consumer warp
    }
    pnx::fence_barrier_init();
  }
  if (!WIN && ntaps < TG) {
    // the Y tiles of the padding taps are zeroed once in every stage and never written again
    constexpr int kPer = kBlk / 16;  // 16-byte words of one block
    const int pad_words = (TG - ntaps) * kYAtoms * kPer;
    for (int i = threadIdx.x; i < kStages * pad_words; i += kThreads) {
      const int s = i / pad_words, w = i - s * pad_words;
      *reinterpret_cast<uint4*>(smem + (size_t)s * C::kStageBytes + (2 + ntaps * kYAtoms) * kBlk + (size_t)w * 16) = make_uint4(0, 0, 0, 0);
    }
    pnx::fence_proxy_async_smem();  // written through the generic proxy, read by wgmma
  }
  __syncthreads();
  if (num_k <= 0) return;

  if (wg == 0 && WIN) {
    // ---------------------------------------------------------------- producer, window path: one thread, TMA only
    pnx::regs_dealloc<56>();
    if (threadIdx.x == 0) {
      const int r = blockIdx.y;  // kernel row of the group: taps 3r .. 3r+2
      constexpr int nblk = XD ? 1 : 2;
      const uint32_t tx = (uint32_t)(nblk * p.chunk + p.chunk + 2) * 128;
      int stage = 0;
      uint32_t phase = 0;
      int m = m_begin;
      for (int kc = 0; kc < num_k; ++kc) {
        const int by = m / p.Wout, x0 = m - by * p.Wout;
        const int len = min(min(m_end, (by + 1) * p.Wout) - m, p.chunk);  // a multiple of 16
        const int y = by % p.Hout, b = by / p.Hout;
        pnx::mbar_wait(&empty[stage], phase ^ 1);
        uint8_t* st = smem + (size_t)stage * C::kStageBytes;
        pnx::mbar_arrive_expect_tx(&full[stage], tx);
        // X in 16-pixel boxes, one per k16 step; the steps past the chunk's length load a box wholly outside the image
        // (x = W), i.e. zeros, and add nothing
#pragma unroll
        for (int i = 0; i < WKS; ++i)
          for (int b2 = 0; b2 < nblk; ++b2)
            pnx::tma_load_4d(&xmap, &full[stage], st + b2 * kWinXAtom + i * 2048, xb * 128 + b2 * 64, 16 * i < len ? x0 + 16 * i : p.Wout, y, b);
        pnx::tma_load_4d(&ymap, &full[stage], st + C::kXBytes, yc * 64, x0 - 1, y + r - 1, b);
        m += len;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (wg == 0) {
    // ---------------------------------------------------------------- producer, gather path
    pnx::regs_dealloc<56>();
    const int warp = threadIdx.x >> 5;
    const int y_ch0 = yc * NYC;
    const int nblk = XD ? 1 : 2;
    const int hw = p.Hout * p.Wout;
    // Warp w gathers rows [16 w, +16) of every tap of the group.  Lane l holds the Y row of (tap 2 n + l / 16,
    // row 16 w + l % 16) in idx[n] (-1 = absent: zero fill) and hands it to the lanes copying that row with a shuffle.
    constexpr int kIdxRegs = (TG + 1) / 2;
    auto load_idx = [&](int kc, int (&idx)[kIdxRegs]) {
      const int m = m_begin + kc * kKS + 16 * warp + (lane & 15);
#pragma unroll
      for (int n = 0; n < kIdxRegs; ++n) {
        const int j = 2 * n + (lane >> 4);
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
        idx[n] = g;
      }
    };
    int idx[kIdxRegs], nxt[kIdxRegs];
    load_idx(0, idx);
    // a warp instruction copies 4 whole 128-byte rows 16 w + 4 qq + rq; their swizzle depends only on rq and qq & 1
    const int sub = lane & 7, rq = lane >> 3;
    const uint32_t row_off = (uint32_t)(16 * warp + rq) * 128;
    const uint32_t swz[2] = {(uint32_t)(sub ^ rq) << 4, (uint32_t)(sub ^ (rq + 4)) << 4};
    int stage = 0;
    uint32_t phase = 0;
    for (int kc = 0; kc < num_k; ++kc) {
      if (kc + 1 < num_k) load_idx(kc + 1, nxt);  // the next stage's indices load while this one waits for its slot
      pnx::mbar_wait(&empty[stage], phase ^ 1);
      uint8_t* st = smem + (size_t)stage * C::kStageBytes;
      if (threadIdx.x == 0) {
        // X: plain 2-D TMA boxes of [64 rows x 64 channels] (rows past M are zero-filled by the tensor map bounds)
        pnx::mbar_arrive_expect_tx(&full[stage], (uint32_t)nblk * kBlk);
        for (int b2 = 0; b2 < nblk; ++b2) pnx::tma_load_2d(&xmap, &full[stage], st + b2 * kBlk, xb * 128 + b2 * 64, m_begin + kc * kKS);
      }
      const uint32_t sy = pnx::smem_u32(st) + 2 * kBlk + row_off;
#pragma unroll
      for (int j = 0; j < TG; ++j) {
        if (j >= ntaps) break;  // padding taps stay zero
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {
          const int g = __shfl_sync(0xffffffffu, idx[j >> 1], ((j & 1) << 4) + 4 * qq + rq);
          const __nv_bfloat16* src = p.Y + (long long)(g < 0 ? 0 : g) * p.ldy + y_ch0 + sub * 8;
#pragma unroll
          for (int a = 0; a < kYAtoms; ++a)
            pnx::cp_async_16(sy + (j * kYAtoms + a) * kBlk + qq * 512 + swz[qq & 1], src + a * 64, g < 0 ? 0u : 16u);
        }
      }
      pnx::cp_async_mbar_arrive(&full[stage]);
#pragma unroll
      for (int n = 0; n < kIdxRegs; ++n) idx[n] = nxt[n];
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
  } else {
    // ---------------------------------------------------------------- consumers
    // X channels [64 * half, +64) of the block over all columns, or (XD) the one X block over columns [kNW * half, +kNW)
    pnx::regs_alloc<224>();
    const int half = wg - 1;
    const uint32_t x_off = XD ? 0u : (uint32_t)half * (WIN ? kWinXAtom : kBlk);
    // window: column block s of the B operand is the window shifted by s pixels (LBO = one 128-byte pixel row)
    const uint32_t y_off = C::kXBytes + (XD ? (uint32_t)half * (kNW / 64) * (WIN ? 128u : kBlk) : 0u);
    const uint32_t y_lbo = WIN ? 128u : kBlk;
    constexpr int ksteps = WIN ? WKS : kKS / 16;
    float acc[kNW / 2];
#pragma unroll
    for (int i = 0; i < kNW / 2; ++i) acc[i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kc = 0; kc < num_k; ++kc) {
      pnx::mbar_wait(&full[stage], phase);
      pnx::fence_proxy_async_smem();  // the cp.async rows were written through the generic proxy; wgmma reads async
      pnx::wgmma_fence();
      pnx::fence_acc(acc);
      const uint32_t st = pnx::smem_u32(smem + (size_t)stage * C::kStageBytes);
#pragma unroll
      for (int k = 0; k < ksteps; ++k)
        pnx::Wgmma<kNW, 1, 1>::mma(acc, pnx::make_smem_desc_sw128(st + x_off + k * 2048, kBlk, 1024),
                                   pnx::make_smem_desc_sw128(st + y_off + k * 2048, y_lbo, 1024), (kc > 0 || k > 0) ? 1u : 0u);
      pnx::wgmma_commit();
      pnx::wgmma_wait<1>();  // the previous stage's MMAs are done: release it
      if (kc > 0 && lane == 0) pnx::mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    pnx::wgmma_wait<0>();
    pnx::fence_acc(acc);
    // ---------------------------------------------------------------- epilogue: registers -> the split's slab
    float* out = p.partials ? p.partials + (size_t)blockIdx.z * ((size_t)p.T * p.X_total * p.Y_total) : p.dW;
    const int x0 = xb * 128 + (XD ? 0 : half * 64);
    const int c0 = XD ? half * kNW : 0;
#pragma unroll
    for (int i = 0; i < kNW / 2; i += 2) {
      const int c = c0 + pnx::acc_col(i), j = c / NYC;
      const int xch = x0 + pnx::acc_row(i);
      if (j >= ntaps || xch >= p.X_total) continue;  // padding taps are not stored
      float* dst = out + ((size_t)(t0 + j) * p.X_total + xch) * p.Y_total + yc * NYC + (c - j * NYC);
      if (p.partials) {  // every (tap, x, y) of a split's slab is written by exactly one CTA
        *reinterpret_cast<float2*>(dst) = make_float2(acc[i], acc[i + 1]);
      } else {
        atomicAdd(dst, acc[i]);
        atomicAdd(dst + 1, acc[i + 1]);
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

// the (NYC, TG) variant pnx_wgrad picks for a shape: the largest Y chunk of 256/192/128/64 dividing y_channels; the taps
// of a 128- or 64-channel chunk are grouped so that one MMA spans N = 192 or 256 columns (3 x 3: 5 groups of 2 taps at
// 128 channels, 3 groups of 3 at 64; ConvTranspose 2 x 2 at 64: one group of 4), with the fewest zero padding taps.
// XD (64-channel X): each consumer warpgroup takes half of the N columns, so N is 128 or 256 (whole atoms per half);
// 3 x 3 at 64 Y channels then runs 3 groups of 4 taps, the last one 1 tap + 3 padding taps.
inline void wgrad_variant(int y_channels, int taps, bool xd, int* NYC, int* TG) {
  if (xd) {
    if (y_channels % 256 == 0) { *NYC = 256; *TG = 1; }
    else if (y_channels % 128 == 0) { *NYC = 128; *TG = taps > 1 ? 2 : 1; }
    else { *NYC = 64; *TG = taps <= 2 ? 2 : 4; }
    return;
  }
  if (y_channels % 256 == 0) { *NYC = 256; *TG = 1; }
  else if (y_channels % 192 == 0) { *NYC = 192; *TG = 1; }
  else if (y_channels % 128 == 0) { *NYC = 128; *TG = taps > 1 ? 2 : 1; }
  else { *NYC = 64; *TG = taps == 1 ? 1 : (4 - taps % 4) % 4 <= (3 - taps % 3) % 3 ? 4 : 3; }
}

// K split plan shared by the launcher and pnx_wgrad_splits.  It depends on the shape alone (it is sized from the grid of
// the full-X-block variant, whatever variant runs), so the order in which every dW element is summed -- the rows of a
// split in order, then the splits in order -- does not depend on how the taps and Y channels are tiled.
struct WPlan { int rows_per_split, splits; };
inline WPlan wgrad_plan(int x_blocks, int Y_total, int T, int M, int sm_count) {
  int NYC, TG;
  wgrad_variant(Y_total, T, false, &NYC, &TG);
  const int ctas_xy = x_blocks * (Y_total / NYC) * ((T + TG - 1) / TG);
  // two full waves of CTAs (one CTA per SM): round DOWN -- 2*132 + a few CTAs would run a third, nearly empty wave
  int splits = (2 * sm_count) / ctas_xy;
  const int max_splits = (M + 8 * kKS - 1) / (8 * kKS);  // at least 8 K-chunks per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  WPlan w;
  w.rows_per_split = ((M + splits - 1) / splits + kKS - 1) / kKS * kKS;
  w.splits = (M + w.rows_per_split - 1) / w.rows_per_split;
  return w;
}

// Window path: most pixels per K chunk for an image row of W pixels.  The chunk is the multiple of 16 (one wgmma k-step)
// in [64, 128] with the fewest zero k16 steps ceil(W / chunk) * chunk - W per whole row, the wider one on a tie (fewer
// windows, and the two extra pixels of each window are a smaller share): 112 for W = 336 (none), 96 for 176.  Rows that a
// split boundary cuts cost up to one more partial chunk each.
inline int wgrad_win_chunk(int W) {
  int best = kWinMaxChunk;
  for (int c = kWinMaxChunk; c >= 64; c -= 16)
    if ((W + c - 1) / c * c < (W + best - 1) / best * best) best = c;
  return best;
}

template <int NYC, int TG, bool XD, int WKS>
int launch_wgrad(const CUtensorMap& xmap, const CUtensorMap& ymap, WgradParams p, int x_blocks, int sm_count, cudaStream_t stream) {
  using C = WCfg<NYC, TG, XD, WKS>;
  constexpr bool WIN = C::WIN;
  static bool attr_set = false;
  if (!attr_set) {
    PNX_CUDA(cudaFuncSetAttribute(wgrad_kernel<NYC, TG, XD, WKS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::kSmem));
    attr_set = true;
  }
  const WPlan w = wgrad_plan(x_blocks, p.Y_total, p.T, p.M, sm_count);  // the window path splits the rows as the gather path does
  p.y_chunks = p.Y_total / NYC;
  p.taps_per_group = WIN ? 3 : TG;
  p.rows_per_split = w.rows_per_split;
  dim3 grid(x_blocks * p.y_chunks, WIN ? 3 : (p.T + TG - 1) / TG, w.splits);
  wgrad_kernel<NYC, TG, XD, WKS><<<grid, kThreads, C::kSmem, stream>>>(xmap, ymap, p);
  PNX_CHECK_LAUNCH();
  if (p.partials) {
    const long long n = (long long)p.T * p.X_total * p.Y_total;
    wgrad_reduce_partials_kernel<<<(int)((n + 255) / 256 < 592 ? (n + 255) / 256 : 592), 256, 0, stream>>>(p.partials, w.splits, n, p.dW);
    PNX_CHECK_LAUNCH();
  }
  return PNX_OK;
}

template <int WKS>
int launch_wgrad_win(const CUtensorMap& xmap, const CUtensorMap& ymap, const WgradParams& p, int x_blocks, int sm_count,
                     cudaStream_t stream) {
  if (p.X_total == 64) return launch_wgrad<64, 4, true, WKS>(xmap, ymap, p, x_blocks, sm_count, stream);
  return launch_wgrad<64, 3, false, WKS>(xmap, ymap, p, x_blocks, sm_count, stream);
}

}  // namespace

// Number of K splits pnx_wgrad uses for a shape (deterministic mode: `partials` holds splits * taps * X * Y floats).
extern "C" int pnx_wgrad_splits(int x_channels, int y_channels, int taps, int M, int sm_count) {
  if (M <= 0 || x_channels <= 0 || y_channels <= 0 || taps <= 0) return 0;
  if (sm_count <= 0) sm_count = 132;
  return wgrad_plan(x_channels == 64 ? 1 : x_channels / 128, y_channels, taps, M, sm_count).splits;
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
  p.y_chunks = 1; p.taps_per_group = 1; p.rows_per_split = M;
  p.chunk = 0;
  const int x_blocks = x_channels == 64 ? 1 : x_channels / 128;
  PNX_CHECK_ARG((reinterpret_cast<uintptr_t>(X) & 15) == 0 && (reinterpret_cast<uintptr_t>(Y) & 15) == 0, "X/Y 16-byte aligned");
  PNX_CHECK_ARG(y_rows >= 1 && y_rows < 0x7fffffffLL, "y_rows = number of rows of Y");
  const long long hw = (long long)p.Hout * p.Wout;
  // W % 16 == 0: no k16 step of 16 consecutive rows straddles an image row, so the window path can run the gather path's
  // k16 steps and sum every dW element in the same order
  const bool window = gathered && !nbr && !shuffle && taps == 9 && kw == 3 && mul == 1 && dil == 1 && pad == 1 && Hin == p.Hout &&
                      Win == p.Wout && p.Wout % 16 == 0 && M % hw == 0 && y_rows >= M;
  if (window) {
    const int B = (int)(M / hw);
    p.chunk = wgrad_win_chunk(p.Wout);
    CUtensorMap xmap, ymap;
    const uint64_t xdims[4] = {(uint64_t)x_channels, (uint64_t)p.Wout, (uint64_t)p.Hout, (uint64_t)B};
    const uint64_t xstr[3] = {(uint64_t)ldx * 2, (uint64_t)p.Wout * ldx * 2, (uint64_t)hw * ldx * 2};
    const uint32_t xbox[4] = {64, 16, 1, 1};
    int rc = pnx_encode_tmap_4d_bf16(&xmap, X, xdims, xstr, xbox);
    if (rc) return rc;
    const uint64_t ydims[4] = {(uint64_t)y_channels, (uint64_t)p.Wout, (uint64_t)p.Hout, (uint64_t)B};
    const uint64_t ystr[3] = {(uint64_t)ldy * 2, (uint64_t)p.Wout * ldy * 2, (uint64_t)hw * ldy * 2};
    const uint32_t ybox[4] = {64, (uint32_t)p.chunk + 2, 1, 1};
    rc = pnx_encode_tmap_4d_bf16(&ymap, Y, ydims, ystr, ybox);
    if (rc) return rc;
    // the k-steps per chunk are a template argument: a run-time trip count around the MMAs would serialize them
    switch (p.chunk / 16) {
      case 4: return launch_wgrad_win<4>(xmap, ymap, p, x_blocks, sm_count, stream);
      case 5: return launch_wgrad_win<5>(xmap, ymap, p, x_blocks, sm_count, stream);
      case 6: return launch_wgrad_win<6>(xmap, ymap, p, x_blocks, sm_count, stream);
      case 7: return launch_wgrad_win<7>(xmap, ymap, p, x_blocks, sm_count, stream);
      default: return launch_wgrad_win<8>(xmap, ymap, p, x_blocks, sm_count, stream);
    }
  }
  CUtensorMap xmap;
  int rc = pnx_encode_tmap_2d_bf16(&xmap, X, (uint64_t)M, (uint64_t)x_channels, (uint64_t)ldx * 2, kKS, 64);
  if (rc) return rc;
  const CUtensorMap& ymap = xmap;  // not read by the gather path
  int NYC, TG;
  if (x_channels == 64) {
    wgrad_variant(y_channels, taps, true, &NYC, &TG);
    if (NYC == 256) return launch_wgrad<256, 1, true, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
    if (NYC == 128) return TG == 2 ? launch_wgrad<128, 2, true, 0>(xmap, ymap, p, x_blocks, sm_count, stream) : launch_wgrad<128, 1, true, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
    return TG == 4 ? launch_wgrad<64, 4, true, 0>(xmap, ymap, p, x_blocks, sm_count, stream) : launch_wgrad<64, 2, true, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
  }
  wgrad_variant(y_channels, taps, false, &NYC, &TG);
  if (NYC == 256) return launch_wgrad<256, 1, false, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
  if (NYC == 192) return launch_wgrad<192, 1, false, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
  if (NYC == 128) return TG == 2 ? launch_wgrad<128, 2, false, 0>(xmap, ymap, p, x_blocks, sm_count, stream) : launch_wgrad<128, 1, false, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
  if (TG == 4) return launch_wgrad<64, 4, false, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
  if (TG == 3) return launch_wgrad<64, 3, false, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
  return launch_wgrad<64, 1, false, 0>(xmap, ymap, p, x_blocks, sm_count, stream);
}
