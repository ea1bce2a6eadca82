// igemm_win.cu -- dense 3x3 'same' convolution (stride 1, dilation 1) on wgmma with the im2col folded into TMA.
//
// The gather engine (igemm.cu) re-reads every input row once per tap: for the head's 336x336 maps with few output
// channels (reference det3d/models/heads/centerhead.py:35-46,108-114 and their data gradients) that makes the
// L2->SM fabric the limit.  Here one M tile = 128 consecutive pixels of ONE image row, and for
// each 64-channel K chunk and each kernel row r the producer issues ONE 4-D TMA load of the 130-pixel window
// (x0-1 .. x0+128, y+r-1) -- out-of-image pixels are zero-filled by the TMA unit, i.e. the padding -- into a
// 128B-swizzled smem buffer.  The three horizontal taps s = 0,1,2 are the SAME buffer read through wgmma descriptors
// whose start address is shifted by s rows (s*128 bytes): 3 window loads feed 9 taps,
// cutting the activation traffic 2.9x, and there are no gather warps at all (one thread issues every load).
//   warpgroup 0: warp 0 is the TMA producer (A windows, 4-D map [C, W, H, B]; weight tiles, 2-D map), warps 1-3 store
//                the staged output tiles and sum their statistics while the next tile's MMAs run (gemm_epilogue.cuh)
//   warpgroups 1-2: wgmma on 64 pixels each, fp32 register accumulators, bias/ReLU/bf16 rounding into the staging buffer
#include "gemm_epilogue.cuh"

extern int g_pnx_deterministic;  // igemm.cu (pnx_set_deterministic)

namespace {

struct WinParams {
  int B, H, W, XC;          // XC = ceil(W / 128) tiles per image row
  int Cin, Cout_total;
  const float* bias;
  int base_off_mode;        // 1: descriptor base offset = (start >> 7) & 7 (PTX ISA), 0: leave 0
  pnx::EpiParams epi;
  const float* bnr_scale; const float* bnr_shift; const float* bnr_mean; const float* bnr_invstd;
  double* bnr_red;
  int bnr_C;
};

constexpr int kThreads = 384;
constexpr uint32_t kWinRows = 130;
constexpr uint32_t kWinBytes = kWinRows * 128;     // bytes written by one window load
constexpr uint32_t kWinSlot = 17 * 1024;           // 1024-aligned slot

// WS = weights stationary: for Cin = 64 the nine [BN x 64] weight tiles (9*BN*128 B) are loaded once per CTA and stay in
// shared memory; a stage is then only the activation window.  Without it every 128-pixel tile re-fetches all nine
// tiles (216 KB at BN = 192 against 50 KB of windows).
template <int BN, bool WS>
struct WCfgWin {
  static constexpr uint32_t kBTap = BN * 128;
  static constexpr uint32_t kWBytes = WS ? 9 * kBTap : 0;
  static constexpr uint32_t kStageBytes = WS ? kWinSlot : kWinSlot + 3 * kBTap;
  static constexpr int kFixed = 1024 + 256 + (2 * pnx::kEpiWarps + 5) * BN * 4;
  static constexpr int kAvail = 227 * 1024 - kFixed - (int)kWBytes;
  // staged epilogue: the whole tile at once, or in two column halves where that would cost pipeline depth below 3 stages
  // (or below what the ring had without staging, if that was less)
  static constexpr int kStagesUnstaged = kAvail / (int)kStageBytes;
  static constexpr int kMinStages = kStagesUnstaged < 3 ? kStagesUnstaged : 3;
  static constexpr int kPasses = (kAvail - pnx::Staging<BN, 1>::kBytes) / (int)kStageBytes >= kMinStages ? 1 : 2;
  static constexpr int kStgBytes = pnx::Staging<BN, kPasses>::kBytes;
  static constexpr int kStagesRaw = (kAvail - kStgBytes) / (int)kStageBytes;
  static constexpr int kStages = kStagesRaw > 6 ? 6 : kStagesRaw;
  static constexpr size_t kSmem = kFixed + kWBytes + (size_t)kStgBytes + (size_t)kStages * kStageBytes;
  static_assert(kStages >= 2, "stages");
  static_assert(kSmem <= 227 * 1024, "shared memory budget");
};

__device__ __forceinline__ uint64_t desc_sw128_off(uint32_t addr, uint32_t base_off) {
  return pnx::make_smem_desc_sw128(addr, 16, 1024) | ((uint64_t)(base_off & 7u) << 49);
}

template <int BN, bool WS, int F>
__global__ void __launch_bounds__(kThreads, 1) igemm_win_kernel(const __grid_constant__ CUtensorMap amap,
                                                                const __grid_constant__ CUtensorMap wmap, WinParams p) {
  using C = WCfgWin<BN, WS>;
  constexpr int kStages = C::kStages;
  constexpr int kPasses = C::kPasses;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem_w = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem = smem_w + C::kWBytes;  // stage ring (the stationary weight tiles, if any, come first)
  uint8_t* stg = smem + (size_t)kStages * C::kStageBytes;  // staged output tile (pnx::Staging)
  uint64_t* full = reinterpret_cast<uint64_t*>(stg + C::kStgBytes);
  uint64_t* empty = full + kStages;
  uint64_t* wfull = empty + kStages;
  uint64_t* staged = wfull + 1;  // the consumers' 256 threads wrote a staging pass
  uint64_t* sfree = staged + 1;  // the 96 store threads have drained it
  float* s_stat = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full) + 256);  // [8 warps][2][BN] per-channel sums
  float* s_bias = s_stat + pnx::kEpiWarps * 2 * BN;
  float* s_bnc = s_bias + BN;   // [4][BN] fused BN-backward: scale, shift, mean, invstd of this CTA's columns

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int n0 = blockIdx.y * BN;
  if (threadIdx.x == 0) {
    pnx::tma_prefetch_desc(&amap);
    pnx::tma_prefetch_desc(&wmap);
    for (int s = 0; s < kStages; ++s) {
      pnx::mbar_init(&full[s], 1);
      pnx::mbar_init(&empty[s], 8);  // one arrival per consumer warp
    }
    pnx::mbar_init(wfull, 1);
    pnx::mbar_init(staged, 256);
    pnx::mbar_init(sfree, 96);
    pnx::fence_barrier_init();
  }
  if (p.bias)
    for (int c = threadIdx.x; c < BN; c += blockDim.x) s_bias[c] = p.bias[n0 + c];
  for (int c = threadIdx.x; c < pnx::kEpiWarps * 2 * BN; c += blockDim.x) s_stat[c] = 0.f;
  if (F == 1)
    for (int c = threadIdx.x; c < BN; c += blockDim.x) {
      const int gc = n0 + c;
      s_bnc[c] = p.bnr_scale[gc]; s_bnc[BN + c] = p.bnr_shift[gc]; s_bnc[2 * BN + c] = p.bnr_mean[gc]; s_bnc[3 * BN + c] = p.bnr_invstd[gc];
    }
  __syncthreads();

  const int num_tiles = p.B * p.H * p.XC;
  const int kcc = p.Cin >> 6;

  if (wg == 0) {
    pnx::regs_dealloc<72>();  // gemm_epilogue_drain must fit in 72 registers: check `ptxas -v` for spills after editing it
    if (threadIdx.x >= 32) {
      // ---------------------------------------------------------------- warps 1-3: drain the staged tiles
      const int stid = threadIdx.x - 32;
      uint32_t spass = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int xc = tile % p.XC, by = tile / p.XC;
        const long long row0 = (long long)by * p.W + xc * 128;
        pnx::gemm_epilogue_drain<BN, F, kPasses>(p.epi, row0, min(128, p.W - xc * 128), n0, stg, s_stat, s_bnc, staged, sfree,
                                                 spass, stid, 96, 2);
      }
      asm volatile("bar.sync 2, 96;" ::: "memory");
      pnx::gemm_epilogue_flush<BN, F>(p.epi, n0, s_stat, p.bnr_red, p.bnr_C, stid, 96);
    } else if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      if (WS) {
        pnx::mbar_arrive_expect_tx(wfull, C::kWBytes);
        for (int t = 0; t < 9; ++t) pnx::tma_load_2d(&wmap, wfull, smem_w + t * C::kBTap, 0, t * p.Cout_total + n0);
      }
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int xc = tile % p.XC, by = tile / p.XC;
        const int y = by % p.H, b = by / p.H;
        for (int cc = 0; cc < kcc; ++cc) {
          for (int r = 0; r < 3; ++r) {
            pnx::mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* st = smem + (size_t)stage * C::kStageBytes;
            pnx::mbar_arrive_expect_tx(&full[stage], WS ? kWinBytes : kWinBytes + 3 * C::kBTap);
            pnx::tma_load_4d(&amap, &full[stage], st, cc * 64, xc * 128 - 1, y + r - 1, b);
#pragma unroll
            for (int s = 0; s < 3; ++s)
              if (!WS) pnx::tma_load_2d(&wmap, &full[stage], st + kWinSlot + s * C::kBTap, cc * 64, (r * 3 + s) * p.Cout_total + n0);
            if (++stage == kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    pnx::regs_alloc<216>();  // 128 * 72 + 256 * 216 <= 65536
    const int half = wg - 1;  // pixels [64 * half, 64 * half + 64) of every tile
    uint32_t spass = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    if (WS) pnx::mbar_wait(wfull, 0);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int xc = tile % p.XC, by = tile / p.XC;
      int prev = 0;
      for (int kc = 0; kc < kcc * 3; ++kc) {
        pnx::mbar_wait(&full[stage], phase);
        pnx::wgmma_fence();
        pnx::fence_acc(acc);
        const uint32_t a_base = pnx::smem_u32(smem + (size_t)stage * C::kStageBytes) + half * 64 * 128;
        // WS: kcc == 1, so stage kc is kernel row r = kc and its taps are weight tiles 3r .. 3r+2
        const uint32_t b_base = WS ? pnx::smem_u32(smem_w) + kc * 3 * C::kBTap : pnx::smem_u32(smem + (size_t)stage * C::kStageBytes) + kWinSlot;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint64_t da = desc_sw128_off(a_base + s * 128 + k * 32, p.base_off_mode ? (uint32_t)s : 0u);
            const uint64_t db = pnx::make_smem_desc_sw128(b_base + s * C::kBTap + k * 32, 16, 1024);
            pnx::Wgmma<BN, 0, 0>::mma(acc, da, db, (kc > 0 || s > 0 || k > 0) ? 1u : 0u);
          }
        }
        pnx::wgmma_commit();
        pnx::wgmma_wait<1>();
        if (kc > 0 && lane == 0) pnx::mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      pnx::wgmma_wait<0>();
      pnx::fence_acc(acc);
      if (lane == 0) pnx::mbar_arrive(&empty[prev]);
      const long long row0 = (long long)by * p.W + xc * 128;  // pixel index of tile row 0 (by = b*H + y)
      pnx::gemm_epilogue_stage<BN, kPasses>(acc, p.epi, row0, min(128, p.W - xc * 128), half, n0, s_bias, stg, staged, sfree, spass);
    }
  }
}

template <int BN, bool WS, int F>
int launch_win_f(const CUtensorMap& amap, const CUtensorMap& wmap, const WinParams& p, int n_blocks, int sm_count,
                 cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    PNX_CUDA(cudaFuncSetAttribute(igemm_win_kernel<BN, WS, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WCfgWin<BN, WS>::kSmem));
    attr_set = true;
  }
  const int num_tiles = p.B * p.H * p.XC;
  int gx = sm_count / n_blocks;
  if (gx < 1) gx = 1;
  if (gx > num_tiles) gx = num_tiles;
  igemm_win_kernel<BN, WS, F><<<dim3(gx, n_blocks), kThreads, WCfgWin<BN, WS>::kSmem, stream>>>(amap, wmap, p);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

template <int BN, bool WS>
int launch_win(const CUtensorMap& amap, const CUtensorMap& wmap, const WinParams& p, int n_blocks, int sm_count,
               cudaStream_t stream) {
  if (p.epi.bnr_raw) return launch_win_f<BN, WS, 1>(amap, wmap, p, n_blocks, sm_count, stream);
  return launch_win_f<BN, WS, 0>(amap, wmap, p, n_blocks, sm_count, stream);
}

}  // namespace

// Contract: include/pnx.h (pnx_conv3x3_win).
extern "C" int pnx_conv3x3_win(const void* A, long long lda, int B, int H, int W, int Cin, const void* Wpacked, int Cout,
                               int block_n, void* out, long long ldc, const float* bias, double* stats, int stats_C,
                               int relu, int base_off_mode, const void* bnr_raw, long long bnr_ld, const float* bnr_scale,
                               const float* bnr_shift, const float* bnr_mean, const float* bnr_invstd, double* bnr_red,
                               int bnr_C, int sm_count, cudaStream_t stream) {
  PNX_CHECK_ARG(B > 0 && H > 0 && W > 0, "shape");
  PNX_CHECK_ARG(Cin % 64 == 0 && Cout % block_n == 0, "Cin % 64, Cout % block_n");
  PNX_CHECK_ARG(lda % 8 == 0 && ldc % 8 == 0, "lda/ldc % 8");
  PNX_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "alignment");
  if (sm_count <= 0) sm_count = 132;
  WinParams p;
  p.B = B; p.H = H; p.W = W; p.XC = (W + 127) / 128;
  p.Cin = Cin; p.Cout_total = Cout;
  p.bias = bias;
  p.base_off_mode = base_off_mode;
  pnx::EpiParams& e = p.epi;
  e.out = out; e.ldc = ldc; e.has_bias = bias != nullptr; e.relu = relu;
  e.addend = nullptr; e.addend_f32 = nullptr; e.ld_add = 0;
  e.stats = stats; e.stats_C = stats_C; e.stats_mod = 1 << 30; e.stats_direct = g_pnx_deterministic;
  e.shuffle = 0; e.Hout = H; e.Wout = W;
  e.bnr_raw = (const __nv_bfloat16*)bnr_raw; e.bnr_ld = bnr_ld;
  p.bnr_scale = bnr_scale; p.bnr_shift = bnr_shift;
  p.bnr_mean = bnr_mean; p.bnr_invstd = bnr_invstd; p.bnr_red = bnr_red; p.bnr_C = bnr_C;
  if (bnr_raw)
    PNX_CHECK_ARG(!stats && bnr_scale && bnr_shift && bnr_mean && bnr_invstd && bnr_red && bnr_C == Cout && bnr_ld % 8 == 0 &&
                      (reinterpret_cast<uintptr_t>(bnr_raw) & 15) == 0, "fused BN-backward reduce: arguments");
  CUtensorMap amap, wmap;
  const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)lda * 2, (uint64_t)W * lda * 2, (uint64_t)H * W * lda * 2};
  const uint32_t box[4] = {64, kWinRows, 1, 1};
  int rc = pnx_encode_tmap_4d_bf16(&amap, A, dims, strides, box);
  if (rc) return rc;
  rc = pnx_encode_tmap_2d_bf16(&wmap, Wpacked, (uint64_t)9 * Cout, (uint64_t)Cin, (uint64_t)Cin * 2, (uint32_t)block_n, 64);
  if (rc) return rc;
  const int n_blocks = Cout / block_n;
  switch (block_n) {
    case 64:
      if (Cin == 64) return launch_win<64, true>(amap, wmap, p, n_blocks, sm_count, stream);
      return launch_win<64, false>(amap, wmap, p, n_blocks, sm_count, stream);
    case 128:
      if (Cin == 64) return launch_win<128, true>(amap, wmap, p, n_blocks, sm_count, stream);
      return launch_win<128, false>(amap, wmap, p, n_blocks, sm_count, stream);
    case 192: return launch_win<192, false>(amap, wmap, p, n_blocks, sm_count, stream);
    default:
      pnx_set_error("pnx_conv3x3_win: unsupported block_n %d (64/128/192)", block_n);
      return PNX_ERR_ARG;
  }
}
