// igemm.cu -- gather implicit-GEMM convolution on wgmma tensor cores (sm_90a).
//
// One engine for every convolution on the path (rows B1-B3, N1, H1 of SURVEY.md section 8a; their
// data-gradients too):   out[m, n] = sum_t sum_c  A[nbr(m,t), c] * W[t, n, c]   (+bias)(relu)
//   * sparse BEV backbone (spconv SparseConv2d / SubMConv2d, reference sparse_conv.py:25-29,50-51,
//     sparse_resnet.py:43-48): rows = active sites, nbr = neighbour table from rulebook.cu
//   * dense neck/head (F.conv2d 3x3 / dilated 3x3 / 1x1, reference aspp.py:19-32, conv.py:9-10,
//     centerhead.py:35-46,108-114): rows = pixels of a channels-last image, nbr computed from geometry
//     (zero padding = absent neighbour), ConvTranspose2d k2 s2 (centerhead.py:26-27) = one GEMM with
//     N = 4*Cout and a pixel-shuffle store.
// CTA persistent over 128-row tiles: warpgroup 0 writes the gathered row of every (tap, row) of a tile into shared
// memory, then per K stage loads the weight tile by TMA and gathers the 128 A rows with 16-byte cp.async (index -1 = zero
// fill) into the 128B-swizzled layout; warpgroups 1-2 each run wgmma on 64 rows into registers.  Staged variants
// (Cfg::kStaged) have a fourth warpgroup: the consumers write the tile into shared memory and go back to their MMAs, and
// warpgroup 3 stores it and sums its statistics meanwhile (gemm_epilogue.cuh).  At BN = 256 (Cfg::kWide) the consumers'
// 128 accumulator registers per thread do not fit the 128 a 512-thread CTA allows: setmaxnreg moves registers from the
// producer and store warpgroups to them, and the store threads keep the statistic slots in registers, which frees the
// shared memory for the whole-tile staging buffer and 3 stages.  Only fp32 output at BN = 192 and 256 (the split mode)
// keeps the whole epilogue on warpgroups 1-2.
#include "gemm_epilogue.cuh"

namespace {

struct IgemmParams {
  const __nv_bfloat16* A;
  long long lda;
  int M, T, Cin, w_rows_per_tap;
  const int* nbr;
  int dense, Hout, Wout, Hin, Win, kw, mul, dil, pad;
  // fp32-grade "split" mode: every value is the sum of P bf16 PIECES (P = 2: hi + lo, 16 mantissa bits; P = 3:
  // hi + mid + lo, 24 bits).  A rows hold piece p of channel c at column p * a_lo_off + c, W rows are
  // [piece 0 (Cin) | piece 1 (Cin) | ...]; the K loop runs nseg (A piece, W piece) segments into the same fp32
  // accumulator, the small correction terms FIRST, while the accumulator is small: the tensor core's fp32
  // accumulation truncates (measured: tools/split_error_probe.py), and adding 2^-9-sized terms to a full-sized
  // accumulator would lose most of their low bits.  nseg = 1 (piece 0 x piece 0): plain bf16.
  int nseg, a_lo_off;
  unsigned long long seg_code;  // 4 bits per segment, in execution order: (A piece << 2) | W piece
  pnx::EpiParams epi;
  int out_fp32;
  const float* bias;
  const float* bnr_scale; const float* bnr_shift; const float* bnr_mean; const float* bnr_invstd;
  double* bnr_red;
  int bnr_C;
};

constexpr uint32_t kABytes = 128 * 128;  // one A stage: 128 rows x 64 bf16
constexpr int kProducerRegs = 56, kConsumerRegs = 224;  // unstaged variants (384 threads): 128 * 56 + 256 * 224 <= 65536
constexpr int kWideStoreRegs = 88, kWideConsumerRegs = 184;  // kWide (512 threads): 128 * (56 + 88) + 256 * 184 = 65536

template <int BN, int F>
struct Cfg {
  static constexpr bool kStaged = F != 2 || BN <= 128;  // fp32 at BN = 192 would spill at 128 registers per thread
  static constexpr bool kWide = kStaged && BN == 256;  // setmaxnreg split, statistic slots in the store threads' registers
  static constexpr int kThreads = kStaged ? 512 : 384;  // + the store warpgroup
  static constexpr uint32_t kBBytes = BN * 128;
  static constexpr int kTbl = 128 * 9;  // ints of the per-tile index table [tap][row]
  static constexpr int kStatFloats = kWide ? 0 : 2 * pnx::kEpiWarps * BN;  // s_stat
  static constexpr int kFixed = 1024 + kTbl * 4 + 256 + (kStatFloats + 5 * BN) * 4;
  static constexpr int kStageBytes = (int)(kABytes + kBBytes);
  static constexpr int kAvail = 227 * 1024 - kFixed;
  // staged epilogue: the whole tile at once, or in two column halves where that would leave fewer than 3 stages
  static constexpr int kPasses = !kStaged ? 1 : ((kAvail - pnx::StagingF<BN, 1, F>::kBytes) / kStageBytes >= 3 ? 1 : 2);
  static constexpr int kStgBytes = !kStaged ? 0 : pnx::StagingF<BN, kPasses, F>::kBytes;
  static constexpr int kStagesRaw = (kAvail - kStgBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr size_t kSmem = (size_t)kFixed + (size_t)kStgBytes + (size_t)kStages * kStageBytes;
  static_assert(kStages >= 3, "pipeline depth");
  static_assert(kSmem <= 227 * 1024, "shared memory budget");
  static_assert(!kWide || kPasses == 1, "register statistic slots need the whole tile staged");
};

__device__ __forceinline__ void named_bar_sync(int id, int n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}

template <int BN, int F>
__global__ void __launch_bounds__(Cfg<BN, F>::kThreads, 1) igemm_kernel(const __grid_constant__ CUtensorMap wmap, IgemmParams p) {
  using C = Cfg<BN, F>;
  constexpr int kStages = C::kStages;
  constexpr int kPasses = C::kPasses;
  constexpr uint32_t kBBytes = C::kBBytes;
  constexpr int kTbl = C::kTbl;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + (size_t)kStages * kABytes;
  uint8_t* stg = sB + (size_t)kStages * kBBytes;                        // staged output tile (pnx::Staging)
  int* s_idx = reinterpret_cast<int*>(stg + C::kStgBytes);              // [T][128 rows] gathered row index, -1 = absent
  uint64_t* full = reinterpret_cast<uint64_t*>(s_idx + kTbl);
  uint64_t* empty = full + kStages;
  uint64_t* staged = empty + kStages;  // the consumers' 256 threads wrote a staging pass
  uint64_t* sfree = staged + 1;        // the store warpgroup has drained it
  float* s_stat = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full) + 256);  // [8 warps][2][BN] per-channel sums
  float* s_bias = s_stat + C::kStatFloats;                                           // [BN] bias of this CTA's columns
  float* s_bnc = s_bias + BN;                                                        // [4][BN] fused BN-backward affine

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int n0 = blockIdx.y * BN;

  if (threadIdx.x == 0) {
    pnx::tma_prefetch_desc(&wmap);
    for (int s = 0; s < kStages; ++s) {
      pnx::mbar_init(&full[s], 1 + 128);  // weight TMA (expect_tx) + the 128 gathering threads (cp.async arrive)
      pnx::mbar_init(&empty[s], 8);       // one arrival per consumer warp
    }
    pnx::mbar_init(staged, 256);
    pnx::mbar_init(sfree, 128);
    pnx::fence_barrier_init();
  }
  if (p.bias)
    for (int c = threadIdx.x; c < BN; c += blockDim.x) s_bias[c] = p.bias[n0 + c];
  for (int c = threadIdx.x; c < C::kStatFloats; c += blockDim.x) s_stat[c] = 0.f;
  if (F == 1)
    for (int c = threadIdx.x; c < BN; c += blockDim.x) {
      const int gc = n0 + c;
      s_bnc[c] = p.bnr_scale[gc]; s_bnc[BN + c] = p.bnr_shift[gc]; s_bnc[2 * BN + c] = p.bnr_mean[gc]; s_bnc[3 * BN + c] = p.bnr_invstd[gc];
    }
  __syncthreads();

  const int num_tiles = (p.M + 127) >> 7;
  const int kpt = p.Cin >> 6;
  const int num_k = p.T * kpt * p.nseg;

  if (wg == 3) {
    // ---------------------------------------------------------------- store warpgroup (staged variants): drains the tiles
    if constexpr (C::kStaged) {
      if constexpr (C::kWide) pnx::regs_dealloc<kWideStoreRegs>();
      const int stid = threadIdx.x - 384;
      uint32_t spass = 0;
      float4 r_stat[pnx::kEpiWarps];  // kWide: the statistic slots of column pair stid
#pragma unroll
      for (int w = 0; w < pnx::kEpiWarps; ++w) r_stat[w] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const long long row0 = (long long)tile * 128;
        pnx::gemm_epilogue_drain<BN, F, kPasses, C::kWide>(p.epi, row0, (int)min((long long)128, (long long)p.M - row0), n0, stg,
                                                           s_stat, s_bnc, staged, sfree, spass, stid, 128, 2, r_stat);
      }
      if constexpr (C::kWide) {
        pnx::gemm_epilogue_flush_regs<BN, F>(p.epi, n0, r_stat, p.bnr_red, p.bnr_C, stid);
      } else {
        named_bar_sync(2, 128);
        pnx::gemm_epilogue_flush<BN, F>(p.epi, n0, s_stat, p.bnr_red, p.bnr_C, stid, 128);
      }
    }
  } else if (wg == 0) {
    // ---------------------------------------------------------------- producer
    if constexpr (!C::kStaged || C::kWide) pnx::regs_dealloc<kProducerRegs>();
    const int ptid = threadIdx.x;
    const int sub = ptid & 7, rsub = ptid >> 3;  // a warp instruction copies 4 whole 128-byte rows
    const int hw = p.Hout * p.Wout;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      named_bar_sync(1, 128);  // every thread is done reading the previous tile's table
      {
        const int r = ptid;
        const int m = tile * 128 + r;
        if (m >= p.M) {
          for (int t = 0; t < p.T; ++t) s_idx[t * 128 + r] = -1;
        } else if (p.nbr) {
          const int* src = p.nbr + (size_t)m * p.T;
          for (int t = 0; t < p.T; ++t) s_idx[t * 128 + r] = src[t];
        } else if (p.dense) {
          const int b = m / hw, rem = m - b * hw, y = rem / p.Wout, x = rem - y * p.Wout;
          const int base = b * p.Hin;
          int t = 0;
          for (int rr = 0; t < p.T; ++rr) {
            const int yi = y * p.mul + rr * p.dil - p.pad;
            const bool yok = yi >= 0 && yi < p.Hin;
            for (int ss = 0; ss < p.kw && t < p.T; ++ss, ++t) {
              const int xi = x * p.mul + ss * p.dil - p.pad;
              s_idx[t * 128 + r] = (yok && xi >= 0 && xi < p.Win) ? (base + yi) * p.Win + xi : -1;
            }
          }
        } else {
          s_idx[r] = m;
        }
      }
      named_bar_sync(1, 128);
      for (int kc = 0; kc < num_k; ++kc) {
        const int ccx = kc / p.T, t = kc - ccx * p.T;  // chunk outer, tap inner: consecutive stages re-read overlapping rows
        const int seg = ccx / kpt, cc = ccx - seg * kpt;
        const int wpiece = (int)((p.seg_code >> (4 * seg)) & 3ull);
        const int acol = cc * 64 + (int)((p.seg_code >> (4 * seg + 2)) & 3ull) * p.a_lo_off + sub * 8;
        pnx::mbar_wait(&empty[stage], phase ^ 1);
        if (ptid == 0) {
          pnx::mbar_arrive_expect_tx(&full[stage], kBBytes);
          pnx::tma_load_2d(&wmap, &full[stage], sB + (size_t)stage * kBBytes, cc * 64 + wpiece * p.Cin, t * p.w_rows_per_tap + n0);
        }
        const uint32_t a_dst = pnx::smem_u32(sA + (size_t)stage * kABytes);
        const int* tbl = s_idx + t * 128;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int r = rsub + 16 * it;
          const int g = tbl[r];
          const __nv_bfloat16* src = p.A + (long long)(g < 0 ? 0 : g) * p.lda + acol;
          pnx::cp_async_16(a_dst + pnx::sw128_offset(r, sub), src, g < 0 ? 0u : 16u);
        }
        pnx::cp_async_mbar_arrive(&full[stage]);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumers: wgmma + epilogue
    if constexpr (!C::kStaged) pnx::regs_alloc<kConsumerRegs>();
    if constexpr (C::kWide) pnx::regs_alloc<kWideConsumerRegs>();
    uint32_t spass = 0;
    const int half = wg - 1;  // rows [64 * half, 64 * half + 64) of every tile
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int prev = 0;
      for (int kc = 0; kc < num_k; ++kc) {
        pnx::mbar_wait(&full[stage], phase);
        pnx::fence_proxy_async_smem();  // the cp.async rows were written through the generic proxy; wgmma reads async
        pnx::wgmma_fence();
        pnx::fence_acc(acc);
        const uint32_t a_base = pnx::smem_u32(sA + (size_t)stage * kABytes) + half * 64 * 128;
        const uint32_t b_base = pnx::smem_u32(sB + (size_t)stage * kBBytes);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t da = pnx::make_smem_desc_sw128(a_base + k * 32, 16, 1024);
          const uint32_t accumulate = (kc > 0 || k > 0) ? 1u : 0u;
          if constexpr (C::kWide) {
            // ptxas sizes one instruction's operands by the launch bound (128 registers at 512 threads), and an
            // m64n256 wgmma needs 154: two m64n128 on the column halves, same per-element sums
#pragma unroll
            for (int nh = 0; nh < 2; ++nh)
              pnx::Wgmma<128, 0, 0>::mma(*reinterpret_cast<float(*)[64]>(acc + 64 * nh), da,
                                         pnx::make_smem_desc_sw128(b_base + nh * 128 * 128 + k * 32, 16, 1024), accumulate);
          } else {
            pnx::Wgmma<BN, 0, 0>::mma(acc, da, pnx::make_smem_desc_sw128(b_base + k * 32, 16, 1024), accumulate);
          }
        }
        pnx::wgmma_commit();
        pnx::wgmma_wait<1>();  // the previous stage's MMAs are done: release it
        if (kc > 0 && lane == 0) pnx::mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      pnx::wgmma_wait<0>();
      pnx::fence_acc(acc);
      if (lane == 0) pnx::mbar_arrive(&empty[prev]);
      const long long row0 = (long long)tile * 128;
      const int nvalid = (int)min((long long)128, (long long)p.M - row0);
      if constexpr (C::kStaged)
        pnx::gemm_epilogue_stage<BN, kPasses, F>(acc, p.epi, row0, nvalid, half, n0, s_bias, stg, staged, sfree, spass);
      else
        pnx::gemm_epilogue<BN, F>(acc, p.epi, row0, nvalid, half, n0, s_bias, s_stat, s_bnc);
    }
    if constexpr (!C::kStaged) {
      named_bar_sync(2, 256);
      pnx::gemm_epilogue_flush<BN, F>(p.epi, n0, s_stat, p.bnr_red, p.bnr_C, threadIdx.x - 128, 256);
    }
  }
}

template <int BN, int F>
int launch_igemm_f(const CUtensorMap& wmap, const IgemmParams& p, int n_blocks, int sm_count, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    PNX_CUDA(cudaFuncSetAttribute(igemm_kernel<BN, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<BN, F>::kSmem));
    attr_set = true;
  }
  const int num_tiles = (p.M + 127) / 128;
  int gx = sm_count / n_blocks;
  if (gx < 1) gx = 1;
  if (gx > num_tiles) gx = num_tiles;
  dim3 grid(gx, n_blocks);
  igemm_kernel<BN, F><<<grid, Cfg<BN, F>::kThreads, Cfg<BN, F>::kSmem, stream>>>(wmap, p);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

template <int BN>
int launch_igemm(const CUtensorMap& wmap, const IgemmParams& p, int n_blocks, int sm_count, cudaStream_t stream) {
  if (p.epi.bnr_raw) {
    if constexpr (BN % 64 == 0) return launch_igemm_f<BN, 1>(wmap, p, n_blocks, sm_count, stream);
  }
  if (p.out_fp32 || p.epi.addend_f32) return launch_igemm_f<BN, 2>(wmap, p, n_blocks, sm_count, stream);
  return launch_igemm_f<BN, 0>(wmap, p, n_blocks, sm_count, stream);
}

}  // namespace

// Deterministic mode (library-wide switch): BatchNorm statistics produced by the GEMM epilogues (pnx_igemm,
// pnx_conv3x3_win) are accumulated in fp64 from per-warp partials instead of through fp32 shared-memory words that four
// warps add to in arrival order.  fp64 adds differ at 1e-16 whatever the order, so the statistics -- and with them the
// whole forward pass -- come out bit-identical from run to run.  Slower (one RED.F64 per warp, tile and channel); meant for
// debugging and regression hunting.  Returns the previous setting.
int g_pnx_deterministic = 0;
extern "C" int pnx_set_deterministic(int on) {
  const int prev = g_pnx_deterministic;
  g_pnx_deterministic = on ? 1 : 0;
  return prev;
}


// Contract: include/pnx.h (pnx_igemm).
extern "C" int pnx_igemm(const void* A, long long lda, long long a_rows, int M, int taps, int Cin, const void* Wpacked, int Cout,
                         int block_n, const int* nbr, int dense, int Hout, int Wout, int Hin, int Win, int kw,
                         int mul, int dil, int pad, void* out, long long ldc, int out_fp32, const float* bias,
                         double* stats, int stats_C, int stats_mod, int shuffle, int relu, const void* addend,
                         long long ld_add, int nseg, long long a_lo_off, long long seg_code, int addend_fp32,
                         const void* bnr_raw, long long bnr_ld, const float* bnr_scale, const float* bnr_shift,
                         const float* bnr_mean, const float* bnr_invstd, double* bnr_red, int bnr_C, int sm_count,
                         cudaStream_t stream) {
  PNX_CHECK_ARG(M >= 0, "M");
  if (M == 0) return PNX_OK;
  PNX_CHECK_ARG(taps >= 1 && taps <= 9, "taps in [1,9]");
  PNX_CHECK_ARG(Cin > 0 && Cin % 64 == 0, "Cin must be a multiple of 64");
  PNX_CHECK_ARG(Cout % block_n == 0, "Cout % block_n");
  PNX_CHECK_ARG(lda % 8 == 0 && ldc % 8 == 0, "lda/ldc must be multiples of 8 elements");
  PNX_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(Wpacked) & 15) == 0,
                "A/out/W must be 16-byte aligned");
  PNX_CHECK_ARG(!(nbr && dense), "nbr table and dense geometry are exclusive");
  PNX_CHECK_ARG(nbr || dense || taps == 1, "taps > 1 needs a neighbour table or dense geometry");
  PNX_CHECK_ARG(!shuffle || (block_n % 64 == 0 || 64 % block_n == 0), "shuffle store needs 64-channel groups");
  if (stats) PNX_CHECK_ARG(stats_C > 0 && stats_mod > 0, "stats_C/stats_mod");
  if (sm_count <= 0) sm_count = 132;
  IgemmParams p;
  p.A = (const __nv_bfloat16*)A;
  p.lda = lda;
  p.M = M; p.T = taps; p.Cin = Cin; p.w_rows_per_tap = Cout;
  p.nbr = nbr; p.dense = dense;
  p.Hout = Hout > 0 ? Hout : 1; p.Wout = Wout > 0 ? Wout : 1; p.Hin = Hin; p.Win = Win;
  p.kw = kw > 0 ? kw : 1; p.mul = mul; p.dil = dil; p.pad = pad;
  p.out_fp32 = out_fp32; p.bias = bias;
  pnx::EpiParams& e = p.epi;
  e.out = out; e.ldc = ldc; e.has_bias = bias != nullptr; e.relu = relu;
  e.stats = stats; e.stats_C = stats_C; e.stats_mod = stats_mod > 0 ? stats_mod : 1 << 30;
  e.stats_direct = g_pnx_deterministic;
  e.shuffle = shuffle; e.Hout = p.Hout; e.Wout = p.Wout;
  e.addend = addend_fp32 ? nullptr : (const __nv_bfloat16*)addend;
  e.addend_f32 = addend_fp32 ? (const float*)addend : nullptr;
  e.ld_add = ld_add;
  e.bnr_raw = (const __nv_bfloat16*)bnr_raw; e.bnr_ld = bnr_ld;
  PNX_CHECK_ARG(!(addend && shuffle), "addend is not supported with the pixel-shuffle store");
  PNX_CHECK_ARG(!addend || (ld_add % 2 == 0 && (reinterpret_cast<uintptr_t>(addend) & 7) == 0), "addend: even row stride, 8-byte aligned");
  PNX_CHECK_ARG(nseg >= 1 && nseg <= 9, "nseg in [1,9]");
  int a_pieces = 1, w_pieces = 1;
  for (int sgi = 0; sgi < nseg; ++sgi) {
    const int ap = (int)((seg_code >> (4 * sgi + 2)) & 3), wp = (int)((seg_code >> (4 * sgi)) & 3);
    PNX_CHECK_ARG(ap <= 2 && wp <= 2, "segment code: piece index <= 2");
    if (ap + 1 > a_pieces) a_pieces = ap + 1;
    if (wp + 1 > w_pieces) w_pieces = wp + 1;
  }
  PNX_CHECK_ARG(nseg > 1 || seg_code == 0, "nseg = 1 is the plain bf16 path (segment code 0)");
  PNX_CHECK_ARG(a_pieces == 1 || (a_lo_off >= Cin && a_lo_off % 64 == 0 && (a_pieces - 1) * a_lo_off + Cin <= lda), "split mode: a_lo_off");
  PNX_CHECK_ARG(!addend_fp32 || out_fp32, "an fp32 addend needs an fp32 output");
  p.nseg = nseg; p.a_lo_off = (int)a_lo_off; p.seg_code = (unsigned long long)seg_code;
  p.bnr_scale = bnr_scale; p.bnr_shift = bnr_shift;
  p.bnr_mean = bnr_mean; p.bnr_invstd = bnr_invstd; p.bnr_red = bnr_red; p.bnr_C = bnr_C;
  if (bnr_raw) {
    PNX_CHECK_ARG(!out_fp32 && !shuffle && !stats && block_n % 64 == 0, "fused BN-backward reduce: bf16 output without forward statistics");
    PNX_CHECK_ARG(bnr_scale && bnr_shift && bnr_mean && bnr_invstd && bnr_red && bnr_C == Cout && bnr_ld % 8 == 0 &&
                      (reinterpret_cast<uintptr_t>(bnr_raw) & 15) == 0, "fused BN-backward reduce: arguments");
  }
  const int wcols = w_pieces * Cin;  // split mode: W rows are [piece 0 | piece 1 | ...]
  CUtensorMap wmap;
  int rc = pnx_encode_tmap_2d_bf16(&wmap, Wpacked, (uint64_t)taps * Cout, (uint64_t)wcols, (uint64_t)wcols * 2,
                                   (uint32_t)block_n, 64);
  if (rc) return rc;
  PNX_CHECK_ARG(a_rows >= 1 && a_rows < 0x7fffffffLL, "a_rows = number of rows of A");
  const int n_blocks = Cout / block_n;
  switch (block_n) {
    case 16: return launch_igemm<16>(wmap, p, n_blocks, sm_count, stream);
    case 32: return launch_igemm<32>(wmap, p, n_blocks, sm_count, stream);
    case 64: return launch_igemm<64>(wmap, p, n_blocks, sm_count, stream);
    case 128: return launch_igemm<128>(wmap, p, n_blocks, sm_count, stream);
    case 192: return launch_igemm<192>(wmap, p, n_blocks, sm_count, stream);
    case 256: return launch_igemm<256>(wmap, p, n_blocks, sm_count, stream);
    default:
      pnx_set_error("pnx_igemm: unsupported block_n %d (16/32/64/128/192/256)", block_n);
      return PNX_ERR_ARG;
  }
}
