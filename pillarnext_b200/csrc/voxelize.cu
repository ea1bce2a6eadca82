// voxelize.cu -- dynamic point->pillar voxelizer (rows V1-V3 of SURVEY.md section 8a) for sm_90a.
//
// Replaces, bit-exactly on the indices, reference det3d/models/readers/pillar_encoder.py:86-125:
//   (xyz-min)/voxel (fp32 sub + IEEE fp32 divide), float-domain range test on x,y only, trunc,
//   torch.unique(dim=0, return_inverse=True) over (b, xi, yi)   [lexicographically sorted]
// WITHOUT a sort: the BEV grid is bounded (B*Gx*Gy cells), so occupancy is a direct-address bitmap
// laid out in the reference's sort order (bit index = (b*Gx + xi)*GyPad + yi); the rank of a set
// bit IS the sorted-unique pillar id, i.e. `unq_inv`.  Ranks are hierarchical so that no dense prefix
// array is ever written: per 32-word block (1024 cells) a count is maintained by the marking kernel
// itself (one extra atomic per NEW pillar), one small scan turns the counts into block offsets, and
//   rank(cell) = blockpref[block] + popc(words before it in the block) + popc(bits below it).
// Index generation = 4 kernels: mark | scan(block counts) | rank | coords.
// pnx_bucketize then groups points by pillar (CSR, ascending point id inside a bucket) so every later
// per-pillar reduction (mean, max) is a plain in-order loop -- no atomics on any reduction.
//
// HBM traffic (algorithmic, SURVEY 8d): 24 B/point read + 4 B/point pillar id + 12 B/pillar coords.
#include "pnx_common.cuh"

namespace {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

__device__ __forceinline__ int warp_incl_scan(int v) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, o);
    if ((int)pnx::lane_id() >= o) v += t;
  }
  return v;
}

// block-wide exclusive scan of one value per thread; returns exclusive prefix, total in *total
template <int kThreads>
__device__ __forceinline__ int block_excl_scan(int v, int* total) {
  __shared__ int wsum[kThreads / 32];
  __shared__ int wtot;
  int incl = warp_incl_scan(v);
  int w = threadIdx.x >> 5;
  if (pnx::lane_id() == 31) wsum[w] = incl;
  __syncthreads();
  if (w == 0) {
    int s = (pnx::lane_id() < kThreads / 32) ? wsum[pnx::lane_id()] : 0;
    int si = warp_incl_scan(s);
    if (pnx::lane_id() < kThreads / 32) wsum[pnx::lane_id()] = si - s;
    if (pnx::lane_id() == kThreads / 32 - 1) wtot = si;
  }
  __syncthreads();
  int r = incl - v + wsum[w];
  *total = wtot;
  __syncthreads();
  return r;
}

template <bool kPopc>
__device__ __forceinline__ int scan_val(const uint32_t* in, int i, int n) {
  if (i >= n) return 0;
  return kPopc ? __popc(in[i]) : (int)in[i];
}

template <bool kPopc>
__global__ void scan_reduce_kernel(const uint32_t* __restrict__ in, int n, int* __restrict__ block_sums) {
  int base = blockIdx.x * kScanTile;
  int s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) s += scan_val<kPopc>(in, base + k * kScanThreads + threadIdx.x, n);
  int tot;
  block_excl_scan<kScanThreads>(s, &tot);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}

__global__ void scan_top_kernel(int* __restrict__ block_sums, int n_blocks, int* __restrict__ total_out) {
  int carry = 0;
  for (int base = 0; base < n_blocks; base += kScanThreads) {
    int i = base + threadIdx.x;
    int v = i < n_blocks ? block_sums[i] : 0;
    int tot;
    int ex = block_excl_scan<kScanThreads>(v, &tot);
    if (i < n_blocks) block_sums[i] = ex + carry;
    carry += tot;
  }
  if (threadIdx.x == 0 && total_out) *total_out = carry;
}

template <bool kPopc>
__global__ void scan_apply_kernel(const uint32_t* __restrict__ in, int n, const int* __restrict__ block_sums,
                                  int* __restrict__ out) {
  // items are distributed so that thread t owns kScanItems CONSECUTIVE elements
  int base = blockIdx.x * kScanTile + threadIdx.x * kScanItems;
  int v[kScanItems];
  int s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    v[k] = scan_val<kPopc>(in, base + k, n);
    s += v[k];
  }
  int tot;
  int ex = block_excl_scan<kScanThreads>(s, &tot) + block_sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) out[base + k] = ex;
    ex += v[k];
  }
  if (base <= n && n < base + kScanItems) out[n] = ex;  // total (exclusive prefix at n)
}

// Exclusive scan of per-block counts, two-level: `counts` holds n_blocks block counts followed (at n_blocks
// rounded up to 4, see super_offset) by one count per superblock of 1024 blocks (maintained by the same atomics /
// warps that produce the block counts).  One CTA per superblock: prefix of the earlier superblocks (<= a few
// hundred adds) + one 1024-wide block scan.  One launch, all SMs.
constexpr int kSuper = 1024;
__host__ __device__ inline int super_offset(int n_blocks) { return (n_blocks + 3) / 4 * 4; }

__global__ void __launch_bounds__(kSuper) scan_blocks_kernel(const int* __restrict__ counts, int n_blocks,
                                                             int* __restrict__ out, int* __restrict__ total_out) {
  __shared__ int s_base;
  const int* supercnt = counts + super_offset(n_blocks);
  const int sb = blockIdx.x;
  if (threadIdx.x < 32) {
    int acc = 0;
    for (int j = threadIdx.x; j < sb; j += 32) acc += supercnt[j];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (threadIdx.x == 0) s_base = acc;
  }
  __syncthreads();
  const int i = sb * kSuper + threadIdx.x;
  const int v = i < n_blocks ? counts[i] : 0;
  int tot;
  const int ex = block_excl_scan<kSuper>(v, &tot) + s_base;
  if (i < n_blocks) out[i] = ex;
  if (sb == gridDim.x - 1 && threadIdx.x == 0) {
    out[n_blocks] = s_base + tot;
    if (total_out) *total_out = s_base + tot;
  }
}

}  // namespace

// Exclusive prefix sum of popcounts (popc=1) or raw int32 values (popc=0).
// out has n+1 entries (out[n] = total); block_sums scratch needs ceil((n+1)/2048)+1 ints.
extern "C" int pnx_scan_u32(const uint32_t* in, int n, int popc, int* out, int* block_sums, int* total_out,
                            cudaStream_t stream) {
  PNX_CHECK_ARG(n >= 0, "n < 0");
  int nb = pnx_cdiv(n + 1, kScanTile);  // +1 so the thread owning index n exists
  if (popc) {
    scan_reduce_kernel<true><<<nb, kScanThreads, 0, stream>>>(in, n, block_sums);
    scan_top_kernel<<<1, kScanThreads, 0, stream>>>(block_sums, nb, total_out);
    scan_apply_kernel<true><<<nb, kScanThreads, 0, stream>>>(in, n, block_sums, out);
  } else {
    scan_reduce_kernel<false><<<nb, kScanThreads, 0, stream>>>(in, n, block_sums);
    scan_top_kernel<<<1, kScanThreads, 0, stream>>>(block_sums, nb, total_out);
    scan_apply_kernel<false><<<nb, kScanThreads, 0, stream>>>(in, n, block_sums, out);
  }
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

// Size (in int32) of a block-count buffer: block counts + superblock counts (see scan_blocks_kernel).
extern "C" int pnx_blockcnt_size(int n_blocks) { return super_offset(n_blocks) + (n_blocks + kSuper - 1) / kSuper + 4; }

// Exclusive scan of the per-block counts of a bitmap in ONE launch.  counts = pnx_blockcnt_size(n_blocks) ints
// (block counts + superblock counts); out [n_blocks+1] (out[n_blocks] = total), total_out optional.
extern "C" int pnx_scan_blocks(const int* counts, int n_blocks, int* out, int* total_out, cudaStream_t stream) {
  PNX_CHECK_ARG(n_blocks >= 1, "n_blocks");
  scan_blocks_kernel<<<(n_blocks + kSuper - 1) / kSuper, kSuper, 0, stream>>>(counts, n_blocks, out, total_out);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

namespace {

struct VoxGeom {
  float min_x, min_y, vs_x, vs_y;
  int gx, gy, vwords, batch;
};

// V1: cell index per point + occupancy bitmap.  Persistent kernel, one CTA of 1024 threads per SM: every CTA streams a
// contiguous chunk of the points through a 3-stage shared-memory ring filled by TMA bulk copies (cp.async.bulk,
// 24 KB = 1024 points per stage, one elected thread issues, mbarrier completion), so HBM requests stay in flight while
// the previous stage is being processed.  One point per thread per stage: bit-exact cell arithmetic, one
// fire-and-forget RED.OR into the bitmap, the cell id stored for the rank pass.
constexpr int kVoxThreads = 1024;
constexpr int kVoxStagePts = 1024;
constexpr int kVoxStages = 3;
constexpr int kVoxStageBytes = kVoxStagePts * 24;

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   pnx::smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(pnx::smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ int vox_cell(const float* p, const VoxGeom& g) {
  const float bf = p[0], x = p[1], y = p[2];
  // pillar_encoder.py:95-96 -- fp32 subtract then true fp32 division (no reciprocal, no FMA)
  const float cx = __fdiv_rn(__fsub_rn(x, g.min_x), g.vs_x);
  const float cy = __fdiv_rn(__fsub_rn(y, g.min_y), g.vs_y);
  // :98-101 -- range test in the float domain, x/y only (NaN fails every comparison)
  bool keep = (cx >= 0.f) && (cx < (float)g.gx) && (cy >= 0.f) && (cy < (float)g.gy);
  const int b = (int)bf;  // :107 .long() truncation
  keep = keep && (b >= 0) && (b < g.batch);
  if (!keep) return -1;
  const int xi = (int)cx, yi = (int)cy;  // :106 trunc
  return ((b * g.gx + xi) * g.vwords + (yi >> 5)) * 32 + (yi & 31);
}

__global__ void __launch_bounds__(kVoxThreads, 1) vox_mark_kernel(const float* __restrict__ points, int n, int pts_per_cta,
                                                                  VoxGeom g, uint32_t* __restrict__ bitmap,
                                                                  int* __restrict__ cell_of_point) {
  extern __shared__ __align__(128) uint8_t vsm[];
  float* ring = reinterpret_cast<float*>(vsm);                                         // [kVoxStages][1024 pts][6]
  uint64_t* full = reinterpret_cast<uint64_t*>(vsm + kVoxStages * kVoxStageBytes);     // [kVoxStages]
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < kVoxStages; ++s) pnx::mbar_init(&full[s], 1);
    pnx::fence_barrier_init();
  }
  __syncthreads();
  const long long p0 = (long long)blockIdx.x * pts_per_cta;
  const long long p1 = min((long long)n, p0 + pts_per_cta);
  const int n_stage = p1 > p0 ? (int)((p1 - p0 + kVoxStagePts - 1) / kVoxStagePts) : 0;
  auto stage_pts = [&](int it) { return (int)min((long long)kVoxStagePts, p1 - (p0 + (long long)it * kVoxStagePts)); };
  auto issue = [&](int it) {   // thread 0: a full stage = one bulk copy
    const int s = it % kVoxStages;
    pnx::mbar_arrive_expect_tx(&full[s], kVoxStageBytes);
    bulk_g2s(ring + (size_t)s * kVoxStagePts * 6, points + (p0 + (long long)it * kVoxStagePts) * 6, kVoxStageBytes, &full[s]);
  };
  if (tid == 0)
    for (int it = 0; it < min(n_stage, kVoxStages); ++it)
      if (stage_pts(it) == kVoxStagePts) issue(it);
  for (int it = 0; it < n_stage; ++it) {
    const int s = it % kVoxStages;
    const int np = stage_pts(it);
    float* st = ring + (size_t)s * kVoxStagePts * 6;
    if (np == kVoxStagePts) {
      pnx::mbar_wait(&full[s], (uint32_t)((it / kVoxStages) & 1));
    } else {  // ragged tail of the whole array (at most one stage of one CTA): plain coalesced loads
      const float* src = points + (p0 + (long long)it * kVoxStagePts) * 6;
      for (int q = tid; q < np * 6; q += kVoxThreads) st[q] = __ldg(src + q);
      __syncthreads();
    }
    if (tid < np) {
      const int cell = vox_cell(st + tid * 6, g);
      // fire-and-forget reduction: `atomicOr` with an unused result still compiles to ATOMG (a round trip per point,
      // measured 3x slower for this pass); red.* is the REDG instruction.  Warp-level aggregation of same-word marks
      // (__match_any_sync + __reduce_or_sync, one RED per distinct word) was measured too: 78 -> 188 us -- MATCH.ANY costs
      // more than the REDs it saves, L2 absorbs the duplicates.
      if (cell >= 0) asm volatile("red.relaxed.gpu.global.or.b32 [%0], %1;" ::"l"(bitmap + (cell >> 5)), "r"(1u << (cell & 31)) : "memory");
      cell_of_point[p0 + (long long)it * kVoxStagePts + tid] = cell;
    }
    __syncthreads();  // everyone has read stage s
    if (tid == 0 && it + kVoxStages < n_stage && stage_pts(it + kVoxStages) == kVoxStagePts) issue(it + kVoxStages);
  }
}

// pillars per 32-word block = popcount of the block, and the in-block exclusive prefix of every word (inblk: used by the
// rank kernel and the rulebook).  One warp per group of kCntU blocks: kCntU coalesced 128-byte reads in flight per warp.
constexpr int kCntU = 4;
__global__ void __launch_bounds__(256) vox_blockcnt_kernel(const uint32_t* __restrict__ bitmap, int n_blocks,
                                                           int* __restrict__ blockcnt, uint16_t* __restrict__ inblk) {
  const int lane = threadIdx.x & 31;
  const long long blk0 = (((long long)blockIdx.x * 256 + threadIdx.x) >> 5) * kCntU;
  if (blk0 >= n_blocks) return;
  uint32_t w[kCntU];
#pragma unroll
  for (int u = 0; u < kCntU; ++u) w[u] = blk0 + u < n_blocks ? __ldg(bitmap + (size_t)(blk0 + u) * 32 + lane) : 0u;
#pragma unroll
  for (int u = 0; u < kCntU; ++u) {
    if (blk0 + u >= n_blocks) break;
    const int c = __popc(w[u]);
    const int incl = warp_incl_scan(c);
    inblk[(size_t)(blk0 + u) * 32 + lane] = (uint16_t)(incl - c);
    if (lane == 31) blockcnt[blk0 + u] = incl;
  }
}

// per-superblock (1024 blocks) totals of the block counts (only ~B*100 counters: atomics from the marking kernel
// would all collide on them)
__global__ void super_reduce_kernel(const int* __restrict__ blockcnt, int n_blocks, int* __restrict__ supercnt) {
  __shared__ int red[8];
  const int base = blockIdx.x * 1024;
  int acc = 0;
  for (int k = threadIdx.x; k < 1024; k += 256) acc += (base + k < n_blocks) ? blockcnt[base + k] : 0;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int k = 0; k < 8; ++k) t += red[k];
    supercnt[blockIdx.x] = t;
  }
}

// V2b: pillar id per point (= hierarchical rank of its bit) and per-pillar point counts.
__global__ void vox_rank_kernel(const int* __restrict__ cell_of_point, int n, const uint32_t* __restrict__ bitmap,
                                const int* __restrict__ blockpref, const uint16_t* __restrict__ inblk,
                                int* __restrict__ pillar_of_point, uint32_t* __restrict__ bucket_cnt) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int cell = cell_of_point[i];
  int pid = -1;
  if (cell >= 0) {
    const int word = cell >> 5, bit = cell & 31;
    pid = blockpref[word >> 5] + (int)inblk[word] + __popc(bitmap[word] & ((1u << bit) - 1u));
    if (bucket_cnt)  // integer count: order-independent; red.* = REDG (atomicAdd with an unused result compiles to ATOMG)
      asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(bucket_cnt + pid) : "memory");
  }
  pillar_of_point[i] = pid;
}

// V2c: coords (b, yi, xi) of every pillar in sorted-unique order.  One warp per kCoU 32-word blocks (coalesced 128-byte
// reads, issued together with the block prefixes).  The pillars of a block are consecutive rows of `coords`: they are
// staged in shared memory and written with coalesced stores.
constexpr int kCoordStage = 128;   // pillars of one block staged per warp (3 ints each); denser blocks take the direct path
constexpr int kCoU = 4;            // blocks per warp, all their loads in flight together (the kernel was load-latency bound:
                                   // blockpref -> bitmap/inblk -> store, one block per warp: 98 us for 452 k blocks)
__global__ void __launch_bounds__(256) vox_coords_kernel(const uint32_t* __restrict__ bitmap, const int* __restrict__ blockpref,
                                                         int n_blocks, VoxGeom g, int* __restrict__ coords, int cap,
                                                         const uint16_t* __restrict__ inblk) {
  __shared__ int s_stage[8 * kCoordStage * 3];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long blk0 = (((long long)blockIdx.x * 256 + threadIdx.x) >> 5) * kCoU;
  if (blk0 >= n_blocks) return;
  int base_idx[kCoU], total[kCoU], pre[kCoU];
  uint32_t bits[kCoU];
#pragma unroll
  for (int u = 0; u < kCoU; ++u) {
    const bool ok = blk0 + u < n_blocks;
    const long long blk = ok ? blk0 + u : blk0;
    base_idx[u] = __ldg(blockpref + blk);
    total[u] = ok ? __ldg(blockpref + blk + 1) : 0;
    bits[u] = __ldg(bitmap + blk * 32 + lane);
    pre[u] = (int)__ldg(inblk + blk * 32 + lane);
  }
#pragma unroll
  for (int u = 0; u < kCoU; ++u) {
    const int tot = total[u] - (blk0 + u < n_blocks ? base_idx[u] : 0);
    if (blk0 + u >= n_blocks || tot <= 0) continue;
    const int w = (int)(blk0 + u) * 32 + lane;
    uint32_t bw = bits[u];
    const int row = w / g.vwords, vw = w - row * g.vwords;
    const int b = row / g.gx, xi = row - b * g.gx;
    if (tot <= kCoordStage && base_idx[u] + tot <= cap) {
      int* cs = s_stage + warp * (kCoordStage * 3);
      int k = pre[u];
      while (bw) {
        const int bit = __ffs(bw) - 1;
        bw &= bw - 1;
        cs[k * 3 + 0] = b;
        cs[k * 3 + 1] = vw * 32 + bit;  // yi
        cs[k * 3 + 2] = xi;
        ++k;
      }
      __syncwarp();
      int* dst = coords + (size_t)base_idx[u] * 3;
      for (int q = lane; q < tot * 3; q += 32) dst[q] = cs[q];
      __syncwarp();
    } else {
      int idx = base_idx[u] + pre[u];
      while (bw) {
        const int bit = __ffs(bw) - 1;
        bw &= bw - 1;
        if (idx < cap) {
          coords[(size_t)idx * 3 + 0] = b;
          coords[(size_t)idx * 3 + 1] = vw * 32 + bit;  // yi
          coords[(size_t)idx * 3 + 2] = xi;
        }
        ++idx;
      }
    }
  }
}

// V3a: place points into their pillar's bucket (slot order is arbitrary here ...)
__global__ void vox_fill_kernel(const int* __restrict__ pillar_of_point, int n, const int* __restrict__ bucket_off,
                                uint32_t* __restrict__ cursor, int* __restrict__ bucket_tmp) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int pid = pillar_of_point[i];
  if (pid < 0) return;
  uint32_t slot = atomicAdd(&cursor[pid], 1u);
  bucket_tmp[bucket_off[pid] + slot] = i;
}
// V3b: ... and made deterministic: each entry is moved to its rank (ascending point id) in the bucket.
__global__ void vox_sort_kernel(const int* __restrict__ bucket_tmp, const int* __restrict__ pillar_of_point,
                                const int* __restrict__ bucket_off, int nv_cap, const int* __restrict__ nv_ptr,
                                int* __restrict__ bucket_pts) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= *nv_ptr || q >= nv_cap) return;
  int i = bucket_tmp[q];
  int pid = pillar_of_point[i];
  int lo = bucket_off[pid], hi = bucket_off[pid + 1];
  int rank = 0;
  for (int k = lo; k < hi; ++k) rank += (bucket_tmp[k] < i);
  bucket_pts[lo + rank] = i;
}

// =====================================================================================================================
// Frame-tiled index generation (round 2).  The global-bitmap pipeline above issues one random RED.OR per point into L2 and
// three random L2 reads per point in the rank pass; both are bounded by the L2 transaction rate (measured ~100 G RED/s,
// ~350 G random reads/s), which caps it near 0.2 of the HBM roofline whatever the streaming side does.  Here a SLICE of one
// frame's occupancy bitmap lives in the shared memory of a CTA (a nuScenes frame is 226 KB = 2 slices of 113 KB), so marking
// and ranking are LOCAL shared-memory operations and HBM/L2 only see streaming traffic:
//   bounds  off[b] = first point of frame b (1024-ary search on the batch column; collate order = grouped by frame)
//   mark    CTA (b, s) streams ALL points of frame b (cp.async.bulk ring; the second slice's read is an L2 hit), ORs the
//           ones that fall into slice s into its bitmap, stores their cell ids, then writes bitmap / in-block prefixes /
//           block counts with coalesced stores (no memset pass, no re-read)
//   scan    exclusive scan of the per-CTA pillar counts (one small CTA)
//   rank    CTA (b, s) reloads its slice (L2), rebuilds the prefixes in shared memory, emits blockpref and the sorted-unique
//           coords, streams the frame's cell ids and turns the ones of its slice into pillar ids with three shared-memory reads
// A first version kept ONE copy of the frame's points per cluster and marked / ranked through distributed shared memory
// (red / ld.shared::cluster): bit-exact, but remote 4-byte transactions retire at only ~50-60 G/s chip-wide -- slower than
// the L2 atomics they were meant to replace (rank 379 us, mark 153 us for 7.68 M points) -- so the slices read the points
// redundantly from L2 instead and every fine-grained access is local.
// Input order is VERIFIED, not assumed: a point whose batch index disagrees with the frame range it lies in, or bounds
// that are not monotone, raise scratch[0] (the caller checks it at its next synchronisation and must then use
// pnx_voxelize, which takes any order).  Outputs are identical to pnx_voxelize (same tests).
constexpr int kFrThreads = 1024;
constexpr int kFrStagePts = 512;                      // points per ring stage (12 KB bulk copy)
constexpr int kFrStageBytes = kFrStagePts * 24;
constexpr int kFrMaxStages = 8;                       // the ring takes what the bitmap slice leaves of the shared memory
constexpr int kFrMinStages = 4;
constexpr int kFrMaxSlices = 8;

struct FrameCfg {
  int W;       // bitmap words per frame (multiple of 32)
  int nblk;    // 32-word blocks per frame
  int bpc;     // blocks per slice
  int cs;      // slices per frame
  int cstage;  // pillars of one block staged per warp for the coords store
  int stages;  // ring depth of the mark kernel
};

__device__ __forceinline__ void red_or_shared(uint32_t* addr, uint32_t v) {
  asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(pnx::smem_u32(addr)), "r"(v) : "memory");
}

__device__ __forceinline__ void frame_range(const int* __restrict__ off, int b, int batch, int n, long long* p0, long long* p1) {
  // frame 0 also owns the points in front of it, the last frame those behind it (batch index outside [0, batch): dropped)
  long long a = b == 0 ? 0 : off[b], e = b == batch - 1 ? n : off[b + 1];
  a = a < 0 ? 0 : (a > n ? n : a);
  e = e < a ? a : (e > n ? n : e);
  *p0 = a;
  *p1 = e;
}

__global__ void __launch_bounds__(1024) vox_frame_bounds_kernel(const float* __restrict__ points, int n, int* __restrict__ off,
                                                               int* __restrict__ status) {
  __shared__ int s_first;
  const int b = blockIdx.x;
  int lo = 0, hi = n;  // the answer lies in [lo, hi]
  while (lo < hi) {
    const int span = hi - lo;
    const int step = (span + 1023) / 1024;
    const int nsamp = (span + step - 1) / step;
    if (threadIdx.x == 0) s_first = 0x7fffffff;
    __syncthreads();
    if ((int)threadIdx.x < nsamp && (int)__ldg(points + ((long long)lo + (long long)threadIdx.x * step) * 6) >= b)
      atomicMin(&s_first, (int)threadIdx.x);
    __syncthreads();
    const int t = s_first;
    __syncthreads();
    if (t == 0x7fffffff) {
      lo = lo + (nsamp - 1) * step + 1;
    } else {
      hi = lo + t * step;
      lo = t > 0 ? hi - step + 1 : hi;
    }
  }
  if (threadIdx.x == 0) {
    off[b] = lo;
    if (b == 0) *status = 0;
  }
}

__global__ void __launch_bounds__(kFrThreads, 1) vox_frame_mark_kernel(const float* __restrict__ points, int n, VoxGeom g, FrameCfg f,
                                                                       const int* __restrict__ off, uint32_t* __restrict__ bitmap,
                                                                       uint16_t* __restrict__ inblk, int* __restrict__ blockcnt,
                                                                       int* __restrict__ cell_of_point, int* __restrict__ cta_cnt,
                                                                       int* __restrict__ status) {
  extern __shared__ __align__(128) uint8_t fsm[];
  const int words = f.bpc * 32;
  uint32_t* bits = reinterpret_cast<uint32_t*>(fsm);
  float* ring = reinterpret_cast<float*>(fsm + (size_t)words * 4);
  uint64_t* full = reinterpret_cast<uint64_t*>(fsm + (size_t)words * 4 + (size_t)f.stages * kFrStageBytes);
  const int S = f.stages;
  __shared__ int s_warp_cnt[kFrThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x / f.cs, r = blockIdx.x - b * f.cs;
  for (int i = tid; i < words / 4; i += kFrThreads) reinterpret_cast<uint4*>(bits)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (tid == 0) {
    for (int s = 0; s < S; ++s) pnx::mbar_init(&full[s], 1);
    pnx::fence_barrier_init();
  }
  __syncthreads();
  long long p0, p1;
  frame_range(off, b, g.batch, n, &p0, &p1);
  const int w_lo = r * words;
  auto process = [&](const float* p, long long i) {
    const float cx = __fdiv_rn(__fsub_rn(p[1], g.min_x), g.vs_x);
    const float cy = __fdiv_rn(__fsub_rn(p[2], g.min_y), g.vs_y);
    const bool inside = (cx >= 0.f) && (cx < (float)g.gx) && (cy >= 0.f) && (cy < (float)g.gy);
    const int pb = (int)p[0];
    if (pb != b) {  // a point of another frame inside this frame's range: the input is not grouped
      if (r == 0) {
        if (pb >= 0 && pb < g.batch) atomicAdd(status, 1);
        cell_of_point[i] = -1;
      }
    } else if (!inside) {
      if (r == 0) cell_of_point[i] = -1;
    } else {
      const int xi = (int)cx, yi = (int)cy;
      const int loc = xi * g.vwords + (yi >> 5) - w_lo;
      if (loc >= 0 && loc < words) {  // this slice owns the cell: mark it and publish the cell id
        red_or_shared(bits + loc, 1u << (yi & 31));
        cell_of_point[i] = ((b * g.gx + xi) * g.vwords + (yi >> 5)) * 32 + (yi & 31);
      }
    }
  };
  if ((p0 & 1) && p0 < p1) {  // odd first point: one plain load, then every stage starts 16-byte aligned (a point is 24 B)
    if (tid == 0) {
      float q[3];
      for (int k = 0; k < 3; ++k) q[k] = __ldg(points + p0 * 6 + k);
      process(q, p0);
    }
    ++p0;
  }
  // ring of S stages of 512 points: S - 1 bulk copies stay in flight while one stage is processed (the loop is otherwise
  // latency-bound: one 1024-point stage per ~1.3 us with a 2-deep ring, measured)
  const int n_stage = p1 > p0 ? (int)((p1 - p0 + kFrStagePts - 1) / kFrStagePts) : 0;
  auto stage_pts = [&](int it) { return (int)min((long long)kFrStagePts, p1 - (p0 + (long long)it * kFrStagePts)); };
  auto issue = [&](int it) {
    const int s = it % S;
    pnx::mbar_arrive_expect_tx(&full[s], kFrStageBytes);
    bulk_g2s(ring + (size_t)s * kFrStagePts * 6, points + (p0 + (long long)it * kFrStagePts) * 6, kFrStageBytes, &full[s]);
  };
  if (tid == 0)
    for (int it = 0; it < min(n_stage, S); ++it)
      if (stage_pts(it) == kFrStagePts) issue(it);
  for (int it = 0; it < n_stage; ++it) {
    const int s = it % S;
    const int np = stage_pts(it);
    float* st = ring + (size_t)s * kFrStagePts * 6;
    if (np == kFrStagePts) {
      pnx::mbar_wait(&full[s], (uint32_t)((it / S) & 1));
    } else {  // ragged last stage of the frame: plain coalesced loads
      const float* src = points + (p0 + (long long)it * kFrStagePts) * 6;
      for (int q = tid; q < np * 6; q += kFrThreads) st[q] = __ldg(src + q);
      __syncthreads();
    }
    if (tid < np) process(st + tid * 6, p0 + (long long)it * kFrStagePts + tid);
    __syncthreads();
    if (tid == 0 && it + S < n_stage && stage_pts(it + S) == kFrStagePts) issue(it + S);
  }
  __syncthreads();
  // ---- block popcounts + in-block prefixes, bitmap written once, coalesced
  int mine = 0;
  for (int lb = warp; lb < f.bpc; lb += kFrThreads / 32) {
    const int fb = r * f.bpc + lb;
    if (fb >= f.nblk) break;
    const uint32_t w = bits[lb * 32 + lane];
    const int c = __popc(w);
    const int incl = warp_incl_scan(c);
    const size_t gw = ((size_t)b * f.nblk + fb) * 32 + lane;
    bitmap[gw] = w;
    inblk[gw] = (uint16_t)(incl - c);
    if (lane == 31) {
      blockcnt[(size_t)b * f.nblk + fb] = incl;
      mine += incl;
    }
  }
  if (lane == 31) s_warp_cnt[warp] = mine;
  __syncthreads();
  if (warp == 0) {
    int v = s_warp_cnt[lane];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) cta_cnt[blockIdx.x] = v;
  }
}

// exclusive scan of the per-CTA pillar counts (n_cta = batch * slices values) + the monotonicity check of the bounds
__global__ void __launch_bounds__(1024) vox_frame_scan_kernel(const int* __restrict__ cta_cnt, int n_cta, int* __restrict__ cta_base,
                                                             const int* __restrict__ off, int batch, int n, int* __restrict__ status,
                                                             int* __restrict__ blockpref_total, int* __restrict__ total_out) {
  int carry = 0;
  for (int base = 0; base < n_cta; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < n_cta ? cta_cnt[i] : 0;
    int tot;
    const int ex = block_excl_scan<1024>(v, &tot);
    if (i < n_cta) cta_base[i] = ex + carry;
    carry += tot;
  }
  if (threadIdx.x == 0) {
    *blockpref_total = carry;
    if (total_out) *total_out = carry;
  }
  int bad = 0;
  for (int b = threadIdx.x; b < batch; b += 1024) bad += (off[b] > off[b + 1]) || off[b] < 0 || off[b + 1] > n;
  if (bad) atomicAdd(status, bad);
}

__global__ void __launch_bounds__(kFrThreads, 1) vox_frame_rank_kernel(int n, VoxGeom g, FrameCfg f, const int* __restrict__ off,
                                                                       const uint32_t* __restrict__ bitmap, const int* __restrict__ cta_base,
                                                                       const int* __restrict__ cell_of_point, int* __restrict__ blockpref,
                                                                       int* __restrict__ pillar_of_point, int* __restrict__ coords, int cap,
                                                                       uint32_t* __restrict__ bucket_cnt) {
  extern __shared__ __align__(128) uint8_t fsm[];
  const int words = f.bpc * 32;
  uint32_t* bits = reinterpret_cast<uint32_t*>(fsm);
  uint16_t* inb = reinterpret_cast<uint16_t*>(fsm + (size_t)words * 4);
  int* bpref = reinterpret_cast<int*>(fsm + (size_t)words * 6);                                   // [bpc + 1]
  int* stage = reinterpret_cast<int*>(fsm + (size_t)words * 6 + ((size_t)f.bpc + 4) / 4 * 16);  // [32 warps][cstage * 3]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x / f.cs, r = blockIdx.x - b * f.cs;
  const int my_blocks = max(0, min(f.bpc, f.nblk - r * f.bpc));
  // A: slice of the bitmap -> shared memory, in-block prefixes, block counts (kA blocks per warp in flight: the loop
  //    is load-latency bound otherwise)
  constexpr int kA = 8;
  for (int lb0 = warp * kA; lb0 < f.bpc; lb0 += (kFrThreads / 32) * kA) {
    uint32_t w[kA];
#pragma unroll
    for (int u = 0; u < kA; ++u)
      w[u] = (lb0 + u < my_blocks) ? __ldg(bitmap + ((size_t)b * f.nblk + r * f.bpc + lb0 + u) * 32 + lane) : 0u;
#pragma unroll
    for (int u = 0; u < kA; ++u) {
      const int lb = lb0 + u;
      if (lb >= f.bpc) break;
      const int c = __popc(w[u]);
      const int incl = warp_incl_scan(c);
      bits[lb * 32 + lane] = w[u];
      inb[lb * 32 + lane] = (uint16_t)(incl - c);
      if (lane == 31) bpref[lb] = incl;
    }
  }
  __syncthreads();
  // B: exclusive scan of the block counts, offset by the pillars in front of this slice
  {
    int carry = __ldg(cta_base + blockIdx.x);
    for (int base = 0; base < f.bpc; base += kFrThreads) {
      const int i = base + tid;
      const int v = i < f.bpc ? bpref[i] : 0;
      int tot;
      const int ex = block_excl_scan<kFrThreads>(v, &tot);
      if (i < f.bpc) {
        bpref[i] = ex + carry;
        if (i < my_blocks) blockpref[(size_t)b * f.nblk + r * f.bpc + i] = ex + carry;
      }
      carry += tot;
    }
    if (tid == 0) bpref[f.bpc] = carry;
  }
  __syncthreads();
  // C: coords (b, yi, xi) of this slice's pillars, rows in sorted-unique order
  for (int lb = warp; lb < my_blocks; lb += kFrThreads / 32) {
    const int base_idx = bpref[lb], total = bpref[lb + 1] - base_idx;
    if (total == 0) continue;
    uint32_t w = bits[lb * 32 + lane];
    const int pre = (int)inb[lb * 32 + lane];
    const int lw = (r * f.bpc + lb) * 32 + lane;
    const int xi = lw / g.vwords, vw = lw - xi * g.vwords;
    if (total <= f.cstage && base_idx + total <= cap) {
      int* cs = stage + warp * (f.cstage * 3);
      int k = pre;
      while (w) {
        const int bit = __ffs(w) - 1;
        w &= w - 1;
        cs[k * 3 + 0] = b;
        cs[k * 3 + 1] = vw * 32 + bit;
        cs[k * 3 + 2] = xi;
        ++k;
      }
      __syncwarp();
      int* dst = coords + (size_t)base_idx * 3;
      for (int q = lane; q < total * 3; q += 32) dst[q] = cs[q];
      __syncwarp();
    } else {
      int idx = base_idx + pre;
      while (w) {
        const int bit = __ffs(w) - 1;
        w &= w - 1;
        if (idx < cap) {
          coords[(size_t)idx * 3 + 0] = b;
          coords[(size_t)idx * 3 + 1] = vw * 32 + bit;
          coords[(size_t)idx * 3 + 2] = xi;
        }
        ++idx;
      }
    }
  }
  // D: pillar ids of the frame's points whose cell lies in this slice (slice 0 also writes the -1 of dropped points)
  long long p0, p1;
  frame_range(off, b, g.batch, n, &p0, &p1);
  const int word0 = b * f.W + r * words;
  constexpr int kU = 8;
  for (long long i0 = p0 + tid; i0 < p1; i0 += (long long)kFrThreads * kU) {
    int cell[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const long long i = i0 + (long long)u * kFrThreads;
      cell[u] = i < p1 ? __ldg(cell_of_point + i) : -2;
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const long long i = i0 + (long long)u * kFrThreads;
      if (cell[u] == -2) break;
      if (cell[u] < 0) {
        if (r == 0) pillar_of_point[i] = -1;
        continue;
      }
      const int loc = (cell[u] >> 5) - word0, bit = cell[u] & 31;
      if (loc < 0 || loc >= words) continue;
      const int pid = bpref[loc >> 5] + (int)inb[loc] + __popc(bits[loc] & ((1u << bit) - 1u));
      if (bucket_cnt) asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(bucket_cnt + pid) : "memory");
      pillar_of_point[i] = pid;
    }
  }
}

constexpr size_t kFrSmemMax = 226 * 1024;
inline size_t frame_mark_smem(int bpc, int stages) { return (size_t)bpc * 128 + (size_t)stages * kFrStageBytes + stages * 8 + 64; }
inline size_t frame_rank_smem(int bpc, int cstage) {
  return (size_t)bpc * 192 + ((size_t)bpc + 4) / 4 * 16 + (size_t)(kFrThreads / 32) * cstage * 12 + 64;
}

// slices per frame: the fewest whose tables fit the shared memory of one CTA per SM (every slice re-reads the frame's
// points from L2, so fewer is better); 0 = the frame does not fit
inline int frame_slices(int nblk) {
  for (int c = 1; c <= kFrMaxSlices; ++c) {
    const int bpc = (nblk + c - 1) / c;
    if (frame_mark_smem(bpc, kFrMinStages) <= kFrSmemMax && frame_rank_smem(bpc, 8) <= kFrSmemMax) return c;
  }
  return 0;
}

}  // namespace

// Scratch (int32 elements) of pnx_voxelize_frames: [0] status, then bounds, per-CTA counts and bases.
extern "C" int pnx_voxelize_frames_scratch(int batch) { return 8 + (batch + 1) + 2 * (batch * kFrMaxSlices + 1); }

// 0: pnx_voxelize_frames cannot run this geometry (a frame must be whole 32-word blocks and its slices must fit shared
// memory); otherwise the number of CTAs it launches (batch * slices) -- the caller compares it with the SM count: with few
// large frames (e.g. 14 frames of 540 k points) the global-bitmap kernels keep more of the machine busy.
extern "C" int pnx_voxelize_frames_supported(int batch, int gx, int gy) {
  if (batch <= 0 || gx <= 0 || gy <= 0) return 0;
  const long long W = (long long)gx * ((gy + 31) / 32);
  if (W % 32 != 0 || W * batch * 32 >= 2147483647LL) return 0;
  return batch * frame_slices((int)(W / 32));
}

// Same outputs as pnx_voxelize for points grouped by frame (ascending batch index, the collate order); see the block
// comment above.  scratch = pnx_voxelize_frames_scratch(batch) ints; scratch[0] != 0 after the call (read it at the next
// synchronisation) means the input was not grouped and the outputs are invalid: call pnx_voxelize instead.
extern "C" int pnx_voxelize_frames(const float* points, int n_points, int batch, float min_x, float min_y, float vs_x,
                                   float vs_y, int gx, int gy, uint32_t* bitmap, uint16_t* inblk, int* blockcnt, int* blockpref,
                                   int* cell_of_point, int* pillar_of_point, int* coords, int cap_pillars,
                                   uint32_t* bucket_cnt, int* counts /* [0]=P */, int* scratch, cudaStream_t stream) {
  PNX_CHECK_ARG(n_points > 0 && batch > 0 && gx > 0 && gy > 0, "bad sizes (n_points must be > 0: use pnx_voxelize for empty input)");
  PNX_CHECK_ARG(vs_x > 0.f && vs_y > 0.f, "voxel size must be positive");
  PNX_CHECK_ARG(pnx_voxelize_frames_supported(batch, gx, gy) > 0, "geometry not supported by the frame-tiled voxelizer");
  PNX_CHECK_ARG((reinterpret_cast<uintptr_t>(points) & 15) == 0, "points must be 16-byte aligned");
  static bool attr_set = false;
  if (!attr_set) {
    PNX_CUDA(cudaFuncSetAttribute(vox_frame_mark_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFrSmemMax));
    PNX_CUDA(cudaFuncSetAttribute(vox_frame_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFrSmemMax));
    attr_set = true;
  }
  VoxGeom g{min_x, min_y, vs_x, vs_y, gx, gy, (gy + 31) / 32, batch};
  FrameCfg f;
  f.W = gx * g.vwords;
  f.nblk = f.W / 32;
  f.cs = frame_slices(f.nblk);
  f.bpc = (f.nblk + f.cs - 1) / f.cs;
  f.cstage = 64;  // coords staging per warp: as much as the slice tables leave
  while (f.cstage > 8 && frame_rank_smem(f.bpc, f.cstage) > kFrSmemMax) f.cstage -= 8;
  f.stages = kFrMaxStages;
  while (f.stages > kFrMinStages && frame_mark_smem(f.bpc, f.stages) > kFrSmemMax) --f.stages;
  int* status = scratch;
  int* off = scratch + 8;
  int* cta_cnt = off + batch + 1;
  int* cta_base = cta_cnt + batch * kFrMaxSlices + 1;
  const int n_cta = batch * f.cs;
  if (bucket_cnt) PNX_CUDA(cudaMemsetAsync(bucket_cnt, 0, (size_t)(cap_pillars + 1) * 4 * 2, stream));
  vox_frame_bounds_kernel<<<batch + 1, 1024, 0, stream>>>(points, n_points, off, status);
  PNX_CHECK_LAUNCH();
  vox_frame_mark_kernel<<<n_cta, kFrThreads, frame_mark_smem(f.bpc, f.stages), stream>>>(points, n_points, g, f, off, bitmap, inblk, blockcnt,
                                                                               cell_of_point, cta_cnt, status);
  PNX_CHECK_LAUNCH();
  vox_frame_scan_kernel<<<1, 1024, 0, stream>>>(cta_cnt, n_cta, cta_base, off, batch, n_points, status,
                                                blockpref + (size_t)batch * f.nblk, counts);
  PNX_CHECK_LAUNCH();
  vox_frame_rank_kernel<<<n_cta, kFrThreads, frame_rank_smem(f.bpc, f.cstage), stream>>>(n_points, g, f, off, bitmap, cta_base, cell_of_point,
                                                                                         blockpref, pillar_of_point, coords, cap_pillars,
                                                                                         bucket_cnt);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

extern "C" size_t pnx_voxelize_bitmap_words(int batch, int gx, int gy) {
  size_t w = (size_t)batch * gx * ((gy + 31) / 32);
  return (w + 31) / 32 * 32;  // whole 32-word blocks
}

// Index generation (V1-V2).  See include/pnx.h for the contract.  All buffers are caller-owned device memory.
extern "C" int pnx_voxelize(const float* points, int n_points, int batch, float min_x, float min_y, float vs_x,
                            float vs_y, int gx, int gy, uint32_t* bitmap, uint16_t* inblk, int* blockcnt, int* blockpref,
                            int* cell_of_point, int* pillar_of_point, int* coords, int cap_pillars,
                            uint32_t* bucket_cnt, int* counts /* [0]=P */, cudaStream_t stream) {
  PNX_CHECK_ARG(n_points >= 0 && batch > 0 && gx > 0 && gy > 0, "bad sizes");
  PNX_CHECK_ARG(vs_x > 0.f && vs_y > 0.f, "voxel size must be positive");
  PNX_CHECK_ARG((long long)batch * gx * ((gy + 31) / 32) * 32 < 2147483647LL, "grid too large for int32 cell ids");
  PNX_CHECK_ARG(cap_pillars >= 0, "cap_pillars");
  VoxGeom g{min_x, min_y, vs_x, vs_y, gx, gy, (gy + 31) / 32, batch};
  const int n_words = (int)pnx_voxelize_bitmap_words(batch, gx, gy);
  const int n_blocks = n_words / 32;
  PNX_CUDA(cudaMemsetAsync(bitmap, 0, (size_t)n_words * 4, stream));
  PNX_CUDA(cudaMemsetAsync(blockcnt, 0, (size_t)pnx_blockcnt_size(n_blocks) * 4, stream));
  int* supercnt = blockcnt + super_offset(n_blocks);
  if (bucket_cnt) PNX_CUDA(cudaMemsetAsync(bucket_cnt, 0, (size_t)(cap_pillars + 1) * 4 * 2, stream));  // counts + cursors
  if (n_points > 0) {
    static int sm_count = 0;
    constexpr int kMarkSmem = kVoxStages * kVoxStageBytes + kVoxStages * 8 + 128;
    if (!sm_count) {
      int dev = 0;
      PNX_CUDA(cudaGetDevice(&dev));
      PNX_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
      PNX_CUDA(cudaFuncSetAttribute(vox_mark_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMarkSmem));
    }
    PNX_CHECK_ARG((reinterpret_cast<uintptr_t>(points) & 15) == 0, "points must be 16-byte aligned");
    // two CTAs' worth of chunks per SM keeps the tail short; chunks are whole stages so every bulk copy is 16-byte aligned
    int ctas = 2 * sm_count;
    int pts_per_cta = (int)((((long long)n_points + ctas - 1) / ctas + kVoxStagePts - 1) / kVoxStagePts * kVoxStagePts);
    ctas = (int)(((long long)n_points + pts_per_cta - 1) / pts_per_cta);
    vox_mark_kernel<<<ctas, kVoxThreads, kMarkSmem, stream>>>(points, n_points, pts_per_cta, g, bitmap, cell_of_point);
    PNX_CHECK_LAUNCH();
    vox_blockcnt_kernel<<<pnx_cdiv((long long)pnx_cdiv(n_blocks, kCntU) * 32, 256), 256, 0, stream>>>(bitmap, n_blocks, blockcnt, inblk);
    PNX_CHECK_LAUNCH();
  }
  super_reduce_kernel<<<(n_blocks + 1023) / 1024, 256, 0, stream>>>(blockcnt, n_blocks, supercnt);
  PNX_CHECK_LAUNCH();
  int rc = pnx_scan_blocks(blockcnt, n_blocks, blockpref, counts, stream);
  if (rc) return rc;
  if (n_points > 0) {
    vox_coords_kernel<<<pnx_cdiv((long long)pnx_cdiv(n_blocks, kCoU) * 32, 256), 256, 0, stream>>>(bitmap, blockpref, n_blocks, g, coords,
                                                                                  cap_pillars, inblk);
  } else {
    PNX_CUDA(cudaMemsetAsync(inblk, 0, (size_t)n_words * 2, stream));
  }
  PNX_CHECK_LAUNCH();
  if (n_points > 0) {
    vox_rank_kernel<<<pnx_cdiv(n_points, 256), 256, 0, stream>>>(cell_of_point, n_points, bitmap, blockpref, inblk,
                                                                 pillar_of_point, bucket_cnt);
    PNX_CHECK_LAUNCH();
  }
  return PNX_OK;
}

// V3 preparation: CSR grouping of the kept points by pillar (ascending point id inside a pillar).
// bucket_cnt comes from pnx_voxelize ([cap+1] counts followed by [cap+1] zeroed cursors); counts[1] receives Nv.
extern "C" int pnx_bucketize(const int* pillar_of_point, int n_points, int cap_pillars, uint32_t* bucket_cnt,
                             int* scan_scratch, int* bucket_off, int* bucket_tmp, int* bucket_pts, int* counts,
                             cudaStream_t stream) {
  PNX_CHECK_ARG(n_points >= 0 && cap_pillars >= 0, "sizes");
  int rc = pnx_scan_u32(bucket_cnt, cap_pillars, 0, bucket_off, scan_scratch, counts + 1, stream);
  if (rc) return rc;
  if (n_points > 0) {
    uint32_t* cursor = bucket_cnt + cap_pillars + 1;
    vox_fill_kernel<<<pnx_cdiv(n_points, 256), 256, 0, stream>>>(pillar_of_point, n_points, bucket_off, cursor,
                                                                 bucket_tmp);
    vox_sort_kernel<<<pnx_cdiv(n_points, 256), 256, 0, stream>>>(bucket_tmp, pillar_of_point, bucket_off, n_points,
                                                                 counts + 1, bucket_pts);
    PNX_CHECK_LAUNCH();
  }
  return PNX_OK;
}
