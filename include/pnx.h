/* pnx.h -- C-ABI of libpnx.so, the H100 (sm_90a) hot path of PillarNeXt-B.
 *
 * Boundary rules (SURVEY.md section 8b): extern "C", plain pointers and sizes, no torch types.
 * The caller owns every buffer (device memory unless stated), kernels never allocate and never
 * synchronise, everything is enqueued on the `stream` argument (the caller passes its current
 * stream; the reference's only native extension, iou3d_nms, uses the legacy default stream and
 * exit()s on error -- /root/reference/det3d/core/iou3d_nms/src/iou3d_nms.cpp:14-38 -- neither is
 * copied).  Every entry point returns 0 on success or a negative PNX_ERR_* code;
 * pnx_last_error() returns the thread-local message.  Variable-size results (pillars, sites)
 * are written into fixed-capacity buffers with the true count in device memory (`counts`).
 *
 * The reference reaches this path through Python modules, not an FFI (its third-party CUDA ops
 * are torch_scatter / spconv / cuDNN); each entry point cites the reference lines it replaces.
 */
#ifndef PNX_H_
#define PNX_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef __CUDA_RUNTIME_H__
typedef struct CUstream_st* cudaStream_t;
#endif

#define PNX_OK 0
#define PNX_ERR_ARG (-1)
#define PNX_ERR_CUDA (-2)
#define PNX_ERR_CAPACITY (-3)

const char* pnx_last_error(void);
int pnx_abi_version(void);
int pnx_sm_count(void);

/* ---------------------------------------------------------------- generic device scan
 * out[i] = sum_{j<i} f(in[j]), i in [0,n]; f = popcount (popc=1) or identity on int32 (popc=0).
 * block_sums: scratch of (n+1)/2048 + 2 ints; total_out (optional) receives out[n]. */
int pnx_scan_u32(const uint32_t* in, int n, int popc, int* out, int* block_sums, int* total_out,
                 cudaStream_t stream);

/* Exclusive scan of the per-32-word-block counts of a bitmap in ONE launch (two-level: the count buffer holds
 * the block counts followed by one count per 1024 blocks; pnx_blockcnt_size() ints).  out [n_blocks+1]. */
int pnx_blockcnt_size(int n_blocks);
int pnx_scan_blocks(const int* counts, int n_blocks, int* out, int* total_out, cudaStream_t stream);

/* ---------------------------------------------------------------- V1-V3 voxelizer
 * Replaces PillarNet.forward index generation, det3d/models/readers/pillar_encoder.py:86-111
 * (range mask, trunc, torch.unique(dim=0, return_inverse=True)) bit-exactly, without a sort.
 *   points        [n_points, 6] fp32 (batch_idx, x, y, z, intensity, time), 16-byte aligned
 *   bitmap        pnx_voxelize_bitmap_words() u32 (padded to whole 32-word blocks), occupancy in (b, xi, yi)
 *                 order (zeroed here)
 *   inblk         [words] u16 OUT: in-block exclusive popcount prefix (also used by the rulebook)
 *   blockcnt      [pnx_blockcnt_size(words/32)] int32: pillars per 32-word block (+ per 1024 blocks), written here
 *   blockpref     [words/32 + 1] exclusive scan of blockcnt; rank of a cell = blockpref[block] +
 *                 popcount of the block's earlier words + popcount of the lower bits of its word
 *   cell_of_point [n_points] scratch
 *   pillar_of_point [n_points] OUT: pillar id (== reference `unq_inv`) or -1 for dropped points
 *   coords        [cap_pillars, 3] OUT int32 (b, yi, xi), rows in the reference's sorted-unique order
 *   bucket_cnt    [2*(cap_pillars+1)] OUT (optional, may be NULL): points per pillar + zeroed cursors for
 *                 pnx_bucketize
 *   counts        [2] device ints: counts[0] = #pillars P (counts[1] = #kept points, set by pnx_bucketize)
 * cap_pillars must be >= min(n_points, batch*gx*gy).  Kernels: mark (persistent, points staged through shared memory by
 * TMA bulk copies, one fire-and-forget RED.OR per point) | block popcounts | scan | coords | rank. */
size_t pnx_voxelize_bitmap_words(int batch, int gx, int gy);
int pnx_voxelize(const float* points, int n_points, int batch, float min_x, float min_y, float vs_x,
                 float vs_y, int gx, int gy, uint32_t* bitmap, uint16_t* inblk, int* blockcnt, int* blockpref,
                 int* cell_of_point, int* pillar_of_point, int* coords, int cap_pillars,
                 uint32_t* bucket_cnt, int* counts, cudaStream_t stream);
/* Frame-tiled variant for points GROUPED BY FRAME in ascending batch index (the collate order, loader/collate.py:17-21):
 * same arguments and bit-identical outputs as pnx_voxelize, but the occupancy bitmap of a frame lives in the shared memory
 * of a thread-block cluster (marking and ranking are shared-memory / DSMEM operations instead of random L2 transactions)
 * and HBM only sees streaming traffic.  Kernels: bounds (1024-ary search of the frame offsets) | mark (cluster per frame)
 * | scan | rank (+ coords, blockpref).  scratch = pnx_voxelize_frames_scratch(batch) int32; the input order is verified on
 * the device: scratch[0] != 0 after the call means the points were not grouped and every output is invalid (use
 * pnx_voxelize).  pnx_voxelize_frames_supported: 1 when the geometry qualifies (whole 32-word blocks per frame, slices
 * that fit shared memory with clusters of at most 8 CTAs). n_points must be > 0. */
int pnx_voxelize_frames_scratch(int batch);
int pnx_voxelize_frames_supported(int batch, int gx, int gy);
int pnx_voxelize_frames(const float* points, int n_points, int batch, float min_x, float min_y, float vs_x,
                        float vs_y, int gx, int gy, uint32_t* bitmap, uint16_t* inblk, int* blockcnt, int* blockpref,
                        int* cell_of_point, int* pillar_of_point, int* coords, int cap_pillars,
                        uint32_t* bucket_cnt, int* counts, int* scratch, cudaStream_t stream);
/* CSR grouping of the kept points by pillar (input of the per-pillar mean / max, pillar_encoder.py:113-114,43):
 * bucket_off [cap_pillars+1], bucket_pts [n_points] (ascending point id inside a pillar), bucket_tmp scratch,
 * scan_scratch [cap_pillars/2048 + 4]; counts[1] receives the number of kept points. */
int pnx_bucketize(const int* pillar_of_point, int n_points, int cap_pillars, uint32_t* bucket_cnt,
                  int* scan_scratch, int* bucket_off, int* bucket_tmp, int* bucket_pts, int* counts,
                  cudaStream_t stream);

/* ---------------------------------------------------------------- BatchNorm statistics
 * stats = [2*C] fp64 (sum, sum of squares) accumulated by the producing kernel.
 * count = (*count_ptr if non-NULL else 1) * count_mult.  Writes scale/shift (y = x*scale+shift),
 * optional mean/invstd (for backward) and updates running_mean/var like torch
 * (nn.BatchNorm1d/2d training forward; pillar_encoder.py:33, sparse_conv.py:31,52, conv.py:27). */
int pnx_bn_finalize(const double* stats, int channels, const int* count_ptr, long long count_mult,
                    const float* gamma, const float* beta, float eps, float momentum,
                    float* running_mean, float* running_var, float* scale, float* shift,
                    float* mean_out, float* invstd_out, cudaStream_t stream);
int pnx_bn_eval_affine(int channels, const float* gamma, const float* beta, const float* running_mean,
                       const float* running_var, float eps, float* scale, float* shift,
                       cudaStream_t stream);

/* ---------------------------------------------------------------- P1-P3 PillarFeatureNet (forward)
 * Replaces pillar_encoder.py:113-123 (scatter_mean + decoration), :35-50 (PFNLayer x2), :180.
 * counts = the voxelizer's device counts.  y0 [cap_points,32], y1 [cap_points,64] fp32 (rows in
 * bucket order), x0max [cap_pillars,32], mean [cap_pillars,3], stats fp64 accumulated in place. */
int pnx_pfn_mean(const float* points, const int* bucket_off, const int* bucket_pts, const int* counts,
                 int cap_pillars, float* mean, cudaStream_t stream);
int pnx_pfn_lin0(const float* points, const int* bucket_pts, const int* pillar_of_point,
                 const int* coords, const float* mean, const int* counts, int cap_points, float min_x,
                 float min_y, float vs_x, float vs_y, const float* w0, float* y0, double* stats,
                 int training, cudaStream_t stream);
int pnx_pfn_max0(const float* y0, const int* bucket_off, const int* counts, int cap_pillars,
                 const float* scale, const float* shift, float* x0max, cudaStream_t stream);
int pnx_pfn_lin1(const float* y0, const float* x0max, const int* bucket_pts, const int* pillar_of_point,
                 const int* counts, int cap_points, const float* scale0, const float* shift0,
                 const float* w1, float* y1, double* stats, int training, cudaStream_t stream);
int pnx_pfn_max1(const float* y1, const int* bucket_off, const int* counts, int cap_pillars,
                 const float* scale, const float* shift, float* feat_f32, void* feat_bf16,
                 cudaStream_t stream);

/* PillarFeatureNet backward (autograd of pillar_encoder.py:35-50,174-182 in the reference).
 * Inputs: the forward's saved buffers (pnx_pfn_* outputs), dfeat [cap_pillars,64] fp32.
 * Scratch: argq1 [cap_pillars,64] int32, d_x0 / dxm_part [cap_points,32] fp32.
 * Outputs (zero them first): red fp64 [64+128] = {dbeta0[32], dgamma0[32], dbeta1[64], dgamma1[64]},
 * dW0 [32,10], dW1 [64,64] fp64 (accumulated by cross-CTA atomics: fp64 makes their order irrelevant at fp32 level). */
int pnx_pfn_backward(const float* points, const int* bucket_off, const int* bucket_pts,
                     const int* pillar_of_point, const int* coords, const int* counts, int cap_points,
                     int cap_pillars, float min_x, float min_y, float vs_x, float vs_y, const float* pmean,
                     const float* y0, const float* y1, const float* x0max, const float* feat,
                     const float* dfeat, const float* w1, const float* scale0, const float* shift0,
                     const float* mean0, const float* invstd0, const float* gamma0, const float* scale1,
                     const float* shift1, const float* mean1, const float* invstd1, const float* gamma1,
                     int* argq1, float* d_x0, float* dxm_part, double* red, double* dW0, double* dW1,
                     int phases, const int* bn_count, cudaStream_t stream);

/* ---------------------------------------------------------------- B1-B4 active sites / rulebook
 * Replaces spconv index-pair generation (sparse_conv.py:25-29,50-51; sparse_resnet.py:43-48,63-64).
 * A level = bitmap in (b, u=x, v=y) order (v padded to 32 bits, words padded to whole 32-word blocks) +
 * inblk [words] u16 (in-block exclusive popcount prefix) + blockpref [words/32+1]; coords are (b, u, v) int32. */
int pnx_sites_out_dim(int in_dim, int stride);
int pnx_sites_dilate(const uint32_t* bm_in, int batch, int u_in, int v_in, int stride, uint32_t* bm_out,
                     uint16_t* inblk, int* blockcnt, cudaStream_t stream);
int pnx_sites_inblock(const uint32_t* bm, int n_words_pad, uint16_t* inblk, cudaStream_t stream);
int pnx_sites_coords(const uint32_t* bm, const int* blockpref, const uint16_t* inblk, int batch, int u, int v,
                     int* coords, int cap, cudaStream_t stream);
/* nbr [cap, 9] int32: row index in the source level feeding site i through tap t = ku*3+kv, -1 = absent.
 * transposed=1 builds the data-gradient table of a (strided) SparseConv2d. */
int pnx_nbr_table(const int* dst_coords, const int* n_dst_ptr, int cap, const uint32_t* src_bm,
                  const int* src_blockpref, const uint16_t* src_inblk, int batch, int src_u, int src_v,
                  int stride, int transposed, int* nbr, cudaStream_t stream);
/* x.dense() (sparse_resnet.py:68): feat [n, C] bf16 -> zeroed channels-last canvas [B, V, U, C]
 * (gather=0) or the reverse (gather=1, used by backward). */
int pnx_scatter_dense(const void* feat, const int* coords, const int* n_ptr, int cap, int channels,
                      int batch, int u, int v, void* canvas, int gather, cudaStream_t stream);

/* ---------------------------------------------------------------- wgmma gather implicit GEMM
 * out[m, n] = sum_{t<taps} sum_{c<Cin} A[nbr(m,t), c] * W[t, n, c]  (+ bias[n]) (relu)
 *   A       [a_rows, lda] bf16 (a_rows = rows really allocated; every gathered row index must be below it)
 *   W       [taps, Cout, Cin] bf16 (packed, K-major)
 *   nbr(m,t): nbr[m*taps+t] if nbr != NULL; computed from the dense geometry if dense != 0
 *             (m -> (b, y, x) over Hout x Wout; source pixel (y*mul + r*dil - pad, x*mul + s*dil - pad)
 *             in an Hin x Win image, t = r*kw + s; out of range = zero);  m itself otherwise (taps==1).
 *   out     bf16 (out_fp32=0) or fp32, row stride ldc elements; shuffle=1: ConvTranspose2d k2 s2
 *           pixel-shuffle store (column n = q*64 + co -> pixel (2y + q/2, 2x + q%2), channel co)
 *   stats   optional fp64 [2*stats_C]: per-channel sum / sum of squares of the stored values
 *           (channel = n % stats_mod), for the BatchNorm that follows the convolution.
 * Replaces spconv SparseConv2d/SubMConv2d (sparse_conv.py:25-29,50-51), F.conv2d/nn.Conv2d
 * (aspp.py:19-32, conv.py:9-10, centerhead.py:35-46,108-114), nn.ConvTranspose2d (centerhead.py:26-27). */
int pnx_igemm(const void* A, long long lda, long long a_rows, int M, int taps, int Cin, const void* Wpacked, int Cout,
              int block_n, const int* nbr, int dense, int Hout, int Wout, int Hin, int Win, int kw,
              int mul, int dil, int pad, void* out, long long ldc, int out_fp32, const float* bias,
              double* stats, int stats_C, int stats_mod, int shuffle, int relu, const void* addend,
              long long ld_add, int nseg, long long a_lo_off, long long seg_code, int addend_fp32,
              const void* bnr_raw, long long bnr_ld, const float* bnr_scale, const float* bnr_shift,
              const float* bnr_mean, const float* bnr_invstd, double* bnr_red, int bnr_C, int sm_count,
              cudaStream_t stream);
/* bnr_raw != NULL fuses the REDUCE pass of a BatchNorm backward into this GEMM (bf16 output, no pixel shuffle, no forward
 * statistics): `out` is dy, the gradient of y = relu(raw*scale + shift) -- the epilogue recomputes the ReLU gate from
 * raw [M, bnr_ld] bf16 with the forward affine, stores g = dy*gate instead of dy and accumulates
 * bnr_red[c] += sum_m g, bnr_red[bnr_C + c] += sum_m g*(raw - mean[c])*invstd[c]  (fp64; zero it first; bnr_C == Cout).
 * pnx_bn_bwd_apply is then called with relu = 0 on g.  Same trailing arguments on pnx_conv3x3_win. */
/* nseg > 1 selects the fp32-grade SPLIT mode (see "split rows" below): every value is a sum of bf16 PIECES, A rows
 * hold piece p of channel c at column p*a_lo_off + c, W is packed [taps, Cout, pieces*Cin] = [piece 0 | piece 1 | ..],
 * and the K loop accumulates nseg (A piece, W piece) segments into the same fp32 register accumulator in the order given
 * by seg_code (4 bits per segment: (A piece << 2) | W piece; callers put the smallest products first).
 * addend_fp32 = 1: `addend` is fp32 [M, ld_add] (requires out_fp32).  nseg = 1, seg_code = 0, a_lo_off = 0,
 * addend_fp32 = 0: the production bf16 path. */

/* ---------------------------------------------------------------- weight repacking (one launch for the whole model)
 * table = device array of n (<= 256) descriptors { const float* src; bf16* dst; int64 start; int64 base; int64 stride[4];
 * int32 dim[4]; } (96 bytes): dst[((a*d1 + b)*d2 + c)*d3 + d] = bf16(src[base + a*s0 + b*s1 + c*s2 + d*s3]); `start` =
 * running element offset of the entry, total = sum of element counts.  Converts the fp32 parameters (reference layouts:
 * nn.Conv2d, spconv [Cout,kH,kW,Cin], nn.ConvTranspose2d) into the [tap, Cout, Cin] / [tap, Cin, Cout] bf16 operands of
 * pnx_igemm / pnx_conv3x3_win after an optimizer step. */
int pnx_pack_weights(const void* table, int n, long long total, cudaStream_t stream);

/* ---------------------------------------------------------------- dense 3x3 conv with TMA-folded im2col
 * out[(b,y,x), n] = sum_{r,s<3} sum_c A[(b, y+r-1, x+s-1), c] * W[r*3+s, n, c] (+bias)(relu), zero padding,
 * on a B x H x W channels-last image (A rows = pixels, row stride lda; W packed [9, Cout, Cin] like pnx_igemm).
 * One 4-D TMA window load per (64-channel chunk, kernel row) feeds the three horizontal taps through shifted
 * shared-memory descriptors.  bf16 output, optional BatchNorm statistics (fp64 [2*stats_C]).  Same layers as
 * pnx_igemm's dense mode (aspp.py/conv.py/centerhead.py 3x3 convs, dilation 1) and their data gradients. */
int pnx_conv3x3_win(const void* A, long long lda, int B, int H, int W, int Cin, const void* Wpacked, int Cout,
                    int block_n, void* out, long long ldc, const float* bias, double* stats, int stats_C, int relu,
                    int base_off_mode, const void* bnr_raw, long long bnr_ld, const float* bnr_scale,
                    const float* bnr_shift, const float* bnr_mean, const float* bnr_invstd, double* bnr_red, int bnr_C,
                    int sm_count, cudaStream_t stream);

/* ---------------------------------------------------------------- wgmma weight gradient
 * dW[t, x, y] += sum_m X[m, x] * Y[g(m,t), y]   (fp32, red.global.add; zero dW first)
 * X = direct operand (output gradient; layer input for ConvTranspose2d, shuffle=1), Y = operand read through
 * the neighbour map: nbr[m*taps+t] if nbr != NULL, else the dense geometry (as pnx_igemm), else row m (taps==1,
 * gathered=0).  x_channels: 64 or a multiple of 128; y_channels: multiple of 64.  Backward of the layers
 * pnx_igemm replaces (autograd in the reference: trainer/trainer/trainer.py:94-108). */
int pnx_wgrad(const void* X, long long ldx, int x_channels, const void* Y, long long ldy, long long y_rows,
              int y_channels, int gathered, int M, int taps, const int* nbr, int Hout, int Wout, int Hin, int Win, int kw,
              int mul, int dil, int pad, int shuffle, float* dW, float* partials, int sm_count, cudaStream_t stream);
/* Deterministic weight gradients: with partials != NULL (pnx_wgrad_splits(...) * taps * x_channels * y_channels floats,
 * 16-byte aligned) every K split stores its own slab with plain stores and one kernel adds the slabs to dW in split order,
 * instead of fp32 red.global.add from all splits.  pnx_wgrad_splits = the number of splits pnx_wgrad uses for the shape. */
int pnx_wgrad_splits(int x_channels, int y_channels, int taps, int M, int sm_count);
/* Library-wide switch: the BatchNorm statistics of the GEMM epilogues (pnx_igemm / pnx_conv3x3_win `stats`) are
 * accumulated in fp64 from per-warp partials (order effects 1e-16) instead of through fp32 shared-memory words added in
 * arrival order (1e-7).  Returns the previous setting. */
int pnx_set_deterministic(int on);

/* ---------------------------------------------------------------- row-wise bf16 kernels
 * y = relu?(x*scale + shift (+ res))  -- BatchNorm apply (+residual)(+ReLU): sparse_conv.py:33-39,55-63,
 * conv.py:29-34; rows = active sites or pixels, C channels, ld* = row strides in elements. */
int pnx_bn_apply(const void* x, long long ldx, long long M, int C, const float* scale, const float* shift,
                 const void* res, long long ldr, int relu, void* y, long long ldy, cudaStream_t stream);
/* BatchNorm backward: red[0:C] += sum g, red[C:2C] += sum g*xhat with g = dy*(y>0 if relu).  y may be NULL when
 * there is no residual: the ReLU mask is then recomputed from x with the forward affine (fscale, fshift). */
int pnx_bn_bwd_reduce(const void* dy, long long lddy, const void* y, long long ldy, const void* x,
                      long long ldx, long long M, int C, const float* mean, const float* invstd, int relu,
                      const float* fscale, const float* fshift, double* red, cudaStream_t stream);
/* ... dx = gamma*invstd*(g - red[c]/count - xhat*red[C+c]/count); optional dres (+)= g (residual branch).
 * count_dev != NULL: the population is read from device memory (SyncBatchNorm: the all-reduced site count of a sparse
 * layer is only known on the device) and `count` is ignored. */
int pnx_bn_bwd_apply(const void* dy, long long lddy, const void* y, long long ldy, const void* x,
                     long long ldx, long long M, int C, const float* mean, const float* invstd,
                     const float* gamma, const double* red, double count, const int* count_dev, int relu,
                     const float* fscale, const float* fshift, void* dx, long long lddx, void* dres,
                     long long lddres, int dres_accumulate, cudaStream_t stream);
int pnx_add_rows(void* a, long long lda, const void* b, long long ldb, long long M, int C, cudaStream_t stream);
/* y = relu(a + b) (BasicBlock tail, conv.py:48-50) and its backward g (+)= dy*(y>0). */
int pnx_add_relu(const void* a, long long lda, const void* b, long long ldb, long long M, int C, void* y,
                 long long ldy, cudaStream_t stream);
int pnx_relu_bwd(const void* dy, long long lddy, const void* y, long long ldy, long long M, int C, void* g,
                 long long ldg, int accumulate, cudaStream_t stream);

/* ---------------------------------------------------------------- fp32-grade "split rows" precision mode
 * The reference is fp32 end to end (aspp.py:19-32, centerhead.py:128-136, sparse_conv.py:31-39; no autocast).  In
 * this mode an activation row matrix stores every value as P bf16 PIECES (pnx_split_set_pieces: 2 = 16 mantissa
 * bits, 3 = 24 bits = an exact fp32): piece 0 = bf16(v) at column c, piece q = bf16(v - pieces before) at column
 * q*lo + c of the same row; the tensor-core kernels run over (piece, piece) segments (pnx_igemm nseg/seg_code; one
 * pnx_wgrad launch per segment, all accumulating into the same dW) and raw convolution outputs, BatchNorm arithmetic
 * and gradient sums stay fp32.  The kernels below are the row-wise glue of the mode
 * (x = fp32 rows, everything named res / y / dy / dx / dres / a / b / g = split rows given as (pointer, ld, lo)).
 * pnx_bn_bwd_reduce_split is two-stage with a fixed order (bit-reproducible): `part` = scratch of
 * pnx_bn_bwd_reduce_split_scratch(C) doubles, `red` [2C] is fully written. */
int pnx_split_set_pieces(int pieces);   /* 2 or 3; process-wide; returns the previous value */
int pnx_split_get_pieces(void);
int pnx_rows_split(const float* x, long long ldx, long long M, int C, void* y, long long ldy, long long lo_y,
                   cudaStream_t stream);
int pnx_rows_merge(const void* x, long long ldx, long long lo_x, long long M, int C, float* y, long long ldy,
                   int accumulate, cudaStream_t stream);
int pnx_bn_apply_split(const float* x, long long ldx, long long M, int C, const float* scale, const float* shift,
                       const void* res, long long ldr, long long lo_r, int relu, void* y, long long ldy, long long lo_y,
                       cudaStream_t stream);
long long pnx_bn_bwd_reduce_split_scratch(int C);
int pnx_bn_bwd_reduce_split(const void* dy, long long lddy, long long lo_dy, const void* y, long long ldy,
                            long long lo_y, const float* x, long long ldx, long long M, int C, const float* mean,
                            const float* invstd, int relu, const float* fscale, const float* fshift, double* part,
                            double* red, cudaStream_t stream);
int pnx_bn_bwd_apply_split(const void* dy, long long lddy, long long lo_dy, const void* y, long long ldy,
                           long long lo_y, const float* x, long long ldx, long long M, int C, const float* mean,
                           const float* invstd, const float* gamma, const double* red, double count, int relu,
                           const float* fscale, const float* fshift, void* dx, long long lddx, long long lo_dx,
                           void* dres, long long lddres, long long lo_dres, cudaStream_t stream);
int pnx_add_relu_split(const void* a, long long lda, long long lo_a, const void* b, long long ldb, long long lo_b,
                       long long M, int C, void* y, long long ldy, long long lo_y, cudaStream_t stream);
int pnx_relu_bwd_split(const float* dy, long long lddy, const void* y, long long ldy, long long lo_y, long long M,
                       int C, void* g, long long ldg, long long lo_g, cudaStream_t stream);

/* ---------------------------------------------------------------- head final 3x3 convs as GEMM + stencil
 * out[m, j] = bias16[j] + sum_{t<9} Z[m + off_t, t*16 + j] on a B x H x W channels-last image (zero padding),
 * Z [M, ldz] fp32 = y . Wz^T from pnx_igemm (taps=1); pnx_tap_scatter is the mirrored backward gather
 * dZ[m', t*cpt+j] = dout[m' - off_t, j] (bf16, columns >= 9*cpt zeroed).  Replaces the `<head>.3` Conv2d(64, c, 3)
 * of SepHead (centerhead.py:44-46) for all sibling heads at once. */
int pnx_tap_gather_sum(const float* Z, long long ldz, int cpt, const float* bias16, int B, int H, int W, float* out,
                       cudaStream_t stream);
/* cpt = channels per tap (4/8/12/16): Z / dZ column = tap*cpt + j; nz = GEMM columns (>= 9*cpt, multiple of 8);
 * lo_off > 0: write all pieces of the split-rows mode (piece q at column q*lo_off + c) */
int pnx_tap_scatter(const float* dout, int B, int H, int W, void* dZ, long long ldz, int nz, int cpt, long long lo_off,
                    cudaStream_t stream);

/* ---------------------------------------------------------------- F3: label assignment on the GPU
 * One task of AssignLabel.__call__ (det3d/datasets/pipelines/assign.py:23-116; gaussian_radius / draw_gaussian:
 * center_utils.py:12-60) for a whole batch, i.e. also the stacking of loader/collate.py:23-33:
 *   boxes [B, N, 9] fp32 (x, y, z, dx, dy, dz, vx, vy, yaw), cls [B, N] int32 global class index (< 0: ignored),
 *   cls_task / cls_id [n_classes] int32 (task of a class, index of the class inside its task)
 *   -> hm [B, C, H, W] fp32, anno_box [B, M, 10] fp32, ind [B, M] i64, mask [B, M] u8, cat [B, M] i64,
 *      gt_boxes [B, M, 7] fp32 (all zeroed by the caller; M = max_objs).
 * Objects keep their order (slot = accepted objects of the task before it); radius/centre/gaussian in float64 and
 * stored as float32 like the numpy reference.  (pc_x, pc_y) = pc_range[0:2], osf = out_size_factor of the task. */
int pnx_assign_labels(const float* boxes, const int* cls, int B, int N, const int* cls_task, const int* cls_id,
                      int n_classes, int task, double vs_x, double vs_y, double pc_x, double pc_y, int osf,
                      double gaussian_overlap, int min_radius, int max_objs, int C, int H, int W, float* hm,
                      float* anno_box, long long* ind, unsigned char* mask, long long* cat, float* gt_boxes,
                      int* obj_scratch /* [B, N, 4] int32 */, cudaStream_t stream);

/* ---------------------------------------------------------------- L1 fused CenterPoint loss (forward + gradient)
 * One task: out/dout [B*H*W, npad] fp32 channels-last head output (columns reg2|height1|dim3|rot2|vel2|hm C|pad)
 * and its gradient (fully written), labels in the reference's collate format (det3d/datasets/pipelines/assign.py:
 * 42-48): hm_gt [B,C,H,W] f32, anno [B,M,10] f32, ind [B,M] i64, mask [B,M] u8, cat [B,M] i64, gt_boxes [B,M,7] f32.
 * acc [16] fp64 (zeroed by the caller) receives the partial sums; pnx_center_loss_finalize turns acc [n_tasks,16]
 * into res [n_tasks,16] = {loss, hm_loss, loc_loss, iou_reg_loss, num_positive, loc_loss_elem[10]} and total[0].
 * Replaces CenterHead.loss (centerhead.py:142-229) + FastFocalLoss/RegLoss/IouRegLoss (centerloss.py:8-176). */
int pnx_center_loss_task(const float* out, float* dout, const float* hm_gt, const float* anno,
                         const long long* ind, const unsigned char* mask, const long long* cat,
                         const float* gt_boxes, int B, int H, int W, int npad, int C, int M, int off_reg,
                         int off_height, int off_dim, int off_rot, int off_vel, int off_hm, float sx, float sy,
                         float ox, float oy, float weight, const float* code_w_host, int with_iou, double* acc,
                         cudaStream_t stream);
int pnx_center_loss_finalize(const double* acc, int n_tasks, const float* weights_dev, const float* code_w_dev,
                             const int* with_iou_dev, float* res, float* total, cudaStream_t stream);

/* ---------------------------------------------------------------- F1 detection decode + rotated NMS (one task)
 * Replaces CenterHead.predict / post_processing (centerhead.py:231-384), rotate_nms_pcdet (box_torch_ops.py:5-31) and
 * the native nms_gpu (iou3d_nms_kernel.cu:280-324, iou3d_nms.cpp:113-159).  `out` is the task's channels-last head
 * output [B*H*W, ld] fp32; offs = HOST ints {reg, height, dim, rot, vel, hm, iou} column offsets (iou < 0: no iou head);
 * range6 (post_center_limit_range), rect (rectifier per class), nms_thr (per class) are HOST float arrays.
 *   pnx_det_keys  : keys [B*H*W] int64 (INT64_MAX = filtered out; else (frame*C + class) << 32 | ~score bits, so an
 *                   ascending sort is segment-major and score-descending), seg_count [B*C] (zeroed here).
 *   pnx_det_nms   : order = argsort(keys) (the caller sorts), seg_start = exclusive prefix of seg_count; for each
 *                   segment the first min(count, pre_max) candidates: suppression mask (scratch [B*C, pre_max,
 *                   ceil(pre_max/64)] u64) and greedy sweep on the device -> keep [B*C, post_max] (positions in the
 *                   segment's sorted run), keep_count [B*C].  pre_max <= 8192 (reference Waymo configs: 4096); mask row stride = ceil(pre_max/64).
 *   pnx_det_gather: det_box [B*C, post_max, 9] (x,y,z,dx,dy,dz,vx,vy,yaw), det_score, det_label (+label_offset, i64).
 * The two *_host entry points evaluate the same inline decode / IoU code on HOST memory (CPU test hooks, no GPU). */
int pnx_det_keys(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf, float vs_x,
                 float vs_y, float pc_x, float pc_y, float score_thr, const float* range6, const float* rect,
                 long long* keys, int* seg_count, cudaStream_t stream);
int pnx_det_nms(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf, float vs_x,
                float vs_y, float pc_x, float pc_y, float score_thr, const float* range6, const float* rect,
                const float* nms_thr, const long long* order, const int* seg_start, const int* seg_count, int pre_max,
                int post_max, unsigned long long* mask, int* keep, int* keep_count, cudaStream_t stream);
int pnx_det_gather(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf, float vs_x,
                   float vs_y, float pc_x, float pc_y, float score_thr, const float* range6, const float* rect,
                   const long long* order, const int* seg_start, const int* keep, const int* keep_count, int post_max,
                   int label_offset, float* det_box, float* det_score, long long* det_label, cudaStream_t stream);
/* F2 helper: out[i] = aligned 3-D IoU (BEV polygon overlap x height overlap / union volume) of a[i], b[i] ([n,7] fp32
 * (x,y,z,dx,dy,dz,heading)); replaces boxes_aligned_iou3d_gpu (det3d/core/iou3d_nms/iou3d_nms_utils.py:45-87 +
 * iou3d_nms_kernel.cu:251-262), the training target of the Waymo `iou` head (centerloss.py:76-87). */
int pnx_aligned_iou3d(const float* a, const float* b, int n, float* out, cudaStream_t stream);
float pnx_aligned_iou3d_host(const float* box7_a, const float* box7_b);
float pnx_det_iou_bev_host(const float* box7_a, const float* box7_b);
int pnx_det_decode_host(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                        float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                        const float* rect, long long m, float* box9, float* score, int* label);

/* ---------------------------------------------------------------- double-flip test-time augmentation
 * pnx_flip4_points: points [n, 6] (batch_idx, x, y, z, intensity, time) -> out [4n, 6]: copy k of point i at row k*n + i
 * with batch index 4b + k; k = 1 negates y, k = 2 negates x, k = 3 both (exact).  The rows are not grouped by frame
 * (voxelize them with pnx_voxelize, not pnx_voxelize_frames); within a frame the input order is kept.
 * pnx_det_*_flip4: the F1 entry points above with the same arguments, on the head output of such a batch: `out` is
 * [4B*H*W, ld] (frame 4b + k = copy k of frame b) and B counts the B merged frames.  Each merged pixel (y, x) reads copy
 * 1 at (H-1-y, x), copy 2 at (y, W-1-x), copy 3 at (H-1-y, W-1-x), undoes the mirror (y: reg_y -> 1 - reg_y, sin -> -sin,
 * vy -> -vy; x: reg_x -> 1 - reg_x, cos -> -cos, vx -> -vx) and merges every quantity as ((v0 + v1) + (v2 + v3)) * 0.25f:
 * hm after the sigmoid (then the first maximum over classes), dim after exp, height / reg / rot / vel / iou raw.  keys,
 * seg_count, masks and results are those of the merged frames ([B*H*W], [B*C], ...).  The host twin takes HOST memory. */
int pnx_flip4_points(const float* points, int n, float* out, cudaStream_t stream);
int pnx_det_keys_flip4(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                       float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                       const float* rect, long long* keys, int* seg_count, cudaStream_t stream);
int pnx_det_nms_flip4(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf, float vs_x,
                      float vs_y, float pc_x, float pc_y, float score_thr, const float* range6, const float* rect,
                      const float* nms_thr, const long long* order, const int* seg_start, const int* seg_count,
                      int pre_max, int post_max, unsigned long long* mask, int* keep, int* keep_count,
                      cudaStream_t stream);
int pnx_det_gather_flip4(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                         float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                         const float* rect, const long long* order, const int* seg_start, const int* keep,
                         const int* keep_count, int post_max, int label_offset, float* det_box, float* det_score,
                         long long* det_label, cudaStream_t stream);
int pnx_det_decode_flip4_host(const float* out, long long ld, int B, int H, int W, int C, const int* offs, float osf,
                              float vs_x, float vs_y, float pc_x, float pc_y, float score_thr, const float* range6,
                              const float* rect, long long m, float* box9, float* score, int* label);

/* ---------------------------------------------------------------- global training augmentation
 * pnx_global_aug: points [n, 6] (batch_idx, x, y, z, intensity, time) and raw boxes [B, M, 9] (x, y, z, dx, dy, dz, vx,
 * vy, yaw) fp32 -> points_out, boxes_out (same shapes, new memory; the inputs are not written).  aug [B, 4, 4] fp64 holds
 * per frame up to four records (code, p0, p1, p2), applied in slot order:
 *   0 empty | 1 rotation (theta, cos theta, sin theta) | 2 scaling (s) | 3 translation (t, added to x, y and z) |
 *   4 flip (fx, fy: nonzero = x flip (y -> -y), y flip (x -> -x)); other codes are no-ops.
 * The results are those of the reference's numpy transforms (det3d/datasets/pipelines/augmentation.py +
 * box_np_ops.rotate / scaling / translate / flip) to the bit, NaN box elements included (csrc/augment.cu lists the
 * rounding rules).  One launch over n + B*M threads; the point order is kept.  A point whose batch index is not an
 * integer in [0, B) is copied unchanged.  The host twin takes HOST memory. */
int pnx_global_aug(const float* points, int n, const float* boxes, int B, int M, const double* aug, float* points_out,
                   float* boxes_out, cudaStream_t stream);
int pnx_global_aug_host(const float* points, int n, const float* boxes, int B, int M, const double* aug,
                        float* points_out, float* boxes_out);

/* ---------------------------------------------------------------- ground-truth database sampling
 * pnx_gt_sample: the reference's DataBaseSamplerV2 acceptance (sample_class_v2) and paste (datasets/base.py:77-96) for a
 * collated batch, given the candidates the data-loader workers drew.
 *   points [n, 6] (batch_idx, x, y, z, intensity, time); scene boxes [B, M, 9], classes [B, M] (-1 = padding),
 *   box_trig [B, M, 2] = numpy's fp32 (cos, sin) of each yaw;
 *   cand_boxes [B, S, 9], cand_classes [B, S] (-1 = padding; a class call is a run of equal ids), cand_trig [B, S, 4] =
 *   (numpy cos, numpy sin, libm cosf, sinf) of each yaw; cand_points [P, 5] (x, y, z relative to the box centre,
 *   intensity, time), candidate (b, s) owning rows cand_off[b S + s] .. cand_off[b S + s + 1] - 1 (cand_off [B S + 1]).
 * Outputs (new memory):
 *   points_out [n + P, 6]: per frame in frame order, the accepted objects' points (xyz + box centre) in acceptance order,
 *     then the frame's scene points outside every accepted box, in their input order; rows [*count, n + P) get batch
 *     index B and zeros.  A scene point whose batch index is not an integer in [0, B) is dropped.
 *   boxes_out [B, M + S, 9], classes_out [B, M + S]: the real scene boxes, the accepted ones, then padding (class -1,
 *     size 1); accepted [B, S] (may be NULL): 1 where the candidate was accepted; count [1]: valid rows of points_out.
 * Arithmetic and quirks: csrc/gt_sample.cu.  Four launches on `stream`, no host sync, no allocation: `workspace` holds
 * pnx_gt_sample_workspace(n, B, S) bytes of device memory (no initialisation needed).  B <= 512.  The host twin takes
 * HOST memory and needs no workspace.  pnx_points_in_boxes_host is the point test alone (box_np_ops.points_in_rbbox):
 * inside [n, m] bytes for points with x, y, z at the start of `stride`-float rows, 9-column boxes, and trig [m, 2] =
 * (cosf, sinf) of each yaw.  pnx_points_in_boxes is its device twin (csrc/det_eval.cu, equal to it to the bit): the same
 * operands in device memory, one launch on `stream`, no host sync, no workspace. */
long long pnx_gt_sample_workspace(int n, int B, int S);
int pnx_gt_sample(const float* points, int n, const float* boxes, const int* classes, const float* box_trig, int B, int M,
                  const float* cand_boxes, const int* cand_classes, const float* cand_trig, int S, const float* cand_points,
                  const int* cand_off, int P, float* points_out, float* boxes_out, int* classes_out, int* accepted,
                  int* count, void* workspace, cudaStream_t stream);
int pnx_gt_sample_host(const float* points, int n, const float* boxes, const int* classes, const float* box_trig, int B,
                       int M, const float* cand_boxes, const int* cand_classes, const float* cand_trig, int S,
                       const float* cand_points, const int* cand_off, int P, float* points_out, float* boxes_out,
                       int* classes_out, int* accepted, int* count);
int pnx_points_in_boxes_host(const float* points, int n, int stride, const float* boxes, const float* trig, int m,
                             unsigned char* inside);
int pnx_points_in_boxes(const float* points, int n, int stride, const float* boxes, const float* trig, int m,
                        unsigned char* inside, cudaStream_t stream);

/* ---------------------------------------------------------------- multi-sweep accumulation
 * pnx_accumulate_sweeps: the reference's NuScenesDataset.load_pointcloud (read_sweep + remove_close) and
 * WaymoDataset.load_pointcloud for a collated batch: past sweeps taken into the key frame and merged behind it.
 *   points [n, 6] (batch_idx, x, y, z, intensity, time): the key frames, frame f owning rows point_off[f] ..
 *   point_off[f + 1] - 1 (point_off [B + 1], from 0 to n);
 *   sweep_points [S, 5] (x, y, z, intensity, time) in each sweep's own frame, time already the reference's fp32 value;
 *   sweep (f, k) owns rows sweep_off[f K + k] .. sweep_off[f K + k + 1] - 1 (sweep_off [B K + 1], from 0 to S; a missing
 *   or dropped sweep is an empty segment); transforms [B, K, 4, 4] fp64 row-major, sweep -> key frame (nuScenes
 *   transform_matrix, Waymo inv(pose) @ sweep_pose); a matrix whose [3][3] entry is NaN marks "no transform" (the xyz is
 *   copied); min_distance: sweep points with |x| < d and |y| < d after the transform are dropped (nuScenes 1.0; 0 = off).
 * Outputs (new memory):
 *   points_out [n + S, 6]: per frame in frame order, its key-frame rows unchanged, then sweep 1, 2, ... (batch index f,
 *     transformed xyz, intensity, time), each in input order; rows [*count, n + S) get batch index B and zeros.
 *   count [1]: valid rows of points_out.
 * Arithmetic: csrc/sweeps.cu.  Three launches on `stream` (two when min_distance = 0), no host sync, no allocation:
 * `workspace` holds pnx_accumulate_sweeps_workspace(S, B) bytes of device memory (no initialisation needed).  The host
 * twin takes HOST memory and needs no workspace. */
long long pnx_accumulate_sweeps_workspace(int S, int B);
int pnx_accumulate_sweeps(const float* points, int n, const int* point_off, int B, const float* sweep_points, int S,
                          const int* sweep_off, int K, const double* transforms, float min_distance, float* points_out,
                          int* count, void* workspace, cudaStream_t stream);
int pnx_accumulate_sweeps_host(const float* points, int n, const int* point_off, int B, const float* sweep_points, int S,
                               const int* sweep_off, int K, const double* transforms, float min_distance,
                               float* points_out, int* count);

/* ---------------------------------------------------------------- Waymo-style evaluation (pillarnext_b200/evaluate_waymo.py)
 * pnx_eval_count_points: counts [B, M] int32 = number of points inside each ground-truth box, with the reference's
 * points_in_boxes_jit test (the one pnx_gt_sample uses).  points [n, stride >= 4] with (batch_idx, x, y, z) in columns
 * 0-3 (a row whose batch index is not an integer in [0, B) is skipped); boxes [B, M, 9] (x, y, z, dx, dy, dz, vx, vy,
 * yaw), classes [B, M] (-1 = padding, count 0), trig [B, M, 2] = libm (cosf, sinf) of each yaw.  Exact integer counts.
 * pnx_eval_match: the greedy score-ordered match of detections to ground truth, per (frame, class) segment s = f C + c.
 *   det_boxes [n_det, 9], det_trig [n_det, 2] = (cos, sin) of each yaw; order [n_det] int64 = detection indices sorted
 *   by segment, then by descending score, ties by lower index; segment s holds order[seg_start[s] ..
 *   seg_start[s] + seg_count[s]) (seg_start / seg_count [B C] int32); gt_boxes [B, M, 9], gt_classes [B, M] in [0, C)
 *   or -1 (padding), gt_trig [B, M, 2] = (cos, sin) of each yaw; thresholds [C] fp32 IoU thresholds; M <= 4096.
 *   Each detection in order takes the unmatched box of its segment with the highest aligned 3-D IoU (boxes_iou3d_gpu
 *   arithmetic, detection first), ties to the lower box index, if that IoU >= thresholds[c].  Outputs per detection
 *   (indexed like det_boxes): match = the box index j within its frame or -1, iou = the highest IoU over the boxes still
 *   unmatched when it was visited (0 if none), heading = 1 - min(|d|, 2 pi - |d|) / pi of the yaw difference d for a
 *   match, else 0.
 * Both run on `stream` with no host sync and no workspace; the _host twins take HOST memory. */
int pnx_eval_count_points(const float* points, long long n, int stride, const float* boxes, const int* classes,
                          const float* trig, int B, int M, int* counts, cudaStream_t stream);
int pnx_eval_count_points_host(const float* points, long long n, int stride, const float* boxes, const int* classes,
                               const float* trig, int B, int M, int* counts);
int pnx_eval_match(const float* det_boxes, const float* det_trig, long long n_det, const long long* order,
                   const int* seg_start, const int* seg_count, const float* gt_boxes, const int* gt_classes,
                   const float* gt_trig, int B, int M, int C, const float* thresholds, int* match, float* iou,
                   float* heading, cudaStream_t stream);
int pnx_eval_match_host(const float* det_boxes, const float* det_trig, long long n_det, const long long* order,
                        const int* seg_start, const int* seg_count, const float* gt_boxes, const int* gt_classes,
                        const float* gt_trig, int B, int M, int C, const float* thresholds, int* match, float* iou,
                        float* heading);

/* The maximum-IoU (Hungarian) matching of evaluate_waymo.py's matching="hungarian", in three passes.
 * pnx_eval_pairs: the feasible pairs (IoU >= thresholds[c], the IoU of pnx_eval_match) of every segment, operands as for
 *   pnx_eval_match.  With edge_start null it writes edge_count [B C] only; with edge_start [B C] (the exclusive prefix
 *   sum of edge_count) it writes segment s's pairs at [edge_start[s], ..): e_det = detection index, e_box = f M + j,
 *   e_iou, e_head = the pair's heading accuracy (as pnx_eval_match's); detections in visit order, each one's boxes in
 *   ascending j.
 * pnx_eval_components: the connected components of each segment's pairs (E = n_edges).  root [E] = the component's
 *   first pair; for a root, comp_start [E] = where its pairs begin in grouped [E] (pair indices, each component's
 *   contiguous, in pair order) and comp_nedge [E] = their number; for any other pair -1 and 0.
 * pnx_eval_assign: every listed component solved exactly for each breakdown b (0 = all pairs, 1 = pairs whose
 *   detection and box share a range: det_range [D], gt_range [B M]) and each score cutoff k < K (a detection takes part
 *   if k < det_pass[d]).  small_roots [n_small] = the roots of the components of at most pnx_eval_assign_warp_pairs()
 *   pairs (one warp each, shared memory); large_roots [n_large] = the others, large_off [n_large] int64 = the exclusive
 *   prefix sum of their pair counts, large_pairs = the total.  The assignment maximises the sum of the fp32 IoUs (exact in 40-bit fixed point, every IoU being >=
 *   2^-17); of several maxima it takes the one chosen detection by detection in visit order, each taking the first
 *   possible of its boxes in ascending j, then "unmatched".  match [2, K, D] int32 = the box index j within the frame or
 *   -1, heading [2, K, D] fp32 = the matched pair's e_head or 0.  `workspace` holds
 *   pnx_eval_assign_workspace(large_pairs) bytes of device memory (no initialisation needed).
 * All three run on `stream` with no host sync; the _host twins take HOST memory and no workspace. */
int pnx_eval_pairs(const float* det_boxes, const float* det_trig, long long n_det, const long long* order,
                   const int* seg_start, const int* seg_count, const float* gt_boxes, const int* gt_classes,
                   const float* gt_trig, int B, int M, int C, const float* thresholds, const int* edge_start,
                   int* edge_count, int* e_det, int* e_box, float* e_iou, float* e_head, cudaStream_t stream);
int pnx_eval_pairs_host(const float* det_boxes, const float* det_trig, long long n_det, const long long* order,
                        const int* seg_start, const int* seg_count, const float* gt_boxes, const int* gt_classes,
                        const float* gt_trig, int B, int M, int C, const float* thresholds, const int* edge_start,
                        int* edge_count, int* e_det, int* e_box, float* e_iou, float* e_head);
int pnx_eval_components(const int* edge_start, const int* edge_count, int B, int M, int C, long long n_edges,
                        const int* e_det, const int* e_box, int* root, int* comp_start, int* comp_nedge, int* grouped,
                        cudaStream_t stream);
int pnx_eval_components_host(const int* edge_start, const int* edge_count, int B, int M, int C, long long n_edges,
                             const int* e_det, const int* e_box, int* root, int* comp_start, int* comp_nedge,
                             int* grouped);
long long pnx_eval_assign_workspace(long long large_pairs);
int pnx_eval_assign_warp_pairs(void);
int pnx_eval_assign(long long n_edges, const int* grouped, const int* comp_start, const int* comp_nedge,
                    const int* e_det, const int* e_box, const float* e_iou, const float* e_head, const int* small_roots,
                    int n_small, const int* large_roots, const long long* large_off, int n_large, long long large_pairs,
                    long long n_det, const int* det_pass, const int* det_range, const int* gt_range, int M, int K,
                    int* match, float* heading, void* workspace, cudaStream_t stream);
int pnx_eval_assign_host(long long n_edges, const int* grouped, const int* comp_start, const int* comp_nedge,
                         const int* e_det, const int* e_box, const float* e_iou, const float* e_head,
                         const int* small_roots, int n_small, const int* large_roots, const long long* large_off,
                         int n_large, long long large_pairs, long long n_det, const int* det_pass, const int* det_range,
                         const int* gt_range, int M, int K, int* match, float* heading);

/* ------------------------------------------------ tracking (pillarnext_b200/track.py, evaluate_waymo_tracking.py)
 * pnx_track_greedy: the velocity-based greedy tracker, per (sequence, class).  boxes [n_det, 9] fp32 (x, y, z, dx, dy,
 *   dz, vx, vy, yaw in the frame's sensor coordinates), scores [n_det]; order [n_det] int64 = detection indices sorted
 *   by segment f C + c, then descending score, ties to the lower index; segment s holds order[seg_start[s] ..
 *   + seg_count[s]) ([F C] int32); poses [F, 4, 4] fp64 sensor -> global; times [F] int64 microseconds; the frames of
 *   sequence q are [seq_start[q], seq_start[q + 1]) ([S + 1] int32), in ascending time; max_dist [C] fp32 metres.
 *   Per frame, each detection with score >= min_score (in order) takes the unclaimed live track nearest to its
 *   back-projected global centre p - v dt, if within max_dist (ties to the older track), else starts a track; matched
 *   tracks take the detection's p and v, the others move by v dt and are dropped after more than max_age misses
 *   (track.py's docstring states every rounding).  Output track_id [n_det] int64: ids consecutive per sequence in
 *   birth order (frame, class, visit order), -1 below min_score.  Scratch: local_id [n_det], births [S C], map
 *   [n_det] int32; row_det_start [S C] int64 = the exclusive prefix sum of the detections per (sequence, class).
 *   status [1] int32 = 0, or 1 + the first (sequence, class) whose live tracks would exceed cap (its ids are then
 *   incomplete, the rest -1).  cap in [1, pnx_track_max_tracks()] = the track slots per (sequence, class) in shared
 *   memory; min(pnx_track_max_tracks(), (max_age + 2) x the largest seg_count) can never run out early, as every live
 *   track was matched or born in the last max_age + 1 frames, plus this frame's births.  C <= 64.  The host twin takes
 *   HOST memory, no scratch, and pnx_track_max_tracks() slots.
 * pnx_eval_mot: the CLEAR-MOT frame matching of evaluate_waymo_tracking.py, one row per (sequence, class, cutoff)
 *   walking the sequence's frames (seq_start [S + 1], frames as for pnx_eval_pairs' segments).  Inputs: the pairs of
 *   pnx_eval_pairs (edge_start / edge_count [B C], e_det, e_box, e_iou), the components of pnx_eval_components
 *   (grouped, comp_start, comp_nedge), det_pass [n_det] (cutoffs each detection passes), det_id [n_det] int32
 *   tracking ids >= 0, gt_obj [B M] int32 object index in [0, n_obj) or -1, gt_points [B M] int32 point counts.
 *   Per frame: carry-over (pairs in order whose detection passes the cutoff and carries the object's last matched id,
 *   each unless its detection or box is already kept), then the tie-ruled maximum-IoU assignment of pnx_eval_assign on
 *   the remaining pairs.  Outputs counts [S, C, K, 5] int64 = matches (every level), L1 matches, L1 mismatches, L2
 *   matches, L2 mismatches (L1: > 5 points, L2: >= 1), dist [S, C, K, 2] fp64 = the sum of 1 - IoU over the L1 / L2
 *   matches in match order, last_id [K, n_obj] int32 scratch.  cap >= max(pnx_eval_assign_warp_pairs() + 2, the
 *   largest component's pair count); workspace = pnx_eval_mot_workspace(S C K, M, cap) bytes, about
 *   S C K (164 cap + 4 M): every row gets room for the largest component anywhere.  The host twin takes
 *   HOST memory and no workspace. */
int pnx_track_max_tracks(void);
int pnx_track_greedy(const float* boxes, const float* scores, long long n_det, const long long* order,
                     const int* seg_start, const int* seg_count, const double* poses, const long long* times,
                     const int* seq_start, int S, int F, int C, const float* max_dist, int max_age, float min_score,
                     int cap, const long long* row_det_start, int* local_id, int* births, int* map,
                     long long* track_id, int* status, cudaStream_t stream);
int pnx_track_greedy_host(const float* boxes, const float* scores, long long n_det, const long long* order,
                          const int* seg_start, const int* seg_count, const double* poses, const long long* times,
                          const int* seq_start, int S, int F, int C, const float* max_dist, int max_age,
                          float min_score, long long* track_id, int* status);
long long pnx_eval_mot_workspace(int rows, int M, int cap);
int pnx_eval_mot(const int* edge_start, const int* edge_count, long long n_edges, const int* grouped,
                 const int* comp_start, const int* comp_nedge, const int* e_det, const int* e_box, const float* e_iou,
                 long long n_det, const int* det_pass, const int* det_id, const int* gt_obj, const int* gt_points,
                 const int* seq_start, int S, int B, int M, int C, int K, int n_obj, int cap, int* last_id,
                 long long* counts, double* dist, void* workspace, cudaStream_t stream);
int pnx_eval_mot_host(const int* edge_start, const int* edge_count, long long n_edges, const int* grouped,
                      const int* comp_start, const int* comp_nedge, const int* e_det, const int* e_box,
                      const float* e_iou, long long n_det, const int* det_pass, const int* det_id, const int* gt_obj,
                      const int* gt_points, const int* seq_start, int S, int B, int M, int C, int K, int n_obj, int cap,
                      int* last_id, long long* counts, double* dist);

/* ------------------------------------------------ nuScenes detection score (pillarnext_b200/evaluate_nuscenes.py)
 * pnx_eval_match_center: the centre-distance match of the nuScenes detection benchmark, per (frame, class) segment
 *   s = f C + c and per distance threshold.  det_boxes [n_det, 9] (x, y first); order [n_det] int64 = detection indices
 *   sorted by segment, then in visit order (descending score, ties to the later detection); segment s holds
 *   order[seg_start[s] .. seg_start[s] + seg_count[s]) (seg_start / seg_count [B C] int32); gt_boxes [B, M, 9],
 *   gt_classes [B, M] in [0, C) or -1 (padding or filtered out); dist_ths [T] fp64 metres, 1 <= T <= 8; M <= 4096.
 *   For each threshold independently, each detection in order takes the not yet matched box of its segment with the
 *   smallest centre distance sqrt(dx^2 + dy^2) (fp64 differences of the fp32 coordinates), ties to the lower box index,
 *   if that distance is < dist_ths[t].  Output match [T, n_det] int32 (column indexed like det_boxes): the box index j
 *   within the frame, or -1.
 * Runs on `stream` with no host sync and no workspace; the _host twin takes HOST memory. */
int pnx_eval_match_center(const float* det_boxes, long long n_det, const long long* order, const int* seg_start,
                          const int* seg_count, const float* gt_boxes, const int* gt_classes, int B, int M, int C,
                          const double* dist_ths, int T, int* match, cudaStream_t stream);
int pnx_eval_match_center_host(const float* det_boxes, long long n_det, const long long* order, const int* seg_start,
                               const int* seg_count, const float* gt_boxes, const int* gt_classes, int B, int M, int C,
                               const double* dist_ths, int T, int* match);

/* ------------------------------------------------ nuScenes tracking (pillarnext_b200/evaluate_nuscenes_tracking.py)
 * pnx_eval_pairs_center: the pairs of every (frame, class) segment whose centre distance (pnx_eval_match_center's
 *   fp64 arithmetic) is < max_dist, 0 < max_dist <= 2 metres.  Operands as for pnx_eval_match_center (order: by
 *   segment, then in visit order); outputs laid out as pnx_eval_pairs': edge_start null -> edge_count [B C] only;
 *   edge_start [B C] -> e_det, e_box = f M + j, e_dist = the distance rounded to fp32, detections in visit order, each
 *   one's boxes in ascending j.
 * pnx_eval_mot_center: pnx_eval_mot's frame walk, rows (S, C, K), carry-over and operands (e_dist in place of e_iou),
 *   with another assignment weight and other counts.  The assignment takes the most pairs, then the smallest sum of
 *   distances, ties by pnx_eval_assign's rule: it maximises 2^40 - round(e_dist 2^26) per pair, and as a component
 *   has at most M <= 2^12 matches of at most 2^27 each, one more match outweighs any distance sum.  gt_prev [B M]
 *   int32 = the frame of the same object's previous box (-1 for its first, or no object).  Outputs counts [S, C, K, 3]
 *   int64 = matches, identity switches (a match whose id differs from the object's last matched id), fragmentations
 *   (a match of an object that was matched before and has a box in a frame after that match); dist [S, C, K] fp64 =
 *   the sum of the matches' e_dist in match order; matched [n_det] uint8 (null, or K = 1 only) = 1 for each matched
 *   detection, else 0.  last_id, last_frame [K, n_obj] int32 scratch.  cap as for pnx_eval_mot; workspace =
 *   pnx_eval_mot_workspace(S C K, M, cap) bytes (the same row layout).
 * Both run on `stream` with no host sync; the _host twins take HOST memory and no workspace, and equal them bit for
 * bit. */
int pnx_eval_pairs_center(const float* det_boxes, long long n_det, const long long* order, const int* seg_start,
                          const int* seg_count, const float* gt_boxes, const int* gt_classes, int B, int M, int C,
                          double max_dist, const int* edge_start, int* edge_count, int* e_det, int* e_box,
                          float* e_dist, cudaStream_t stream);
int pnx_eval_pairs_center_host(const float* det_boxes, long long n_det, const long long* order, const int* seg_start,
                               const int* seg_count, const float* gt_boxes, const int* gt_classes, int B, int M, int C,
                               double max_dist, const int* edge_start, int* edge_count, int* e_det, int* e_box,
                               float* e_dist);
int pnx_eval_mot_center(const int* edge_start, const int* edge_count, long long n_edges, const int* grouped,
                        const int* comp_start, const int* comp_nedge, const int* e_det, const int* e_box,
                        const float* e_dist, long long n_det, const int* det_pass, const int* det_id, const int* gt_obj,
                        const int* gt_prev, const int* seq_start, int S, int B, int M, int C, int K, int n_obj, int cap,
                        int* last_id, int* last_frame, long long* counts, double* dist, unsigned char* matched,
                        void* workspace, cudaStream_t stream);
int pnx_eval_mot_center_host(const int* edge_start, const int* edge_count, long long n_edges, const int* grouped,
                             const int* comp_start, const int* comp_nedge, const int* e_det, const int* e_box,
                             const float* e_dist, long long n_det, const int* det_pass, const int* det_id,
                             const int* gt_obj, const int* gt_prev, const int* seq_start, int S, int B, int M, int C,
                             int K, int n_obj, int cap, int* last_id, int* last_frame, long long* counts, double* dist,
                             unsigned char* matched);

#ifdef __cplusplus
}
#endif
#endif /* PNX_H_ */
