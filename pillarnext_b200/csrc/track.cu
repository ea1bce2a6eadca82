// track.cu -- the velocity-based greedy tracker of pillarnext_b200/track.py on sm_90a.
//   pnx_track_greedy  two kernels.  track_greedy_kernel: one warp per (sequence, class) walks the sequence's frames in
//                     order.  The live tracks (global BEV position, velocity, id, misses) live in shared memory, in a
//                     table of `cap` <= kMaxTracks slots the caller sizes to what the input can need, so that small
//                     inputs keep several warps per SM.  The frame's detections are visited in the order of the caller's key sort
//                     (descending score, ties to the lower index); for each, the lanes compute the distance of its
//                     back-projected global centre to their unclaimed tracks and a shuffle arg-min picks the nearest,
//                     ties to the older track, as eval_match_center_kernel does.  The result is a per-(sequence, class)
//                     track number in birth order.  track_renumber_kernel: one warp per sequence turns those numbers
//                     into ids consecutive over the sequence, in birth order (frame, then class, then visit order).
// Every floating-point step is a __host__ __device__ routine shared with the host twin, and the file is compiled with
// -fmad=false (pillarnext_b200/build.py), so the kernels equal pnx_track_greedy_host to the bit.  No host sync inside.
#include <limits.h>
#include <math.h>

#include <vector>

#include "pnx_common.cuh"

namespace {

constexpr int kMaxTracks = 4096;   // live tracks per (sequence, class), those born in the current frame included
constexpr int kNone = 0x7fffffff;

struct TrackArgs {
  const float* boxes;         // [D, 9] x, y, z, dx, dy, dz, vx, vy, yaw in the frame's sensor coordinates
  const float* scores;        // [D]
  const long long* order;     // [D] detection indices sorted by segment f C + c, then descending score
  const int* seg_start;       // [F C]
  const int* seg_count;       // [F C]
  const double* poses;        // [F, 4, 4] sensor -> global, row-major
  const long long* times;     // [F] microseconds
  const int* seq_start;       // [S + 1] the frames of sequence s are [seq_start[s], seq_start[s + 1])
  int S, F, C;
  const float* max_dist;      // [C] metres
  int max_age;
  float min_score;
  int* local_id;              // [D] OUT the track's number within its (sequence, class), -1 below min_score
  int* births;                // [S C] OUT tracks born per (sequence, class)
  int* status;                // [1] OUT 0, or 1 + the first (sequence, class) row that ran out of track slots
  int cap;                    // track slots per (sequence, class): <= kMaxTracks
};

// BEV centre and velocity of box b in the global frame of pose T: fp64 products and sums in this order, one fp32 rounding.
__host__ __device__ inline void to_global(const double* T, const float* b, float* p, float* v) {
  const double x = b[0], y = b[1], z = b[2], vx = b[6], vy = b[7];
  p[0] = (float)(T[0] * x + T[1] * y + T[2] * z + T[3]);
  p[1] = (float)(T[4] * x + T[5] * y + T[6] * z + T[7]);
  v[0] = (float)(T[0] * vx + T[1] * vy);
  v[1] = (float)(T[4] * vx + T[5] * vy);
}

// Frame gap in seconds: the exact integer difference of the microsecond stamps, times 1e-6 in fp64, rounded to fp32.
__host__ __device__ inline float frame_dt(const long long* times, int f, int first) {
  return f == first ? 0.0f : (float)((double)(times[f] - times[f - 1]) * 1e-6);
}

// fp32 distance of the back-projected centre b = p - v dt to track position (qx, qy)
__host__ __device__ inline float track_distance(const float* p, const float* v, float dt, float qx, float qy) {
  const float bx = p[0] - v[0] * dt, by = p[1] - v[1] * dt;
  const float dx = bx - qx, dy = by - qy;
  return sqrtf(dx * dx + dy * dy);
}

// Track table of one (sequence, class): structure of arrays, slots [0, n) in birth order.
struct Tracks {
  float *qx, *qy, *vx, *vy;
  int *id, *misses, *match;   // match: the detection holding the slot this frame, -1 = none
};

__host__ __device__ inline Tracks carve_tracks(void* base, int cap) {
  float* f = (float*)base;
  int* i = (int*)(f + 4 * (size_t)cap);
  return Tracks{f, f + cap, f + 2 * cap, f + 3 * cap, i, i + cap, i + 2 * cap};
}

constexpr size_t kTrackBytes = 4 * sizeof(float) + 3 * sizeof(int);

// End of a frame: matched tracks take the detection's position and velocity, the others coast (q += v dt) and age.
__host__ __device__ inline void update_slot(const TrackArgs& a, const Tracks& t, int q, const double* T, float dt) {
  const int di = t.match[q];
  if (di >= 0) {
    float p[2], v[2];
    to_global(T, a.boxes + (long long)di * 9, p, v);
    t.qx[q] = p[0]; t.qy[q] = p[1]; t.vx[q] = v[0]; t.vy[q] = v[1];
    t.misses[q] = 0;
  } else if (di == -1) {
    t.qx[q] = t.qx[q] + t.vx[q] * dt;
    t.qy[q] = t.qy[q] + t.vy[q] * dt;
    t.misses[q] += 1;
  }                                                            // -2: born this frame, already in place
}

__host__ __device__ inline void move_slot(const Tracks& t, int from, int to) {
  t.qx[to] = t.qx[from]; t.qy[to] = t.qy[from]; t.vx[to] = t.vx[from]; t.vy[to] = t.vy[from];
  t.id[to] = t.id[from]; t.misses[to] = t.misses[from];
}

__global__ void __launch_bounds__(32) track_greedy_kernel(TrackArgs a) {
  extern __shared__ float smem[];
  __shared__ int sh_n, sh_born, sh_next, sh_full;
  const Tracks t = carve_tracks(smem, a.cap);
  const int row = blockIdx.x, lane = threadIdx.x;
  const int s = row / a.C, c = row - s * a.C;
  const float maxd = a.max_dist[c];
  if (lane == 0) { sh_n = 0; sh_next = 0; sh_full = 0; }
  __syncwarp();
  const int f0 = a.seq_start[s], f1 = a.seq_start[s + 1];
  for (int f = f0; f < f1; ++f) {
    const double* T = a.poses + (long long)f * 16;
    const float dt = frame_dt(a.times, f, f0);
    const int n = sh_n;
    for (int q = lane; q < n; q += 32) t.match[q] = -1;
    if (lane == 0) sh_born = 0;
    __syncwarp();
    const int seg = f * a.C + c, base = a.seg_start[seg], cnt = a.seg_count[seg];
    for (int k = 0; k < cnt; ++k) {
      const long long di = a.order[base + k];
      if (!(a.scores[di] >= a.min_score)) {
        if (lane == 0) a.local_id[di] = -1;
        continue;
      }
      float p[2], v[2];
      to_global(T, a.boxes + di * 9, p, v);
      float best = INFINITY;
      int bq = kNone;
      for (int q = lane; q < n; q += 32) {                     // ascending q: the first minimum of the lane
        if (t.match[q] != -1) continue;
        const float d = track_distance(p, v, dt, t.qx[q], t.qy[q]);
        if (d <= maxd && d < best) { best = d; bq = q; }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oq = __shfl_xor_sync(0xffffffffu, bq, off);
        if (ob < best || (ob == best && oq < bq)) { best = ob; bq = oq; }
      }
      if (lane == 0) {
        if (bq != kNone) {
          t.match[bq] = (int)di;
          a.local_id[di] = t.id[bq];
        } else if (n + sh_born < a.cap) {
          const int q = n + sh_born++;
          t.qx[q] = p[0]; t.qy[q] = p[1]; t.vx[q] = v[0]; t.vy[q] = v[1];
          t.id[q] = sh_next++; t.misses[q] = 0; t.match[q] = -2;
          a.local_id[di] = t.id[q];
        } else {
          sh_full = 1;
        }
      }
      __syncwarp();
      if (sh_full) break;
    }
    if (sh_full) break;
    const int total = n + sh_born;
    for (int q = lane; q < n; q += 32) update_slot(a, t, q, T, dt);
    __syncwarp();
    // stable compaction of the survivors (misses <= max_age): read a chunk, then write it at or below where it was
    int kept = 0;
    for (int q0 = 0; q0 < total; q0 += 32) {
      const int q = q0 + lane;
      const bool live = q < total && t.misses[q] <= a.max_age;
      const unsigned bal = __ballot_sync(0xffffffffu, live);
      float r0 = 0, r1 = 0, r2 = 0, r3 = 0;
      int r4 = 0, r5 = 0;
      if (live) { r0 = t.qx[q]; r1 = t.qy[q]; r2 = t.vx[q]; r3 = t.vy[q]; r4 = t.id[q]; r5 = t.misses[q]; }
      __syncwarp();
      if (live) {
        const int to = kept + __popc(bal & ((1u << lane) - 1u));
        t.qx[to] = r0; t.qy[to] = r1; t.vx[to] = r2; t.vy[to] = r3; t.id[to] = r4; t.misses[to] = r5;
      }
      kept += __popc(bal);
      __syncwarp();
    }
    if (lane == 0) sh_n = kept;
    __syncwarp();
  }
  if (lane == 0) {
    a.births[row] = sh_next;
    if (sh_full) atomicMax(a.status, INT_MAX - row);          // the lowest overflowing row wins
  }
}

// One warp per sequence: every birth, in (frame, class, visit) order, takes the sequence's next id (map, indexed from
// row_det_start[row], the row's first detection slot); then every detection reads its track's id.
__global__ void __launch_bounds__(32) track_renumber_kernel(TrackArgs a, const long long* row_det_start, int* map,
                                                            long long* track_id) {
  __shared__ int next_local[64];
  const int s = blockIdx.x, lane = threadIdx.x;
  // the tracker left INT_MAX - (lowest overflowing row), or 0: turn it into the contract's 1 + row
  if (s == 0 && lane == 0 && *a.status) *a.status = 1 + (INT_MAX - *a.status);
  for (int c = lane; c < a.C; c += 32) next_local[c] = 0;
  __syncwarp();
  int next = 0;
  for (int pass = 0; pass < 2; ++pass)
    for (int f = a.seq_start[s]; f < a.seq_start[s + 1]; ++f)
      for (int c = 0; c < a.C; ++c) {
        const int seg = f * a.C + c, base = a.seg_start[seg], cnt = a.seg_count[seg];
        int* m = map + row_det_start[s * a.C + c];
        const int first = next_local[c];
        int born = 0;
        for (int k0 = 0; k0 < cnt; k0 += 32) {
          const int k = k0 + lane;
          const long long di = k < cnt ? a.order[base + k] : -1;
          const int l = di >= 0 ? a.local_id[di] : -1;
          if (pass == 0) {
            // this frame's births carry the row's next numbers, first, first + 1, .. in visit order
            if (l >= first) m[l] = next + (l - first);
            born += __popc(__ballot_sync(0xffffffffu, l >= first));
          } else if (di >= 0) {
            track_id[di] = l >= 0 ? (long long)m[l] : -1LL;
          }
        }
        next += born;
        __syncwarp();
        if (lane == 0) next_local[c] = first + born;
        __syncwarp();
      }
}

int check_track_args(const TrackArgs& a, long long D) {
  PNX_CHECK_ARG(a.S >= 0 && a.F >= 0 && a.C >= 1 && a.C <= 64 && a.max_age >= 0, "S / F / 1 to 64 classes / max_age");
  PNX_CHECK_ARG(D >= 0 && D < (1LL << 31) && (long long)a.F * a.C < (1LL << 31), "number of detections / segments");
  PNX_CHECK_ARG(a.seq_start && a.max_dist && a.status, "seq_start / max_dist / status");
  PNX_CHECK_ARG(a.F == 0 || (a.seg_start && a.seg_count && a.poses && a.times), "frame pointers");
  PNX_CHECK_ARG(D == 0 || (a.boxes && a.scores && a.order), "detection pointers");
  return PNX_OK;
}

}  // namespace

extern "C" int pnx_track_max_tracks(void) { return kMaxTracks; }

// Contract: include/pnx.h.
extern "C" int pnx_track_greedy(const float* boxes, const float* scores, long long n_det, const long long* order,
                                const int* seg_start, const int* seg_count, const double* poses, const long long* times,
                                const int* seq_start, int S, int F, int C, const float* max_dist, int max_age,
                                float min_score, int cap, const long long* row_det_start, int* local_id, int* births,
                                int* map, long long* track_id, int* status, cudaStream_t stream) {
  const TrackArgs a{boxes, scores, order, seg_start, seg_count, poses, times, seq_start, S, F, C, max_dist, max_age,
                    min_score, local_id, births, status, cap};
  int rc = check_track_args(a, n_det);
  if (rc) return rc;
  PNX_CHECK_ARG(S == 0 || births, "births");
  PNX_CHECK_ARG(cap >= 1 && cap <= kMaxTracks, "1 <= cap <= pnx_track_max_tracks()");
  PNX_CHECK_ARG(n_det == 0 || (row_det_start && map && track_id), "renumbering pointers");
  PNX_CUDA(cudaMemsetAsync(status, 0, sizeof(int), stream));
  if ((long long)S * C == 0 || n_det == 0) return PNX_OK;
  // every detection starts untracked: a row that runs out of slots stops early and leaves the rest at -1
  PNX_CUDA(cudaMemsetAsync(local_id, 0xff, (size_t)n_det * sizeof(int), stream));
  const size_t smem = (size_t)cap * kTrackBytes;
  PNX_CUDA(cudaFuncSetAttribute(track_greedy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  track_greedy_kernel<<<S * C, 32, smem, stream>>>(a);
  PNX_CHECK_LAUNCH();
  track_renumber_kernel<<<S, 32, 0, stream>>>(a, row_det_start, map, track_id);
  PNX_CHECK_LAUNCH();
  return PNX_OK;
}

// Host twin: the same per-(sequence, class) walk and renumbering on HOST memory, sequentially.
extern "C" int pnx_track_greedy_host(const float* boxes, const float* scores, long long n_det, const long long* order,
                                     const int* seg_start, const int* seg_count, const double* poses,
                                     const long long* times, const int* seq_start, int S, int F, int C,
                                     const float* max_dist, int max_age, float min_score, long long* track_id,
                                     int* status) {
  const TrackArgs a{boxes, scores, order, seg_start, seg_count, poses, times, seq_start, S, F, C, max_dist, max_age,
                    min_score, nullptr, nullptr, status, kMaxTracks};
  int rc = check_track_args(a, n_det);
  if (rc) return rc;
  PNX_CHECK_ARG(n_det == 0 || track_id, "track_id");
  std::vector<int> local_id(n_det > 0 ? n_det : 1);
  *status = 0;
  void* mem = new char[kMaxTracks * kTrackBytes];
  const Tracks t = carve_tracks(mem, kMaxTracks);
  std::vector<int> next_local(C);
  for (int s = 0; s < S && !*status; ++s) {
    // the tracker, one class at a time
    for (int c = 0; c < C && !*status; ++c) {
      int n = 0, next = 0;
      for (int f = seq_start[s]; f < seq_start[s + 1]; ++f) {
        const double* T = poses + (long long)f * 16;
        const float dt = frame_dt(times, f, seq_start[s]);
        for (int q = 0; q < n; ++q) t.match[q] = -1;
        int born = 0;
        const int seg = f * C + c;
        for (int k = 0; k < seg_count[seg]; ++k) {
          const long long di = order[seg_start[seg] + k];
          if (!(scores[di] >= min_score)) { local_id[di] = -1; continue; }
          float p[2], v[2];
          to_global(T, boxes + di * 9, p, v);
          float best = INFINITY;
          int bq = -1;
          for (int q = 0; q < n; ++q) {
            if (t.match[q] != -1) continue;
            const float d = track_distance(p, v, dt, t.qx[q], t.qy[q]);
            if (d <= max_dist[c] && d < best) { best = d; bq = q; }
          }
          if (bq >= 0) {
            t.match[bq] = (int)di;
            local_id[di] = t.id[bq];
          } else if (n + born < kMaxTracks) {
            const int q = n + born++;
            t.qx[q] = p[0]; t.qy[q] = p[1]; t.vx[q] = v[0]; t.vy[q] = v[1];
            t.id[q] = next++; t.misses[q] = 0; t.match[q] = -2;
            local_id[di] = t.id[q];
          } else {
            *status = 1 + s * C + c;
            break;
          }
        }
        if (*status) break;
        for (int q = 0; q < n; ++q) update_slot(a, t, q, T, dt);
        int kept = 0;
        for (int q = 0; q < n + born; ++q)
          if (t.misses[q] <= max_age) move_slot(t, q, kept++);
        n = kept;
      }
    }
    if (*status) break;
    // ids over the sequence in birth order: frame, then class, then visit order
    std::vector<std::vector<int>> map(C);
    for (int c = 0; c < C; ++c) next_local[c] = 0;
    int next = 0;
    for (int f = seq_start[s]; f < seq_start[s + 1]; ++f)
      for (int c = 0; c < C; ++c) {
        const int seg = f * C + c;
        const int first = next_local[c];
        for (int k = 0; k < seg_count[seg]; ++k) {
          const int l = local_id[order[seg_start[seg] + k]];
          if (l >= first) {
            if ((int)map[c].size() <= l) map[c].resize(l + 1, -1);
            map[c][l] = next++;
            next_local[c] = l + 1;
          }
        }
      }
    for (int f = seq_start[s]; f < seq_start[s + 1]; ++f)
      for (int c = 0; c < C; ++c) {
        const int seg = f * C + c;
        for (int k = 0; k < seg_count[seg]; ++k) {
          const long long di = order[seg_start[seg] + k];
          track_id[di] = local_id[di] >= 0 ? (long long)map[c][local_id[di]] : -1LL;
        }
      }
  }
  delete[] (char*)mem;
  return PNX_OK;
}
