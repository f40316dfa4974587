// Place recognition by randomized ferns (omnidata_b200/places.py FernDatabase; Glocker et al. 2015, as ElasticFusion
// uses it): a compact code per frame from a 60 x 80 thumbnail of depth and colour, and a Hamming-style lookup of one
// code against a database of codes.  Definition in DESIGN.md §3 "Place recognition and relocalisation" and
// include/omnidata_b200.h; oracle/places_oracle.py restates it in float64.
//
//   fern_cells_kernel    one thread per (cell, channel, frame): the mean of the channel's usable samples in the cell,
//                        summed in fp64 in row-major pixel order and rounded to fp32 (NaN where a cell has none)
//   fern_stats_kernel    one CTA per (frame, channel): m = the lower median of the finite cells and s = the lower
//                        median of |v - m| (fp32 round-to-nearest difference), both exact order statistics from
//                        block_radix_select's integer histograms
//   fern_code_kernel     one thread per (frame, fern): bit c = (v_c - m_c) > theta_c s_c in round-to-nearest fp64
//   fern_distance_kernel one warp per database entry: the number of ferns whose codes differ (integer warp sum)
//   fern_select_kernel   one CTA: the k smallest distances from a (F + 1)-bin integer histogram, ties to the lower
//                        index, entries in index order through block-wide integer scans, padded with -1
//
// Integer shared-memory atomics only (histograms), no floating-point atomics; built without fast-math; every output is
// bit-reproducible.  Launch sequences are fixed for the arguments (3 launches to encode, 2 to query) with no host
// synchronisation, so both calls can be captured in a CUDA graph.
#include <cmath>

#include "common.cuh"
#include "host_util.h"
#include "select.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kFernRows = ODB_FERN_GRID_ROWS, kFernCols = ODB_FERN_GRID_COLS;
constexpr int kFernCells = kFernRows * kFernCols;
constexpr int kFernChannels = 4;                  // depth, R, G, B
constexpr int kCellThreads = 128;
constexpr int kStatThreads = 512;
constexpr int kCodeThreads = 128;
constexpr int kDistThreads = 256;                 // 8 entries (warps) per CTA
constexpr int kSelThreads = 1024;

// workspace of odb_fern_encode: cells fp32 [n][4][4800], then (m, s) fp32 [n][4][2]
static int64_t fern_encode_bytes(int32_t n) {
  const int64_t floats = (int64_t)n * kFernChannels * (kFernCells + 2);
  return (floats * 4 + 7) / 8 * 8;
}

__global__ void __launch_bounds__(kCellThreads) fern_cells_kernel(int h, int w, const float* __restrict__ depth,
                                                                  const float* __restrict__ rgb,
                                                                  float* __restrict__ cells) {
  const int cell = blockIdx.x * kCellThreads + threadIdx.x;
  const int q = blockIdx.y;                       // channel: 0 depth, 1..3 R, G, B
  const int img = blockIdx.z;
  if (cell >= kFernCells) return;
  const int r = cell / kFernCols, c = cell - r * kFernCols;
  const int y0 = (int)((long long)r * h / kFernRows), y1 = (int)((long long)(r + 1) * h / kFernRows);
  const int x0 = (int)((long long)c * w / kFernCols), x1 = (int)((long long)(c + 1) * w / kFernCols);
  const long long plane = (long long)h * w;
  const float* src = q == 0 ? depth + img * plane : rgb + (img * 3LL + q - 1) * plane;
  double sum = 0.0;
  int cnt = 0;
  for (int y = y0; y < y1; ++y) {
    for (int x = x0; x < x1; ++x) {
      const float v = __ldg(src + (long long)y * w + x);
      if (isfinite(v) && (q != 0 || v > 0.0f)) {
        sum = __dadd_rn(sum, (double)v);
        ++cnt;
      }
    }
  }
  cells[((long long)img * kFernChannels + q) * kFernCells + cell] =
      cnt ? __double2float_rn(__ddiv_rn(sum, (double)cnt)) : __int_as_float(0x7fc00000);
}

__global__ void __launch_bounds__(kStatThreads) fern_stats_kernel(const float* __restrict__ cells,
                                                                  float* __restrict__ stats) {
  __shared__ float v[kFernCells];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t bcast[2];
  __shared__ int nfinite;
  const float* src = cells + (long long)blockIdx.x * kFernCells;     // blockIdx.x = frame * 4 + channel
  if (threadIdx.x == 0) nfinite = 0;
  __syncthreads();
  int mine = 0;
  for (int i = threadIdx.x; i < kFernCells; i += kStatThreads) {
    v[i] = src[i];
    mine += isnan(v[i]) ? 0 : 1;
  }
  atomicAdd(&nfinite, mine);
  __syncthreads();
  const int nf = nfinite;
  if (nf == 0) {
    if (threadIdx.x == 0) stats[2 * blockIdx.x] = stats[2 * blockIdx.x + 1] = __int_as_float(0x7fc00000);
    return;
  }
  auto usable = [&](long long i) { return !isnan(v[i]); };
  const unsigned long long rank = (unsigned long long)(nf - 1) / 2;
  const float m = key_to_float(block_radix_select(v, kFernCells, rank, usable, hist, bcast));
  for (int i = threadIdx.x; i < kFernCells; i += kStatThreads)
    if (!isnan(v[i])) v[i] = fabsf(__fsub_rn(v[i], m));
  __syncthreads();
  const float s = key_to_float(block_radix_select(v, kFernCells, rank, usable, hist, bcast));
  if (threadIdx.x == 0) {
    stats[2 * blockIdx.x] = m;
    stats[2 * blockIdx.x + 1] = s;
  }
}

__global__ void __launch_bounds__(kCodeThreads) fern_code_kernel(int n_ferns, const int32_t* __restrict__ fern_cells,
                                                                 const double* __restrict__ thresholds,
                                                                 const float* __restrict__ cells,
                                                                 const float* __restrict__ stats,
                                                                 uint8_t* __restrict__ codes) {
  const int f = blockIdx.x * kCodeThreads + threadIdx.x;
  const int img = blockIdx.y;
  if (f >= n_ferns) return;
  const int p = fern_cells[f];
  uint32_t code = 0;
  if (p >= 0 && p < kFernCells) {
#pragma unroll
    for (int q = 0; q < kFernChannels; ++q) {
      const int ch = img * kFernChannels + q;
      const float x = cells[(long long)ch * kFernCells + p];
      const float m = stats[2 * ch], s = stats[2 * ch + 1];
      // a NaN cell, a channel without finite cells (m, s NaN) or with s = 0 gives 0
      if (!isnan(x) && s > 0.0f &&
          __dsub_rn((double)x, (double)m) > __dmul_rn(thresholds[kFernChannels * f + q], (double)s))
        code |= 1u << q;
    }
  }
  codes[(long long)img * n_ferns + f] = (uint8_t)code;
}

__global__ void __launch_bounds__(kDistThreads) fern_distance_kernel(int n_ferns, int limit,
                                                                     const uint8_t* __restrict__ db,
                                                                     const uint8_t* __restrict__ code,
                                                                     int32_t* __restrict__ dist) {
  const int lane = threadIdx.x & 31;
  const long long i = (long long)blockIdx.x * (kDistThreads / 32) + (threadIdx.x >> 5);
  if (i >= limit) return;
  const uint8_t* row = db + i * n_ferns;
  unsigned diff = 0;
  for (int f = lane; f < n_ferns; f += 32) diff += __ldg(row + f) != __ldg(code + f) ? 1u : 0u;
  diff = __reduce_add_sync(0xffffffffu, diff);
  if (lane == 0) dist[i] = (int32_t)diff;
}

// exclusive block-wide prefix count of `flag` in thread order, and the block's total; warp_tot [32] shared
ODB_DEVINL int block_scan_flag(bool flag, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ballot = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_tot[warp] = __popc(ballot);
  __syncthreads();
  int before = 0, all = 0;
  for (int q = 0; q < kSelThreads / 32; ++q) {
    before += q < warp ? warp_tot[q] : 0;
    all += warp_tot[q];
  }
  __syncthreads();
  *total = all;
  return before + __popc(ballot & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(kSelThreads) fern_select_kernel(int n_ferns, int limit, int k,
                                                                  const int32_t* __restrict__ dist,
                                                                  int32_t* __restrict__ out_index,
                                                                  int32_t* __restrict__ out_distance) {
  __shared__ uint32_t hist[ODB_FERN_MAX_FERNS + 1];
  __shared__ int32_t s_idx[ODB_FERN_MAX_K], s_dist[ODB_FERN_MAX_K];
  __shared__ int warp_tot[2][kSelThreads / 32];
  __shared__ int sh[3];                           // D, entries below D, entries at D to take
  for (int d = threadIdx.x; d <= n_ferns; d += kSelThreads) hist[d] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < limit; i += kSelThreads) atomicAdd(&hist[dist[i]], 1u);
  __syncthreads();
  if (threadIdx.x == 0) {
    // D: the smallest distance with at least k entries at or below it (n_ferns + 1 when there are fewer than k)
    int D = 0, below = 0;
    for (; D <= n_ferns; ++D) {
      if (below + (int)hist[D] >= k) break;
      below += (int)hist[D];
    }
    sh[0] = D;
    sh[1] = below;
    sh[2] = D <= n_ferns ? k - below : 0;
  }
  __syncthreads();
  const int D = sh[0], n_less = sh[1], n_eq = sh[2];
  // gather, in index order: every entry below D at [0, n_less), the first n_eq entries at D at [n_less, n_less + n_eq)
  int got_less = 0, got_eq = 0;
  for (int c = 0; c < limit && (got_less < n_less || got_eq < n_eq); c += kSelThreads) {
    const int i = c + threadIdx.x;
    const int d = i < limit ? dist[i] : -1;
    const bool lt = i < limit && d < D, eq = i < limit && d == D;
    int t_lt, t_eq;
    const int r_lt = block_scan_flag(lt, warp_tot[0], &t_lt);
    const int r_eq = block_scan_flag(eq, warp_tot[1], &t_eq);
    if (lt) {
      s_idx[got_less + r_lt] = i;
      s_dist[got_less + r_lt] = d;
    }
    if (eq && got_eq + r_eq < n_eq) {
      s_idx[n_less + got_eq + r_eq] = i;
      s_dist[n_less + got_eq + r_eq] = d;
    }
    got_less += t_lt;
    got_eq += t_eq;
  }
  __syncthreads();
  // entries below D to (distance, index) order by rank; those at D are already in index order after them
  const int t = threadIdx.x;
  if (t < n_less) {
    const int dt = s_dist[t], it = s_idx[t];
    int rank = 0;
    for (int u = 0; u < n_less; ++u) rank += (s_dist[u] < dt || (s_dist[u] == dt && s_idx[u] < it)) ? 1 : 0;
    out_index[rank] = it;
    out_distance[rank] = dt;
  } else if (t < n_less + n_eq) {
    out_index[t] = s_idx[t];
    out_distance[t] = s_dist[t];
  } else if (t < k) {
    out_index[t] = -1;
    out_distance[t] = -1;
  }
}

static bool fern_count_ok(int32_t n_ferns) { return n_ferns >= 1 && n_ferns <= ODB_FERN_MAX_FERNS; }

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_fern_encode_workspace_bytes(int32_t n) {
  if (n < 1 || n > 65535) return -1;
  return fern_encode_bytes(n);
}

extern "C" int odb_fern_encode(int32_t n, int32_t h, int32_t w, const float* depth, const float* rgb, int32_t n_ferns,
                               const int32_t* fern_cells, const double* fern_thresholds, uint8_t* codes,
                               void* workspace, void* stream_) {
  if (!planes_ok(n, h, w) || h < kFernRows || w < kFernCols || !fern_count_ok(n_ferns) || !depth || !rgb ||
      !fern_cells || !fern_thresholds || !codes || !workspace || !aligned(depth, 4) || !aligned(rgb, 4) ||
      !aligned(fern_cells, 4) || !aligned(fern_thresholds, 8) || !aligned(workspace, 8))
    return fail(ODB_ERR_INVALID, "fern_encode: bad argument");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  float* cells = static_cast<float*>(workspace);
  float* stats = cells + (int64_t)n * kFernChannels * kFernCells;
  fern_cells_kernel<<<dim3((kFernCells + kCellThreads - 1) / kCellThreads, kFernChannels, n), kCellThreads, 0,
                      stream>>>(
      h, w, depth, rgb, cells);
  count_launch();
  fern_stats_kernel<<<n * kFernChannels, kStatThreads, 0, stream>>>(cells, stats);
  count_launch();
  fern_code_kernel<<<dim3((n_ferns + kCodeThreads - 1) / kCodeThreads, n), kCodeThreads, 0, stream>>>(
      n_ferns, fern_cells, fern_thresholds, cells, stats, codes);
  count_launch();
  return check_launch("fern_encode");
}

extern "C" int64_t odb_fern_query_workspace_bytes(int32_t n_db) {
  if (n_db < 1 || n_db > ODB_FERN_MAX_ENTRIES) return -1;
  return ((int64_t)n_db * 4 + 7) / 8 * 8;
}

extern "C" int odb_fern_query(int32_t n_db, int32_t n_ferns, const uint8_t* db_codes, const uint8_t* code,
                              int32_t limit, int32_t k, int32_t* out_index, int32_t* out_distance, void* workspace,
                              void* stream_) {
  if (n_db < 1 || n_db > ODB_FERN_MAX_ENTRIES || !fern_count_ok(n_ferns) || limit < 0 || limit > n_db || k < 1 ||
      k > ODB_FERN_MAX_K || !db_codes || !code || !out_index || !out_distance || !workspace ||
      !aligned(out_index, 4) || !aligned(out_distance, 4) || !aligned(workspace, 8))
    return fail(ODB_ERR_INVALID, "fern_query: bad argument");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int32_t* dist = static_cast<int32_t*>(workspace);
  const int64_t per = kDistThreads / 32;         // n_db <= 2^28: at most 2^25 CTAs
  fern_distance_kernel<<<(unsigned)(((int64_t)n_db + per - 1) / per), kDistThreads, 0, stream>>>(
      n_ferns, limit, db_codes, code, dist);
  count_launch();
  fern_select_kernel<<<1, kSelThreads, 0, stream>>>(n_ferns, limit, k, dist, out_index, out_distance);
  count_launch();
  return check_launch("fern_query");
}
