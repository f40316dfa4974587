// Tiled inference for images of any size (omnidata_b200/tiled.py TiledPredictor): the image is cut into overlapping
// tiles the network accepts, every tile goes through the DPT forward (dpt_depth.py:67-85,107), and the tile predictions
// are merged back at the image's own size.
//
// Tile grid, per axis of length L, tile length t, overlap v (tile_grid in omnidata_b200/tiled.py restates it):
//   L <= t : one tile at origin 0 (the gather replicates the last row / column up to t);
//   L >  t : n = ceil((L - v) / (t - v)) tiles at o_k = round(k (L - t) / (n - 1)) (halves up); every tile lies inside
//            the image and neighbours overlap by >= v.
// Tiles are numbered row-major, i = ty * nx + tx.  Neighbour pairs (4-neighbourhood): the ny (nx - 1) horizontal pairs
// (ty, tx)-(ty, tx + 1) row-major, then the (ny - 1) nx vertical pairs (ty, tx)-(ty + 1, tx) row-major; in a pair, "a" is
// the first (left / upper) tile's prediction and "b" the second's.
//
// Kernels (no floating-point atomics; every result is bit-reproducible and independent of the batch):
//   tile_gather_kernel        image fp32 NCHW -> tiles [B*T][3][th][tw], 16-byte stores (HBM-bound)
//   tile_moments_kernel       depth: per (pair, image) n, Sa, Sb, Saa, Sbb, Sab over the overlap, fp64 (rect_moments)
//   tile_align_solve_kernel   depth: per image the per-tile scale / shift minimising
//                               E(s,t) = sum_pairs sum_overlap (s_i a + t_i - s_j b - t_j)^2
//                                        + lambda Nbar sum_i ((s_i - 1)^2 + t_i^2)
//                             (fp64 band_cholesky_solve, fp64.cuh, of the 2T x 2T normal equations; anchored form at
//                             the end)
//   tile_blend_kernel         each output pixel: sum_i w_i (s_i d_i + t_i) / sum_i w_i over its covering tiles
//
// The alignment follows the MiDaS scale-and-shift alignment of losses/midas_loss.py:10-30 (compute_scale_and_shift: a
// 2 x 2 least-squares system per image), generalised to all tiles of an image at once.  Built without fast-math: the
// merge promises IEEE fp32 / fp64 arithmetic that oracle/tiled_oracle.py restates.
#include <cmath>

#include "common.cuh"
#include "fp64.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr double kAlignLambda = 1e-3, kAnchorKappa = 1e-6;     // kappa: the ridge's share in the anchored solve
constexpr int kSolveThreads = 256;
constexpr size_t kSolveSmemMax = kBandSmemMax;

__host__ __device__ inline int tile_count(int L, int t, int v) {
  return L <= t ? 1 : (L - v + (t - v) - 1) / (t - v);
}
__host__ __device__ inline int tile_origin(int k, int n, int L, int t) {
  return n == 1 ? 0 : (2 * k * (L - t) + (n - 1)) / (2 * (n - 1));
}
// half-bandwidth + 1 of the interleaved (s_i, t_i) system: neighbours at tile distance 1 and nx
__host__ __device__ inline int band_width(int ny, int nx) { return ny > 1 ? 2 * nx + 2 : 4; }

// tiles[b*T + i][c][y][x] = image[b][c][min(oy_i + y, H - 1)][min(ox_i + x, W - 1)];  grid (chunks, 3 T, B), tw % 4 == 0
__global__ void __launch_bounds__(256) tile_gather_kernel(const float* __restrict__ img, int H, int W, int th, int tw,
                                                          int ny, int nx, float4* __restrict__ tiles) {
  const int tw4 = tw >> 2;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= th * tw4) return;
  const int y = e / tw4, x0 = (e - y * tw4) * 4;
  const int c = blockIdx.y % 3, ti = blockIdx.y / 3, b = blockIdx.z;
  const int T = ny * nx;
  const int oy = tile_origin(ti / nx, ny, H, th), ox = tile_origin(ti % nx, nx, W, tw);
  const float* row = img + (((long long)b * 3 + c) * H + min(oy + y, H - 1)) * W;
  const int sx = ox + x0;
  float4 v;
  if (sx + 3 < W && (reinterpret_cast<uintptr_t>(row + sx) & 15) == 0) {
    v = __ldg(reinterpret_cast<const float4*>(row + sx));
  } else {
    v.x = __ldg(row + min(sx, W - 1));
    v.y = __ldg(row + min(sx + 1, W - 1));
    v.z = __ldg(row + min(sx + 2, W - 1));
    v.w = __ldg(row + min(sx + 3, W - 1));
  }
  tiles[((((long long)b * T + ti) * 3 + c) * th * tw >> 2) + e] = v;
}

// Moments of two fp32 planes over an rh x rw rectangle, a at A[y * lda + x] and b at B[y * ldb + x]: returns
// S(a, b, a^2, b^2, a b)[q] in fp64 to thread q < 5 of the (256-thread) CTA.  Pixel e = y rw + x is summed by thread
// e % 256, each thread's pixels in increasing order; the 256 per-thread partials are combined by ordered_sum8.  The
// walk steps (y, x) by 256 pixels without divisions, and each thread loads kMomentBatch pixels before summing them, to
// keep loads in flight (a grid has few pairs and tiles: 12 and 9 at 1024^2); the zeros past the end add nothing.
constexpr int kMomentBatch = 8;
ODB_DEVINL double rect_moments(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb, int rh,
                               int rw) {
  __shared__ double part[5][256];
  double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  if (rw > 0) {
    const int dy = blockDim.x / rw, dx = blockDim.x - dy * rw;
    int y = threadIdx.x / rw, x = threadIdx.x - y * rw;
    while (y < rh) {
      float av[kMomentBatch], bv[kMomentBatch];
#pragma unroll
      for (int k = 0; k < kMomentBatch; ++k) {
        av[k] = bv[k] = 0.0f;
        if (y < rh) {
          av[k] = __ldg(A + (long long)y * lda + x);
          bv[k] = __ldg(B + (long long)y * ldb + x);
        }
        x += dx;
        y += dy;
        if (x >= rw) {
          x -= rw;
          ++y;
        }
      }
#pragma unroll
      for (int k = 0; k < kMomentBatch; ++k) {
        const double a = av[k], b = bv[k];
        s[0] += a;
        s[1] += b;
        s[2] = fma(a, a, s[2]);
        s[3] = fma(b, b, s[3]);
        s[4] = fma(a, b, s[4]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 5; ++q) part[q][threadIdx.x] = s[q];
  __syncthreads();
  const int col = threadIdx.x & 31;
  return ordered_sum8(256, col < 5, [&](int q) { return part[col][q]; });
}

// One CTA per (pair, image): moments[b][p] = (n, Sa, Sb, Saa, Sbb, Sab) over the pair's overlap inside the image.
__global__ void __launch_bounds__(256) tile_moments_kernel(const float* __restrict__ pred, int H, int W, int th, int tw,
                                                           int ny, int nx, double* __restrict__ moments) {
  const int p = blockIdx.x, b = blockIdx.y;
  const int T = ny * nx, nh = ny * (nx - 1), P = nh + (ny - 1) * nx;
  int i, j, y0, y1, x0, x1;                          // tiles and the overlap rectangle, image coordinates
  if (p < nh) {
    const int ty = p / (nx - 1), tx = p - ty * (nx - 1);
    i = ty * nx + tx;
    j = i + 1;
    y0 = tile_origin(ty, ny, H, th);
    y1 = y0 + min(th, H);
    x0 = tile_origin(tx + 1, nx, W, tw);
    x1 = tile_origin(tx, nx, W, tw) + tw;
  } else {
    const int q = p - nh, ty = q / nx, tx = q - ty * nx;
    i = ty * nx + tx;
    j = i + nx;
    x0 = tile_origin(tx, nx, W, tw);
    x1 = x0 + min(tw, W);
    y0 = tile_origin(ty + 1, ny, H, th);
    y1 = tile_origin(ty, ny, H, th) + th;
  }
  const int rw = max(x1 - x0, 0), rh = max(y1 - y0, 0);
  const int oyi = tile_origin(i / nx, ny, H, th), oxi = tile_origin(i % nx, nx, W, tw);
  const int oyj = tile_origin(j / nx, ny, H, th), oxj = tile_origin(j % nx, nx, W, tw);
  const float* A = pred + ((long long)b * T + i) * th * tw + (y0 - oyi) * tw + (x0 - oxi);
  const float* B = pred + ((long long)b * T + j) * th * tw + (y0 - oyj) * tw + (x0 - oxj);
  const double s = rect_moments(A, tw, B, tw, rh, rw);
  double* m = moments + ((long long)b * P + p) * 6;
  if (threadIdx.x < 5) m[1 + threadIdx.x] = s;
  if (threadIdx.x == 0) m[0] = (double)rw * (double)rh;
}

// One CTA per image.  Unknowns interleaved (s_0, t_0, s_1, t_1, ...): the normal equations are SPD and banded with
// half-bandwidth w - 1 (2 nx + 1; 3 for a single row of tiles).  The lower band is stored row-wise,
// band[r * w + q] = A[r][r - q], in shared memory when it fits, else in the image's slice of `workspace`.
__global__ void __launch_bounds__(kSolveThreads) tile_align_solve_kernel(const double* __restrict__ moments,
                                                                         const double* __restrict__ anchor, int ny,
                                                                         int nx, int band_in_smem, double* workspace,
                                                                         double* __restrict__ scale_shift) {
  extern __shared__ double sm[];
  __shared__ double s_ridge;
  const int b = blockIdx.x;
  const int T = ny * nx, n = 2 * T, w = band_width(ny, nx);
  const int nh = ny * (nx - 1), P = nh + (ny - 1) * nx;
  const double* mom = moments + (long long)b * P * 6;
  double* rhs = sm;
  double* band = band_in_smem ? sm + n : workspace + (long long)b * n * w;
  if (threadIdx.x == 0) {                            // ridge weight lambda * Nbar, Nbar = mean overlap pixel count (>= 1)
    double s = 0.0;
    for (int p = 0; p < P; ++p) s += mom[p * 6];
    s_ridge = kAlignLambda * (P > 0 ? fmax(s / P, 1.0) : 1.0);
  }
  __syncthreads();
  const double ridge = s_ridge, r0 = anchor != nullptr ? kAnchorKappa * ridge : ridge;     // anchored: kappa ridge
  // assembly: tile i writes rows 2i (s_i) and 2i + 1 (t_i): its diagonal 2 x 2 block, and the blocks coupling it to its
  // left and upper neighbour j < i (where i is the pair's second tile, b)
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    double* rs = band + (long long)(2 * i) * w;
    double* rt = rs + w;
    for (int q = 0; q < w; ++q) rs[q] = rt[q] = 0.0;
    const int ty = i / nx, tx = i - ty * nx;
    double ass = r0, ast = 0.0, att = r0, bs = r0, bt = 0.0;
    if (anchor != nullptr) {                          // mu_i (Saa, Sa; Sa, n), rhs mu_i (Sag, Sg), mu_i = ridge / n_i
      const double* g = anchor + ((long long)b * T + i) * 5;
      const double mu = ridge / g[0];
      ass = fma(mu, g[2], ass); ast = mu * g[1]; att = fma(mu, g[0], att);
      bs = fma(mu, g[4], bs); bt = mu * g[3];
    }
    if (tx < nx - 1) {                                // i is "a" of its right pair
      const double* m = mom + (ty * (nx - 1) + tx) * 6;
      ass += m[3]; ast += m[1]; att += m[0];
    }
    if (ty < ny - 1) {                                // ... and of its lower pair
      const double* m = mom + (nh + ty * nx + tx) * 6;
      ass += m[3]; ast += m[1]; att += m[0];
    }
    for (int side = 0; side < 2; ++side) {            // i is "b" of its left pair, then of its upper pair
      if (side == 0 ? tx == 0 : ty == 0) continue;
      const double* m = mom + (side == 0 ? ty * (nx - 1) + tx - 1 : nh + (ty - 1) * nx + tx) * 6;
      const int d = side == 0 ? 2 : 2 * nx;           // 2 (i - j)
      ass += m[4]; ast += m[2]; att += m[0];
      rs[d] = -m[5];                                  // (s_i, s_j)
      rs[d - 1] = -m[2];                              // (s_i, t_j)
      rt[d + 1] = -m[1];                              // (t_i, s_j)
      rt[d] = -m[0];                                  // (t_i, t_j)
    }
    rs[0] = ass;
    rt[1] = ast;
    rt[0] = att;
    rhs[2 * i] = bs;
    rhs[2 * i + 1] = bt;
  }
  __syncthreads();
  band_cholesky_solve(band, rhs, n, w);
  for (int e = threadIdx.x; e < n; e += blockDim.x) scale_shift[(long long)b * n + e] = rhs[e];
}

// tiles k0..k1 covering position p of an axis (consecutive: origins increase)
ODB_DEVINL void tile_cover(int p, int L, int t, int n, int& k0, int& k1) {
  int k = n == 1 ? 0 : min(n - 1, (int)((long long)p * (n - 1) / (L - t)));
  while (k + 1 < n && tile_origin(k + 1, n, L, t) <= p) ++k;
  while (k > 0 && tile_origin(k, n, L, t) > p) --k;
  k1 = k;
  while (k > 0 && tile_origin(k - 1, n, L, t) + t > p) --k;
  k0 = k;
}

// rho(d) = min(1, (d + 1) / (v + 1)), d = distance of p to the nearest edge of tile k that is not on the image border
ODB_DEVINL float tile_ramp(int p, int k, int n, int o, int t, int v) {
  int d = 0x7fffffff;
  if (k > 0) d = p - o;
  if (k < n - 1) d = min(d, o + t - 1 - p);
  return d >= v ? 1.0f : __fdiv_rn((float)(d + 1), (float)(v + 1));
}

// out[b][c][y][x] = sum_i w_i (s_i d_i + t_i) / sum_i w_i over the covering tiles in row-major order, fp32;
// w_i = rho_y * rho_x; without scale_shift s = 1, t = 0.  grid (ceil(W / 256), H, B)
__global__ void __launch_bounds__(256) tile_blend_kernel(const float* __restrict__ pred,
                                                         const double* __restrict__ scale_shift, int C, int H, int W,
                                                         int th, int tw, int v, int ny, int nx, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= W) return;
  const int T = ny * nx;
  int ky0, ky1, kx0, kx1;
  tile_cover(y, H, th, ny, ky0, ky1);
  tile_cover(x, W, tw, nx, kx0, kx1);
  for (int c = 0; c < C; ++c) {
    float acc = 0.0f, wsum = 0.0f;
    for (int ty = ky0; ty <= ky1; ++ty) {
      const int oy = tile_origin(ty, ny, H, th);
      const float wy = tile_ramp(y, ty, ny, oy, th, v);
      for (int tx = kx0; tx <= kx1; ++tx) {
        const int ox = tile_origin(tx, nx, W, tw);
        const float wt = __fmul_rn(wy, tile_ramp(x, tx, nx, ox, tw, v));
        const int i = ty * nx + tx;
        const float d = pred[((((long long)b * T + i) * C + c) * th + (y - oy)) * tw + (x - ox)];
        float val = d;
        if (scale_shift != nullptr) {
          const double* st = scale_shift + ((long long)b * T + i) * 2;
          val = __fmaf_rn((float)st[0], d, (float)st[1]);
        }
        acc = __fmaf_rn(wt, val, acc);
        wsum = __fadd_rn(wsum, wt);
      }
    }
    out[(((long long)b * C + c) * H + y) * W + x] = __fdiv_rn(acc, wsum);
  }
}

// Anchored alignment (TiledPredictor(anchor=...)): g, a whole-image prediction resampled to the image's size, replaces
// the ridge.  tile_align_solve_kernel with anchor moments (its nullable `anchor`, [b][T][5]) minimises
//   E(s,t) = sum_pairs sum_overlap (s_i a + t_i - s_j b - t_j)^2
//            + lambda Nbar sum_i (1/n_i) sum_tile (s_i a + t_i - g)^2 + kappa lambda Nbar sum_i ((s_i - 1)^2 + t_i^2).
// tile_anchor_moments_kernel, one CTA per (tile, image): moments[b][i] = (n, Sa, Saa, Sg, Sag) over the tile's pixels
// inside the image, a the tile's prediction, g the anchor [b][H][W].  In the solve, each tile's anchor term adds
// mu_i = lambda Nbar / n_i times its moments to the tile's diagonal 2 x 2 block and right-hand side only, so the band,
// the workspace and the tile cap are those of the ridge solve.  oracle/tiled_anchor_oracle.py restates it in float64.
__global__ void __launch_bounds__(256) tile_anchor_moments_kernel(const float* __restrict__ pred,
                                                                  const float* __restrict__ anchor, int H, int W,
                                                                  int th, int tw, int ny, int nx,
                                                                  double* __restrict__ moments) {
  const int i = blockIdx.x, b = blockIdx.y;
  const int T = ny * nx;
  const int oy = tile_origin(i / nx, ny, H, th), ox = tile_origin(i % nx, nx, W, tw);
  const int rh = min(th, H), rw = min(tw, W);
  const float* A = pred + ((long long)b * T + i) * th * tw;
  const float* G = anchor + ((long long)b * H + oy) * W + ox;
  const double s = rect_moments(A, tw, G, W, rh, rw);          // thread q: (Sa, Sg, Saa, Sgg, Sag)[q]
  double* m = moments + ((long long)b * T + i) * 5;
  const int q = threadIdx.x;
  if (q < 5 && q != 3) m[q == 0 ? 1 : q == 1 ? 3 : q] = s;
  if (q == 0) m[0] = (double)(rh * rw);
}

static bool tile_geometry_ok(int32_t b, int32_t h, int32_t w, int32_t th, int32_t tw, int32_t overlap) {
  if (!planes_ok(b, h, w) || th < 32 || tw < 32 || th % 32 || tw % 32 || overlap < 0 || 2 * overlap >= min(th, tw))
    return false;
  return (long long)tile_count(h, th, overlap) * tile_count(w, tw, overlap) <= ODB_TILE_MAX_TILES;
}

static size_t solve_smem_bytes(int ny, int nx) {
  const size_t n = 2 * (size_t)ny * nx;
  return (n + n * band_width(ny, nx)) * sizeof(double);
}

}  // namespace odb

using namespace odb;

extern "C" int odb_tile_gather(const float* image, int32_t b, int32_t h, int32_t w, int32_t tile_h, int32_t tile_w,
                               int32_t overlap, float* tiles, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!image || !tiles || !tile_geometry_ok(b, h, w, tile_h, tile_w, overlap) || !aligned(tiles, 16))
    return fail(ODB_ERR_INVALID, "tile_gather: bad argument");
  const int ny = tile_count(h, tile_h, overlap), nx = tile_count(w, tile_w, overlap);
  const dim3 grid((tile_h * (tile_w / 4) + 255) / 256, 3 * ny * nx, b);
  tile_gather_kernel<<<grid, 256, 0, stream>>>(image, h, w, tile_h, tile_w, ny, nx, reinterpret_cast<float4*>(tiles));
  count_launch();
  return check_launch("tile_gather");
}

extern "C" int odb_tile_overlap_moments(const float* pred, int32_t b, int32_t h, int32_t w, int32_t tile_h,
                                        int32_t tile_w, int32_t overlap, double* moments, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!pred || !moments || !tile_geometry_ok(b, h, w, tile_h, tile_w, overlap))
    return fail(ODB_ERR_INVALID, "tile_overlap_moments: bad argument");
  const int ny = tile_count(h, tile_h, overlap), nx = tile_count(w, tile_w, overlap);
  const int pairs = ny * (nx - 1) + (ny - 1) * nx;
  if (pairs == 0) return ODB_OK;                      // a single tile: nothing to compare
  tile_moments_kernel<<<dim3(pairs, b), 256, 0, stream>>>(pred, h, w, tile_h, tile_w, ny, nx, moments);
  count_launch();
  return check_launch("tile_overlap_moments");
}

extern "C" int64_t odb_tile_align_workspace_bytes(int32_t b, int32_t tiles_y, int32_t tiles_x) {
  if (b < 1 || tiles_y < 1 || tiles_x < 1 || (long long)tiles_y * tiles_x > ODB_TILE_MAX_TILES) return -1;
  if (solve_smem_bytes(tiles_y, tiles_x) <= kSolveSmemMax) return 0;
  return (int64_t)b * 2 * tiles_y * tiles_x * band_width(tiles_y, tiles_x) * (int64_t)sizeof(double);
}

extern "C" int odb_tile_anchor_moments(const float* pred, const float* anchor, int32_t b, int32_t h, int32_t w,
                                       int32_t tile_h, int32_t tile_w, int32_t overlap, double* moments,
                                       void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!pred || !anchor || !moments || !tile_geometry_ok(b, h, w, tile_h, tile_w, overlap))
    return fail(ODB_ERR_INVALID, "tile_anchor_moments: bad argument");
  const int ny = tile_count(h, tile_h, overlap), nx = tile_count(w, tile_w, overlap);
  tile_anchor_moments_kernel<<<dim3(ny * nx, b), 256, 0, stream>>>(pred, anchor, h, w, tile_h, tile_w, ny, nx,
                                                                   moments);
  count_launch();
  return check_launch("tile_anchor_moments");
}

static int align_solve(const char* name, const char* bad_argument, const double* moments, const double* anchor,
                       int32_t b, int32_t tiles_y, int32_t tiles_x, void* workspace, double* scale_shift,
                       cudaStream_t stream) {
  const int64_t ws = odb_tile_align_workspace_bytes(b, tiles_y, tiles_x);
  const bool single = tiles_y == 1 && tiles_x == 1;
  if (ws < 0 || !scale_shift || (!moments && !single) || (ws > 0 && !workspace) || b > 65535)
    return fail(ODB_ERR_INVALID, bad_argument);
  const bool in_smem = ws == 0;
  const size_t n = 2 * (size_t)tiles_y * tiles_x;
  const size_t smem = in_smem ? solve_smem_bytes(tiles_y, tiles_x) : n * sizeof(double);
  static bool configured[kMaxDevices] = {};
  const int dev = current_device();
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(tile_align_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)kSolveSmemMax);
    if (e != cudaSuccess) return fail_cuda(e, "tile_align_solve: cudaFuncSetAttribute");
    configured[dev] = true;
  }
  tile_align_solve_kernel<<<b, kSolveThreads, smem, stream>>>(moments, anchor, tiles_y, tiles_x, in_smem ? 1 : 0,
                                                              static_cast<double*>(workspace), scale_shift);
  count_launch();
  return check_launch(name);
}

extern "C" int odb_tile_align_solve(const double* moments, int32_t b, int32_t tiles_y, int32_t tiles_x,
                                    void* workspace, double* scale_shift, void* stream_) {
  return align_solve("tile_align_solve", "tile_align_solve: bad argument", moments, nullptr, b, tiles_y, tiles_x,
                     workspace, scale_shift, static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_tile_align_solve_anchored(const double* moments, const double* anchor_moments, int32_t b,
                                             int32_t tiles_y, int32_t tiles_x, void* workspace, double* scale_shift,
                                             void* stream_) {
  if (!anchor_moments) return fail(ODB_ERR_INVALID, "tile_align_solve_anchored: anchor_moments is required");
  return align_solve("tile_align_solve_anchored", "tile_align_solve_anchored: bad argument", moments, anchor_moments,
                     b, tiles_y, tiles_x, workspace, scale_shift, static_cast<cudaStream_t>(stream_));
}

extern "C" int odb_tile_blend(const float* pred, const double* scale_shift, int32_t b, int32_t c, int32_t h, int32_t w,
                              int32_t tile_h, int32_t tile_w, int32_t overlap, float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!pred || !out || c < 1 || !tile_geometry_ok(b, h, w, tile_h, tile_w, overlap))
    return fail(ODB_ERR_INVALID, "tile_blend: bad argument");
  const int ny = tile_count(h, tile_h, overlap), nx = tile_count(w, tile_w, overlap);
  tile_blend_kernel<<<dim3((w + 255) / 256, h, b), 256, 0, stream>>>(pred, scale_shift, c, h, w, tile_h, tile_w,
                                                                     overlap, ny, nx, out);
  count_launch();
  return check_launch("tile_blend");
}
