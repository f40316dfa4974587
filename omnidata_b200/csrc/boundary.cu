// Depth-boundary errors of a depth prediction against ground truth (omnidata_b200/metrics.py BoundaryMetrics;
// definitions in DESIGN.md §3 "Depth-boundary metrics" and include/omnidata_b200.h, restated in float64 by
// oracle/boundary_oracle.py).
//
// Edge detector E(f, V), per map (ground truth, then prediction), all in fp64 with explicit round-to-nearest operations:
//   edge_stats_kernel (slabs) -> launch_slab_reduce (n, non-finite, min, max over V)
//   -> smooth_h_kernel (masked Gaussian along rows: numerator and denominator)
//   -> smooth_v_kernel (along columns, s = num / den)
//   -> sobel_nms_kernel (shared-memory tile with a two-pixel halo: Sobel, magnitude, non-maximum suppression, weak /
//      strong bytes, union-find labels; the magnitude never leaves shared memory)
//   -> ccl_merge_kernel -> ccl_resolve_kernel -> edge_select_kernel (hysteresis as 8-connected labelling: union-find
//      with integer atomicMin, so every component's root is its least linear index; integer atomicOr marks the roots
//      of components with a strong pixel)
// Distances and errors, both maps in each launch:
//   edt_col_kernel (one thread per column, two integer sweeps) -> edt_row_kernel (one thread per row, lower envelope
//   of parabolas in integers) -> chamfer_kernel (slabs) -> launch_slab_reduce -> boundary_fold_kernel (one thread,
//   image order).
// No floating-point atomics, no fast-math: results are bit-reproducible and independent of the batch.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "host_util.h"
#include "select.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kBThreads = 256;
constexpr int kBSlabIters = kSlab / kBThreads;
constexpr int kMaxRadius = 16;                          // R = floor(4 sigma + 0.5) for sigma <= 4
constexpr uint32_t kNoLabel = 0xFFFFFFFFu;              // > every linear index (h w <= 65535^2 < 2^32 - 1)
constexpr int kNoSite = -1;                             // column pass: no edge in the column
constexpr unsigned long long kNoEdge = ~0ull;           // squared distance in a map without edges
constexpr uint8_t kWeak = 1, kStrong = 2, kRootStrong = 4;
constexpr int kTileW = 32, kTileH = 8;                  // sobel_nms_kernel outputs per CTA
constexpr int kRowThreads = 64;                         // edt_row_kernel rows per CTA

struct EdgeParams {
  double taps[2 * kMaxRadius + 1];                      // normalised Gaussian, k = -R .. R
  int radius;
  double low, high, min_depth, max_depth;
};

ODB_DEVINL bool mask_on(const void* mask, int kind, long long i) {
  if (kind == ODB_MASK_U8) return static_cast<const uint8_t*>(mask)[i] != 0;
  if (kind == ODB_MASK_F32) return static_cast<const float*>(mask)[i] != 0.0f;
  return true;
}

// V: mask != 0, g finite, min_depth < g <= max_depth
ODB_DEVINL bool in_v(const float* g, const void* mask, int kind, long long i, const EdgeParams& p) {
  if (!mask_on(mask, kind, i)) return false;
  const double v = g[i];
  return isfinite(v) && v > p.min_depth && v <= p.max_depth;
}

// per-image statistics st[8] = (|V|, #non-finite f on V, min, max of the finite f on V)
ODB_DEVINL bool usable(const double* st) { return st[0] > 0.0 && st[1] == 0.0 && st[3] > st[2]; }

// Slab partials [b][slab][8] = (|V|, #non-finite f on V, min f, max f).  grid (slabs, b)
__global__ void __launch_bounds__(kBThreads) edge_stats_kernel(const float* __restrict__ f, const float* __restrict__ g,
                                                               const void* mask, int kind, long long hw, EdgeParams p,
                                                               double* __restrict__ part) {
  __shared__ double scratch[32];
  const long long base = (long long)blockIdx.y * hw;
  double n = 0.0, bad = 0.0, lo = INFINITY, hi = -INFINITY;
  for (int k = 0; k < kBSlabIters; ++k) {
    const long long i = blockIdx.x * kSlab + k * kBThreads + threadIdx.x;
    if (i >= hw || !in_v(g, mask, kind, base + i, p)) continue;
    const double v = f[base + i];
    n += 1.0;
    if (isfinite(v)) {
      lo = fmin(lo, v);
      hi = fmax(hi, v);
    } else {
      bad += 1.0;
    }
  }
  double* out = part + ((long long)blockIdx.y * gridDim.x + blockIdx.x) * kPartStride;
  const double r0 = block_sum_d(n, scratch);
  const double r1 = block_sum_d(bad, scratch);
  const double r2 = block_min_d(lo, scratch);
  const double r3 = block_max_d(hi, scratch);
  if (threadIdx.x == 0) {
    out[0] = r0;
    out[1] = r1;
    out[2] = r2;
    out[3] = r3;
  }
}

// Horizontal pass: num[i] = S_k w_k fhat(x + k) 1_V(x + k), den[i] = S_k w_k 1_V(x + k), k = -R .. R in order, zeros
// outside the image; fhat = (f - lo) / (hi - lo).  grid (ceil(w / 256), h, b)
__global__ void __launch_bounds__(kBThreads) smooth_h_kernel(const float* __restrict__ f, const float* __restrict__ g,
                                                             const void* mask, int kind, int h, int w, EdgeParams p,
                                                             const double* __restrict__ st, double* __restrict__ num,
                                                             double* __restrict__ den) {
  __shared__ double sf[kBThreads + 2 * kMaxRadius], sv[kBThreads + 2 * kMaxRadius];
  const int R = p.radius;
  const double* s = st + (long long)blockIdx.z * kPartStride;
  const double lo = s[2], range = __dsub_rn(s[3], s[2]);
  const long long row = ((long long)blockIdx.z * h + blockIdx.y) * w;
  const int x0 = blockIdx.x * kBThreads;
  for (int j = threadIdx.x; j < kBThreads + 2 * R; j += kBThreads) {
    const int x = x0 - R + j;
    double fv = 0.0, vv = 0.0;
    if (x >= 0 && x < w && in_v(g, mask, kind, row + x, p)) {
      fv = __ddiv_rn(__dsub_rn((double)f[row + x], lo), range);
      vv = 1.0;
    }
    sf[j] = fv;
    sv[j] = vv;
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= w) return;
  double a = 0.0, d = 0.0;
  for (int k = 0; k <= 2 * R; ++k) {
    a = __dadd_rn(a, __dmul_rn(p.taps[k], sf[threadIdx.x + k]));
    d = __dadd_rn(d, __dmul_rn(p.taps[k], sv[threadIdx.x + k]));
  }
  num[row + x] = a;
  den[row + x] = d;
}

// Vertical pass of both sums (rows outside the image add nothing: every sum is >= +0, so a zero term changes no bit),
// s = num / den where den > 0, else 0.  grid (ceil(w / 256), h, b)
__global__ void __launch_bounds__(kBThreads) smooth_v_kernel(const double* __restrict__ num,
                                                             const double* __restrict__ den, int h, int w,
                                                             EdgeParams p, double* __restrict__ s) {
  const int x = blockIdx.x * kBThreads + threadIdx.x;
  if (x >= w) return;
  const int y = blockIdx.y, R = p.radius;
  const long long img = (long long)blockIdx.z * h * w;
  double a = 0.0, d = 0.0;
  for (int k = -R; k <= R; ++k) {
    const int yy = y + k;
    if (yy < 0 || yy >= h) continue;
    const long long i = img + (long long)yy * w + x;
    a = __dadd_rn(a, __dmul_rn(p.taps[k + R], num[i]));
    d = __dadd_rn(d, __dmul_rn(p.taps[k + R], den[i]));
  }
  s[img + (long long)y * w + x] = d > 0.0 ? __ddiv_rn(a, d) : 0.0;
}

// Sobel at tile position (r, c) of the s tile: gx = (dx(-1) + 2 dx(0)) + dx(1), dx(j) = s[y+j][x+1] - s[y+j][x-1];
// gy = (dy(-1) + 2 dy(0)) + dy(1), dy(j) = s[y+1][x+j] - s[y-1][x+j]
ODB_DEVINL void sobel(const double (*t)[kTileW + 4], int r, int c, double& gx, double& gy) {
  const double d0 = __dsub_rn(t[r - 1][c + 1], t[r - 1][c - 1]);
  const double d1 = __dsub_rn(t[r][c + 1], t[r][c - 1]);
  const double d2 = __dsub_rn(t[r + 1][c + 1], t[r + 1][c - 1]);
  gx = __dadd_rn(__dadd_rn(d0, __dmul_rn(2.0, d1)), d2);
  const double e0 = __dsub_rn(t[r + 1][c - 1], t[r - 1][c - 1]);
  const double e1 = __dsub_rn(t[r + 1][c], t[r - 1][c]);
  const double e2 = __dsub_rn(t[r + 1][c + 1], t[r - 1][c + 1]);
  gy = __dadd_rn(__dadd_rn(e0, __dmul_rn(2.0, e1)), e2);
}

// m1 (1 - w) + m2 w
ODB_DEVINL double lerp_rn(double m1, double m2, double w) {
  return __dadd_rn(__dmul_rn(m1, __dsub_rn(1.0, w)), __dmul_rn(m2, w));
}

// Sobel, magnitude, non-maximum suppression and thresholds of one kTileH x kTileW tile: flags = weak | strong << 1,
// label = the pixel's linear index where weak, kNoLabel elsewhere.  Nothing is weak in an image whose statistics are
// not usable (no valid pixel, a non-finite f on V, or a flat f).  grid (ceil(w / 32), ceil(h / 8), b), block (32, 8)
__global__ void __launch_bounds__(kTileW * kTileH, 1) sobel_nms_kernel(const double* __restrict__ s,
                                                                    const float* __restrict__ g, const void* mask,
                                                                    int kind, int h, int w, EdgeParams p,
                                                                    const double* __restrict__ st,
                                                                    uint8_t* __restrict__ flags,
                                                                    uint32_t* __restrict__ labels) {
  __shared__ double ts[kTileH + 4][kTileW + 4];
  __shared__ double tm[kTileH + 2][kTileW + 2];
  __shared__ uint8_t tv[kTileH + 2][kTileW + 2];
  const int tid = threadIdx.y * kTileW + threadIdx.x;
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  const long long img = (long long)blockIdx.z * h * w;
  for (int j = tid; j < (kTileH + 4) * (kTileW + 4); j += kTileW * kTileH) {
    const int r = j / (kTileW + 4), c = j % (kTileW + 4);
    const int y = y0 - 2 + r, x = x0 - 2 + c;
    ts[r][c] = (y >= 0 && y < h && x >= 0 && x < w) ? s[img + (long long)y * w + x] : 0.0;
  }
  for (int j = tid; j < (kTileH + 2) * (kTileW + 2); j += kTileW * kTileH) {
    const int r = j / (kTileW + 2), c = j % (kTileW + 2);
    const int y = y0 - 1 + r, x = x0 - 1 + c;
    tv[r][c] = (y >= 0 && y < h && x >= 0 && x < w && in_v(g, mask, kind, img + (long long)y * w + x, p)) ? 1 : 0;
  }
  __syncthreads();
  for (int j = tid; j < (kTileH + 2) * (kTileW + 2); j += kTileW * kTileH) {
    const int r = j / (kTileW + 2), c = j % (kTileW + 2);
    const int y = y0 - 1 + r, x = x0 - 1 + c;
    double m = 0.0;                                                 // 0 on the image's border and outside it
    if (y >= 1 && y < h - 1 && x >= 1 && x < w - 1) {
      double gx, gy;
      sobel(ts, r + 1, c + 1, gx, gy);
      m = __dsqrt_rn(__dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy)));
    }
    tm[r][c] = m;
  }
  __syncthreads();
  const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  if (x >= w || y >= h) return;
  const int r = threadIdx.y + 1, c = threadIdx.x + 1;
  const double m = tm[r][c];
  bool cand = usable(st + (long long)blockIdx.z * kPartStride) && x >= 1 && x < w - 1 && y >= 1 && y < h - 1 &&
              m > 0.0;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) cand = cand && tv[r + dy][c + dx];
  uint8_t fl = 0;
  if (cand) {
    double gx, gy;
    sobel(ts, r + 1, c + 1, gx, gy);
    const double ax = fabs(gx), ay = fabs(gy);
    const int sx = gx >= 0.0 ? 1 : -1, sy = gy >= 0.0 ? 1 : -1;
    double pa, pb;
    if (ax >= ay) {                                                 // the points lie on the columns x +- 1
      const double wt = __ddiv_rn(ay, ax);
      pa = lerp_rn(tm[r][c + sx], tm[r + sy][c + sx], wt);
      pb = lerp_rn(tm[r][c - sx], tm[r - sy][c - sx], wt);
    } else {                                                        // on the rows y +- 1
      const double wt = __ddiv_rn(ax, ay);
      pa = lerp_rn(tm[r + sy][c], tm[r + sy][c + sx], wt);
      pb = lerp_rn(tm[r - sy][c], tm[r - sy][c - sx], wt);
    }
    if (m >= pa && m >= pb && m >= p.low) fl = m >= p.high ? (kWeak | kStrong) : kWeak;
  }
  const long long i = img + (long long)y * w + x;
  flags[i] = fl;
  labels[i] = fl ? (uint32_t)((long long)y * w + x) : kNoLabel;
}

// flags[i] = the weak / strong bits of a given map (bit 0 weak, bit 1 strong; a strong pixel is weak), labels as
// sobel_nms_kernel writes them.  grid (ceil(w / 256), h, b)
__global__ void __launch_bounds__(kBThreads) hysteresis_init_kernel(const uint8_t* __restrict__ in, int h, int w,
                                                                    uint8_t* __restrict__ flags,
                                                                    uint32_t* __restrict__ labels) {
  const int x = blockIdx.x * kBThreads + threadIdx.x;
  if (x >= w) return;
  const long long j = (long long)blockIdx.y * w + x, i = (long long)blockIdx.z * h * w + j;
  const uint8_t v = in[i];
  const uint8_t fl = (v & kStrong) ? (kWeak | kStrong) : (v & kWeak);
  flags[i] = fl;
  labels[i] = fl ? (uint32_t)j : kNoLabel;
}

// Root of x, halving the path on the way (integer atomicMin: a label only ever decreases, to an ancestor).
ODB_DEVINL uint32_t uf_find(uint32_t* L, uint32_t x) {
  while (true) {
    const uint32_t p = *(volatile uint32_t*)(L + x);
    if (p == x) return x;
    const uint32_t gp = *(volatile uint32_t*)(L + p);
    if (gp != p) atomicMin(L + x, gp);
    x = gp;
  }
}

// Playne & Hawick (2018): links the larger root under the smaller one with atomicMin and retries from the value it
// found when another thread relinked that root first.
ODB_DEVINL void uf_union(uint32_t* L, uint32_t a, uint32_t b) {
  bool done = false;
  while (!done) {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a < b) {
      const uint32_t old = atomicMin(L + b, a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const uint32_t old = atomicMin(L + a, b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  }
}

// Every weak pixel joins its weak neighbours W, NW, N and NE (each 8-neighbour pair once).  grid (ceil(w / 256), h, b)
__global__ void __launch_bounds__(kBThreads) ccl_merge_kernel(const uint8_t* __restrict__ flags, int h, int w,
                                                              uint32_t* __restrict__ labels) {
  const int x = blockIdx.x * kBThreads + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const long long img = (long long)blockIdx.z * h * w;
  const uint8_t* F = flags + img;
  uint32_t* L = labels + img;
  const long long i = (long long)y * w + x;
  if (!(F[i] & kWeak)) return;
  if (x > 0 && (F[i - 1] & kWeak)) uf_union(L, (uint32_t)i, (uint32_t)(i - 1));
  if (y > 0) {
    const long long u = i - w;
    if (x > 0 && (F[u - 1] & kWeak)) uf_union(L, (uint32_t)i, (uint32_t)(u - 1));
    if (F[u] & kWeak) uf_union(L, (uint32_t)i, (uint32_t)u);
    if (x < w - 1 && (F[u + 1] & kWeak)) uf_union(L, (uint32_t)i, (uint32_t)(u + 1));
  }
}

// labels[i] = root of i (the least linear index of its component); a strong pixel sets kRootStrong in its root's
// flags byte (integer atomicOr on the aligned word holding it).  grid (ceil(w / 256), h, b)
__global__ void __launch_bounds__(kBThreads) ccl_resolve_kernel(uint8_t* __restrict__ flags, int h, int w,
                                                                uint32_t* __restrict__ labels) {
  const int x = blockIdx.x * kBThreads + threadIdx.x;
  if (x >= w) return;
  const long long img = (long long)blockIdx.z * h * w;
  const long long i = (long long)blockIdx.y * w + x;
  const uint8_t fl = flags[img + i];
  if (!(fl & kWeak)) return;
  const uint32_t r = uf_find(labels + img, (uint32_t)i);
  labels[img + i] = r;
  if (fl & kStrong) {
    const unsigned long long byte = (unsigned long long)(img + r);
    atomicOr(reinterpret_cast<unsigned int*>(flags) + (byte >> 2), (unsigned int)kRootStrong << (8 * (byte & 3)));
  }
}

// edges[i] = 1 where i is weak and its component holds a strong pixel, else 0.  grid (ceil(w / 256), h, b)
__global__ void __launch_bounds__(kBThreads) edge_select_kernel(const uint8_t* __restrict__ flags,
                                                                const uint32_t* __restrict__ labels, int h, int w,
                                                                uint8_t* __restrict__ edges) {
  const int x = blockIdx.x * kBThreads + threadIdx.x;
  if (x >= w) return;
  const long long img = (long long)blockIdx.z * h * w;
  const long long i = img + (long long)blockIdx.y * w + x;
  edges[i] = (flags[i] & kWeak) && (flags[img + labels[i]] & kRootStrong) ? 1 : 0;
}

// Column pass of the squared distance transform: col[y][x] = rows to the nearest edge pixel of column x (nonzero
// byte), kNoSite where the column has none.  One thread per column, a down and an up sweep.  Map z of the launch reads
// e0 (z = 0) or e1 and writes col + z b h w.  grid (ceil(w / 256), b, maps)
__global__ void __launch_bounds__(kBThreads) edt_col_kernel(const uint8_t* __restrict__ e0,
                                                            const uint8_t* __restrict__ e1, int b, int h, int w,
                                                            int* __restrict__ col) {
  const int x = blockIdx.x * kBThreads + threadIdx.x;
  if (x >= w) return;
  const long long img = (long long)blockIdx.y * h * w;
  const uint8_t* E = (blockIdx.z ? e1 : e0) + img + x;
  int* G = col + (long long)blockIdx.z * b * h * w + img + x;
  int d = kNoSite;
  for (int y = 0; y < h; ++y) {
    if (E[(long long)y * w]) d = 0;
    else if (d != kNoSite) ++d;
    G[(long long)y * w] = d;
  }
  int below = d;
  for (int y = h - 2; y >= 0; --y) {
    int cur = G[(long long)y * w];
    if (below != kNoSite && (cur == kNoSite || below + 1 < cur)) {
      cur = below + 1;
      G[(long long)y * w] = cur;
    }
    below = cur;
  }
}

ODB_DEVINL long long floor_div(long long n, long long d) { return n >= 0 ? n / d : -((-n + d - 1) / d); }

// Row pass: d2[y][x] = min over the columns q with an edge of (x - q)^2 + col[y][q]^2, exact in 64-bit integers;
// kNoEdge in every pixel of a map without edges (no column has a site).  The lower envelope of the parabolas is a
// stack of (site, first column it wins) packed in one 64-bit word per entry; it is kept in the output row itself
// (entry k <= the column being written, and the fill runs right to left with the live entry in registers), so it
// takes no shared memory or workspace at any width.  One thread per row.  grid (ceil(h / 64), b, maps)
__global__ void __launch_bounds__(kRowThreads) edt_row_kernel(const int* __restrict__ col, int b, int h, int w,
                                                              unsigned long long* __restrict__ d2) {
  const int y = blockIdx.x * kRowThreads + threadIdx.x;
  if (y >= h) return;
  const long long base = (((long long)blockIdx.z * b + blockIdx.y) * h + y) * w;
  const int* G = col + base;
  unsigned long long* out = d2 + base;
  int k = -1, tv = 0, tz = 0;                                       // top entry: site tv from column tz on
  long long tg = 0;                                                 // its col^2
  for (int q = 0; q < w; ++q) {
    const int gq = G[q];
    if (gq == kNoSite) continue;
    const long long Gq = (long long)gq * gq;
    long long s = 0;
    while (k >= 0) {                                                // q beats tv from column s on
      s = floor_div((long long)q * q - (long long)tv * tv + Gq - tg, 2ll * (q - tv)) + 1;
      if (s > tz) break;
      if (--k >= 0) {
        const unsigned long long e = out[k];
        tv = (int)(e & 0xffffffffu);
        tz = (int)(e >> 32);
        tg = (long long)G[tv] * G[tv];
      }
    }
    if (k < 0) {
      k = 0;
      tv = q;
      tz = 0;
      tg = Gq;
    } else if (s < w) {
      ++k;
      tv = q;
      tz = (int)s;
      tg = Gq;
    } else {
      continue;
    }
    out[k] = (unsigned long long)(uint32_t)tv | ((unsigned long long)(uint32_t)tz << 32);
  }
  if (k < 0) {
    for (int x = 0; x < w; ++x) out[x] = kNoEdge;
    return;
  }
  for (int x = w - 1; x >= 0; --x) {
    while (tz > x) {                                                // entry k - 1 lies in slot k - 1 <= x: not yet written
      const unsigned long long e = out[--k];
      tv = (int)(e & 0xffffffffu);
      tz = (int)(e >> 32);
      tg = (long long)G[tv] * G[tv];
    }
    const long long dx = x - tv;
    out[x] = (unsigned long long)(dx * dx + tg);
  }
}

ODB_DEVINL double dist(unsigned long long d2) { return d2 == kNoEdge ? INFINITY : __dsqrt_rn((double)d2); }

// Slab partials [b][slab][8] = (S_A D_g, |A|, S_{E_g} D_p, |E_p|, |E_g|), A = {p in E_p : D_g(p) < max_dist}.
// grid (slabs, b)
__global__ void __launch_bounds__(kBThreads) chamfer_kernel(const uint8_t* __restrict__ eg,
                                                            const uint8_t* __restrict__ ep,
                                                            const unsigned long long* __restrict__ dg2,
                                                            const unsigned long long* __restrict__ dp2, long long hw,
                                                            double max_dist, double* __restrict__ part) {
  __shared__ double scratch[32];
  const long long base = (long long)blockIdx.y * hw;
  double acc[5] = {0, 0, 0, 0, 0};
  for (int k = 0; k < kBSlabIters; ++k) {
    const long long i = blockIdx.x * kSlab + k * kBThreads + threadIdx.x;
    if (i >= hw) continue;
    if (ep[base + i]) {
      acc[3] += 1.0;
      const double d = dist(dg2[base + i]);
      if (d < max_dist) {
        acc[0] += d;
        acc[1] += 1.0;
      }
    }
    if (eg[base + i]) {
      acc[4] += 1.0;
      acc[2] += dist(dp2[base + i]);
    }
  }
  double* out = part + ((long long)blockIdx.y * gridDim.x + blockIdx.x) * kPartStride;
  for (int q = 0; q < 5; ++q) {
    const double r = block_sum_d(acc[q], scratch);
    if (threadIdx.x == 0) out[q] = r;
  }
}

// One thread, images in order: records[b][ODB_BOUNDARY_RECORD] = (accuracy, completeness, |E_p|, |E_g|, |A|,
// non-finite predictions on V, |E_g| = 0, A empty); sums[2] += (accuracy, completeness) and counts[5] += (1, |E_g| = 0,
// A empty, |E_p|, |E_g|).  A non-finite prediction on V makes the image's errors NaN.
__global__ void boundary_fold_kernel(const double* __restrict__ cham, const double* __restrict__ pst, int b_n,
                                     double max_dist, double* __restrict__ records, double* __restrict__ sums,
                                     long long* __restrict__ counts) {
  if (threadIdx.x != 0) return;
  for (int b = 0; b < b_n; ++b) {
    const double* c = cham + (long long)b * kPartStride;
    const double bad = pst[(long long)b * kPartStride + 1] > 0.0 ? NAN : 0.0;
    double* r = records + (long long)b * ODB_BOUNDARY_RECORD;
    const bool no_gt = c[4] == 0.0, no_pred = !no_gt && c[1] == 0.0;
    double acc = NAN, comp = NAN;
    if (!no_gt) {
      acc = (no_pred ? max_dist : c[0] / c[1]) + bad;
      comp = (no_pred ? max_dist : c[2] / c[4]) + bad;
      sums[0] += acc;
      sums[1] += comp;
    }
    r[0] = acc;
    r[1] = comp;
    r[2] = c[3];
    r[3] = c[4];
    r[4] = c[1];
    r[5] = pst[(long long)b * kPartStride + 1];
    r[6] = no_gt ? 1.0 : 0.0;
    r[7] = no_pred ? 1.0 : 0.0;
    counts[0] += 1;
    counts[1] += no_gt ? 1 : 0;
    counts[2] += no_pred ? 1 : 0;
    counts[3] += (long long)c[3];
    counts[4] += (long long)c[4];
  }
}

// ---------------------------------------------------------------------------------------------------- host side
// Workspace (8-byte aligned), for b images of hw pixels:
//   dg2, dp2   uint64 [b][hw] each    squared distances (during detection: the row-pass numerator / denominator)
//   sm         fp64 [b][hw]           smoothed map (during the distance transform: int32 [2][b][hw] column pass)
//   part       fp64 [b][slabs][8]     slab partials;  st fp64 [2][b][8] map statistics;  cham fp64 [b][8]
//   labels     uint32 [b][hw]
//   flags      uint8 [b][hw], padded to a multiple of 4 bytes (word atomics)
//   eg, ep     uint8 [b][hw] each     detected edge maps
struct Layout {
  unsigned long long *dg2, *dp2;
  double *sm, *part, *st, *cham;
  uint32_t* labels;
  uint8_t *flags, *eg, *ep;
};

static long long pad4(long long n) { return (n + 3) & ~3ll; }

static int64_t workspace_bytes(int32_t b, int32_t h, int32_t w) {
  const long long n = (long long)b * h * w;
  return 3 * 8 * n + 8ll * kPartStride * ((long long)b * slab_count(h, w) + 3ll * b) + 4 * n + pad4(n) + 2 * n;
}

static Layout layout(void* ws, int32_t b, int32_t h, int32_t w) {
  const long long n = (long long)b * h * w;
  Layout L;
  char* p = static_cast<char*>(ws);
  L.dg2 = reinterpret_cast<unsigned long long*>(p);
  L.dp2 = L.dg2 + n;
  L.sm = reinterpret_cast<double*>(L.dp2 + n);
  L.part = L.sm + n;
  L.st = L.part + (long long)b * slab_count(h, w) * kPartStride;
  L.cham = L.st + 2ll * b * kPartStride;
  L.labels = reinterpret_cast<uint32_t*>(L.cham + (long long)b * kPartStride);
  L.flags = reinterpret_cast<uint8_t*>(L.labels + n);
  L.eg = L.flags + pad4(n);
  L.ep = L.eg + n;
  return L;
}

static bool mask_arg_ok(const void* mask, int32_t kind) {
  if (kind == ODB_MASK_NONE) return mask == nullptr;
  if (kind == ODB_MASK_U8) return mask != nullptr;
  return kind == ODB_MASK_F32 && mask != nullptr && aligned(mask, 4);
}

// sigma in (0, 4], low / high finite with 0 <= low <= high, 0 <= min_depth < max_depth (max_depth = +inf: none)
static bool edge_params(double sigma, double low, double high, double min_depth, double max_depth, EdgeParams& p) {
  if (!(sigma > 0.0 && sigma <= 4.0) || !std::isfinite(low) || !std::isfinite(high) || !(low >= 0.0) ||
      !(low <= high) || !std::isfinite(min_depth) || !(min_depth >= 0.0) || std::isnan(max_depth) ||
      !(max_depth > min_depth))
    return false;
  const int R = (int)std::floor(4.0 * sigma + 0.5);
  double sum = 0.0;
  for (int k = -R; k <= R; ++k) {
    p.taps[k + R] = std::exp(-(double)(k * k) / (2.0 * sigma * sigma));
    sum += p.taps[k + R];
  }
  for (int k = 0; k <= 2 * R; ++k) p.taps[k] /= sum;
  for (int k = 2 * R + 1; k <= 2 * kMaxRadius; ++k) p.taps[k] = 0.0;
  p.radius = R;
  p.low = low;
  p.high = high;
  p.min_depth = min_depth;
  p.max_depth = max_depth;
  return true;
}

static dim3 row_grid(int32_t b, int32_t h, int32_t w) { return dim3((w + kBThreads - 1) / kBThreads, h, b); }

// ccl_merge -> ccl_resolve -> edge_select on flags / labels already initialised
static void hysteresis(const Layout& L, int32_t b, int32_t h, int32_t w, uint8_t* edges, cudaStream_t stream) {
  ccl_merge_kernel<<<row_grid(b, h, w), kBThreads, 0, stream>>>(L.flags, h, w, L.labels);
  count_launch();
  ccl_resolve_kernel<<<row_grid(b, h, w), kBThreads, 0, stream>>>(L.flags, h, w, L.labels);
  count_launch();
  edge_select_kernel<<<row_grid(b, h, w), kBThreads, 0, stream>>>(L.flags, L.labels, h, w, edges);
  count_launch();
}

// E(f, V) into edges; st: the map's statistics [b][8].  Eight launches.
static void detect(const float* f, const float* g, const void* mask, int32_t kind, int32_t b, int32_t h, int32_t w,
                   const EdgeParams& p, const Layout& L, double* st, uint8_t* edges, cudaStream_t stream) {
  const int slabs = slab_count(h, w);
  const long long hw = (long long)h * w;
  edge_stats_kernel<<<dim3(slabs, b), kBThreads, 0, stream>>>(f, g, mask, kind, hw, p, L.part);
  count_launch();
  launch_slab_reduce(L.part, b, slabs, 4, 1u << 2, 1u << 3, st, stream);
  double* num = reinterpret_cast<double*>(L.dg2);
  double* den = reinterpret_cast<double*>(L.dp2);
  smooth_h_kernel<<<row_grid(b, h, w), kBThreads, 0, stream>>>(f, g, mask, kind, h, w, p, st, num, den);
  count_launch();
  smooth_v_kernel<<<row_grid(b, h, w), kBThreads, 0, stream>>>(num, den, h, w, p, L.sm);
  count_launch();
  sobel_nms_kernel<<<dim3((w + kTileW - 1) / kTileW, (h + kTileH - 1) / kTileH, b), dim3(kTileW, kTileH), 0,
                     stream>>>(L.sm, g, mask, kind, h, w, p, st, L.flags, L.labels);
  count_launch();
  hysteresis(L, b, h, w, edges, stream);
}

// squared distance transforms of maps e0 -> d0 and (maps = 2) e1 -> d1 = d0 + b h w.  Two launches.
static void distance2(const uint8_t* e0, const uint8_t* e1, int maps, int32_t b, int32_t h, int32_t w,
                      const Layout& L, unsigned long long* d0, cudaStream_t stream) {
  int* col = reinterpret_cast<int*>(L.sm);
  edt_col_kernel<<<dim3((w + kBThreads - 1) / kBThreads, b, maps), kBThreads, 0, stream>>>(e0, e1, b, h, w, col);
  count_launch();
  edt_row_kernel<<<dim3((h + kRowThreads - 1) / kRowThreads, b, maps), kRowThreads, 0, stream>>>(col, b, h, w, d0);
  count_launch();
}

}  // namespace odb

using namespace odb;

extern "C" int64_t odb_boundary_workspace_bytes(int32_t b, int32_t h, int32_t w) {
  if (!planes_ok(b, h, w)) return -1;
  return workspace_bytes(b, h, w);
}

extern "C" int odb_depth_edges(const float* depth, const void* mask, int32_t mask_dtype, int32_t b, int32_t h,
                               int32_t w, double sigma, double low, double high, double min_depth, double max_depth,
                               void* workspace, uint8_t* edges, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  EdgeParams p;
  if (!depth || !workspace || !edges || !planes_ok(b, h, w) || !mask_arg_ok(mask, mask_dtype) || !aligned(depth, 4) ||
      !aligned(workspace, 8) || !edge_params(sigma, low, high, min_depth, max_depth, p))
    return fail(ODB_ERR_INVALID, "depth_edges: bad argument");
  const Layout L = layout(workspace, b, h, w);
  detect(depth, depth, mask, mask_dtype, b, h, w, p, L, L.st, edges, stream);
  return check_launch("depth_edges");
}

extern "C" int odb_edge_hysteresis(const uint8_t* weak_strong, int32_t b, int32_t h, int32_t w, void* workspace,
                                   uint8_t* edges, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!weak_strong || !workspace || !edges || !planes_ok(b, h, w) || !aligned(workspace, 8))
    return fail(ODB_ERR_INVALID, "edge_hysteresis: bad argument");
  const Layout L = layout(workspace, b, h, w);
  hysteresis_init_kernel<<<row_grid(b, h, w), kBThreads, 0, stream>>>(weak_strong, h, w, L.flags, L.labels);
  count_launch();
  hysteresis(L, b, h, w, edges, stream);
  return check_launch("edge_hysteresis");
}

extern "C" int odb_edge_distance2(const uint8_t* edges, int32_t b, int32_t h, int32_t w, void* workspace,
                                  uint64_t* dist2, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!edges || !workspace || !dist2 || !planes_ok(b, h, w) || !aligned(workspace, 8) || !aligned(dist2, 8))
    return fail(ODB_ERR_INVALID, "edge_distance2: bad argument");
  const Layout L = layout(workspace, b, h, w);
  distance2(edges, edges, 1, b, h, w, L, reinterpret_cast<unsigned long long*>(dist2), stream);
  return check_launch("edge_distance2");
}

extern "C" int odb_boundary_metrics_update(const float* pred, const float* gt, const void* mask, int32_t mask_dtype,
                                           const uint8_t* gt_edges, int32_t b, int32_t h, int32_t w, double sigma,
                                           double low, double high, double max_dist, double min_depth,
                                           double max_depth, void* workspace, double* records, double* state_sums,
                                           int64_t* state_counts, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  EdgeParams p;
  if (!pred || !gt || !workspace || !records || !state_sums || !state_counts || !planes_ok(b, h, w) ||
      !mask_arg_ok(mask, mask_dtype) || !aligned(pred, 4) || !aligned(gt, 4) || !aligned(workspace, 8) ||
      !aligned(records, 8) || !aligned(state_sums, 8) || !aligned(state_counts, 8) || !std::isfinite(max_dist) ||
      !(max_dist > 0.0) || !edge_params(sigma, low, high, min_depth, max_depth, p))
    return fail(ODB_ERR_INVALID, "boundary_metrics_update: bad argument");
  const Layout L = layout(workspace, b, h, w);
  double* st_g = L.st;
  double* st_p = L.st + (long long)b * kPartStride;
  const uint8_t* eg = gt_edges;
  if (!eg) {
    detect(gt, gt, mask, mask_dtype, b, h, w, p, L, st_g, L.eg, stream);
    eg = L.eg;
  }
  detect(pred, gt, mask, mask_dtype, b, h, w, p, L, st_p, L.ep, stream);
  distance2(eg, L.ep, 2, b, h, w, L, L.dg2, stream);
  const int slabs = slab_count(h, w);
  chamfer_kernel<<<dim3(slabs, b), kBThreads, 0, stream>>>(eg, L.ep, L.dg2, L.dp2, (long long)h * w, max_dist, L.part);
  count_launch();
  launch_slab_reduce(L.part, b, slabs, 5, 0u, 0u, L.cham, stream);
  boundary_fold_kernel<<<1, 32, 0, stream>>>(L.cham, st_p, b, max_dist, records, state_sums,
                                             reinterpret_cast<long long*>(state_counts));
  count_launch();
  return check_launch("boundary_metrics_update");
}
