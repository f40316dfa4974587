// Sparse TSDF volumes (omnidata_b200/volume.py SparseTSDFVolume): the dense volume's points X(p) = origin + voxel p,
// p in Z^3, stored only in allocated blocks of 8^3 points, found through a hash table of block coordinates.
// Definitions in DESIGN.md §3 "Sparse TSDF volumes" and include/omnidata_b200.h; oracle/sparse_volume_oracle.py
// restates them in float64.
//
//   spv_clear_kernel / spv_insert_kernel   rebuild the hash table from the allocated blocks (ids kept)
//   spv_mark_kernel       one thread per pixel and frame: inserts the blocks of the pixel's truncation segment, the
//                         earliest frame by integer atomicMin; a new slot is appended to a list
//   spv_sort_*_kernel     bitonic sort of the new slots by (birth frame, block key), so ids never depend on scheduling
//   spv_assign_kernel     ids in sorted order, block keys, birth stamps, the bounding box (integer atomics)
//   spv_zero_kernel       zeroes the new blocks' data
//   spv_nbr_kernel        per block, the ids of the 7 blocks at +x, +y, +z offsets (-1: unallocated)
//   spv_integrate_kernel  one thread per allocated point, frames from its block's birth stamp on
//   spv_raycast_kernel    the dense raycast's march over the blocks' bounding box, skipping unallocated blocks
//   spv_mesh_*_kernel     the dense extraction's count / scan / base / emit, one CTA per block
//
// The per-point arithmetic restates tsdf_integrate_kernel, tsdf_raycast_kernel and mesh_emit_kernel (csrc/volume.cu)
// operation for operation: explicit round-to-nearest fp64 and fp32, no contraction, no floating-point atomics.
#include <climits>
#include <cmath>
#include <string>

#include "common.cuh"
#include "fp64.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {
namespace {

constexpr int kB = 8;                         // block edge in points
constexpr int kBP = kB * kB * kB;             // points per block
constexpr int kFrames = 16;                   // poses per launch, by value (as csrc/volume.cu)
constexpr int kSortTile = 1024;
constexpr long long kEmpty = -1;

struct Poses {
  double m[kFrames][12];                      // R row-major (9), then t (3), camera-to-world
};
struct Cam {
  double fx, fy, cx, cy;
};

// the view of a volume the kernels read
struct Vol {
  float* data;
  long long* keys;
  int* birth;
  int* nbr;
  long long* tkeys;
  int* tids;
  int* tbirth;
  int* bbox;
  int* scratch;
  int blocks, ch;
  unsigned tmask;
  int tshift;
  double o[3], voxel;
};

ODB_DEVINL long long pack_key(long long bx, long long by, long long bz) {
  return ((bz + ODB_SPARSE_TSDF_BLOCK_RANGE) << 42) | ((by + ODB_SPARSE_TSDF_BLOCK_RANGE) << 21) |
         (bx + ODB_SPARSE_TSDF_BLOCK_RANGE);
}
ODB_DEVINL void unpack_key(long long k, int b[3]) {
  b[0] = (int)(k & 0x1FFFFF) - ODB_SPARSE_TSDF_BLOCK_RANGE;
  b[1] = (int)((k >> 21) & 0x1FFFFF) - ODB_SPARSE_TSDF_BLOCK_RANGE;
  b[2] = (int)(k >> 42) - ODB_SPARSE_TSDF_BLOCK_RANGE;
}
ODB_DEVINL unsigned slot_of(long long key, int shift) {
  return (unsigned)(((unsigned long long)key * 0x9E3779B97F4A7C15ull) >> shift);
}
// the id of block key, -1 when unallocated (the table is at most half full outside spv_mark_kernel)
ODB_DEVINL int find(const Vol& V, long long key) {
  unsigned h = slot_of(key, V.tshift);
  for (unsigned probe = 0; probe <= V.tmask; ++probe) {
    const long long k = V.tkeys[h];
    if (k == key) return V.tids[h];
    if (k == kEmpty) return -1;
    h = (h + 1) & V.tmask;
  }
  return -1;
}

// ---------------------------------------------------------------------------------------------------- table
__global__ void __launch_bounds__(256) spv_clear_kernel(Vol V) {
  const unsigned s = blockIdx.x * 256u + threadIdx.x;
  if (s > V.tmask) return;
  V.tkeys[s] = kEmpty;
  V.tids[s] = -1;
  V.tbirth[s] = INT_MAX;
}

__global__ void __launch_bounds__(256) spv_insert_kernel(Vol V) {
  const int id = blockIdx.x * 256 + threadIdx.x;
  if (id >= V.blocks) return;
  const long long key = V.keys[id];
  unsigned h = slot_of(key, V.tshift);
  for (;;) {
    const long long prev = (long long)atomicCAS((unsigned long long*)&V.tkeys[h], (unsigned long long)kEmpty,
                                                (unsigned long long)key);
    if (prev == kEmpty) {
      V.tids[h] = id;
      V.tbirth[h] = V.birth[id];
      return;
    }
    h = (h + 1) & V.tmask;
  }
}

// scratch[0]: slots inserted by this call (also the list length), scratch[1]: set when the table passed half full,
// scratch[2..]: the inserted slots
ODB_DEVINL void mark_block(const Vol& V, long long key, int g) {
  int* count = V.scratch;
  unsigned h = slot_of(key, V.tshift);
  for (unsigned probe = 0; probe <= V.tmask; ++probe) {
    long long k = *(volatile long long*)&V.tkeys[h];
    if (k == kEmpty) {
      if ((long long)V.blocks + *(volatile int*)count >= (long long)(V.tmask + 1) / 2) {
        V.scratch[1] = 1;
        return;
      }
      k = (long long)atomicCAS((unsigned long long*)&V.tkeys[h], (unsigned long long)kEmpty, (unsigned long long)key);
      if (k == kEmpty) {
        atomicMin(&V.tbirth[h], g);
        V.scratch[2 + atomicAdd(count, 1)] = (int)h;
        return;
      }
    }
    if (k == key) {
      if (V.tids[h] < 0) atomicMin(&V.tbirth[h], g);
      return;
    }
    h = (h + 1) & V.tmask;
  }
  V.scratch[1] = 1;
}

__global__ void __launch_bounds__(128) spv_mark_kernel(Vol V, const float* __restrict__ depth, int h, int w, Cam K,
                                                       Poses P, double trunc, double max_depth, int frame0) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y, fr = blockIdx.z;
  if (x >= w) return;
  const double d = (double)depth[(long long)fr * h * w + (long long)y * w + x];
  if (!(isfinite(d) && d > 0.0 && d <= max_depth)) return;
  const double* m = P.m[fr];
  const double rx = __ddiv_rn(__dsub_rn((double)x, K.cx), K.fx), ry = __ddiv_rn(__dsub_rn((double)y, K.cy), K.fy);
  double lo[3], hi[3];
#pragma unroll 1
  for (int e = 0; e < 2; ++e) {
    const double z = e ? __dadd_rn(d, trunc) : __dsub_rn(d, trunc);
    const double xc = __dmul_rn(z, rx), yc = __dmul_rn(z, ry);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double X = __dadd_rn(
          __dadd_rn(__dadd_rn(__dmul_rn(m[3 * a], xc), __dmul_rn(m[3 * a + 1], yc)), __dmul_rn(m[3 * a + 2], z)),
          m[9 + a]);
      const double b = floor(__dmul_rn(__ddiv_rn(__dsub_rn(X, V.o[a]), V.voxel), 0.125));
      lo[a] = e ? fmin(lo[a], b) : b;
      hi[a] = e ? fmax(hi[a], b) : b;
    }
  }
  const double lim = (double)ODB_SPARSE_TSDF_BLOCK_RANGE;
#pragma unroll
  for (int a = 0; a < 3; ++a)
    if (!(lo[a] > -lim && hi[a] < lim)) return;         // never allocated: outside the block range
  const int g = frame0 + fr;
  for (int bz = (int)lo[2]; bz <= (int)hi[2]; ++bz)
    for (int by = (int)lo[1]; by <= (int)hi[1]; ++by)
      for (int bx = (int)lo[0]; bx <= (int)hi[0]; ++bx) mark_block(V, pack_key(bx, by, bz), g);
}

// ---------------------------------------------------------------------------------------------------- sort
struct NewBlock {
  long long key;
  int birth, slot;
};
ODB_DEVINL bool before(const NewBlock& a, const NewBlock& b) {
  return a.birth < b.birth || (a.birth == b.birth && a.key < b.key);
}

__global__ void __launch_bounds__(256) spv_sort_fill_kernel(Vol V, int n, int padded, NewBlock* __restrict__ s) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= padded) return;
  NewBlock e;
  if (i < n) {
    const int slot = V.scratch[2 + i];
    e.key = V.tkeys[slot];
    e.birth = V.tbirth[slot];
    e.slot = slot;
  } else {
    e.key = LLONG_MAX;
    e.birth = INT_MAX;
    e.slot = -1;
  }
  s[i] = e;
}

ODB_DEVINL void exchange(NewBlock& a, NewBlock& b, bool up) {
  if (before(b, a) == up) {
    const NewBlock t = a;
    a = b;
    b = t;
  }
}

// the bitonic stages j = min(k / 2, kSortTile / 2) .. 1 of merge size k (every k when k_first), in shared memory
__global__ void __launch_bounds__(kSortTile / 2) spv_sort_tile_kernel(NewBlock* __restrict__ s, int k_first,
                                                                      int k_last) {
  __shared__ NewBlock sh[kSortTile];
  const int base = blockIdx.x * kSortTile;
  sh[threadIdx.x] = s[base + threadIdx.x];
  sh[threadIdx.x + kSortTile / 2] = s[base + threadIdx.x + kSortTile / 2];
  __syncthreads();
  for (int k = k_first; k <= k_last; k <<= 1)
    for (int j = min(k, kSortTile) >> 1; j > 0; j >>= 1) {
      const int i = 2 * threadIdx.x - (threadIdx.x & (j - 1));      // the lower index of this thread's pair
      exchange(sh[i], sh[i + j], ((base + i) & k) == 0);
      __syncthreads();
    }
  s[base + threadIdx.x] = sh[threadIdx.x];
  s[base + threadIdx.x + kSortTile / 2] = sh[threadIdx.x + kSortTile / 2];
}

__global__ void __launch_bounds__(256) spv_sort_global_kernel(NewBlock* __restrict__ s, int k, int j) {
  const int t = blockIdx.x * 256 + threadIdx.x;
  const int i = 2 * t - (t & (j - 1));
  NewBlock a = s[i], b = s[i + j];
  exchange(a, b, (i & k) == 0);
  s[i] = a;
  s[i + j] = b;
}

// ---------------------------------------------------------------------------------------------------- commit
__global__ void __launch_bounds__(256) spv_assign_kernel(Vol V, int n, const NewBlock* __restrict__ s) {
  const int r = blockIdx.x * 256 + threadIdx.x;
  if (r >= n) return;
  const NewBlock e = s[r];
  const int id = V.blocks + r;
  V.keys[id] = e.key;
  V.birth[id] = e.birth;
  V.tids[e.slot] = id;
  int b[3];
  unpack_key(e.key, b);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    atomicMin(&V.bbox[a], b[a]);
    atomicMax(&V.bbox[3 + a], b[a]);
  }
}

__global__ void __launch_bounds__(256) spv_zero_kernel(Vol V, int n) {
  const long long q = (long long)blockIdx.x * 256 + threadIdx.x, per = (long long)V.ch * kBP;
  if (q >= n * per) return;
  V.data[(long long)V.blocks * per + q] = 0.f;
}

__global__ void __launch_bounds__(256) spv_nbr_kernel(Vol V, int total) {
  const long long q = (long long)blockIdx.x * 256 + threadIdx.x;
  if (q >= 8LL * total) return;
  const int id = (int)(q >> 3), c = (int)(q & 7);
  int b[3];
  unpack_key(V.keys[id], b);
  const long long nb[3] = {(long long)b[0] + (c & 1), (long long)b[1] + ((c >> 1) & 1), (long long)b[2] + (c >> 2)};
  bool in = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) in &= nb[a] < ODB_SPARSE_TSDF_BLOCK_RANGE;
  V.nbr[q] = in ? find(V, pack_key(nb[0], nb[1], nb[2])) : -1;
}

// ---------------------------------------------------------------------------------------------------- integrate
// tsdf_integrate_kernel's per-frame update, restated; a point updates from frame g only when g >= its block's birth
__global__ void __launch_bounds__(256) spv_integrate_kernel(Vol V, const float* __restrict__ depth,
                                                            const float* __restrict__ rgb, int h, int w, int frames,
                                                            int frame0, Cam K, double trunc, Poses P) {
  const int id = blockIdx.x >> 1, l = ((blockIdx.x & 1) << 8) | threadIdx.x;
  int b[3];
  unpack_key(V.keys[id], b);
  const int born = V.birth[id];
  const double X = __dadd_rn(V.o[0], __dmul_rn(V.voxel, (double)(kB * (long long)b[0] + (l & 7))));
  const double Y = __dadd_rn(V.o[1], __dmul_rn(V.voxel, (double)(kB * (long long)b[1] + ((l >> 3) & 7))));
  const double Z = __dadd_rn(V.o[2], __dmul_rn(V.voxel, (double)(kB * (long long)b[2] + (l >> 6))));
  float* p = V.data + (long long)id * V.ch * kBP + l;
  const bool col = V.ch == 5;
  const long long plane = (long long)h * w;
  float f = p[0], wt = p[kBP];
  float c0 = 0.f, c1 = 0.f, c2 = 0.f;
  if (col) {
    c0 = p[2 * kBP];
    c1 = p[3 * kBP];
    c2 = p[4 * kBP];
  }
  bool seen = false;
  for (int fr = 0; fr < frames; ++fr) {
    if (frame0 + fr < born) continue;
    const double* m = P.m[fr];
    const double dx = __dsub_rn(X, m[9]), dy = __dsub_rn(Y, m[10]), dz = __dsub_rn(Z, m[11]);
    const double zc = __dadd_rn(__dadd_rn(__dmul_rn(m[2], dx), __dmul_rn(m[5], dy)), __dmul_rn(m[8], dz));
    if (!(zc > 0.0)) continue;
    const double xc = __dadd_rn(__dadd_rn(__dmul_rn(m[0], dx), __dmul_rn(m[3], dy)), __dmul_rn(m[6], dz));
    const double yc = __dadd_rn(__dadd_rn(__dmul_rn(m[1], dx), __dmul_rn(m[4], dy)), __dmul_rn(m[7], dz));
    const double u = floor(__dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(K.fx, xc), zc), K.cx), 0.5));
    const double v = floor(__dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(K.fy, yc), zc), K.cy), 0.5));
    if (!(u >= 0.0 && u <= (double)(w - 1) && v >= 0.0 && v <= (double)(h - 1))) continue;
    const long long off = (long long)v * w + (long long)u;
    const float d = depth[fr * plane + off];
    if (!(isfinite(d) && d > 0.f)) continue;
    const double eta = __dsub_rn((double)d, zc);
    if (eta < -trunc) continue;
    const float fo = (float)fmin(1.0, __ddiv_rn(eta, trunc));
    const float w1 = __fadd_rn(wt, 1.f);
    f = __fdiv_rn(__fadd_rn(__fmul_rn(f, wt), fo), w1);
    if (col) {
      const float* px = rgb + 3 * fr * plane + off;
      c0 = __fdiv_rn(__fadd_rn(__fmul_rn(c0, wt), px[0]), w1);
      c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c1, wt), px[plane]), w1);
      c2 = __fdiv_rn(__fadd_rn(__fmul_rn(c2, wt), px[2 * plane]), w1);
    }
    wt = w1;
    seen = true;
  }
  if (seen) {
    p[0] = f;
    p[kBP] = wt;
    if (col) {
      p[2 * kBP] = c0;
      p[3 * kBP] = c1;
      p[4 * kBP] = c2;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- raycast
// The march box is the allocated blocks' bounding box [bmin, bmax]: its points are lo + voxel c, c in [0, n - 1]^3 with
// lo = origin + voxel 8 bmin and n = 8 (bmax - bmin + 1), exactly the grid SparseTSDFVolume.to_dense() returns.
struct Marcher {
  Vol V;
  double lo[3];
  int n[3], bmin[3];
  long long last_key;
  int last_id;

  // the trilinear cell of o + t d in box indices (tsdf_raycast_kernel's locate)
  ODB_DEVINL void locate(const double o[3], const double d[3], double t, int c[3], double fr[3]) const {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double g = __ddiv_rn(__dsub_rn(__dadd_rn(o[a], __dmul_rn(t, d[a])), lo[a]), V.voxel);
      const double fl = fmin(fmax(floor(g), 0.0), (double)(n[a] - 2));
      c[a] = (int)fl;
      fr[a] = fmin(fmax(__dsub_rn(g, fl), 0.0), 1.0);
    }
  }
  // the id of the block holding cell corner c, -1: unallocated (the last lookup is remembered)
  ODB_DEVINL int block_id(const int c[3]) {
    const long long key = pack_key(bmin[0] + (c[0] >> 3), bmin[1] + (c[1] >> 3), bmin[2] + (c[2] >> 3));
    if (key != last_key) {
      last_key = key;
      last_id = find(V, key);
    }
    return last_id;
  }
  // offsets into data of the cell's 8 corners (corner code bit 0 x, bit 1 y, bit 2 z); false when one is unallocated
  ODB_DEVINL bool corners(int id0, const int c[3], long long off[8]) const {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int lx = (c[0] & 7) + (q & 1), ly = (c[1] & 7) + ((q >> 1) & 1), lz = (c[2] & 7) + (q >> 2);
      const int id = V.nbr[8 * id0 + ((lx >> 3) | ((ly >> 3) << 1) | ((lz >> 3) << 2))];
      if (id < 0) return false;
      off[q] = (long long)id * V.ch * kBP + (lx & 7) + kB * (ly & 7) + kB * kB * (lz & 7);
    }
    return true;
  }
  ODB_DEVINL double trilinear(int chan, const long long off[8], const double fr[3]) const {
    const float* P = V.data + chan * kBP;
    double cv[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) cv[q] = lerp_rn((double)P[off[2 * q]], (double)P[off[2 * q + 1]], fr[0]);
    return lerp_rn(lerp_rn(cv[0], cv[1], fr[1]), lerp_rn(cv[2], cv[3], fr[1]), fr[2]);
  }
  // trilinear F at cell c, false when a corner is unallocated or has W = 0
  ODB_DEVINL bool sample(int id0, const int c[3], const double fr[3], double& val) const {
    long long off[8];
    if (!corners(id0, c, off)) return false;
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if (!(V.data[kBP + off[q]] > 0.f)) return false;
    val = trilinear(0, off, fr);
    return true;
  }
  ODB_DEVINL double color(const double o[3], const double d[3], double t, int a) {
    int c[3];
    double fr[3];
    locate(o, d, t, c, fr);
    long long off[8];
    corners(block_id(c), c, off);
    return trilinear(2 + a, off, fr);
  }
};

template <bool kColor>
__global__ void __launch_bounds__(128) spv_raycast_kernel(Vol V, Cam K, Poses P, int h, int w, double step,
                                                          float* __restrict__ out, float* __restrict__ rgb) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const double* m = P.m[0];
  const double rx = __ddiv_rn(__dsub_rn((double)x, K.cx), K.fx), ry = __ddiv_rn(__dsub_rn((double)y, K.cy), K.fy);
  const double nrm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(rx, rx), __dmul_rn(ry, ry)), 1.0));
  const double ux = __ddiv_rn(rx, nrm), uy = __ddiv_rn(ry, nrm), uz = __ddiv_rn(1.0, nrm);
  double d[3], o[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    d[a] = __dadd_rn(__dadd_rn(__dmul_rn(m[3 * a], ux), __dmul_rn(m[3 * a + 1], uy)), __dmul_rn(m[3 * a + 2], uz));
    o[a] = m[9 + a];
  }
  Marcher M;
  M.V = V;
  M.last_key = kEmpty;
  M.last_id = -1;
  bool miss = false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    M.bmin[a] = V.bbox[a];
    const int bmax = V.bbox[3 + a];
    miss |= bmax < M.bmin[a];                       // no block allocated
    M.n[a] = kB * (bmax - M.bmin[a] + 1);
    M.lo[a] = __dadd_rn(V.o[a], __dmul_rn(V.voxel, (double)(kB * (long long)M.bmin[a])));
  }
  double t0 = 0.0, t1 = INFINITY;
  if (!miss) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double lo = M.lo[a], hi = __dadd_rn(lo, __dmul_rn(V.voxel, (double)(M.n[a] - 1)));
      if (d[a] == 0.0) {
        miss |= o[a] < lo || o[a] > hi;
      } else {
        const double ta = __ddiv_rn(__dsub_rn(lo, o[a]), d[a]), tb = __ddiv_rn(__dsub_rn(hi, o[a]), d[a]);
        t0 = fmax(t0, fmin(ta, tb));
        t1 = fmin(t1, fmax(ta, tb));
      }
    }
  }
  float z = 0.f;
  bool hit = false;
  double t_lo = 0.0, t_hi = 0.0, frac = 0.0;
  if (!miss && t0 <= t1) {
    bool prev_ok = false;
    double prev = 0.0, tp = t0;
    // reciprocals for the skip estimate only (its result is confirmed by an exact locate)
    const double inv_step = __drcp_rn(step), inv_d[3] = {__drcp_rn(d[0]), __drcp_rn(d[1]), __drcp_rn(d[2])};
    for (long long s = 0;; ++s) {
      const double t = __dadd_rn(t0, __dmul_rn((double)s, step));
      if (!(t <= t1)) break;
      int c[3];
      double fr[3], val = 0.0;
      M.locate(o, d, t, c, fr);
      const int id0 = M.block_id(c);
      bool ok = false;
      if (id0 >= 0) {
        ok = M.sample(id0, c, fr, val);
      } else {
        // Every sample whose cell's lowest corner lies in this unallocated block is invalid.  The cell index is
        // monotone in s along each axis, so when sample s2 > s is in the same block, so is every sample between:
        // estimate the block's exit from its faces, step one sample back for rounding, confirm, and jump.
        double tx = INFINITY;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const int cb = c[a] >> 3;
          if (d[a] != 0.0) {
            const double face = __dadd_rn(M.lo[a], __dmul_rn(V.voxel, (double)(kB * (d[a] > 0.0 ? cb + 1 : cb))));
            tx = fmin(tx, __dmul_rn(__dsub_rn(face, o[a]), inv_d[a]));
          }
        }
        const double ks = floor(__dmul_rn(__dsub_rn(tx, t0), inv_step)) - 1.0;
        if (ks > (double)s && ks < 9.0e15) {
          const long long s2 = (long long)ks;
          int c2[3];
          double fr2[3];
          M.locate(o, d, __dadd_rn(t0, __dmul_rn((double)s2, step)), c2, fr2);
          if ((c2[0] >> 3) == (c[0] >> 3) && (c2[1] >> 3) == (c[1] >> 3) && (c2[2] >> 3) == (c[2] >> 3)) s = s2;
        }
      }
      if (ok && prev_ok && prev > 0.0 && val <= 0.0) {
        frac = __ddiv_rn(prev, __dsub_rn(prev, val));
        const double th = __dadd_rn(tp, __dmul_rn(step, frac));
        z = (float)__dmul_rn(th, uz);
        hit = true;
        t_lo = tp;
        t_hi = t;
        break;
      }
      prev_ok = ok;
      prev = val;
      tp = t;
    }
  }
  const long long px = (long long)y * w + x, plane = (long long)h * w;
  out[px] = z;
  if constexpr (kColor) {
#pragma unroll 1
    for (int a = 0; a < 3; ++a)
      rgb[a * plane + px] = hit ? (float)lerp_rn(M.color(o, d, t_lo, a), M.color(o, d, t_hi, a), frac) : NAN;
  }
}

// ---------------------------------------------------------------------------------------------------- mesh
// Kuhn split and marching-tetrahedra tables: csrc/volume.cu's, restated
__constant__ unsigned char kTetCorner[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7},
                                               {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};
__constant__ unsigned char kTetOdd[6] = {0, 1, 1, 0, 0, 1};
__constant__ unsigned char kTetEdge[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
__constant__ signed char kTetTri[16][2][3] = {
    {{-1, -1, -1}, {-1, -1, -1}}, {{0, 1, 2}, {-1, -1, -1}}, {{0, 4, 3}, {-1, -1, -1}}, {{1, 2, 4}, {1, 4, 3}},
    {{1, 3, 5}, {-1, -1, -1}},    {{0, 5, 2}, {0, 3, 5}},    {{0, 4, 5}, {0, 5, 1}},    {{2, 4, 5}, {-1, -1, -1}},
    {{2, 5, 4}, {-1, -1, -1}},    {{0, 1, 5}, {0, 5, 4}},    {{0, 5, 3}, {0, 2, 5}},    {{1, 5, 3}, {-1, -1, -1}},
    {{1, 3, 4}, {1, 4, 2}},       {{0, 3, 4}, {-1, -1, -1}}, {{0, 2, 1}, {-1, -1, -1}}, {{-1, -1, -1}, {-1, -1, -1}}};

struct MeshWs {                 // odb_sparse_tsdf_mesh_workspace_bytes
  long long* base;              // [2][blocks]: exclusive vertex / face base of each block
  int* vbase;                   // [blocks][512]: first vertex id of each point
  int* blk;                     // [2][blocks]: vertex / face count of each block
  unsigned char *mask, *ntri;   // [blocks][512]
};

MeshWs mesh_ws(void* workspace, long long nb) {
  MeshWs M;
  M.base = static_cast<long long*>(workspace);
  M.vbase = reinterpret_cast<int*>(M.base + 2 * nb);
  M.blk = M.vbase + nb * kBP;
  M.mask = reinterpret_cast<unsigned char*>(M.blk + 2 * nb);
  M.ntri = M.mask + nb * kBP;
  return M;
}

// the block id and in-block index of corner c of point l of block id, -1 when the corner's block is unallocated
ODB_DEVINL long long corner_ref(const Vol& V, int id, int l, int c) {
  const int lx = (l & 7) + (c & 1), ly = ((l >> 3) & 7) + ((c >> 1) & 1), lz = (l >> 6) + (c >> 2);
  const int nid = V.nbr[8 * id + ((lx >> 3) | ((ly >> 3) << 1) | ((lz >> 3) << 2))];
  return nid < 0 ? -1 : (long long)nid * kBP + ((lx & 7) + kB * (ly & 7) + kB * kB * (lz & 7));
}

ODB_DEVINL void load_corners(const Vol& V, int id, int l, float f[8], float wt[8]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const long long r = corner_ref(V, id, l, c);
    const float* p = V.data + (r / kBP) * V.ch * kBP + (r % kBP);
    f[c] = r < 0 ? 0.f : p[0];
    wt[c] = r < 0 ? 0.f : p[kBP];
  }
}

ODB_DEVINL int edge_mask(const float f[8], const float wt[8]) {
  int mask = 0;
  if (wt[0] > 0.f) {
#pragma unroll
    for (int c = 1; c < 8; ++c)
      if (wt[c] > 0.f && ((f[0] < 0.f) != (f[c] < 0.f))) mask |= 1 << (c - 1);
  }
  return mask;
}

ODB_DEVINL void corner_bits(const float f[8], const float wt[8], int& obs, int& neg) {
  obs = neg = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    obs |= (wt[c] > 0.f ? 1 : 0) << c;
    neg |= (f[c] < 0.f ? 1 : 0) << c;
  }
}

ODB_DEVINL int tet_inside(int q, int obs, int neg) {
  int m = 0;
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    const int c = kTetCorner[q][v];
    if (!((obs >> c) & 1)) return -1;
    m |= ((neg >> c) & 1) << v;
  }
  return m;
}

ODB_DEVINL int tet_triangles(int inside) { return (inside == 0 || inside == 15) ? 0 : (__popc(inside) == 2 ? 2 : 1); }

// exclusive scan of v over the CTA (kBP threads); total = the CTA's sum
ODB_DEVINL int block_exclusive_scan(int v, int& total) {
  __shared__ int warp_sum[kBP / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int s = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, s, o);
    if (lane >= o) s += t;
  }
  if (lane == 31) warp_sum[wid] = s;
  __syncthreads();
  int before = 0;
  total = 0;
#pragma unroll
  for (int q = 0; q < kBP / 32; ++q) {
    const int t = warp_sum[q];
    before += q < wid ? t : 0;
    total += t;
  }
  __syncthreads();
  return before + s - v;
}

__global__ void __launch_bounds__(kBP) spv_mesh_count_kernel(Vol V, MeshWs M) {
  const int id = blockIdx.x, l = threadIdx.x;
  const long long p = (long long)id * kBP + l;
  float f[8], wt[8];
  load_corners(V, id, l, f, wt);
  const int mask = edge_mask(f, wt);
  int obs, neg, tris = 0;
  corner_bits(f, wt, obs, neg);
  for (int q = 0; q < 6; ++q) {
    const int m = tet_inside(q, obs, neg);
    if (m >= 0) tris += tet_triangles(m);
  }
  M.mask[p] = (unsigned char)mask;
  M.ntri[p] = (unsigned char)tris;
  int tv, tf;
  block_exclusive_scan(__popc(mask), tv);
  block_exclusive_scan(tris, tf);
  if (threadIdx.x == 0) {
    M.blk[id] = tv;
    M.blk[gridDim.x + id] = tf;
  }
}

// one CTA of 1024 threads: each scans a contiguous run of block totals (mesh_scan_kernel, restated)
__global__ void __launch_bounds__(1024) spv_mesh_scan_kernel(MeshWs M, long long nb, long long* __restrict__ counts) {
  __shared__ long long run[2][1024];
  const long long per = (nb + 1023) / 1024, b0 = min(nb, threadIdx.x * per), b1 = min(nb, b0 + per);
  for (int s = 0; s < 2; ++s) {
    long long sum = 0;
    for (long long b = b0; b < b1; ++b) sum += M.blk[s * nb + b];
    run[s][threadIdx.x] = sum;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    long long acc = 0;
    for (int t = 0; t < 1024; ++t) {
      const long long v = run[threadIdx.x][t];
      run[threadIdx.x][t] = acc;
      acc += v;
    }
    counts[threadIdx.x] = acc;
  }
  __syncthreads();
  for (int s = 0; s < 2; ++s) {
    long long acc = run[s][threadIdx.x];
    for (long long b = b0; b < b1; ++b) {
      M.base[s * nb + b] = acc;
      acc += M.blk[s * nb + b];
    }
  }
}

__global__ void __launch_bounds__(kBP) spv_mesh_base_kernel(MeshWs M) {
  const long long p = (long long)blockIdx.x * kBP + threadIdx.x;
  int total;
  const int local = block_exclusive_scan(__popc(M.mask[p]), total);
  M.vbase[p] = (int)(M.base[blockIdx.x] + local);
}

__global__ void __launch_bounds__(kBP) spv_mesh_emit_kernel(Vol V, MeshWs M, float* __restrict__ verts,
                                                            int* __restrict__ faces, float* __restrict__ colors) {
  const int id = blockIdx.x, l = threadIdx.x;
  const long long p = (long long)id * kBP + l;
  const int tris = M.ntri[p];
  int total;
  const long long fbase = M.base[gridDim.x + id] + block_exclusive_scan(tris, total);
  const int mask = M.mask[p];
  if (mask == 0 && tris == 0) return;
  float f[8], wt[8];
  load_corners(V, id, l, f, wt);
  int b[3];
  unpack_key(V.keys[id], b);
  const double gp[3] = {(double)(kB * (long long)b[0] + (l & 7)), (double)(kB * (long long)b[1] + ((l >> 3) & 7)),
                        (double)(kB * (long long)b[2] + (l >> 6))};
  const float* cp = V.data + (long long)id * V.ch * kBP + 2 * kBP + l;
  long long vid = M.vbase[p];
#pragma unroll
  for (int c = 1; c < 8; ++c) {
    if (!((mask >> (c - 1)) & 1)) continue;
    const double fp = f[0], s = __ddiv_rn(fp, __dsub_rn(fp, (double)f[c]));
#pragma unroll
    for (int a = 0; a < 3; ++a)
      verts[3 * vid + a] =
          (float)__dadd_rn(V.o[a], __dmul_rn(V.voxel, __dadd_rn(gp[a], ((c >> a) & 1) ? s : 0.0)));
    if (colors) {
      const long long r = corner_ref(V, id, l, c);
      const float* cq = V.data + (r / kBP) * V.ch * kBP + 2 * kBP + (r % kBP);
#pragma unroll
      for (int a = 0; a < 3; ++a)
        colors[3 * vid + a] = (float)lerp_rn((double)cp[a * kBP], (double)cq[a * kBP], s);
    }
    ++vid;
  }
  if (tris == 0) return;
  int obs, neg;
  corner_bits(f, wt, obs, neg);
  long long fo = fbase;
  for (int q = 0; q < 6; ++q) {
    const int m = tet_inside(q, obs, neg);
    if (m < 0) continue;
    for (int t = 0; t < 2; ++t) {
      if (kTetTri[m][t][0] < 0) break;
      int vi[3];
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        const int edge = kTetTri[m][t][e];
        const int ca = kTetCorner[q][kTetEdge[edge][0]], cb = kTetCorner[q][kTetEdge[edge][1]];
        const long long owner = corner_ref(V, id, l, ca);
        const int dir = (ca ^ cb) - 1;
        vi[e] = M.vbase[owner] + __popc(M.mask[owner] & ((1 << dir) - 1));
      }
      const int odd = kTetOdd[q];
      faces[3 * fo] = vi[0];
      faces[3 * fo + 1] = vi[odd ? 2 : 1];
      faces[3 * fo + 2] = vi[odd ? 1 : 2];
      ++fo;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- host
bool vol_ok(const odb_sparse_tsdf* s, Vol& V) {
  if (!s || !s->data || !s->keys || !s->birth || !s->nbr || !s->table_keys || !s->table_ids || !s->table_birth ||
      !s->bbox || !s->scratch || !(s->channels == 2 || s->channels == 5) || s->blocks < 0 ||
      s->blocks > s->capacity || s->capacity > ODB_SPARSE_TSDF_MAX_BLOCKS || s->table_size < 1024 ||
      s->table_size > (1 << 30) || (s->table_size & (s->table_size - 1)) || s->blocks > s->table_size / 2 ||
      !(std::isfinite(s->ox) && std::isfinite(s->oy) && std::isfinite(s->oz) && std::isfinite(s->voxel) &&
        s->voxel > 0.0) ||
      !aligned(s->data, 4) || !aligned(s->keys, 8) || !aligned(s->birth, 4) || !aligned(s->nbr, 4) ||
      !aligned(s->table_keys, 8) || !aligned(s->table_ids, 4) || !aligned(s->table_birth, 4) ||
      !aligned(s->bbox, 4) || !aligned(s->scratch, 4))
    return false;
  V.data = s->data;
  V.keys = reinterpret_cast<long long*>(s->keys);
  V.birth = s->birth;
  V.nbr = s->nbr;
  V.tkeys = reinterpret_cast<long long*>(s->table_keys);
  V.tids = s->table_ids;
  V.tbirth = s->table_birth;
  V.bbox = s->bbox;
  V.scratch = s->scratch;
  V.blocks = s->blocks;
  V.ch = s->channels;
  V.tmask = (unsigned)s->table_size - 1u;
  int bits = 0;
  while ((1 << bits) < s->table_size) ++bits;
  V.tshift = 64 - bits;
  V.o[0] = s->ox;
  V.o[1] = s->oy;
  V.o[2] = s->oz;
  V.voxel = s->voxel;
  return true;
}

bool cam_ok(double fx, double fy, double cx, double cy, Cam& K) {
  if (!(std::isfinite(fx) && fx > 0.0 && std::isfinite(fy) && fy > 0.0 && std::isfinite(cx) && std::isfinite(cy)))
    return false;
  K.fx = fx; K.fy = fy; K.cx = cx; K.cy = cy;
  return true;
}

unsigned cdiv(long long a, long long b) { return (unsigned)((a + b - 1) / b); }

int sort_pad(int n) {
  int p = kSortTile;
  while (p < n) p <<= 1;
  return p;
}

}  // namespace
}  // namespace odb

using namespace odb;

extern "C" int odb_sparse_tsdf_rebuild(const odb_sparse_tsdf* vol, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Vol V;
  if (!vol_ok(vol, V)) return fail(ODB_ERR_INVALID, "sparse_tsdf_rebuild: bad argument");
  spv_clear_kernel<<<cdiv((long long)V.tmask + 1, 256), 256, 0, stream>>>(V);
  count_launch();
  if (V.blocks > 0) {
    spv_insert_kernel<<<cdiv(V.blocks, 256), 256, 0, stream>>>(V);
    count_launch();
  }
  return check_launch("sparse_tsdf_rebuild");
}

extern "C" int odb_sparse_tsdf_mark(const odb_sparse_tsdf* vol, double trunc, double max_depth, const float* depth,
                                    int32_t b, int32_t h, int32_t w, double fx, double fy, double cx, double cy,
                                    const double* cam_to_world, int32_t frame0, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Vol V;
  Cam K;
  if (!vol_ok(vol, V) || !depth || !cam_to_world || !(std::isfinite(trunc) && trunc > 0.0) ||
      !(std::isfinite(max_depth) && max_depth > 0.0) || !planes_ok(b, h, w) || !cam_ok(fx, fy, cx, cy, K) ||
      frame0 < 0 || (int64_t)frame0 + b > INT_MAX || !aligned(depth, 4))
    return fail(ODB_ERR_INVALID, "sparse_tsdf_mark: bad argument");
  double tmp[12];
  for (int32_t f = 0; f < b; ++f)
    if (!pose_ok(cam_to_world + 16 * (int64_t)f, tmp))
      return fail(ODB_ERR_INVALID, "sparse_tsdf_mark: a pose is not a finite rigid camera-to-world matrix");
  cudaMemsetAsync(V.scratch, 0, 2 * sizeof(int), stream);
  const long long plane = (long long)h * w;
  for (int32_t f0 = 0; f0 < b; f0 += kFrames) {
    const int frames = b - f0 < kFrames ? b - f0 : kFrames;
    Poses P;
    for (int f = 0; f < frames; ++f) pose_ok(cam_to_world + 16 * (int64_t)(f0 + f), P.m[f]);
    spv_mark_kernel<<<dim3(cdiv(w, 128), h, frames), 128, 0, stream>>>(V, depth + f0 * plane, h, w, K, P, trunc,
                                                                        max_depth, frame0 + f0);
    count_launch();
  }
  return check_launch("sparse_tsdf_mark");
}

extern "C" int64_t odb_sparse_tsdf_commit_workspace_bytes(int32_t n_new) {
  if (n_new < 0 || n_new > ODB_SPARSE_TSDF_MAX_BLOCKS) return -1;
  return (int64_t)sort_pad(n_new) * (int64_t)sizeof(NewBlock);
}

extern "C" int odb_sparse_tsdf_commit(const odb_sparse_tsdf* vol, int32_t n_new, void* workspace, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Vol V;
  if (!vol_ok(vol, V) || n_new < 0 || (int64_t)V.blocks + n_new > vol->capacity ||
      (int64_t)V.blocks + n_new > (int64_t)vol->table_size / 2 || !workspace || !aligned(workspace, 16))
    return fail(ODB_ERR_INVALID, "sparse_tsdf_commit: bad argument");
  if (n_new == 0) return 0;
  NewBlock* s = static_cast<NewBlock*>(workspace);
  const int pad = sort_pad(n_new);
  spv_sort_fill_kernel<<<cdiv(pad, 256), 256, 0, stream>>>(V, n_new, pad, s);
  count_launch();
  spv_sort_tile_kernel<<<pad / kSortTile, kSortTile / 2, 0, stream>>>(s, 2, kSortTile);
  count_launch();
  for (int k = 2 * kSortTile; k <= pad; k <<= 1) {
    for (int j = k >> 1; j >= kSortTile; j >>= 1) {
      spv_sort_global_kernel<<<pad / 2 / 256, 256, 0, stream>>>(s, k, j);
      count_launch();
    }
    spv_sort_tile_kernel<<<pad / kSortTile, kSortTile / 2, 0, stream>>>(s, k, k);
    count_launch();
  }
  spv_assign_kernel<<<cdiv(n_new, 256), 256, 0, stream>>>(V, n_new, s);
  count_launch();
  spv_zero_kernel<<<cdiv((long long)n_new * V.ch * kBP, 256), 256, 0, stream>>>(V, n_new);
  count_launch();
  const int total = V.blocks + n_new;
  V.blocks = total;
  spv_nbr_kernel<<<cdiv(8LL * total, 256), 256, 0, stream>>>(V, total);
  count_launch();
  return check_launch("sparse_tsdf_commit");
}

extern "C" int odb_sparse_tsdf_integrate(const odb_sparse_tsdf* vol, double trunc, const float* depth,
                                         const float* rgb, int32_t b, int32_t h, int32_t w, double fx, double fy,
                                         double cx, double cy, const double* cam_to_world, int32_t frame0,
                                         void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Vol V;
  Cam K;
  if (!vol_ok(vol, V) || !depth || !cam_to_world || (V.ch == 5) != (rgb != nullptr) ||
      !(std::isfinite(trunc) && trunc > 0.0) || !planes_ok(b, h, w) || !cam_ok(fx, fy, cx, cy, K) || frame0 < 0 ||
      (int64_t)frame0 + b > INT_MAX || !aligned(depth, 4) || !aligned(rgb, 4))
    return fail(ODB_ERR_INVALID, "sparse_tsdf_integrate: bad argument");
  double tmp[12];
  for (int32_t f = 0; f < b; ++f)
    if (!pose_ok(cam_to_world + 16 * (int64_t)f, tmp))
      return fail(ODB_ERR_INVALID, "sparse_tsdf_integrate: a pose is not a finite rigid camera-to-world matrix");
  if (V.blocks == 0) return 0;
  const long long plane = (long long)h * w;
  for (int32_t f0 = 0; f0 < b; f0 += kFrames) {
    const int frames = b - f0 < kFrames ? b - f0 : kFrames;
    Poses P;
    for (int f = 0; f < frames; ++f) pose_ok(cam_to_world + 16 * (int64_t)(f0 + f), P.m[f]);
    spv_integrate_kernel<<<2u * (unsigned)V.blocks, 256, 0, stream>>>(
        V, depth + f0 * plane, rgb ? rgb + 3 * f0 * plane : nullptr, h, w, frames, frame0 + f0, K, trunc, P);
    count_launch();
  }
  return check_launch("sparse_tsdf_integrate");
}

extern "C" int odb_sparse_tsdf_raycast(const odb_sparse_tsdf* vol, const double* cam_to_world, int32_t h, int32_t w,
                                       double fx, double fy, double cx, double cy, double step, float* out, float* rgb,
                                       void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Vol V;
  Cam K;
  Poses P;
  if (!vol_ok(vol, V) || !cam_to_world || !out || (rgb && V.ch != 5) || !planes_ok(1, h, w) ||
      !cam_ok(fx, fy, cx, cy, K) || !(std::isfinite(step) && step >= V.voxel / 64.0 && step <= V.voxel) ||
      !aligned(out, 4) || !aligned(rgb, 4))
    return fail(ODB_ERR_INVALID, "sparse_tsdf_raycast: bad argument");
  if (!pose_ok(cam_to_world, P.m[0]))
    return fail(ODB_ERR_INVALID, "sparse_tsdf_raycast: the pose is not a finite rigid camera-to-world matrix");
  const dim3 grid(cdiv(w, 128), h);
  if (rgb)
    spv_raycast_kernel<true><<<grid, 128, 0, stream>>>(V, K, P, h, w, step, out, rgb);
  else
    spv_raycast_kernel<false><<<grid, 128, 0, stream>>>(V, K, P, h, w, step, out, nullptr);
  count_launch();
  return check_launch("sparse_tsdf_raycast");
}

extern "C" int64_t odb_sparse_tsdf_mesh_workspace_bytes(int32_t blocks) {
  if (blocks < 0 || blocks > ODB_SPARSE_TSDF_MAX_BLOCKS) return -1;
  const long long nb = blocks > 0 ? blocks : 1;
  return 2 * nb * 8 + nb * kBP * 4 + 2 * nb * 4 + 2 * nb * kBP;
}

extern "C" int odb_sparse_tsdf_mesh_count(const odb_sparse_tsdf* vol, void* workspace, int64_t* counts,
                                          void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Vol V;
  if (!vol_ok(vol, V) || !workspace || !counts || !aligned(workspace, 8) || !aligned(counts, 8))
    return fail(ODB_ERR_INVALID, "sparse_tsdf_mesh_count: bad argument");
  if (V.blocks == 0) {
    cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), stream);
    return check_launch("sparse_tsdf_mesh_count");
  }
  const MeshWs M = mesh_ws(workspace, V.blocks);
  spv_mesh_count_kernel<<<(unsigned)V.blocks, kBP, 0, stream>>>(V, M);
  count_launch();
  spv_mesh_scan_kernel<<<1, 1024, 0, stream>>>(M, V.blocks, reinterpret_cast<long long*>(counts));
  count_launch();
  spv_mesh_base_kernel<<<(unsigned)V.blocks, kBP, 0, stream>>>(M);
  count_launch();
  return check_launch("sparse_tsdf_mesh_count");
}

extern "C" int odb_sparse_tsdf_mesh_emit(const odb_sparse_tsdf* vol, const void* workspace, float* vertices,
                                         int32_t* faces, float* colors, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Vol V;
  if (!vol_ok(vol, V) || !workspace || (colors && V.ch != 5) || !aligned(workspace, 8) || !aligned(vertices, 4) ||
      !aligned(faces, 4) || !aligned(colors, 4))
    return fail(ODB_ERR_INVALID, "sparse_tsdf_mesh_emit: bad argument");
  if (V.blocks == 0) return 0;
  const MeshWs M = mesh_ws(const_cast<void*>(workspace), V.blocks);
  spv_mesh_emit_kernel<<<(unsigned)V.blocks, kBP, 0, stream>>>(V, M, vertices, faces, colors);
  count_launch();
  return check_launch("sparse_tsdf_mesh_emit");
}
