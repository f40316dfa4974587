// wgmma fused attention for the ViT blocks of the DPTs (d = 64, up to 4 097 tokens):
//   out = softmax(q k^T * scale) v        (timm Attention.forward; block loop at M/vit.py:150-151)
//
// Two instances of one kernel, chosen by the host from the token count:
//   resident (<= 640 tokens)  one persistent CTA per SM; a work unit is one (image, head).  K and V of the unit
//                             (<= 5 blocks of 128 keys x 64 d each) are TMA-loaded once into shared memory and stay
//                             resident; the 128-query tiles of the unit stream through a double-buffered Q slot.
//   streaming (> 640 tokens)  a work item is one (image, head, 128-query tile), items of one (image, head) adjacent so
//                             that the CTAs running at the same time share K and V through L2.  K and V blocks stream
//                             through a ring of 10 slots of 128 keys (the shared memory of the resident K and V) in
//                             the order the consumers read them: K_0..K_{n-1} for pass 1, then K_j, V_j for pass 2.
//                             Every query tile reads K twice and V once from L2.
//   warpgroup 0      TMA producer (K, V blocks; Q tiles)
//   warpgroups 1, 2  64 query rows of the tile each:  S = Q K_j^T  (wgmma M=64, N=128, K=64, both operands K-major)
//                                                     O += P_j V_j (M=64, N=64, K=128, P from registers,
//                                                                  V the MN-major B operand)
// Softmax is two-pass and exact: pass 1 computes the S blocks for the row maximum, pass 2 re-computes them,
// turns them into P = exp2(s*c - m*c) (bf16, straight from the accumulator registers into the A-operand registers
// of the PV product) and accumulates the fp32 row sum of the unrounded P.  O therefore never needs rescaling and
// stays in registers until the epilogue.  A row of S lives in the four lanes of a quad: row reductions are two
// shuffles.  Both instances compute the same function with the same rounding points; only the data movement differs.
#include "common.cuh"
#include "host_util.h"
#include "wgmma.cuh"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kTcBlk = 128;         // queries per tile == keys per block
constexpr int kTcMaxBlocks = 5;     // 640 keys: the resident instance
constexpr int kTcStreamMaxTokens = 4097;   // 64 x 64 patches + cls: the streaming instance
constexpr int kTcRing = 2 * kTcMaxBlocks;  // streaming K / V ring slots: the resident K and V space
constexpr int kTcTileBytes = kTcBlk * 128;   // 128 rows x 64 bf16
constexpr int kTcThreads = 384;
constexpr int kTcConsumerWarps = 8;

constexpr int kTcOffK = 0;
constexpr int kTcOffV = kTcMaxBlocks * kTcTileBytes;
constexpr int kTcOffQ = 2 * kTcMaxBlocks * kTcTileBytes;
constexpr int kTcOffBar = kTcOffQ + 2 * kTcTileBytes;
constexpr int kTcSmemBytes = kTcOffBar + 256 + 1024;
static_assert(kTcSmemBytes <= 232448, "attention smem plan exceeds 227 KiB");

struct AttnTcParams {
  CUtensorMap qkv_map;   // dims {64 d, 3*heads, tokens, batch}; box {64, 1, 128, 1}
  bf16* out;
  float* lse;            // optional [batch][heads][tokens]: log2 sum_j exp2(s_j c) per query row (training)
  int tokens, heads, batch;
  float scale_log2e;
  unsigned long long* trace;   // diagnostics: per CTA kTraceSlots stamps; per q tile i < 8 at 8 + 12 i:
                               // first S seen, maxima known, P block 0..4 done, sums known, O ready, tile stored
};
#define ODB_ATRACE(i, k)                                                                           \
  do {                                                                                             \
    if (p.trace != nullptr && (i) < 8u && warp == 4 && lane == 0) {                                \
      unsigned long long t_;                                                                       \
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));                                       \
      p.trace[static_cast<long long>(blockIdx.x) * kTraceSlots + 8 + 12 * static_cast<int>(i) + (k)] = t_; \
    }                                                                                              \
  } while (0)

ODB_DEVINL float fast_exp2_tc(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <bool STREAM>
__global__ void __launch_bounds__(kTcThreads, 1) attention_tc_kernel(const __grid_constant__ AttnTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar0 = sbase + kTcOffBar;
  const uint32_t kv_empty = bar0;
  auto q_full = [&](int i) { return bar0 + 16u + 8u * i; };
  auto q_empty = [&](int i) { return bar0 + 32u + 8u * i; };
  // K and V arrive block by block (own barrier each): the first S block of a unit starts after 16 KiB
  // instead of after the whole 160 KiB, the rest of the fetch hides behind pass 1
  auto k_full = [&](int j) { return bar0 + 136u + 8u * j; };
  auto v_full = [&](int j) { return bar0 + 176u + 8u * j; };
  // streaming: slot i of the K / V ring at sbase + i * kTcTileBytes, full / empty barrier pair of its own
  auto ring_full = [&](uint32_t i) { return bar0 + 48u + 8u * i; };
  auto ring_empty = [&](uint32_t i) { return bar0 + 128u + 8u * i; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nblk = (p.tokens + kTcBlk - 1) / kTcBlk;     // key blocks == query tiles
  const int units = p.batch * p.heads;
  const int items = units * nblk;                         // streaming work items: (image, head, query tile)

  if (threadIdx.x == 0) {
    if constexpr (STREAM) {
      for (uint32_t i = 0; i < kTcRing; ++i) { mbar_init(ring_full(i), 1); mbar_init(ring_empty(i), kTcConsumerWarps); }
    } else {
      mbar_init(kv_empty, kTcConsumerWarps);
      for (int j = 0; j < kTcMaxBlocks; ++j) { mbar_init(k_full(j), 1); mbar_init(v_full(j), 1); }
    }
    for (int i = 0; i < 2; ++i) { mbar_init(q_full(i), 1); mbar_init(q_empty(i), kTcConsumerWarps); }
    mbar_fence_init();
    tma_prefetch_desc(&p.qkv_map);
  }
  __syncthreads();
  grid_dep_wait();
  grid_dep_launch();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      if constexpr (STREAM) {
        uint32_t slot = 0, phase = 0, qt_iter = 0;
        auto ring_load = [&](int row, int j, int b) {
          mbar_wait(ring_empty(slot), phase ^ 1u);
          mbar_expect_tx(ring_full(slot), kTcTileBytes);
          tma_load_4d(sbase + slot * kTcTileBytes, &p.qkv_map, ring_full(slot), 0, row, j * kTcBlk, b);
          if (++slot == kTcRing) { slot = 0; phase ^= 1u; }
        };
        for (int item = blockIdx.x; item < items; item += gridDim.x, ++qt_iter) {
          const int unit = item / nblk, qt = item - unit * nblk;
          const int b = unit / p.heads, h = unit % p.heads;
          const int qb = qt_iter & 1u;
          mbar_wait(q_empty(qb), ((qt_iter >> 1) & 1u) ^ 1u);
          mbar_expect_tx(q_full(qb), kTcTileBytes);
          tma_load_4d(sbase + kTcOffQ + qb * kTcTileBytes, &p.qkv_map, q_full(qb), 0, h, qt * kTcBlk, b);
          for (int j = 0; j < nblk; ++j) ring_load(p.heads + h, j, b);             // pass 1: K
          for (int j = 0; j < nblk; ++j) {                                         // pass 2: K, V
            ring_load(p.heads + h, j, b);
            ring_load(2 * p.heads + h, j, b);
          }
        }
      } else {
        uint32_t u_iter = 0, qt_iter = 0;
        for (int unit = blockIdx.x; unit < units; unit += gridDim.x, ++u_iter) {
          const int b = unit / p.heads, h = unit % p.heads;
          mbar_wait(kv_empty, (u_iter & 1u) ^ 1u);
          for (int j = 0; j < nblk; ++j) {
            mbar_expect_tx(k_full(j), kTcTileBytes);
            tma_load_4d(sbase + kTcOffK + j * kTcTileBytes, &p.qkv_map, k_full(j), 0, p.heads + h, j * kTcBlk, b);
          }
          for (int j = 0; j < nblk; ++j) {
            mbar_expect_tx(v_full(j), kTcTileBytes);
            tma_load_4d(sbase + kTcOffV + j * kTcTileBytes, &p.qkv_map, v_full(j), 0, 2 * p.heads + h, j * kTcBlk, b);
          }
          for (int qt = 0; qt < nblk; ++qt, ++qt_iter) {
            const int qb = qt_iter & 1u;
            mbar_wait(q_empty(qb), ((qt_iter >> 1) & 1u) ^ 1u);
            mbar_expect_tx(q_full(qb), kTcTileBytes);
            tma_load_4d(sbase + kTcOffQ + qb * kTcTileBytes, &p.qkv_map, q_full(qb), 0, h, qt * kTcBlk, b);
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ softmax + PV + epilogue
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = (warp - 4) >> 2;
    const int r0 = wg * 64 + 16 * (warp & 3) + (lane >> 2);   // tile rows r0 and r0 + 8 of this thread
    const int cl = 2 * (lane & 3);                             // first of the two columns per 8-column block
    const float c = p.scale_log2e;
    uint32_t u_iter = 0, qt_iter = 0;
    float s[64];
    auto compute_s = [&](uint32_t koff, uint32_t qb) {
      const uint64_t adesc = gmma_desc_sw128(sbase + kTcOffQ + qb * kTcTileBytes + static_cast<uint32_t>(wg) * 8192u);
      const uint64_t bdesc = gmma_desc_sw128(sbase + koff);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) Wgmma<128>::ss<0, 0>(s, adesc + 2u * k, bdesc + 2u * k, k != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<64>(s);
    };
    // streaming: the next ring slot in the producer's order, released once this warp's MMAs have read it
    uint32_t r_slot = 0, r_phase = 0;
    auto ring_acquire = [&]() {
      mbar_wait(ring_full(r_slot), r_phase);
      return r_slot;
    };
    auto ring_release = [&](uint32_t slot) {
      __syncwarp();
      if (lane == 0) mbar_arrive(ring_empty(slot));
      if (++r_slot == kTcRing) { r_slot = 0; r_phase ^= 1u; }
    };
    // resident: work unit = (image, head), all its query tiles; streaming: work item = one query tile
    for (int unit = blockIdx.x; unit < (STREAM ? items : units); unit += gridDim.x, ++u_iter) {
      const int bh = STREAM ? unit / nblk : unit;
      const int b = bh / p.heads, h = bh % p.heads;
      const int qt_end = STREAM ? unit - bh * nblk + 1 : nblk;
      for (int qt = STREAM ? qt_end - 1 : 0; qt < qt_end; ++qt, ++qt_iter) {
        const uint32_t qb = qt_iter & 1u;
        mbar_wait(q_full(qb), (qt_iter >> 1) & 1u);
        // ---- pass 1: row maximum over all valid keys
        float mx0 = -INFINITY, mx1 = -INFINITY;
        for (int j = 0; j < nblk; ++j) {
          if constexpr (STREAM) {
            const uint32_t slot = ring_acquire();
            compute_s(slot * kTcTileBytes, qb);
            ring_release(slot);
          } else {
            mbar_wait(k_full(j), u_iter & 1u);
            compute_s(kTcOffK + j * kTcTileBytes, qb);
          }
          if (j == 0) ODB_ATRACE(qt_iter, 0);
          const int key0 = j * kTcBlk + cl;
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (key0 + 8 * jj + e < p.tokens) {
                mx0 = fmaxf(mx0, s[4 * jj + e]);
                mx1 = fmaxf(mx1, s[4 * jj + 2 + e]);
              }
            }
          }
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mc0 = mx0 * c, mc1 = mx1 * c;
        ODB_ATRACE(qt_iter, 1);
        // ---- pass 2: P = exp2(s*c - m*c) -> bf16 A operand, fp32 row sum, O += P V
        float o[32];
        float l0 = 0.f, l1 = 0.f;
        for (int j = 0; j < nblk; ++j) {
          if constexpr (STREAM) {
            const uint32_t slot = ring_acquire();
            compute_s(slot * kTcTileBytes, qb);
            ring_release(slot);
          } else {
            compute_s(kTcOffK + j * kTcTileBytes, qb);
          }
          const int key0 = j * kTcBlk + cl;
          uint32_t a[32];
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            float p00 = fast_exp2_tc(fmaf(s[4 * jj + 0], c, -mc0));
            float p01 = fast_exp2_tc(fmaf(s[4 * jj + 1], c, -mc0));
            float p10 = fast_exp2_tc(fmaf(s[4 * jj + 2], c, -mc1));
            float p11 = fast_exp2_tc(fmaf(s[4 * jj + 3], c, -mc1));
            if (key0 + 8 * jj >= p.tokens) { p00 = 0.f; p10 = 0.f; }
            if (key0 + 8 * jj + 1 >= p.tokens) { p01 = 0.f; p11 = 0.f; }
            l0 += p00 + p01;
            l1 += p10 + p11;
            // 8-column block jj is half (jj & 1) of the 16-key slice jj / 2: registers {0, 1} or {2, 3} of that slice
            a[4 * (jj >> 1) + 2 * (jj & 1) + 0] = pack_bf16x2(p00, p01);
            a[4 * (jj >> 1) + 2 * (jj & 1) + 1] = pack_bf16x2(p10, p11);
          }
          uint32_t voff, vslot = 0;
          if constexpr (STREAM) {
            vslot = ring_acquire();
            voff = vslot * kTcTileBytes;
          } else {
            mbar_wait(v_full(j), u_iter & 1u);
            voff = kTcOffV + j * kTcTileBytes;
          }
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 8; ++kk)   // B = V_j rows 16 kk.. (MN-major: +16 rows = 2048 B)
            Wgmma<64>::rs<1>(o, a + 4 * kk, gmma_desc_sw128(sbase + voff + kk * 2048), (j | kk) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs<32>(o);
          if constexpr (STREAM) ring_release(vslot);
          if (!STREAM || j < kTcMaxBlocks) ODB_ATRACE(qt_iter, 2 + j);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(q_empty(qb));                 // this warp no longer reads the Q tile
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
        l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
        const int q0 = qt * kTcBlk + r0, q1 = q0 + 8;
        if (p.lse != nullptr && (lane & 3) == 0) {
          const long long base = ((long long)b * p.heads + h) * p.tokens;
          if (q0 < p.tokens) p.lse[base + q0] = mc0 + log2f(l0);
          if (q1 < p.tokens) p.lse[base + q1] = mc1 + log2f(l1);
        }
        ODB_ATRACE(qt_iter, 7);
        ODB_ATRACE(qt_iter, 8);
        // ---- epilogue: O / l -> bf16 -> global
        bf16* dst0 = p.out + ((long long)b * p.tokens + q0) * (p.heads * 64) + h * 64 + cl;
        bf16* dst1 = dst0 + 8LL * (p.heads * 64);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          if (q0 < p.tokens)
            *reinterpret_cast<uint32_t*>(dst0 + 8 * jj) = pack_bf16x2(o[4 * jj] * inv0, o[4 * jj + 1] * inv0);
          if (q1 < p.tokens)
            *reinterpret_cast<uint32_t*>(dst1 + 8 * jj) = pack_bf16x2(o[4 * jj + 2] * inv1, o[4 * jj + 3] * inv1);
        }
        ODB_ATRACE(qt_iter, 9);
      }
      if constexpr (!STREAM) {
        __syncwarp();
        if (lane == 0) mbar_arrive(kv_empty);                    // K / V of this unit are no longer read
      }
    }
  }
}

}  // namespace odb

using namespace odb;

extern "C" int odb_attention(const void* qkv, void* out, float* lse, int32_t b, int32_t tokens, int32_t heads,
                             float scale, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!qkv || !out || b < 1 || heads < 1 || tokens < 1)
    return fail(ODB_ERR_INVALID, "attention: bad argument");
  if (tokens > kTcStreamMaxTokens) return fail(ODB_ERR_UNSUPPORTED, "attention: at most 4097 tokens");
  const bool stream_kv = tokens > kTcBlk * kTcMaxBlocks;   // K / V no longer fit in shared memory
  const long long units = (long long)b * heads;
  const long long items = stream_kv ? units * ((tokens + kTcBlk - 1) / kTcBlk) : units;
  if (items > 0x7fffffffLL) return fail(ODB_ERR_UNSUPPORTED, "attention: too many (image, head, query tile) items");
  if (reinterpret_cast<uintptr_t>(qkv) & 15u) return fail(ODB_ERR_INVALID, "attention: qkv must be 16-byte aligned");
  AttnTcParams p;
  memset(&p, 0, sizeof(p));
  {
    cuuint64_t dims[4] = {64, (cuuint64_t)(3 * heads), (cuuint64_t)tokens, (cuuint64_t)b};
    cuuint64_t strides[3] = {128, (cuuint64_t)(3 * heads) * 128, (cuuint64_t)tokens * (3 * heads) * 128};
    cuuint32_t box[4] = {64, 1, (cuuint32_t)kTcBlk, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    int rc = encode_tiled(&p.qkv_map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(qkv), dims,
                          strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  p.out = static_cast<bf16*>(out);
  p.lse = lse;
  p.tokens = tokens; p.heads = heads; p.batch = b;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.trace = debug_trace();
  static bool configured[2][kMaxDevices] = {};
  const int dev_ = current_device();
  const auto kernel = stream_kv ? attention_tc_kernel<true> : attention_tc_kernel<false>;
  if (!configured[stream_kv][dev_]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmemBytes);
    if (e != cudaSuccess) return fail_cuda(e, "attention: cudaFuncSetAttribute");
    configured[stream_kv][dev_] = true;
  }
  const int grid = items < num_sms() ? (int)items : num_sms();
  cudaError_t le = launch_pdl(kernel, dim3(grid), dim3(kTcThreads), kTcSmemBytes, stream, p);
  count_launch();
  if (le != cudaSuccess) return fail_cuda(le, "attention_tc: launch");
  return check_launch("attention_tc");
}
