// Implicit-GEMM convolution / linear layer for sm_90a: TMA -> shared memory -> wgmma -> registers
// -> fused epilogue -> TMA store.  One persistent CTA per SM, warp-specialised:
//   warpgroup 0     TMA producer (one lane)
//   warpgroups 1-2  consumers: each issues the wgmma of 64 of the 128 tile rows, then all eight warps run the
//                   epilogue (accumulator chunk -> shared memory -> one row per thread -> bias/act/residual
//                   -> bf16 -> swizzled smem -> TMA store), two warps per 32-row quarter, each owning 32 of
//                   the 64 columns of a chunk (EPI_BIAS_RES_F32: each thread adds its accumulator fragment
//                   into the staged fp32 residual instead)
//
// The A operand of the GEMM (rows = output pixels, K = taps x input channels) is never
// materialised: each K block is a 4-D TMA box {64 ch, tile_w, tile_h, 1} of the channels-last
// input, shifted by the tap offset; out-of-bounds rows/columns are zero-filled by the TMA unit,
// which is exactly the convolution zero padding.  The box lands in shared memory as dense
// 128-byte rows with the 128B swizzle, i.e. directly in the canonical K-major wgmma operand layout.
//
// What this replaces in the reference is listed in include/omnidata_b200.h (odb_conv_gemm).
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"
#include "host_util.h"
#include "../../include/omnidata_b200.h"

namespace odb {

constexpr int kTileRows = 128;                 // two wgmma M = 64 halves
constexpr int kKBlock = 64;                    // bf16 elements per K block = one 128B swizzle row
constexpr int kABytes = kTileRows * 128;       // 16 KiB per stage
constexpr int kStagingBytes = kTileRows * 128; // one 128 x 64 bf16 output chunk
constexpr int kNumThreads = 384;  // warpgroup 0 TMA, warpgroups 1-2 MMA + epilogue
constexpr int kEpiThreads = 256;
constexpr int kConsumerWarps = 8;

struct ConvGemmParams {
  CUtensorMap a_map[ODB_MAX_VIEWS];
  CUtensorMap b_map;
  CUtensorMap out_map;
  CUtensorMap out2_map;
  int num_taps;
  int kb_per_tap;
  int8_t tap_view[12];
  int8_t tap_dx[12];
  int8_t tap_dy[12];
  int tiles_n, tiles_x, tiles_y, tiles_b;
  int tile_w, tile_h;
  int out_w, out_h, out_b, n_total;
  const float* bias;
  long long bias_sb;
  const bf16* residual;
  long long res_sx, res_sy, res_sb;
  int act;
  int has_out2;
  int out2_gelu;       // out2 = gelu(value) instead of relu(value)
  const float* head_w;
  const float* head_b;
  int head_c;
  int head_relu;
  float* head_out;
  int halo_w;          // HALO mode: tile_w + 2 (row pitch of the halo tile), else 0
  int a_stages;        // HALO + HEAD (resident weights): halo ring depth and stage size chosen by the host
  int a_stage_bytes;
  float* gn_partial;   // optional GroupNorm partial sums, [b][tiles_y*tiles_x][4 quadrants][groups][2]
  int gn_cpg;          // channels per group (2..32, power of two)
  int gn_groups;
  CUtensorMap res_map;        // EPI_BIAS_RES: the residual, boxed like out_map
  unsigned long long* trace;  // diagnostics (odb_debug_conv_trace): kTraceSlots globaltimer stamps per CTA
};

// Parameters of the e4m3 instances (odb_conv_gemm_scaled).  `trace` is hidden by a null constant: the diagnostics
// trace is compiled out of these instances, whose bookkeeping would not fit beside the accumulator without spilling.
struct ConvGemmParamsFp8 : ConvGemmParams {
  const float* row_scale;     // fp32 [rows]: the A operand's per-row dequantisation scale
  const float* col_scale;     // fp32 [n]: the weight's per-output-channel dequantisation scale
  static constexpr unsigned long long* trace = nullptr;
};

// trace slots per CTA: 0 prologue done, 1 dependency wait done, 2 kernel end, 3 tiles of this CTA;
// per tile i < kTraceTiles at 8 + 5 i: MMA start, first stage full, accumulator complete, epilogue start, epilogue end
constexpr int kTraceTiles = 24;
ODB_DEVINL unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define ODB_TRACE(slot)                                                                      \
  do {                                                                                       \
    if (p.trace != nullptr) p.trace[static_cast<long long>(blockIdx.x) * kTraceSlots + (slot)] = global_ns(); \
  } while (0)
#define ODB_TRACE_TILE(i, k)                                   \
  do {                                                         \
    if (p.trace != nullptr && (i) < kTraceTiles) ODB_TRACE(8 + 5 * static_cast<int>(i) + (k)); \
  } while (0)

// Epilogue specialisations.  EPI_GENERIC handles every flag combination at run time (GroupNorm
// statistics, relu copy, residual with arbitrary strides / batch broadcast, missing bias).  The
// others are straight-line bodies for the combinations that carry the ViT blocks and most decoder
// convolutions: ~4x fewer instructions per 64-column chunk, and (EPI_BIAS_RES) the residual fetched by TMA into the output
// staging slot a few chunks ahead instead of 1024 scattered 16-byte loads per chunk.
// EPI_BIAS_RES_F32: fp32 residual in, fp32 out (the ViT residual stream: attn.proj / mlp.fc2 / patch proj).  A
// 64-column chunk is two 128-row x 32-fp32 TMA boxes (128-byte swizzled rows), so a chunk occupies TWO 16 KiB staging
// units.  Each consumer thread adds its own accumulator fragment elements into the staged residual in place: this
// epilogue needs no accumulator chunk buffer, and the shared memory it frees holds one more operand stage.
enum : int { EPI_GENERIC = 0, EPI_BIAS = 1, EPI_BIAS_RELU = 2, EPI_BIAS_GELU = 3, EPI_BIAS_RES = 4, EPI_GN = 5,
             EPI_BIAS_RES_F32 = 6 };

// ---- GroupNorm partial statistics of one epilogue warp (32 rows x 32 columns of a tile):
// per-thread group sums over its row, then a transposing butterfly over the 32 lanes: V values are
// reduced with V-1 + (5 - log2 V) shuffles in a FIXED order (deterministic), value i ending on the
// lanes whose top log2(V) bits equal i.
template <int CPG>
ODB_DEVINL void gn_row_group_sums(const float* v, float* vals) {
  constexpr int NG = 32 / CPG;
#pragma unroll
  for (int g = 0; g < NG; ++g) {
    float sm = 0.f, sq = 0.f;
#pragma unroll
    for (int j = 0; j < CPG; ++j) {
      const float x = v[g * CPG + j];
      sm += x;
      sq = fmaf(x, x, sq);
    }
    vals[2 * g] = sm;
    vals[2 * g + 1] = sq;
  }
}
template <int V>
ODB_DEVINL void gn_lane_butterfly(float* vals, int lane) {
  int n = V;
#pragma unroll
  for (int sft = 16; sft >= 1; sft >>= 1) {
    if (n > 1) {
      const int half = n >> 1;
      const bool upper = (lane & sft) != 0;
#pragma unroll
      for (int i = 0; i < V / 2; ++i) {
        if (i < half) {
          const float send = upper ? vals[i] : vals[i + half];
          const float keep = upper ? vals[i + half] : vals[i];
          vals[i] = keep + __shfl_xor_sync(0xffffffffu, send, sft);
        }
      }
      n = half;
    } else {
      vals[0] += __shfl_xor_sync(0xffffffffu, vals[0], sft);
    }
  }
}
template <int CPG>
ODB_DEVINL void gn_warp_partials(const float* v, int lane, float* dst /* [groups*2] at group gidx0 */) {
  constexpr int V = 2 * (32 / CPG);
  constexpr int LOGV = V == 32 ? 5 : V == 16 ? 4 : V == 8 ? 3 : V == 4 ? 2 : 1;
  float vals[V];
  gn_row_group_sums<CPG>(v, vals);
  gn_lane_butterfly<V>(vals, lane);
  if ((lane & ((1 << (5 - LOGV)) - 1)) == 0) dst[lane >> (5 - LOGV)] = vals[0];
}

// HALO = true (3x3 stride-1 convolutions): instead of nine shifted 128-row boxes per K block, ONE
// halo box {64 ch, tile_w + 2, tile_h + 2} is loaded per K block into its own ring and the nine taps
// are nine wgmma descriptors into it (start address shifted by whole 128-byte rows; the operand
// swizzle is address-based, so no base-offset correction is needed).  Accumulator row r is halo position
// (r / (tile_w+2), r % (tile_w+2)); the two junk columns per halo row are masked in the epilogue.
// L2 -> smem traffic for A drops from 9 x 16 KiB to <= 49 KiB per K block.  The weights keep their
// own (tap, K block) ring.
constexpr int kHaloAutoMaxN = 0;             // per-tap boxes (deeper ring) are the default, halo stays opt-in
constexpr int kHaloStageBytes = 49 * 1024;   // >= 390 rows x 128 B (tile_w = 128, tile_h = 1)

// HALO + HEAD (the DPT head's 128 -> 32 convolution at full resolution): the whole weight matrix
// (<= 18 K blocks x 32 rows = 72 KiB) stays resident in shared memory for the lifetime of the CTA and
// only input halos stream through a (run-time sized) ring.  Without this the layer re-reads its
// weights for every 128-pixel tile and its input nine times.
constexpr int kResidentBTiles = 18;
constexpr int kMaxAStages = 8;
constexpr int kHaloAreaBytes = 2 * kHaloStageBytes;

// The accumulator lives in the registers of the two consumer warpgroups (64 rows each).  The epilogue works on one
// accumulator row per thread, so each chunk of up to 64 columns is handed over through an fp32 buffer in shared
// memory: row pitch W + 4 floats (16-byte aligned rows, conflict-free row reads).
template <int BLOCK_N>
struct AccChunk {
  static constexpr int kCols = BLOCK_N < 64 ? BLOCK_N : 64;
  static constexpr int kPitch = kCols + 4;
  static constexpr int kBytes = kTileRows * kPitch * 4;
};

// ACC_BUF = false (EPI_BIAS_RES_F32): no accumulator chunk buffer
template <int BLOCK_N, int STAGES, int NSTAGING, bool HALO, bool HEAD, bool ACC_BUF>
struct SmemPlan {
  static constexpr bool kBResident = HALO && HEAD;
  static constexpr int kBBytes = BLOCK_N * 128;
  static constexpr int kAStages = HALO ? 2 : STAGES;
  static constexpr int kAStageBytes = HALO ? kHaloStageBytes : kABytes;
  static constexpr int kAOff = 0;
  static constexpr int kBOff = kAStages * kAStageBytes;
  static constexpr int kCOff = kBOff + (kBResident ? kResidentBTiles : STAGES) * kBBytes;
  static constexpr int kAccOff = kCOff + NSTAGING * kStagingBytes;
  static constexpr int kBarOff = kAccOff + (ACC_BUF ? AccChunk<BLOCK_N>::kBytes : 0);
  // full[STAGES], empty[STAGES], a_full[8], a_empty[8], res_full[4], b_resident
  static constexpr int kBarBytes = (2 * STAGES + 2 * kMaxAStages + 4 + 1) * 8;
  static constexpr int kTotal = kBarOff + kBarBytes + 1024;  // +1024: manual 1 KiB alignment
  static_assert(kTotal <= 232448, "shared memory plan exceeds 227 KiB");
};

// ---- FP8 epilogue pieces (conv_gemm_kernel<..., FP8 = true>).  The scaled GEMM takes [rows][C] operands (h = b = 1):
// tile row r is output row x0 + r; rows outside the output get scale 0.
ODB_DEVINL float fp8_row_scale(const ConvGemmParamsFp8& p, int x0, int r) {
  return r < p.tile_w && x0 + r < p.out_w ? __ldg(p.row_scale + x0 + r) : 0.f;
}
// v[j] = src[j] * (sa * cs[j]) + b[j] for the 32 staged accumulator values of one row (the row-per-thread epilogues).
// The scale products are formed in v first, so that the column scales and the bias are never in registers together
// beside the accumulator columns still to be staged.
ODB_DEVINL void fp8_read_row_scaled(const float* src_row, const float* b, const float* cs, float sa, float* v) {
  const float4* src = reinterpret_cast<const float4*>(src_row);
  const float4* bp = reinterpret_cast<const float4*>(b);
  const float4* sp = reinterpret_cast<const float4*>(cs);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 s4 = __ldg(sp + j);
    v[4 * j + 0] = sa * s4.x; v[4 * j + 1] = sa * s4.y; v[4 * j + 2] = sa * s4.z; v[4 * j + 3] = sa * s4.w;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 q = src[j];
    const float4 b4 = __ldg(bp + j);
    v[4 * j + 0] = fmaf(q.x, v[4 * j + 0], b4.x); v[4 * j + 1] = fmaf(q.y, v[4 * j + 1], b4.y);
    v[4 * j + 2] = fmaf(q.z, v[4 * j + 2], b4.z); v[4 * j + 3] = fmaf(q.w, v[4 * j + 3], b4.w);
  }
}
// EPI_BIAS_RES_F32 with e4m3 operands: as the kernel's add_frag_res_f32 (same fragment rows, columns and swizzled
// staging addresses), adding res + (acc * (sa[h] * cs[c]) + bias[c]); sa[h] = the scales of rows r and r + 8.
template <int C0>
ODB_DEVINL void fp8_add_frag_res_f32(const float* dacc, uint32_t buf, const float* b, const float* cs, const float* sa,
                                     int r, int lane) {
  const uint32_t rbase = buf + static_cast<uint32_t>(r) * 128u + (static_cast<uint32_t>(lane & 1) << 3);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float2 b2 = __ldg(reinterpret_cast<const float2*>(b + C0 + 8 * j + 2 * (lane & 3)));
    const float2 s2 = __ldg(reinterpret_cast<const float2*>(cs + C0 + 8 * j + 2 * (lane & 3)));
    const uint32_t unit = static_cast<uint32_t>(2 * (j & 3) + ((lane & 3) >> 1));
    const uint32_t addr = rbase + static_cast<uint32_t>(j >> 2) * kStagingBytes + ((unit ^ (r & 7)) << 4);
    const float* a = dacc + 4 * (C0 / 8 + j);
#pragma unroll
    for (int h = 0; h < 2; ++h) {                   // rows r, r + 8
      const uint32_t ad = addr + h * 8u * 128u;
      float q0, q1;
      asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(q0), "=f"(q1) : "r"(ad) : "memory");
      q0 += fmaf(a[2 * h], sa[h] * s2.x, b2.x);
      q1 += fmaf(a[2 * h + 1], sa[h] * s2.y, b2.y);
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(ad), "f"(q0), "f"(q1) : "memory");
    }
  }
}
template <int BLOCK_N>
ODB_DEVINL void fp8_add_frag_res_f32_rt(int c, const float* dacc, uint32_t buf, const float* b, const float* cs,
                                        const float* sa, int r, int lane) {   // run-time chunk index
  if (c == 0) fp8_add_frag_res_f32<0>(dacc, buf, b, cs, sa, r, lane);
  if constexpr (BLOCK_N > 64) {
    if (c == 1) fp8_add_frag_res_f32<64>(dacc, buf, b, cs, sa, r, lane);
  }
  if constexpr (BLOCK_N > 128) {
    if (c == 2) fp8_add_frag_res_f32<128>(dacc, buf, b, cs, sa, r, lane);
    else if (c == 3) fp8_add_frag_res_f32<192>(dacc, buf, b, cs, sa, r, lane);
  }
}

// The row scales of one thread's rows for a tile, read once per tile: x = the row of the row-per-thread epilogues, or
// (x, y) = the fragment rows r and r + 8 (EPI_BIAS_RES_F32).  bf16 instances get an empty object.
struct Fp8NoScale {};
template <bool FP8, bool F32, typename P>
ODB_DEVINL auto fp8_tile_scales(const P& p, int x0, int row, int frag_row) {
  if constexpr (!FP8) {
    return Fp8NoScale{};
  } else if constexpr (F32) {
    return make_float2(fp8_row_scale(p, x0, frag_row), fp8_row_scale(p, x0, frag_row + 8));
  } else {
    return make_float2(fp8_row_scale(p, x0, row), 0.f);
  }
}

// K elements per 128-byte operand row: 64 bf16, 128 e4m3.  (A class constant: a constexpr local in the kernel
// body changes the register allocation of the bf16 instances.)
template <bool FP8> struct KBlock { static constexpr int value = FP8 ? 2 * kKBlock : kKBlock; };

// Named barriers of the consumer warpgroups (barrier 0 is __syncthreads)
constexpr uint32_t kBarEpilogue = 1;   // staging slot hand-over to the TMA store
constexpr uint32_t kBarAccChunk = 2;   // accumulator chunk buffer written / read

// PAIR = true: the two CTAs of a cluster take two vertically adjacent 128-row M tiles against the same N tile.  Each
// CTA TMA-loads its own A rows and HALF of the B rows, multicast into both CTAs, so the pair reads each weight tile
// from L2 once.  A B stage is refilled only after the consumers of BOTH CTAs released it (each consumer warp arrives
// on the empty barrier of both CTAs).  The MMAs and their order are those of the single-CTA kernel.
//
// FP8 = true (odb_conv_gemm_scaled, the ViT blocks' linear layers in the fp8 inference mode): e4m3 operands.  A
// 128-byte swizzled row holds 128 e4m3 elements instead of 64 bf16 ones, so a stage has the same bytes and layout and
// carries twice the K; each of its four wgmma steps is one m64nNk32 e4m3 instruction (32 bytes, as k16 bf16).  The
// epilogue dequantises before the bias: v = acc * (row_scale[r] * col_scale[c]) + bias[c] (one fma), then the
// layer's epilogue as in bf16.  1-tap linear layers with EPI_BIAS / EPI_BIAS_GELU / EPI_BIAS_RES_F32 only.  Every
// FP8 difference sits in an `if constexpr (FP8)` branch: the FP8 = false instances are the code they were before.
template <int BLOCK_N, int STAGES, int NSTAGING, bool HEAD, bool HALO, bool PAIR, int EPI = EPI_GENERIC,
          bool FP8 = false>
__global__ void __launch_bounds__(kNumThreads, 1)
conv_gemm_kernel(const __grid_constant__ std::conditional_t<FP8, ConvGemmParamsFp8, ConvGemmParams> p) {
  static_assert(EPI == EPI_GENERIC || (!HEAD && !HALO && NSTAGING >= 2), "fast epilogues: plain tiles only");
  static_assert(!PAIR || !HEAD, "CTA pairs: no head tail");
  static_assert(EPI != EPI_BIAS_RES_F32 || NSTAGING >= 4, "fp32 epilogue: two staging slots of two 16 KiB units");
  static_assert(!FP8 || (!PAIR && (EPI == EPI_BIAS || EPI == EPI_BIAS_GELU || EPI == EPI_BIAS_RES_F32)),
                "e4m3 operands: single-CTA linear layers with a bias, bias + GELU or fp32-residual epilogue");
  using Plan = SmemPlan<BLOCK_N, STAGES, NSTAGING, HALO, HEAD, EPI != EPI_BIAS_RES_F32>;
  using Acc = AccChunk<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + Plan::kBarOff;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  auto afull_bar = [&](int a) { return bar_base + 8u * (2 * STAGES + a); };
  auto aempty_bar = [&](int a) { return bar_base + 8u * (2 * STAGES + kMaxAStages + a); };
  auto rfull_bar = [&](int a) { return bar_base + 8u * (2 * STAGES + 2 * kMaxAStages + a); };
  const uint32_t bres_bar = bar_base + 8u * (2 * STAGES + 2 * kMaxAStages + 4);
  float* acc_buf = reinterpret_cast<float*>(smem_raw + (smem_base + Plan::kAccOff - smem_u32(smem_raw)));
  // halo ring geometry: compile-time, except for the resident-weights head variant
  const int a_stages = Plan::kBResident ? p.a_stages : Plan::kAStages;
  const uint32_t a_stage_bytes = Plan::kBResident ? static_cast<uint32_t>(p.a_stage_bytes)
                                                  : static_cast<uint32_t>(Plan::kAStageBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), (PAIR ? 2 : 1) * kConsumerWarps);    // one arrive per consumer warp (of both CTAs)
    }
    for (int a = 0; a < kMaxAStages; ++a) {
      mbar_init(afull_bar(a), 1);
      mbar_init(aempty_bar(a), kConsumerWarps);
    }
    for (int a = 0; a < 4; ++a) mbar_init(rfull_bar(a), 1);
    mbar_init(bres_bar, 1);
    mbar_fence_init();
    if (EPI == EPI_BIAS_RES || EPI == EPI_BIAS_RES_F32) tma_prefetch_desc(&p.res_map);
    for (int v = 0; v < ODB_MAX_VIEWS; ++v) tma_prefetch_desc(&p.a_map[v]);
    tma_prefetch_desc(&p.b_map);
    if (!HEAD) tma_prefetch_desc(&p.out_map);
  }
  if constexpr (PAIR) cluster_sync_all(); else __syncthreads();   // the peer's barriers exist before any multicast
  if (threadIdx.x == 0) ODB_TRACE(0);
  // everything above overlapped the tail of the previous kernel (programmatic dependent launch)
  grid_dep_wait();
  grid_dep_launch();
  if (threadIdx.x == 0) ODB_TRACE(1);

  // work units: (n tile, m tile) for a single CTA, (n tile, pair of m tiles) for a CTA pair
  const uint32_t cta_rank = PAIR ? cluster_ctarank() : 0u;
  // the unit schedule, computed by each role after its setmaxnreg: values live across the role split must fit the
  // producer's 40 registers, and ptxas keeps them in local memory instead
  auto m_tiles = [&]() { return p.tiles_x * p.tiles_y * p.tiles_b; };
  auto schedule = [&](int& total_tiles, int& unit0, int& unit_stride) {
    total_tiles = p.tiles_n * (PAIR ? (m_tiles() + 1) / 2 : m_tiles());
    unit0 = PAIR ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
    unit_stride = PAIR ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);
  };
  const int num_kb = p.num_taps * p.kb_per_tap;
  const uint32_t a_bytes =
      HALO ? static_cast<uint32_t>(p.halo_w * (p.tile_h + 2)) * 128u
           : static_cast<uint32_t>(p.tile_w * p.tile_h) * 128u;
  // unit -> (tn, tx, ty, tb); an M tile past the end (odd tile count, second CTA of a pair) maps to batch index
  // tiles_b: every TMA box is then out of bounds (zero fill on load, nothing stored)
  auto decode = [&](int unit, int& tn, int& tx, int& ty, int& tb) {
    tn = unit % p.tiles_n;
    int m = unit / p.tiles_n;
    if (PAIR) m = 2 * m + static_cast<int>(cta_rank);
    if (m >= m_tiles()) { tx = 0; ty = 0; tb = p.tiles_b; return; }
    tx = m % p.tiles_x; m /= p.tiles_x;
    ty = m % p.tiles_y;
    tb = m / p.tiles_y;
  };

  // B tile of K coordinate kcoord, N tile tn into stage `stage` (a pair: this CTA's half, multicast to both CTAs)
  auto load_b = [&](int stage, int kcoord, int tn) {
    const uint32_t sb = smem_base + Plan::kBOff + stage * Plan::kBBytes;
    if constexpr (PAIR)
      tma_load_2d_multicast(sb + cta_rank * (Plan::kBBytes / 2), &p.b_map, full_bar(stage), kcoord,
                            tn * BLOCK_N + static_cast<int>(cta_rank) * (BLOCK_N / 2), 0x3);
    else
      tma_load_2d(sb, &p.b_map, full_bar(stage), kcoord, tn * BLOCK_N);
  };
  // a consumer warp is done with B stage `stage` (lane 0)
  const uint32_t peer_empty0 = PAIR ? mapa_shared(empty_bar(0), cta_rank ^ 1u) : 0u;
  auto release_b = [&](int stage) {
    mbar_arrive(empty_bar(stage));
    if constexpr (PAIR) mbar_arrive_cluster(peer_empty0 + 8u * stage);
  };

  if (warp < 4) {
    // ------------------------------------------------------------ TMA producer (warpgroup 0, one lane)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    int total_tiles, unit0, unit_stride;
    schedule(total_tiles, unit0, unit_stride);
    if (warp == 0 && lane == 0) {
      int stage = 0, astage = 0;
      uint32_t phase = 0, aphase = 0;
      for (int tile = unit0; tile < total_tiles; tile += unit_stride) {
        int tn, tx, ty, tb;
        decode(tile, tn, tx, ty, tb);
        const int x0 = tx * p.tile_w, y0 = ty * p.tile_h;
        if constexpr (Plan::kBResident) {
          if (tile == unit0) {
            // the whole weight matrix, once (K blocks in (tap, kb) order, 32 rows each)
            mbar_expect_tx(bres_bar, static_cast<uint32_t>(num_kb) * Plan::kBBytes);
            for (int t = 0; t < num_kb; ++t)
              tma_load_2d(smem_base + Plan::kBOff + t * Plan::kBBytes, &p.b_map, bres_bar, t * kKBlock, 0);
          }
          for (int kb = 0; kb < p.kb_per_tap; ++kb) {
            mbar_wait(aempty_bar(astage), aphase ^ 1u);
            mbar_expect_tx(afull_bar(astage), a_bytes);
            tma_load_4d(smem_base + Plan::kAOff + astage * a_stage_bytes, &p.a_map[0], afull_bar(astage),
                        kb * kKBlock, x0 - 1, y0 - 1, tb);
            if (++astage == a_stages) { astage = 0; aphase ^= 1u; }
          }
        } else if constexpr (HALO) {
          for (int kb = 0; kb < p.kb_per_tap; ++kb) {
            // ---- one halo box of the input per K block ...
            mbar_wait(aempty_bar(astage), aphase ^ 1u);
            mbar_expect_tx(afull_bar(astage), a_bytes);
            tma_load_4d(smem_base + Plan::kAOff + astage * Plan::kAStageBytes, &p.a_map[0], afull_bar(astage),
                        kb * kKBlock, x0 - 1, y0 - 1, tb);
            if (++astage == Plan::kAStages) { astage = 0; aphase ^= 1u; }
            // ---- ... and the nine weight tiles of that K block
            for (int tap = 0; tap < p.num_taps; ++tap) {
              mbar_wait(empty_bar(stage), phase ^ 1u);
              mbar_expect_tx(full_bar(stage), Plan::kBBytes);
              load_b(stage, (tap * p.kb_per_tap + kb) * kKBlock, tn);
              if (++stage == STAGES) { stage = 0; phase ^= 1u; }
            }
          }
        } else {
          for (int tap = 0; tap < p.num_taps; ++tap) {
            const CUtensorMap* amap = &p.a_map[p.tap_view[tap]];
            const int ax = x0 + p.tap_dx[tap], ay = y0 + p.tap_dy[tap];
            for (int kb = 0; kb < p.kb_per_tap; ++kb) {
              mbar_wait(empty_bar(stage), phase ^ 1u);
              mbar_expect_tx(full_bar(stage), a_bytes + Plan::kBBytes);
              tma_load_4d(smem_base + Plan::kAOff + stage * kABytes, amap, full_bar(stage), kb * KBlock<FP8>::value, ax, ay, tb);
              load_b(stage, (tap * p.kb_per_tap + kb) * KBlock<FP8>::value, tn);
              if (++stage == STAGES) { stage = 0; phase ^= 1u; }
            }
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers (warpgroups 1, 2): wgmma + epilogue
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    int total_tiles, unit0, unit_stride;
    schedule(total_tiles, unit0, unit_stride);
    const int wg = (warp - 4) >> 2;                              // 64-row half of the 128-row tile
    const uint32_t a_half = static_cast<uint32_t>(wg) * 64u * 128u;
    float dacc[BLOCK_N / 2];
    int stage = 0, astage = 0;
    uint32_t phase = 0, aphase = 0;
    uint32_t tap_off[9];                   // resident-weights halo kernel: tap shift in bytes
#pragma unroll
    for (int t = 0; t < 9; ++t)
      tap_off[t] = Plan::kBResident ? static_cast<uint32_t>((p.tap_dy[t] + 1) * p.halo_w + (p.tap_dx[t] + 1)) * 128u : 0u;
    // the MMA half of a tile: the accumulator of tile `iter` complete in `acc`
    auto mainloop = [&](uint32_t iter) {
      if (lane == 0 && warp == 4) ODB_TRACE_TILE(iter, 0);
      // The first wgmma of a tile ignores the accumulator (scale-d 0), but its asm operands are read-write: without
      // this the previous tile's accumulator registers count as live through that tile's whole epilogue, and the
      // 256-wide epilogues spill.  Overwriting them here frees each chunk's registers once it has been staged.
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) dacc[i] = 0.f;
      if constexpr (Plan::kBResident) {
        if (iter == 0) mbar_wait(bres_bar, 0);
        const uint32_t b_tap_step = static_cast<uint32_t>(p.kb_per_tap) * Plan::kBBytes;
        for (int kb = 0; kb < p.kb_per_tap; ++kb) {
          mbar_wait(afull_bar(astage), aphase);
          const uint32_t a0 = smem_base + Plan::kAOff + astage * a_stage_bytes + a_half;
          const uint32_t b0 = smem_base + Plan::kBOff + kb * Plan::kBBytes;
          wgmma_fence();
#pragma unroll
          for (int tap = 0; tap < 9; ++tap) {
            const uint64_t adesc = gmma_desc_sw128(a0 + tap_off[tap]);
            const uint64_t bdesc = gmma_desc_sw128(b0 + static_cast<uint32_t>(tap) * b_tap_step);
#pragma unroll
            for (int k = 0; k < kKBlock / 16; ++k)
              Wgmma<BLOCK_N>::template ss<0, 0>(dacc, adesc + 2u * k, bdesc + 2u * k, (kb | tap | k) != 0 ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          if (lane == 0) mbar_arrive(aempty_bar(astage));     // the halo stage is free
          if (++astage == a_stages) { astage = 0; aphase ^= 1u; }
        }
      } else if constexpr (HALO) {
        for (int kb = 0; kb < p.kb_per_tap; ++kb) {
          mbar_wait(afull_bar(astage), aphase);
          const uint32_t a_base = smem_base + Plan::kAOff + astage * Plan::kAStageBytes + a_half;
          for (int tap = 0; tap < p.num_taps; ++tap) {
            mbar_wait(full_bar(stage), phase);
            // tap (dy, dx) = the halo tile shifted by whole 128-byte rows
            const uint64_t adesc = gmma_desc_sw128(
                a_base + static_cast<uint32_t>((p.tap_dy[tap] + 1) * p.halo_w + (p.tap_dx[tap] + 1)) * 128u);
            const uint64_t bdesc = gmma_desc_sw128(smem_base + Plan::kBOff + stage * Plan::kBBytes);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kKBlock / 16; ++k)
              Wgmma<BLOCK_N>::template ss<0, 0>(dacc, adesc + 2u * k, bdesc + 2u * k, (kb | tap | k) != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            if (lane == 0) release_b(stage);
            if (++stage == STAGES) { stage = 0; phase ^= 1u; }
          }
          if (lane == 0) mbar_arrive(aempty_bar(astage));
          if (++astage == Plan::kAStages) { astage = 0; aphase ^= 1u; }
        }
      } else {
        // one wgmma group in flight: the stage of K block kb-1 is released once group kb has been issued
        int prev = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(full_bar(stage), phase);
          if (kb == 0 && lane == 0 && warp == 4) ODB_TRACE_TILE(iter, 1);
          const uint64_t adesc = gmma_desc_sw128(smem_base + Plan::kAOff + stage * kABytes + a_half);
          const uint64_t bdesc = gmma_desc_sw128(smem_base + Plan::kBOff + stage * Plan::kBBytes);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kKBlock / 16; ++k) {  // +32 bytes (= 2 in 16-byte units) per K step of 16 (FP8: 32)
            if constexpr (FP8)
              WgmmaE4M3<BLOCK_N>::ss(dacc, adesc + 2u * k, bdesc + 2u * k, (kb | k) != 0 ? 1u : 0u);
            else
              Wgmma<BLOCK_N>::template ss<0, 0>(dacc, adesc + 2u * k, bdesc + 2u * k, (kb | k) != 0 ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && lane == 0) release_b(prev);
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        if (prev >= 0 && lane == 0) release_b(prev);
      }
      wgmma_fence_regs<BLOCK_N / 2>(dacc);
      if (lane == 0 && warp == 4) ODB_TRACE_TILE(iter, 2);
    };
    // columns [C0, C0 + kCols) of the accumulator -> acc_buf; every consumer thread then reads its own row
    auto stage_chunk = [&](auto c0_tag) {
      constexpr int C0 = decltype(c0_tag)::value;
      named_bar_sync(kBarAccChunk, kEpiThreads);        // the previous chunk has been read
      wgmma_frag_to_smem<BLOCK_N, C0, Acc::kCols>(dacc, acc_buf, Acc::kPitch, wg * 64);
      named_bar_sync(kBarAccChunk, kEpiThreads);
    };
    auto stage_chunk_rt = [&](int c) {                  // run-time chunk index
      if constexpr (BLOCK_N <= 64) {
        stage_chunk(std::integral_constant<int, 0>{});
      } else {
        if (c == 0) stage_chunk(std::integral_constant<int, 0>{});
        else if (c == 1) stage_chunk(std::integral_constant<int, 64>{});
        if constexpr (BLOCK_N > 128) {
          if (c == 2) stage_chunk(std::integral_constant<int, 128>{});
          else if (c == 3) stage_chunk(std::integral_constant<int, 192>{});
        }
      }
    };
    // v[j] = accumulator (row, col + j) + b[j] for 32 columns (b == nullptr: + 0.f).  The bias is read four values at
    // a time after the chunk hand-over, so that beside the accumulator registers still to be staged only the 32 row
    // values and one float4 of bias are live: the 256-wide tiles then fit without spilling.
    auto read_row_bias = [&](int row, int col, const float* b, float* v) {
      const float4* src = reinterpret_cast<const float4*>(acc_buf + row * Acc::kPitch + col);
      const float4* bp = reinterpret_cast<const float4*>(b);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 q = src[j];
        const float4 b4 = b != nullptr ? __ldg(bp + j) : make_float4(0.f, 0.f, 0.f, 0.f);
        v[4 * j + 0] = q.x + b4.x; v[4 * j + 1] = q.y + b4.y;
        v[4 * j + 2] = q.z + b4.z; v[4 * j + 3] = q.w + b4.w;
      }
    };
    // EPI_BIAS_RES_F32: the accumulator columns [C0, C0 + 64) of this thread's fragment (rows r and r + 8 of its
    // warpgroup's 64-row half) added in place into the fp32 residual chunk staged at `buf`, two 32-column TMA boxes
    // of 128-byte rows whose 16-byte unit u sits at u ^ (row & 7).  The sum is res + (acc + bias), as the row
    // epilogues round it.  A quad covers 32 contiguous bytes of a row: 8-byte accesses.
    auto add_frag_res_f32 = [&](auto c0_tag, uint32_t buf, const float* b) {
      constexpr int C0 = decltype(c0_tag)::value;
      const int r = wg * 64 + 16 * (warp & 3) + (lane >> 2);
      const uint32_t rbase = buf + static_cast<uint32_t>(r) * 128u + (static_cast<uint32_t>(lane & 1) << 3);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 b2 = __ldg(reinterpret_cast<const float2*>(b + C0 + 8 * j + 2 * (lane & 3)));
        const uint32_t unit = static_cast<uint32_t>(2 * (j & 3) + ((lane & 3) >> 1));
        const uint32_t addr = rbase + static_cast<uint32_t>(j >> 2) * kStagingBytes + ((unit ^ (r & 7)) << 4);
        const float* a = dacc + 4 * (C0 / 8 + j);
#pragma unroll
        for (int h = 0; h < 2; ++h) {                   // rows r, r + 8
          const uint32_t ad = addr + h * 8u * 128u;
          float q0, q1;
          asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(q0), "=f"(q1) : "r"(ad) : "memory");
          q0 += a[2 * h] + b2.x;
          q1 += a[2 * h + 1] + b2.y;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(ad), "f"(q0), "f"(q1) : "memory");
        }
      }
    };
    auto add_frag_res_f32_rt = [&](int c, uint32_t buf, const float* b) {   // run-time chunk index
      if (c == 0) add_frag_res_f32(std::integral_constant<int, 0>{}, buf, b);
      if constexpr (BLOCK_N > 64) {
        if (c == 1) add_frag_res_f32(std::integral_constant<int, 64>{}, buf, b);
      }
      if constexpr (BLOCK_N > 128) {
        if (c == 2) add_frag_res_f32(std::integral_constant<int, 128>{}, buf, b);
        else if (c == 3) add_frag_res_f32(std::integral_constant<int, 192>{}, buf, b);
      }
    };
    // ------------------------------------------------------------ epilogue
    const int ew = warp - 4;               // epilogue warp 0..7
    const int quad = (ew + 2) & 3;         // 32-row quarter of the tile this warp owns
    const int half = ew >> 2;              // which 32 of the 64 chunk columns this warp owns
    const int row = quad * 32 + lane;      // accumulator row == pixel within the tile
    const bool store_leader = (ew == 0 && lane == 0);
    const int tw = p.tile_w;
    if constexpr (EPI != EPI_GENERIC) {
      // ---------------------------------------------------------- specialised epilogues
      constexpr int kChunks = BLOCK_N / 64;
      constexpr bool F32 = (EPI == EPI_BIAS_RES_F32);
      constexpr bool RES = (EPI == EPI_BIAS_RES || EPI == EPI_BIAS_RES_F32);
      constexpr int kSlotBytes = F32 ? 2 * kStagingBytes : kStagingBytes;
      constexpr int NS = F32 ? NSTAGING / 2 : NSTAGING;   // staging slots of one 128 x 64 chunk each
      constexpr int D = NS >= 4 ? NS / 2 : (NS >= 2 ? NS - 1 : 0);   // residual prefetch distance in chunks
      static_assert(!RES || NS >= 2, "residual epilogues need two staging slots");
      const int cofs = half * 32;
      const uint32_t rowoff = static_cast<uint32_t>(row) * 128u;
      uint32_t g = 0;                   // chunks this CTA has processed
      // residual loader (store leader): chunk ld_g of the CTA's static schedule -> slot ld_g % NS
      int ld_tile = unit0, ld_c = 0;
      uint32_t ld_g = 0;
      auto issue_res_load = [&]() {
        if (ld_tile < total_tiles) {
          int tn, tx, ty, tb;
          decode(ld_tile, tn, tx, ty, tb);
          const uint32_t slot = ld_g % NS;
          mbar_expect_tx(rfull_bar(slot), F32 ? 2u * a_bytes : a_bytes);
          tma_load_4d(smem_base + Plan::kCOff + slot * kSlotBytes, &p.res_map, rfull_bar(slot),
                      tn * BLOCK_N + ld_c * 64, tx * p.tile_w, ty * p.tile_h, tb);
          if constexpr (F32)
            tma_load_4d(smem_base + Plan::kCOff + slot * kSlotBytes + kStagingBytes, &p.res_map, rfull_bar(slot),
                        tn * BLOCK_N + ld_c * 64 + 32, tx * p.tile_w, ty * p.tile_h, tb);
          ++ld_g;
          if (++ld_c == kChunks) { ld_c = 0; ld_tile += unit_stride; }
        }
      };
      if (RES && store_leader) {
        for (int i = 0; i < D; ++i) issue_res_load();
      }
      uint32_t iter = 0;
      for (int tile = unit0; tile < total_tiles; tile += unit_stride, ++iter) {
        mainloop(iter);      // first: the per-tile values below need no registers beside the accumulator
        if (store_leader) ODB_TRACE_TILE(iter, 3);
        int tn, tx, ty, tb;
        decode(tile, tn, tx, ty, tb);
        const int x0 = tx * p.tile_w, y0 = ty * p.tile_h;
        const int n0 = tn * BLOCK_N;
        const float* bias_n0 = EPI == EPI_GN ? nullptr
                                             : p.bias + static_cast<long long>(tb < p.out_b ? tb : 0) * p.bias_sb + n0;
        const float* bias = EPI == EPI_GN ? nullptr : bias_n0 + cofs;
        // EPI_GN: rows of this thread that really exist (ragged tiles)
        const int gx = x0 + (row % p.tile_w), gy = y0 + (row / p.tile_w);
        const bool valid = row < p.tile_w * p.tile_h && gx < p.out_w && gy < p.out_h && tb < p.out_b;
        [[maybe_unused]] const auto sa = fp8_tile_scales<FP8, F32>(p, x0, row, wg * 64 + 16 * (warp & 3) + (lane >> 2));
#pragma unroll
        for (int c = 0; c < kChunks; ++c, ++g) {
          float v[32];
          if constexpr (!F32) {
            stage_chunk_rt(c);
            if constexpr (FP8)
              fp8_read_row_scaled(acc_buf + row * Acc::kPitch + cofs, bias + c * 64, p.col_scale + n0 + cofs + c * 64,
                                  sa.x, v);
            else
              read_row_bias(row, cofs, EPI == EPI_GN ? nullptr : bias + c * 64, v);
          }
          if constexpr (EPI == EPI_BIAS_GELU) {
#pragma unroll
            for (int j = 0; j < 16; ++j) gelu_erf_x2(v[2 * j], v[2 * j + 1]);
          } else if constexpr (EPI == EPI_BIAS_RELU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
          }
          const uint32_t slot = g % NS;
          const uint32_t buf = smem_base + Plan::kCOff + slot * kSlotBytes;
          if constexpr (F32) {
            mbar_wait(rfull_bar(slot), (g / NS) & 1u);
            if constexpr (FP8) {
              const int r = wg * 64 + 16 * (warp & 3) + (lane >> 2);      // the fragment rows r and r + 8
              const float sa2[2] = {sa.x, sa.y};
              fp8_add_frag_res_f32_rt<BLOCK_N>(c, dacc, buf, bias_n0, p.col_scale + n0, sa2, r, lane);
            } else {
              add_frag_res_f32_rt(c, buf, bias_n0);
            }
          } else {
          if constexpr (EPI == EPI_BIAS_RES) {
            // the residual rows of this chunk were TMA-loaded into the staging slot (same swizzled
            // layout as the output): read own 64 bytes, add, write the result back in place
            mbar_wait(rfull_bar(slot), (g / NS) & 1u);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint32_t addr = buf + rowoff + (static_cast<uint32_t>((half * 4 + j) ^ (row & 7)) << 4);
              uint32_t q0, q1, q2, q3;
              asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                           : "=r"(q0), "=r"(q1), "=r"(q2), "=r"(q3) : "r"(addr) : "memory");
              float2 t2;
              t2 = unpack_bf16x2(q0); v[8 * j + 0] += t2.x; v[8 * j + 1] += t2.y;
              t2 = unpack_bf16x2(q1); v[8 * j + 2] += t2.x; v[8 * j + 3] += t2.y;
              t2 = unpack_bf16x2(q2); v[8 * j + 4] += t2.x; v[8 * j + 5] += t2.y;
              t2 = unpack_bf16x2(q3); v[8 * j + 6] += t2.x; v[8 * j + 7] += t2.y;
            }
          }
          uint32_t packed[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) packed[j] = pack_bf16x2(v[2 * j], v[2 * j + 1]);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint32_t addr = buf + rowoff + (static_cast<uint32_t>((half * 4 + j) ^ (row & 7)) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(packed[4 * j]),
                         "r"(packed[4 * j + 1]), "r"(packed[4 * j + 2]), "r"(packed[4 * j + 3])
                         : "memory");
          }
          if constexpr (EPI == EPI_GN) {
            // fused GroupNorm statistics over the UNROUNDED fp32 accumulators (the reference normalises the fp32
            // conv output: timm GroupNormAct after StdConv2dSame); same order of operations as the generic
            // epilogue: bit-identical partial sums
            float rq[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) rq[j] = valid ? v[j] : 0.f;
            if (tb < p.out_b) {
              const int cpg = p.gn_cpg;
              float* dst = p.gn_partial +
                           ((((long long)tb * (p.tiles_x * p.tiles_y) + (ty * p.tiles_x + tx)) * 4 + quad) *
                                p.gn_groups + (n0 + c * 64 + cofs) / cpg) * 2;
              if (cpg == 2) gn_warp_partials<2>(rq, lane, dst);
              else if (cpg == 4) gn_warp_partials<4>(rq, lane, dst);
              else if (cpg == 8) gn_warp_partials<8>(rq, lane, dst);
              else if (cpg == 16) gn_warp_partials<16>(rq, lane, dst);
              else gn_warp_partials<32>(rq, lane, dst);
            }
          }
          }  // !F32
          fence_proxy_async_smem();
          // slot reuse without a residual: the store of chunk g+1-NS must have read its slot before any
          // thread passes this barrier and starts writing chunk g+1 (with a residual the TMA load of
          // chunk g+1, issued after that store was read, orders it)
          if (!RES && store_leader) tma_store_wait_read<(NS >= 2 ? NS - 2 : 0)>();
          named_bar_sync(kBarEpilogue, kEpiThreads);
          if (store_leader) {
            tma_store_4d(&p.out_map, buf, n0 + c * 64, x0, y0, tb);
            if constexpr (F32) tma_store_4d(&p.out_map, buf + kStagingBytes, n0 + c * 64 + 32, x0, y0, tb);
            tma_store_commit();
            if constexpr (RES) {
              tma_store_wait_read<NS - D>();     // the store of chunk g+D-NS has read its slot
              issue_res_load();                  // residual of chunk g+D -> that slot
            }
          }
        }
        if (store_leader) ODB_TRACE_TILE(iter, 4);
      }
      if (store_leader) tma_store_wait_all();
    } else {
    uint32_t iter = 0;
    uint32_t chunk_counter = 0;
    const int bufs_per_chunk = p.has_out2 ? 2 : 1;
    const int slots = NSTAGING > 0 ? NSTAGING / bufs_per_chunk : 1;

    for (int tile = unit0; tile < total_tiles; tile += unit_stride, ++iter) {
      mainloop(iter);
      if (store_leader) ODB_TRACE_TILE(iter, 3);
      // the row geometry is recomputed per tile: kept across the MMA loop it would not fit beside the accumulator
      const int rpitch = HALO ? p.halo_w : tw;            // accumulator rows per tile row
      const int ly = row / rpitch, lx = row - ly * rpitch;
      const bool row_in_tile = HALO ? (lx < tw && ly < p.tile_h) : (row < p.tile_w * p.tile_h);
      const int srow = HALO ? (row_in_tile ? ly * tw + lx : 0) : row;   // dense row in the store staging tile
      int tn, tx, ty, tb;
      decode(tile, tn, tx, ty, tb);
      const int x0 = tx * p.tile_w, y0 = ty * p.tile_h;
      const int x = x0 + lx, y = y0 + ly;
      const bool valid = row_in_tile && x < p.out_w && y < p.out_h && tb < p.out_b;

      if constexpr (HEAD) {
        // ---- DPT head tail: relu(conv + bias) (32 ch) -> 1x1 conv to head_c channels -> relu -> NCHW fp32
        stage_chunk_rt(0);
        float v[32];
        read_row_bias(row, 0, p.bias, v);
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
        if (valid) {
          for (int k = half; k < p.head_c; k += 2) {   // the two warp halves share the output channels
            const float4* wk = reinterpret_cast<const float4*>(p.head_w + k * 32);
            float o0 = __ldg(p.head_b + k), o1 = 0.f, o2 = 0.f, o3 = 0.f;     // four independent chains
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 w4 = __ldg(wk + j);
              o0 = fmaf(v[4 * j + 0], w4.x, o0);
              o1 = fmaf(v[4 * j + 1], w4.y, o1);
              o2 = fmaf(v[4 * j + 2], w4.z, o2);
              o3 = fmaf(v[4 * j + 3], w4.w, o3);
            }
            float o = (o0 + o1) + (o2 + o3);
            if (p.head_relu) o = fmaxf(o, 0.f);
            p.head_out[((static_cast<long long>(tb) * p.head_c + k) * p.out_h + y) * p.out_w + x] = o;
          }
        }
      } else {
        const int n0 = tn * BLOCK_N;
        const int cofs = half * 32;
        const float* bias =
            p.bias ? p.bias + static_cast<long long>(tb < p.out_b ? tb : 0) * p.bias_sb + n0 + cofs
                   : nullptr;
        const bf16* res = (p.residual && valid)
                              ? p.residual + tb * p.res_sb + y * p.res_sy + x * p.res_sx + n0 + cofs
                              : nullptr;
        constexpr int kChunks = BLOCK_N / 64;
        // unrolled: the chunk index is a compile-time constant, so the accumulator registers of a staged chunk are
        // free for the epilogue of the chunks after it
#pragma unroll
        for (int c = 0; c < kChunks; ++c, ++chunk_counter) {
          stage_chunk_rt(c);
          // ---- bias + activation (specialised per activation: a straight-line block keeps the 32
          //      independent elements of a thread in flight), residual, bf16 packing
          float v[32];
          read_row_bias(row, cofs, bias != nullptr ? bias + c * 64 : nullptr, v);
          if (p.act == ODB_ACT_GELU) {
#pragma unroll
            for (int j = 0; j < 16; ++j) gelu_erf_x2(v[2 * j], v[2 * j + 1]);
          } else if (p.act == ODB_ACT_RELU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
          }
          uint4 rv[4];
          if (res != nullptr) {
            const uint4* rp = reinterpret_cast<const uint4*>(res + c * 64);
#pragma unroll
            for (int j = 0; j < 4; ++j) rv[j] = rp[j];  // plain ld.global: out may alias residual
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) rv[j] = make_uint4(0, 0, 0, 0);
          }
          const uint32_t* ru = reinterpret_cast<const uint32_t*>(rv);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float2 rr = unpack_bf16x2(ru[j]);
            v[2 * j] += rr.x;
            v[2 * j + 1] += rr.y;
          }
          // ---- staging: two slots alternate.  Slot (c & 1) was last read by the TMA store of chunk
          //      c-2, whose completion the store leader awaited before the barrier of chunk c-1, so
          //      one block barrier per chunk suffices.  (With a relu copy and only two staging
          //      buffers there is a single slot: wait for the previous store first.)
          const int slot = slots >= 2 ? static_cast<int>(chunk_counter & 1u) : 0;
          if (slots < 2) {
            if (store_leader) tma_store_wait_read<0>();
            named_bar_sync(kBarEpilogue, kEpiThreads);
          }
          const uint32_t buf0 = smem_base + Plan::kCOff + (slot * bufs_per_chunk) * kStagingBytes;
          const uint32_t rowoff = static_cast<uint32_t>(srow) * 128u;
          const bool do_store = !HALO || row_in_tile;       // halo junk columns own no staging row
          if (do_store) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint32_t addr =
                  buf0 + rowoff + (static_cast<uint32_t>((half * 4 + j) ^ (srow & 7)) << 4);
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr),
                           "r"(pack_bf16x2(v[8 * j + 0], v[8 * j + 1])), "r"(pack_bf16x2(v[8 * j + 2], v[8 * j + 3])),
                           "r"(pack_bf16x2(v[8 * j + 4], v[8 * j + 5])), "r"(pack_bf16x2(v[8 * j + 6], v[8 * j + 7]))
                           : "memory");
            }
          }
          if (p.has_out2 && do_store) {
            // the stored pre-activation `out` stays as it is; the copy is relu / gelu of the same fp32 value, taken
            // two elements at a time so that v stays intact for the GroupNorm statistics
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              uint32_t q[4];
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                float a = v[8 * j + 2 * i], b = v[8 * j + 2 * i + 1];
                if (p.out2_gelu) {
                  gelu_erf_x2(a, b);
                } else {
                  a = fmaxf(a, 0.f);
                  b = fmaxf(b, 0.f);
                }
                q[i] = pack_bf16x2(a, b);
              }
              const uint32_t addr = buf0 + kStagingBytes + rowoff +
                                    (static_cast<uint32_t>((half * 4 + j) ^ (srow & 7)) << 4);
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(q[0]), "r"(q[1]), "r"(q[2]),
                           "r"(q[3])
                           : "memory");
            }
          }
          // ---- fused GroupNorm statistics over the unrounded fp32 values (before the bf16 store); v is not
          //      needed after this, so the rows outside the output are zeroed in place
          if (p.gn_partial != nullptr) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = valid ? v[j] : 0.f;
            if (tb < p.out_b) {
              const int cpg = p.gn_cpg;
              float* dst = p.gn_partial +
                           ((((long long)tb * (p.tiles_x * p.tiles_y) + (ty * p.tiles_x + tx)) * 4 + quad) *
                                p.gn_groups + (n0 + c * 64 + cofs) / cpg) * 2;
              if (cpg == 2) gn_warp_partials<2>(v, lane, dst);
              else if (cpg == 4) gn_warp_partials<4>(v, lane, dst);
              else if (cpg == 8) gn_warp_partials<8>(v, lane, dst);
              else if (cpg == 16) gn_warp_partials<16>(v, lane, dst);
              else gn_warp_partials<32>(v, lane, dst);
            }
          }
          fence_proxy_async_smem();
          if (slots >= 2 && store_leader) tma_store_wait_read<0>();  // store of chunk c-1 has read its slot
          named_bar_sync(kBarEpilogue, kEpiThreads);
          if (store_leader) {
            tma_store_4d(&p.out_map, buf0, n0 + c * 64, x0, y0, tb);
            if (p.has_out2) tma_store_4d(&p.out2_map, buf0 + kStagingBytes, n0 + c * 64, x0, y0, tb);
            tma_store_commit();
          }
        }
      }
      if (store_leader) ODB_TRACE_TILE(iter, 4);
    }
    if (store_leader) tma_store_wait_all();
    }  // EPI_GENERIC
  }
  // a CTA of a pair stays resident until its peer no longer multicasts into it or arrives on its barriers
  if constexpr (PAIR) cluster_sync_all();
  if (threadIdx.x == 0) ODB_TRACE(2);
}

// ------------------------------------------------------------------------------------------ host

// esz: element size in bytes, 2 = bf16, 4 = fp32, 1 = e4m3 (encoded as UINT8: TMA moves bytes)
static int encode_view_map(CUtensorMap* map, const odb_view& v, int box_c, int box_w, int box_h,
                           CUtensorMapSwizzle swz, int esz = 2) {
  if (v.ptr == nullptr) return fail(ODB_ERR_INVALID, "conv_gemm: null view pointer");
  if ((reinterpret_cast<uintptr_t>(v.ptr) & 15u) != 0)
    return fail(ODB_ERR_INVALID, "conv_gemm: view pointer must be 16-byte aligned");
  if (v.c % 8 != 0) return fail(ODB_ERR_INVALID, "conv_gemm: channel count must be a multiple of 8");
  cuuint64_t dims[4] = {(cuuint64_t)v.c, (cuuint64_t)v.w, (cuuint64_t)v.h, (cuuint64_t)v.b};
  // strides of dims 1..3 in bytes; a unit extent may carry any (16B-multiple) stride
  long long sx = v.sx, sy = v.sy, sb = v.sb;
  if (v.w == 1 && sx == 0) sx = v.c;
  if (v.h == 1 && sy == 0) sy = (long long)v.w * sx;
  if (v.b == 1 && sb == 0) sb = (long long)v.h * sy;
  if (sx % 8 != 0 || sy % 8 != 0 || sb % 8 != 0 || sx <= 0 || sy <= 0 || sb <= 0)
    return fail(ODB_ERR_INVALID, "conv_gemm: view strides must be positive multiples of 8 elements");
  if (esz == 1 && (sx % 16 != 0 || sy % 16 != 0 || sb % 16 != 0 || v.c % 16 != 0))
    return fail(ODB_ERR_INVALID, "conv_gemm: e4m3 views need channel counts and strides that are multiples of 16");
  cuuint64_t strides[3] = {(cuuint64_t)sx * esz, (cuuint64_t)sy * esz, (cuuint64_t)sb * esz};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUtensorMapDataType dt = esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : esz == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  return encode_tiled(map, dt, 4, const_cast<void*>(v.ptr), dims, strides, box, estr, swz);
}

template <int BLOCK_N, int STAGES, int NSTAGING, bool HEAD, bool HALO, int EPI = EPI_GENERIC, bool PAIR = false,
          bool FP8 = false>
static int launch_instance(const std::conditional_t<FP8, ConvGemmParamsFp8, ConvGemmParams>& p, long long units,
                           cudaStream_t stream) {
  using Plan = SmemPlan<BLOCK_N, STAGES, NSTAGING, HALO, HEAD, EPI != EPI_BIAS_RES_F32>;
  auto kernel = conv_gemm_kernel<BLOCK_N, STAGES, NSTAGING, HEAD, HALO, PAIR, EPI, FP8>;
  static bool configured[kMaxDevices] = {};      // the opt-in is per device
  const int dev = current_device();
  if (!configured[dev]) {
    cudaError_t e =
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Plan::kTotal);
    if (e != cudaSuccess) return fail_cuda(e, "conv_gemm: cudaFuncSetAttribute");
    configured[dev] = true;
  }
  const int sms = num_sms();
  cudaError_t e;
  if constexpr (PAIR) {
    // units = pairs of M tiles x N tiles; one cluster of two CTAs per unit slot
    const long long pairs = units < sms / 2 ? units : sms / 2;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = 2;
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 2;
    cfg.gridDim = dim3((unsigned)(2 * pairs));
    cfg.blockDim = dim3(kNumThreads);
    cfg.dynamicSmemBytes = Plan::kTotal;
    cfg.stream = stream;
    e = cudaLaunchKernelEx(&cfg, kernel, p);
  } else {
    e = launch_pdl(kernel, dim3((unsigned)(units < sms ? units : sms)), dim3(kNumThreads), Plan::kTotal, stream, p);
  }
  count_launch();
  if (e != cudaSuccess) return fail_cuda(e, "conv_gemm: launch");
  return check_launch("conv_gemm");
}

// the plain-tile kernels (no halo, no head tail) with a specialised epilogue.  Stage counts: the operand ring, the
// output staging slots and the accumulator chunk buffer share the 227 KiB of shared memory.  `units`: M tiles (pairs
// of M tiles for a CTA pair) x N tiles.
template <int EPI>
static int launch_fast(const ConvGemmParams& p, int block_n, bool pair, long long units, cudaStream_t stream) {
  if constexpr (EPI == EPI_BIAS_RES_F32) {
    // fp32 residual stream: a chunk needs two 16 KiB staging units, and there is no accumulator chunk buffer
    // (256 wide: 3 x 48 KiB of operands + 64 KiB of staging = 208 KiB)
    if (pair && block_n == 128) return launch_instance<128, 4, 4, false, false, EPI, true>(p, units, stream);
    if (pair) return launch_instance<256, 3, 4, false, false, EPI, true>(p, units, stream);
    switch (block_n) {
      case 256: return launch_instance<256, 3, 4, false, false, EPI>(p, units, stream);
      case 128: return launch_instance<128, 4, 4, false, false, EPI>(p, units, stream);
      default: return launch_instance<64, 4, 4, false, false, EPI>(p, units, stream);
    }
  } else {
    if (pair && block_n == 128) return launch_instance<128, 4, 2, false, false, EPI, true>(p, units, stream);
    if (pair) return launch_instance<256, 3, 2, false, false, EPI, true>(p, units, stream);
    switch (block_n) {
      case 256: return launch_instance<256, 3, 2, false, false, EPI>(p, units, stream);
      case 128: return launch_instance<128, 4, 2, false, false, EPI>(p, units, stream);
      default: return launch_instance<64, 4, 4, false, false, EPI>(p, units, stream);
    }
  }
}

// the e4m3 instances (odb_conv_gemm_scaled): the bf16 instances' shared-memory plans, each stage carrying twice the K.
// EPI_BIAS has no 256-wide instance (it does not fit in registers without spilling); the host plans it at 128.
template <int EPI>
static int launch_fp8(const ConvGemmParamsFp8& p, int block_n, long long units, cudaStream_t stream) {
  constexpr int NS = EPI == EPI_BIAS_RES_F32 ? 4 : 2;
  if constexpr (EPI != EPI_BIAS) {
    if (block_n == 256) return launch_instance<256, 3, NS, false, false, EPI, false, true>(p, units, stream);
  }
  switch (block_n) {
    case 128: return launch_instance<128, 4, NS, false, false, EPI, false, true>(p, units, stream);
    case 64: return launch_instance<64, 4, 4, false, false, EPI, false, true>(p, units, stream);
    default: return fail(ODB_ERR_UNSUPPORTED, "conv_gemm_scaled: no instance for this block_n");
  }
}

}  // namespace odb

namespace odb { int conv_gemm_f32(const odb_conv_gemm_desc* d, cudaStream_t stream); }   // fp32_path.cu

using namespace odb;

struct HostPlan {
  int tw, th, tiles_x, tiles_y, block_n;
  bool pair, head, halo;
  long long m_tiles;
};

// the canonical 3x3 / stride 1 / pad 1 pattern over a single view (tap t = (ky, kx) row-major)
static bool is_canonical_3x3(const odb_conv_gemm_desc* d) {
  if (d->num_views != 1 || d->num_taps != 9) return false;
  for (int t = 0; t < 9; ++t)
    if (d->tap_view[t] != 0 || d->tap_dx[t] != t % 3 - 1 || d->tap_dy[t] != t / 3 - 1) return false;
  return d->views[0].w == d->out.w && d->views[0].h == d->out.h && d->views[0].b == d->out.b;
}

static int make_plan(const odb_conv_gemm_desc* d, HostPlan* hp) {
  if (d == nullptr) return fail(ODB_ERR_INVALID, "conv_gemm: null descriptor");
  if (d->num_views < 1 || d->num_views > ODB_MAX_VIEWS || d->num_taps < 1 ||
      d->num_taps > ODB_MAX_TAPS)
    return fail(ODB_ERR_INVALID, "conv_gemm: bad view/tap count");
  const int C = d->views[0].c;
  for (int v = 0; v < d->num_views; ++v)
    if (d->views[v].c != C) return fail(ODB_ERR_INVALID, "conv_gemm: views disagree on channels");
  for (int t = 0; t < d->num_taps; ++t)
    if (d->tap_view[t] < 0 || d->tap_view[t] >= d->num_views)
      return fail(ODB_ERR_INVALID, "conv_gemm: tap refers to a missing view");
  const bool head = d->head_out != nullptr;
  const int N = d->n;
  if (head) {
    if (N != 32 || d->head_c < 1 || d->head_w == nullptr || d->head_b == nullptr)
      return fail(ODB_ERR_INVALID, "conv_gemm: head tail needs n == 32, head_w, head_b");
  } else {
    if (N % 64 != 0) return fail(ODB_ERR_INVALID, "conv_gemm: n must be a multiple of 64");
  }
  const int ow = d->out.w, oh = d->out.h, ob = d->out.b;
  if (ow < 1 || oh < 1 || ob < 1) return fail(ODB_ERR_INVALID, "conv_gemm: empty output extent");
  int tw = d->tile_w, th = d->tile_h;
  bool halo = false;
  if (d->halo == 1) {
    if (!is_canonical_3x3(d)) return fail(ODB_ERR_INVALID, "conv_gemm: halo mode needs a 3x3 stride-1 pad-1 conv");
    halo = true;
  } else if (d->halo == 0) {
    // automatic only for the head tail (resident weights: 3x faster there); for the other layers the
    // deeper per-tap ring measured faster
    halo = is_canonical_3x3(d) && (tw <= 0 || th <= 0) &&
           (d->n <= kHaloAutoMaxN || (d->head_out != nullptr && d->num_taps * ((d->views[0].c + 63) / 64) <= kResidentBTiles));
  }
  if (halo && (tw <= 0 || th <= 0)) {
    if (ow <= 126) { tw = ow; th = 130 / (ow + 2); if (th > oh) th = oh; }
    else {
      // wide images: the (tile_w, tile_h) with tile_h * (tile_w + 2) - 2 <= 128 accumulator rows that
      // wastes the fewest MMA rows (ragged right / bottom edges included); ties -> smaller halo
      double best = -1.0;
      for (int h_ = 1; h_ <= 8 && h_ <= oh; ++h_) {
        const int w_ = 130 / h_ - 2;
        if (w_ < 8) break;
        const double eff = (double)(w_ * h_) / 128.0 * (double)ow / (double)(((ow + w_ - 1) / w_) * w_) *
                           (double)oh / (double)(((oh + h_ - 1) / h_) * h_);
        if (eff > best + 1e-9) { best = eff; tw = w_; th = h_; }
      }
    }
  }
  if (halo && (th * (tw + 2) - 2 > kTileRows || (tw + 2) * (th + 2) * 128 > kHaloStageBytes))
    return fail(ODB_ERR_INVALID, "conv_gemm: halo tile does not fit (tile_h * (tile_w + 2) - 2 <= 128)");
  hp->halo = halo;
  if (tw <= 0 || th <= 0) {
    if (oh == 1) { tw = 128; th = 1; }
    else if (ow % 16 == 0 && oh % 8 == 0) { tw = 16; th = 8; }
    else if (ow % 32 == 0 && oh % 4 == 0) { tw = 32; th = 4; }
    else if (ow <= 128) { tw = ow; th = 128 / ow; if (th > oh) th = oh; }
    else { tw = 128; th = 1; }
  }
  if (tw * th > kTileRows || tw > 256 || th > 256)
    return fail(ODB_ERR_INVALID, "conv_gemm: tile_w * tile_h must be <= 128");
  hp->tw = tw; hp->th = th;
  hp->tiles_x = (ow + tw - 1) / tw;
  hp->tiles_y = (oh + th - 1) / th;
  hp->m_tiles = (long long)hp->tiles_x * hp->tiles_y * ob;
  int block_n = d->block_n;
  if (head) block_n = 32;
  if (block_n == 0) {
    block_n = (N % 256 == 0) ? 256 : (N % 128 == 0) ? 128 : 64;
    const int sms = num_sms();
    while (block_n > 64 && hp->m_tiles * (N / block_n) < sms) block_n /= 2;
  }
  if (!(block_n == 256 || block_n == 128 || block_n == 64 || block_n == 32) || N % block_n != 0)
    return fail(ODB_ERR_INVALID, "conv_gemm: unsupported block_n");
  if (hp->m_tiles * (N / block_n) > 0x7fffffffLL)
    return fail(ODB_ERR_INVALID, "conv_gemm: too many tiles");
  // CTA pairs (2-CTA clusters sharing the weight tile by TMA multicast): on explicit request only
  const bool pair = d->cta_pair == 1;
  if (pair && (!(block_n == 256 || (block_n == 128 && !halo)) || head))
    return fail(ODB_ERR_UNSUPPORTED, "conv_gemm: cta_pair needs block_n 256 (or 128 without halo) and no head tail");
  hp->block_n = block_n; hp->pair = pair; hp->head = head;
  return ODB_OK;
}

extern "C" int odb_conv_gemm_plan(const odb_conv_gemm_desc* d, int32_t* out4) {
  HostPlan hp;
  int rc = make_plan(d, &hp);
  if (rc) return rc;
  if (out4) {
    out4[0] = hp.tiles_x; out4[1] = hp.tiles_y; out4[2] = hp.block_n;
    out4[3] = (hp.pair ? 1 : 0) | (hp.halo ? 2 : 0);
  }
  return ODB_OK;
}

extern "C" int odb_conv_gemm(const odb_conv_gemm_desc* d, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (d != nullptr && d->in_dtype == ODB_DTYPE_F32) return conv_gemm_f32(d, stream);   // fp32 correctness mode
  HostPlan hp;
  int rc = make_plan(d, &hp);
  if (rc) return rc;
  const bool head = hp.head, pair = hp.pair;
  const int block_n = hp.block_n, tw = hp.tw, th = hp.th;
  const int C = d->views[0].c;
  const int N = d->n;
  if (!head && d->out.ptr == nullptr) return fail(ODB_ERR_INVALID, "conv_gemm: null output");
  if (d->weight == nullptr || (reinterpret_cast<uintptr_t>(d->weight) & 15u) != 0)
    return fail(ODB_ERR_INVALID, "conv_gemm: weight must be non-null and 16-byte aligned");
  const long long K = (long long)d->num_taps * C;

  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  const int ow = d->out.w, oh = d->out.h, ob = d->out.b;
  p.tile_w = tw; p.tile_h = th;
  p.tiles_x = hp.tiles_x;
  p.tiles_y = hp.tiles_y;
  p.tiles_b = ob;
  p.out_w = ow; p.out_h = oh; p.out_b = ob; p.n_total = N;
  const long long m_tiles = hp.m_tiles;
  p.tiles_n = N / block_n;
  const long long total = m_tiles * p.tiles_n;
  const long long units = pair ? ((m_tiles + 1) / 2) * p.tiles_n : total;

  p.num_taps = d->num_taps;
  p.kb_per_tap = (C + kKBlock - 1) / kKBlock;
  for (int t = 0; t < d->num_taps; ++t) {
    p.tap_view[t] = d->tap_view[t];
    p.tap_dx[t] = d->tap_dx[t];
    p.tap_dy[t] = d->tap_dy[t];
  }
  for (int v = 0; v < ODB_MAX_VIEWS; ++v) {
    // unused slots alias view 0 so that prefetch.tensormap always sees a valid descriptor
    const odb_view& src = d->views[v < d->num_views ? v : 0];
    rc = encode_view_map(&p.a_map[v], src, kKBlock, hp.halo ? tw + 2 : tw, hp.halo ? th + 2 : th,
                         CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    if ((K * 2) % 16 != 0) return fail(ODB_ERR_INVALID, "conv_gemm: K must be a multiple of 8");
    cuuint32_t box[2] = {(cuuint32_t)kKBlock, (cuuint32_t)(pair ? block_n / 2 : block_n)};
    cuuint32_t estr[2] = {1, 1};
    rc = encode_tiled(&p.b_map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(d->weight),
                      dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  const bool out_f32 = d->out_dtype == ODB_DTYPE_F32;
  if (d->in_dtype != ODB_DTYPE_BF16) return fail(ODB_ERR_INVALID, "conv_gemm: tensor-core path takes bf16 operands");
  if (out_f32) {
    // fp32 residual stream (ViT attn.proj / mlp.fc2 / patch projection): out = residual + (acc + bias), all fp32
    if (head || hp.halo || d->out2.ptr || d->gn_partial || d->act != ODB_ACT_NONE || !d->bias || !d->residual.ptr ||
        d->epilogue != 0)
      return fail(ODB_ERR_UNSUPPORTED, "conv_gemm: fp32 output needs bias + fp32 residual and no act/out2/gn/head/halo");
    if (d->out.c != N || d->residual.c != N || d->residual.w < ow || d->residual.h < oh || d->residual.b < ob)
      return fail(ODB_ERR_INVALID, "conv_gemm: fp32 out/residual extent mismatch");
    rc = encode_view_map(&p.out_map, d->out, 32, tw, th, CU_TENSOR_MAP_SWIZZLE_128B, 4);
    if (rc) return rc;
    rc = encode_view_map(&p.res_map, d->residual, 32, tw, th, CU_TENSOR_MAP_SWIZZLE_128B, 4);
    if (rc) return rc;
    p.out2_map = p.out_map;
    p.bias = d->bias;
    p.bias_sb = d->bias_sb;
    p.trace = debug_trace();
    return launch_fast<EPI_BIAS_RES_F32>(p, block_n, pair, units, stream);
  }
  if (!head) {
    if (d->out.c != N) return fail(ODB_ERR_INVALID, "conv_gemm: out.c must equal n");
    rc = encode_view_map(&p.out_map, d->out, 64, tw, th, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    if (d->out2.ptr) {
      odb_view o2 = d->out2;
      if (o2.c != N || o2.w != ow || o2.h != oh || o2.b != ob)
        return fail(ODB_ERR_INVALID, "conv_gemm: out2 extent mismatch");
      rc = encode_view_map(&p.out2_map, o2, 64, tw, th, CU_TENSOR_MAP_SWIZZLE_128B);
      if (rc) return rc;
      p.has_out2 = 1;
      if (d->out2_act != ODB_ACT_NONE && d->out2_act != ODB_ACT_RELU && d->out2_act != ODB_ACT_GELU)
        return fail(ODB_ERR_INVALID, "conv_gemm: out2_act must be ODB_ACT_NONE / RELU (relu copy) or ODB_ACT_GELU");
      p.out2_gelu = d->out2_act == ODB_ACT_GELU;
    } else {
      p.out2_map = p.out_map;
    }
  } else {
    p.out_map = p.a_map[0];
    p.out2_map = p.a_map[0];
  }
  p.bias = d->bias;
  p.bias_sb = d->bias_sb;
  if (d->residual.ptr) {
    if ((reinterpret_cast<uintptr_t>(d->residual.ptr) & 15u) || d->residual.sx % 8 ||
        d->residual.sy % 8 || d->residual.sb % 8)
      return fail(ODB_ERR_INVALID, "conv_gemm: residual must be 16-byte aligned / strided");
    p.residual = static_cast<const bf16*>(d->residual.ptr);
    p.res_sx = d->residual.sx; p.res_sy = d->residual.sy; p.res_sb = d->residual.sb;
  }
  p.act = d->act;
  p.head_w = d->head_w; p.head_b = d->head_b; p.head_c = d->head_c; p.head_relu = d->head_relu;
  p.head_out = d->head_out;
  if (d->gn_partial != nullptr) {
    const int g = d->gn_groups;
    const int cpg = g > 0 ? N / g : 0;
    if (head || g < 1 || N % g != 0 || !(cpg == 2 || cpg == 4 || cpg == 8 || cpg == 16 || cpg == 32))
      return fail(ODB_ERR_INVALID, "conv_gemm: gn_partial needs n / gn_groups in {2,4,8,16,32}");
    p.gn_partial = d->gn_partial;
    p.gn_cpg = cpg;
    p.gn_groups = g;
  }
  p.trace = debug_trace();

  // specialised epilogue when the flag combination allows it (see the EPI_* comment)
  if (!hp.halo && !head && block_n >= 64 && p.bias == nullptr && !p.has_out2 && p.gn_partial != nullptr &&
      p.residual == nullptr && p.act == ODB_ACT_NONE && d->epilogue == 0)
    return launch_fast<EPI_GN>(p, block_n, pair, units, stream);
  if (!hp.halo && !head && block_n >= 64 && p.bias != nullptr && !p.has_out2 && p.gn_partial == nullptr &&
      d->epilogue == 0) {
    if (p.residual == nullptr) {
      if (p.act == ODB_ACT_NONE) return launch_fast<EPI_BIAS>(p, block_n, pair, units, stream);
      if (p.act == ODB_ACT_RELU) return launch_fast<EPI_BIAS_RELU>(p, block_n, pair, units, stream);
      if (p.act == ODB_ACT_GELU) return launch_fast<EPI_BIAS_GELU>(p, block_n, pair, units, stream);
    } else if (p.act == ODB_ACT_NONE && d->residual.c == N && d->residual.w >= ow && d->residual.h >= oh &&
               d->residual.b >= ob && (d->residual.sb > 0 || ob == 1) && (d->residual.sy > 0 || oh == 1)) {
      rc = encode_view_map(&p.res_map, d->residual, 64, tw, th, CU_TENSOR_MAP_SWIZZLE_128B);
      if (rc) return rc;
      return launch_fast<EPI_BIAS_RES>(p, block_n, pair, units, stream);
    }
  }
  if (hp.halo) {
    p.halo_w = tw + 2;
    if (head) {
      if (p.num_taps * p.kb_per_tap > kResidentBTiles)
        return fail(ODB_ERR_UNSUPPORTED, "conv_gemm: halo head tail needs taps * ceil(C / 64) <= 18");
      p.a_stage_bytes = (((tw + 2) * (th + 2) * 128) + 1023) & ~1023;
      p.a_stages = kHaloAreaBytes / p.a_stage_bytes;
      if (p.a_stages > kMaxAStages) p.a_stages = kMaxAStages;
    }
    if (pair) return launch_instance<256, 1, 2, false, true, EPI_GENERIC, true>(p, units, stream);
    switch (block_n) {
      case 256: return launch_instance<256, 1, 2, false, true>(p, total, stream);
      case 128: return launch_instance<128, 3, 2, false, true>(p, total, stream);
      case 64: return launch_instance<64, 4, 2, false, true>(p, total, stream);
      case 32:
        if (!head) return fail(ODB_ERR_UNSUPPORTED, "conv_gemm: block_n 32 only with the head tail");
        return launch_instance<32, 8, 0, true, true>(p, total, stream);
    }
  }
  if (pair && block_n == 128) return launch_instance<128, 4, 2, false, false, EPI_GENERIC, true>(p, units, stream);
  if (pair) return launch_instance<256, 3, 2, false, false, EPI_GENERIC, true>(p, units, stream);
  switch (block_n) {
    case 256: return launch_instance<256, 3, 2, false, false>(p, total, stream);
    case 128: return launch_instance<128, 4, 2, false, false>(p, total, stream);
    case 64: return launch_instance<64, 4, 4, false, false>(p, total, stream);
    case 32:
      if (!head) return fail(ODB_ERR_UNSUPPORTED, "conv_gemm: block_n 32 only with the head tail");
      return launch_instance<32, 8, 0, true, false>(p, total, stream);
  }
  return fail(ODB_ERR_INVALID, "conv_gemm: unreachable");
}


extern "C" int odb_conv_gemm_scaled(const odb_conv_gemm_desc* d, const float* row_scale, const float* col_scale,
                                    void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (d == nullptr || d->in_dtype != ODB_DTYPE_E4M3)
    return fail(ODB_ERR_INVALID, "conv_gemm_scaled: needs a descriptor with in_dtype ODB_DTYPE_E4M3");
  if (row_scale == nullptr || col_scale == nullptr || (reinterpret_cast<uintptr_t>(row_scale) & 3u) != 0 ||
      (reinterpret_cast<uintptr_t>(col_scale) & 15u) != 0)
    return fail(ODB_ERR_INVALID, "conv_gemm_scaled: row_scale (4-byte) and col_scale (16-byte aligned) are required");
  if (d->num_views != 1 || d->num_taps != 1 || d->tap_view[0] != 0 || d->tap_dx[0] != 0 || d->tap_dy[0] != 0)
    return fail(ODB_ERR_UNSUPPORTED, "conv_gemm_scaled: linear layers only (one view, one tap at offset 0)");
  if (d->views[0].w != d->out.w || d->views[0].h != 1 || d->views[0].b != 1 || d->out.h != 1 || d->out.b != 1)
    return fail(ODB_ERR_INVALID, "conv_gemm_scaled: [rows][C] operands (h = b = 1) with equal input and output rows");
  if (d->head_out != nullptr || d->halo == 1 || d->cta_pair == 1 || d->gn_partial != nullptr || d->out2.ptr != nullptr ||
      d->bias == nullptr || d->epilogue != 0)
    return fail(ODB_ERR_UNSUPPORTED, "conv_gemm_scaled: needs a bias; no head, halo, CTA pair, GroupNorm or out2");
  const bool out_f32 = d->out_dtype == ODB_DTYPE_F32;
  if (out_f32 ? (d->act != ODB_ACT_NONE || d->residual.ptr == nullptr)
              : (d->out_dtype != ODB_DTYPE_BF16 || d->residual.ptr != nullptr ||
                 (d->act != ODB_ACT_NONE && d->act != ODB_ACT_GELU)))
    return fail(ODB_ERR_UNSUPPORTED,
                "conv_gemm_scaled: bf16 output with bias [+ GELU], or fp32 output with bias + fp32 residual");
  HostPlan hp;
  int rc = make_plan(d, &hp);
  if (rc) return rc;
  if (d->out.ptr == nullptr) return fail(ODB_ERR_INVALID, "conv_gemm_scaled: null output");
  if (d->weight == nullptr || (reinterpret_cast<uintptr_t>(d->weight) & 15u) != 0)
    return fail(ODB_ERR_INVALID, "conv_gemm_scaled: weight must be non-null and 16-byte aligned");
  const bool bias_only = !out_f32 && d->act == ODB_ACT_NONE;
  if (bias_only && hp.block_n == 256) {
    if (d->block_n == 256) return fail(ODB_ERR_UNSUPPORTED, "conv_gemm_scaled: bias-only epilogue: block_n 64 or 128");
    hp.block_n = 128;
  }
  const int C = d->views[0].c, N = d->n, tw = hp.tw, th = hp.th, block_n = hp.block_n;
  if (block_n < 64) return fail(ODB_ERR_UNSUPPORTED, "conv_gemm_scaled: block_n must be 64, 128 or 256");
  const int ow = d->out.w, oh = d->out.h, ob = d->out.b;

  ConvGemmParamsFp8 p;
  memset(&p, 0, sizeof(p));
  p.tile_w = tw; p.tile_h = th;
  p.tiles_x = hp.tiles_x; p.tiles_y = hp.tiles_y; p.tiles_b = ob;
  p.out_w = ow; p.out_h = oh; p.out_b = ob; p.n_total = N;
  p.tiles_n = N / block_n;
  const long long units = hp.m_tiles * p.tiles_n;
  p.num_taps = 1;
  p.kb_per_tap = (C + 127) / 128;        // 128 e4m3 elements per K block
  for (int v = 0; v < ODB_MAX_VIEWS; ++v) {
    rc = encode_view_map(&p.a_map[v], d->views[0], 128, tw, th, CU_TENSOR_MAP_SWIZZLE_128B, 1);
    if (rc) return rc;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)N};
    cuuint64_t strides[1] = {(cuuint64_t)C};
    cuuint32_t box[2] = {128u, (cuuint32_t)block_n};
    cuuint32_t estr[2] = {1, 1};
    rc = encode_tiled(&p.b_map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(d->weight), dims, strides, box,
                      estr, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  if (d->out.c != N) return fail(ODB_ERR_INVALID, "conv_gemm_scaled: out.c must equal n");
  p.bias = d->bias;
  p.bias_sb = d->bias_sb;
  p.row_scale = row_scale;
  p.col_scale = col_scale;
  if (out_f32) {
    if (d->residual.c != N || d->residual.w < ow || d->residual.h < oh || d->residual.b < ob)
      return fail(ODB_ERR_INVALID, "conv_gemm_scaled: fp32 out/residual extent mismatch");
    rc = encode_view_map(&p.out_map, d->out, 32, tw, th, CU_TENSOR_MAP_SWIZZLE_128B, 4);
    if (rc) return rc;
    rc = encode_view_map(&p.res_map, d->residual, 32, tw, th, CU_TENSOR_MAP_SWIZZLE_128B, 4);
    if (rc) return rc;
    p.out2_map = p.out_map;
    return launch_fp8<EPI_BIAS_RES_F32>(p, block_n, units, stream);
  }
  rc = encode_view_map(&p.out_map, d->out, 64, tw, th, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  p.out2_map = p.out_map;
  p.res_map = p.out_map;
  p.act = d->act;
  return d->act == ODB_ACT_GELU ? launch_fp8<EPI_BIAS_GELU>(p, block_n, units, stream)
                                : launch_fp8<EPI_BIAS>(p, block_n, units, stream);
}
