// Implicit-GEMM convolution for sm_90a: TMA -> shared memory -> wgmma -> registers -> fused epilogue.
//
// Replaces every nn.Conv2d (+ folded eval BatchNorm / bias / residual add / ReLU / GroupNorm statistics)
// on the SipMask inference path (reference: SipMask-mmdetection/mmdet/models/backbones/resnet.py:203-239,
// models/necks/fpn.py:138-178, ops/conv_module.py:124-132, models/anchor_heads/sipmask_head.py:241-287;
// the reference runs them through cuDNN + separate ATen kernels).
//
//   D[pixel, co] = sum_{tap, ci} A[pixel (+) tap, ci] * Wt[co, tap*Cin + ci]
//
//  * A (activations) is NHWC fp16.  One M-tile is a BH x BW patch of output pixels (BH*BW = 128); for every
//    filter tap the producer issues ONE 4-D TMA box {64 ch, BW, BH, 1} at the tap-shifted coordinate, so
//    im2col never exists in memory and zero padding is TMA out-of-bounds fill.  Stride-2 convolutions use
//    parity-split tensor maps (doubled global strides), the 7x7/2 stem a sliding-window map.
//  * W is [Cout, taps*Cin] fp16, K-major, loaded as {64, N} boxes (rows past Cout are zero-filled).  Both operands
//    use the 128-byte swizzle, the canonical K-major wgmma layout (8-row groups 1024 B apart).
//  * Persistent CTAs (one per SM), warp-specialised: warps 0..7 are two consumer warpgroups, each issuing
//    wgmma.m64nNk16 (fp32 accumulators in registers) for 64 of the tile's 128 pixels and then running the epilogue
//    (scale / bias / residual / GN statistics / ReLU -> global NHWC store) on its own accumulators; warp 8 is the TMA
//    producer, which runs ahead into the next tile while the consumers drain the current one.
//  * fp16-output plans without an upsampled residual (epi_tma) take the epilogue through shared memory: warp 9 loads the
//    residual of each 64-pixel x 32-channel chunk by TMA into a slot, the consumer warps read it with ldmatrix, write their
//    results over it with stmatrix and hand the slot back, and warp 9 stores it by TMA.  The consumers never wait on a
//    global load or store.  fp32-output (head) and nearest-upsampled-residual (FPN lateral) plans store from registers.
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"

namespace smb {

constexpr int kMaxTaps = 9;
constexpr int kMaxMaps = 8;
constexpr int kMaxLevels = 5;
constexpr int kConsumerWarps = 8;
// + a producer warpgroup: warp 8 issues the operand TMA loads, warp 9 the epilogue's residual loads and output stores
// (epi_tma plans), warps 10-11 exist only so that the CTA is whole warpgroups, which setmaxnreg needs to move registers
// from the producer (40 per thread) to the consumers (232 instead of 168)
constexpr int kThreads = 32 * (kConsumerWarps + 4);
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kEpiWarp = kConsumerWarps + 1;
constexpr int kABytes = 128 * 64 * 2;                // one A stage: 128 pixels x 64 channels fp16
constexpr size_t kSmemBudget = 220 * 1024;           // epilogue slots + operand stages + barriers (227 KB per block on sm_90)
// Epilogue slots (epi_tma plans): per consumer warpgroup a ring of kEpiSlots chunks of 64 pixels x 32 channels fp16, one
// 64-byte row per pixel in the TMA 64-byte swizzle.  32 channels keep every N at its operand ring (static_asserts below).
constexpr int kEpiSlots = 3;
constexpr int kEpiSlotBytes = 64 * 32 * 2;
constexpr int kEpiBytes = 2 * kEpiSlots * kEpiSlotBytes;

// operand stages of an N-channel tile: what is left of the budget after the epilogue slots, 1 KB alignment slack and
// 256 B of epilogue barriers, 16 B of barriers per stage, at most 8
constexpr int ring_stages(int n_tile) {
  const int s = (int)((kSmemBudget - kEpiBytes - 1024 - 256) / ((size_t)kABytes + (size_t)n_tile * 128 + 16));
  return s > 8 ? 8 : s;
}
static_assert(ring_stages(256) == 4 && ring_stages(128) == 6 && ring_stages(64) == 8,
              "the epilogue slots must not cost any N tile an operand stage");
static_assert(4 * kEpiSlots * 8 <= 256, "epilogue barriers exceed their reserve");

// One pyramid level (or the only tensor) of a launch.  Convolutions whose weights are shared by several feature-pyramid
// levels (the FCOS towers and heads, sipmask_head.py:250-257) run as ONE launch over the union of the levels' tiles.
struct LevelDesc {
  int H_out, W_out, BH, BW, tiles_x, tiles_y;
  int tile_start;                 // first M-tile of this level in the launch-wide tile order
  int map0;                       // index of this level's first A tensor map
  void* out;
  const __half* residual;
  long long* gn_stats;            // fixed-point per-(image,group) {sum * 2^20, sumsq * 2^16}
  int res_h, res_w;
};

struct ConvParams {
  CUtensorMap amap[kMaxMaps];
  CUtensorMap bmap;
  // epi_tma plans: output per level and the same-shape residual (single-level plans, encoded per launch), as boxes of
  // {32 ch, min(BW, 64), max(BH / 2, 1), 1}: one consumer warpgroup's 64 pixels of a chunk, rows in accumulator order
  CUtensorMap omap[kMaxLevels];
  CUtensorMap rmap;
  LevelDesc lv[kMaxLevels];
  int num_levels;
  int tap_map[kMaxTaps], tap_dx[kMaxTaps], tap_dy[kMaxTaps];
  int num_taps, kb_per_tap;       // k-blocks (64 channels) per tap
  int n_img, tiles_m;
  int Cout, n_tile, n_tiles_n, stages;
  int out_pitch, out_f32;
  const float* bias;
  float alpha;
  int res_pitch, res_mode;        // res_mode: 0 none, 1 same shape, 2 nearest-upsampled coarser map
  int gn_group;                   // channels per GroupNorm group (8 or 16), 0 = no statistics
  int relu;
  int epi_tma;                    // epilogue through shared memory and TMA (fp16 output, res_mode 0 / 1)
};
static_assert(sizeof(ConvParams) <= 4096, "ConvParams must fit the 4 KB kernel-parameter space");

// ------------------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// generic-proxy writes to shared memory (stmatrix) -> visible to a later TMA store
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// lane l addresses row l % 8 of 8x8 matrix l / 8; register m holds row lane / 4, columns 2 (lane % 4) + {0, 1} of matrix m
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t* r) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]),
               "r"(r[2]), "r"(r[3])
               : "memory");
}

// K-major, 128-byte swizzle wgmma shared-memory matrix descriptor (sm_90):
//   [0,14) start>>4 | [16,30) LBO>>4 (unused for swizzled K-major, 1) | [32,46) SBO>>4 = 1024>>4 | [62,64) 1 = SWIZZLE_128B
__device__ __forceinline__ uint64_t make_sdesc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// The accumulators are "+f" operands of the asm statements that issue the MMAs; this one pins them below the wait so that
// no read of an accumulator can be scheduled before the MMA that writes it has completed.
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory, fp32 accumulators in registers:
// d[4j + 2i + c] is row (warp%4)*16 + lane/4 + 8i, column 8j + 2*(lane%4) + c.
template <int N>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t a, uint64_t b, int scale_d);

template <>
__device__ __forceinline__ void wgmma_f16<64>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d)
      : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<128>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d)
      : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<256>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a), "l"(b), "r"(scale_d)
      : "memory");
}

// ------------------------------------------------------------------------------------------------ kernel
// work unit -> tile.  Units of the same M-tile with different N-tiles are adjacent, so concurrently running CTAs share the
// activation patch in L2.
struct TileCoord {
  int lvl, img, x0, y0, n0;
};

// n / d and n % d for small non-negative n (< 2^22) without the ~30-instruction integer division: float reciprocal estimate
// plus one correction step (exact: the estimate is off by at most one).
__device__ __forceinline__ int fast_divmod(int n, int d, int& rem) {
  int q = __float2int_rz(__int2float_rn(n) * __frcp_rn(__int2float_rn(d)));
  int r = n - q * d;
  if (r >= d) { ++q; r -= d; }
  if (r < 0) { --q; r += d; }
  rem = r;
  return q;
}

__device__ __forceinline__ TileCoord decode_tile(const ConvParams& p, int unit) {
  TileCoord t;
  int nt = 0, mt = unit;
  if (p.n_tiles_n > 1) mt = fast_divmod(unit, p.n_tiles_n, nt);
  int l = 0;
#pragma unroll
  for (int i = 1; i < kMaxLevels; ++i)
    if (i < p.num_levels && mt >= p.lv[i].tile_start) l = i;
  mt -= p.lv[l].tile_start;
  int tx, ty;
  mt = fast_divmod(mt, p.lv[l].tiles_x, tx);
  t.img = fast_divmod(mt, p.lv[l].tiles_y, ty);
  t.lvl = l;
  t.x0 = tx * p.lv[l].BW;
  t.y0 = ty * p.lv[l].BH;
  t.n0 = nt * p.n_tile;
  return t;
}

// Epilogue of one consumer warp: rows (warp%4)*16 + lane/4 + {0, 8} of its warpgroup's 64-pixel half of the tile.
// Per element: acc + bias, * alpha, + residual -> GroupNorm statistics (pre-activation) -> ReLU -> fp16 / fp32 store.
// GroupNorm partials of one tile: [consumer warp][group within the N tile (<= 256 / 8)][sum, sum of squares], fixed point
typedef unsigned long long GnPart[kConsumerWarps][32][2];

// After every consumer warp has written its partials of the tile: one global atomic per (group, statistic) of the tile
// instead of one per warp.  When all SMs run tower convolutions, per-warp atomics on the same few addresses serialised
// in L2 and stretched every tile.  Integer sums are exact, so the statistics are the same bits.
__device__ __forceinline__ void gn_flush(const ConvParams& p, const TileCoord& tc, GnPart& gn_part, int N) {
  asm volatile("bar.sync 1, %0;" ::"n"(32 * kConsumerWarps) : "memory");       // partials of all consumer warps written
  const int t = threadIdx.x, ngl = min(N, p.Cout - tc.n0) / p.gn_group;
  if (t < 2 * ngl) {
    unsigned long long v = 0;
#pragma unroll
    for (int w = 0; w < kConsumerWarps; ++w) v += gn_part[w][t >> 1][t & 1];
    const int ngroups = p.Cout / p.gn_group;
    atomicAdd(reinterpret_cast<unsigned long long*>(p.lv[tc.lvl].gn_stats) +
                  ((size_t)tc.img * ngroups + tc.n0 / p.gn_group + (t >> 1)) * 2 + (t & 1), v);
  }
  asm volatile("bar.sync 1, %0;" ::"n"(32 * kConsumerWarps) : "memory");       // read before the next tile overwrites
}

template <int N>
__device__ __forceinline__ void epilogue(const ConvParams& p, const TileCoord& tc, const float* acc, int wg, int warp, int lane,
                                         GnPart& gn_part) {
  const LevelDesc& L = p.lv[tc.lvl];
  const int bw_shift = 31 - __clz(L.BW);            // BW is a power of two (choose_patch)
  bool valid[2];
  size_t pix[2];
  const __half* res_row[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
    const int x = tc.x0 + (row & (L.BW - 1)), y = tc.y0 + (row >> bw_shift);
    valid[i] = (x < L.W_out) && (y < L.H_out);
    pix[i] = ((size_t)tc.img * L.H_out + y) * L.W_out + x;
    res_row[i] = nullptr;
    if (valid[i]) {
      if (p.res_mode == 1) {
        res_row[i] = L.residual + pix[i] * p.res_pitch;
      } else if (p.res_mode == 2) {
        // F.interpolate(mode='nearest', size=...) : src = min(floor(dst * in/out), in-1)   (fpn.py:149-152)
        const int sy = min((int)floorf((float)y * ((float)L.res_h / (float)L.H_out)), L.res_h - 1);
        const int sx = min((int)floorf((float)x * ((float)L.res_w / (float)L.W_out)), L.res_w - 1);
        res_row[i] = L.residual + (((size_t)tc.img * L.res_h + sy) * L.res_w + sx) * p.res_pitch;
      }
    }
  }
  const int cq = 2 * (lane & 3);
  float gsum = 0.f, gsq = 0.f;                       // GroupNorm partials of the current 16-channel group (gn_group 16)
  // The output may alias the residual as far as the compiler knows, so a residual load written after a store cannot be
  // issued before it: one 8-channel block at a time, every residual load would wait a full memory round trip.  The
  // bias and residual operands of kEpiChunk blocks are therefore loaded together, then combined and stored (at N = 256
  // next to 128 accumulators: this is what the consumers' 232 registers are for).
  constexpr int kEpiChunk = 8;
#pragma unroll
  for (int j0 = 0; j0 < N / 8; j0 += kEpiChunk) {
    if (tc.n0 + 8 * j0 >= p.Cout) break;
    float2 bb[kEpiChunk], rr[kEpiChunk][2];
#pragma unroll
    for (int jj = 0; jj < kEpiChunk; ++jj) {
      const int ch = tc.n0 + 8 * (j0 + jj) + cq;
      bb[jj] = make_float2(0.f, 0.f);
      rr[jj][0] = rr[jj][1] = make_float2(0.f, 0.f);
      if (ch - cq >= p.Cout) continue;
      if (p.bias) bb[jj] = make_float2(__ldg(p.bias + ch), __ldg(p.bias + ch + 1));
#pragma unroll
      for (int i = 0; i < 2; ++i)
        if (res_row[i]) rr[jj][i] = __half22float2(*reinterpret_cast<const __half2*>(res_row[i] + ch));
    }
#pragma unroll
    for (int jj = 0; jj < kEpiChunk; ++jj) {
      const int j = j0 + jj;
      const int ch0 = tc.n0 + 8 * j;                 // first channel of this 8-channel block (warp-uniform)
      if (ch0 >= p.Cout) break;
      const int ch = ch0 + cq;
      float s = 0.f, q = 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float f0 = acc[4 * j + 2 * i] + bb[jj].x, f1 = acc[4 * j + 2 * i + 1] + bb[jj].y;
        if (p.alpha != 1.0f) { f0 *= p.alpha; f1 *= p.alpha; }
        if (res_row[i]) { f0 += rr[jj][i].x; f1 += rr[jj][i].y; }
        if (valid[i]) { s += f0 + f1; q += f0 * f0 + f1 * f1; }
        if (p.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
        if (valid[i]) {
          if (p.out_f32) {
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(L.out) + pix[i] * p.out_pitch + ch) = make_float2(f0, f1);
          } else {
            *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(L.out) + pix[i] * p.out_pitch + ch) = __floats2half2_rn(f0, f1);
          }
        }
      }
      if (p.gn_group) {
        // per-(image, group) sum / sum of squares of the conv output (pre-activation): fp32 over the warp's 16 rows, then
        // 64-bit fixed point, summed over the tile by gn_flush (integer sums: bit-reproducible whatever the tile order).
        gsum += s; gsq += q;
        if (p.gn_group == 8 || (j & 1)) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            gsum += __shfl_xor_sync(0xffffffffu, gsum, o);
            gsq += __shfl_xor_sync(0xffffffffu, gsq, o);
          }
          if (lane == 0) {
            unsigned long long* part = gn_part[warp][(ch0 - tc.n0) / p.gn_group];
            part[0] = (unsigned long long)__float2ll_rn(gsum * kGnSumScale);
            part[1] = (unsigned long long)__float2ll_rn(gsq * kGnSqScale);
          }
          gsum = 0.f; gsq = 0.f;
        }
      }
    }
  }
}

// The same per-element arithmetic and GroupNorm partials as epilogue(), for epi_tma plans, one 32-channel chunk at a time
// through the warpgroup's slot ring (slot es, phase eph, carried across tiles): wait until warp 9 has filled the slot
// (residual) or freed it, ldmatrix the residual, stmatrix the fp16 results over it, hand the slot to warp 9's TMA store.
// Slot layout: pixel row r (0..63, accumulator row order) at r * 64 bytes, its 16-byte channel quad q at
// ((q ^ (r >> 1) & 3) * 16): the TMA 64-byte swizzle (address bits [4,6) ^= bits [7,9)).
template <int N>
__device__ __forceinline__ void epilogue_tma(const ConvParams& p, const TileCoord& tc, const float* acc, int wg, int warp,
                                             int lane, GnPart& gn_part, uint32_t slots, uint64_t* epi_full,
                                             uint64_t* epi_ready, int& es, uint32_t& eph) {
  const LevelDesc& L = p.lv[tc.lvl];
  const int bw_shift = 31 - __clz(L.BW);
  bool valid[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
    valid[i] = (tc.x0 + (row & (L.BW - 1)) < L.W_out) && (tc.y0 + (row >> bw_shift) < L.H_out);
  }
  // ldmatrix / stmatrix x4 number h covers the warp's 16 rows x 8-channel blocks 2h, 2h + 1 of the chunk: lane supplies
  // row (lane & 7) + 8 * ((lane >> 3) & 1) of block 2h + (lane >> 4); register m = 2 * (block & 1) + i of that call.
  const int mrow = (warp & 3) * 16 + 8 * ((lane >> 3) & 1) + (lane & 7);
  const uint32_t row_addr = slots + (uint32_t)wg * (kEpiSlots * kEpiSlotBytes) + (uint32_t)mrow * 64;
  const uint32_t q0 = (uint32_t)((0 + (lane >> 4)) ^ ((mrow >> 1) & 3)) << 4;
  const uint32_t q1 = (uint32_t)((2 + (lane >> 4)) ^ ((mrow >> 1) & 3)) << 4;
  const int cq = 2 * (lane & 3);
  const int nchunks = (min(N, p.Cout - tc.n0) + 31) >> 5;
  float gsum = 0.f, gsq = 0.f;
#pragma unroll
  for (int c = 0; c < N / 32; ++c) {
    if (c >= nchunks) break;
    mbar_wait(&epi_full[wg * kEpiSlots + es], eph);
    const uint32_t sa = row_addr + (uint32_t)es * kEpiSlotBytes;
    uint32_t rh[8], oh[8];                           // residual / output: block jj, row half i in register 2 jj + i
    if (p.res_mode) { ldmatrix_x4(sa + q0, rh); ldmatrix_x4(sa + q1, rh + 4); }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * c + jj;
      const int ch0 = tc.n0 + 8 * j;                 // warp-uniform; blocks past Cout are clipped by the TMA store
      const int ch = ch0 + cq;
      float2 bb = make_float2(0.f, 0.f);
      if (p.bias && ch0 < p.Cout) bb = make_float2(__ldg(p.bias + ch), __ldg(p.bias + ch + 1));
      float s = 0.f, q = 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float f0 = acc[4 * j + 2 * i] + bb.x, f1 = acc[4 * j + 2 * i + 1] + bb.y;
        if (p.alpha != 1.0f) { f0 *= p.alpha; f1 *= p.alpha; }
        if (p.res_mode) {
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(&rh[2 * jj + i]));
          f0 += r.x; f1 += r.y;
        }
        if (valid[i]) { s += f0 + f1; q += f0 * f0 + f1 * f1; }
        if (p.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
        const __half2 h = __floats2half2_rn(f0, f1);
        oh[2 * jj + i] = *reinterpret_cast<const uint32_t*>(&h);
      }
      if (p.gn_group && ch0 < p.Cout) {
        gsum += s; gsq += q;
        if (p.gn_group == 8 || (j & 1)) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            gsum += __shfl_xor_sync(0xffffffffu, gsum, o);
            gsq += __shfl_xor_sync(0xffffffffu, gsq, o);
          }
          if (lane == 0) {
            unsigned long long* part = gn_part[warp][(ch0 - tc.n0) / p.gn_group];
            part[0] = (unsigned long long)__float2ll_rn(gsum * kGnSumScale);
            part[1] = (unsigned long long)__float2ll_rn(gsq * kGnSqScale);
          }
          gsum = 0.f; gsq = 0.f;
        }
      }
    }
    stmatrix_x4(sa + q0, oh);
    stmatrix_x4(sa + q1, oh + 4);
    fence_proxy_async_smem();
    mbar_arrive(&epi_ready[wg * kEpiSlots + es]);
    if (++es == kEpiSlots) { es = 0; eph ^= 1; }
  }
}

// Box origin of warpgroup wg's 64 pixels of a tile: the lower / upper half of the patch rows, or of the 1 x 128 row.
__device__ __forceinline__ void epi_box_origin(const LevelDesc& L, int x0, int y0, int wg, int& x, int& y) {
  if (L.BW > 64) { x = x0 + 64 * wg; y = y0; }
  else { x = x0; y = y0 + wg * (L.BH >> 1); }
}

template <int N>
__global__ void __launch_bounds__(kThreads, 1) conv_gemm_kernel(const __grid_constant__ ConvParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ GnPart gn_part;                         // 4 KB beside the <= 220 KB of operand stages
  // the 128-byte swizzle atoms (8 rows x 128 B) must start on 1024-byte boundaries
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kBBytes = N * 128;                   // one B stage: N output channels x 64 k fp16
  constexpr uint32_t kStageBytes = kABytes + kBBytes;
  const int nstages = p.stages;
  uint8_t* epi_slots = smem;                         // [warpgroup][kEpiSlots] x 4 KB, 1024-byte aligned
  uint8_t* sA = smem + kEpiBytes;
  uint8_t* sB = sA + (size_t)nstages * kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sB + (size_t)nstages * kBBytes);
  uint64_t* empty_bar = full_bar + nstages;
  uint64_t* epi_full = empty_bar + nstages;          // [warpgroup][slot]: residual landed / slot free (warp 9)
  uint64_t* epi_ready = epi_full + 2 * kEpiSlots;    // [warpgroup][slot]: results written (the warpgroup's 128 threads)

  if (threadIdx.x == 0) {
    for (int i = 0; i < nstages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumerWarps); }
    for (int i = 0; i < 2 * kEpiSlots; ++i) { mbar_init(&epi_full[i], 1); mbar_init(&epi_ready[i], 128); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: the prologue above may overlap the tail of the previous kernel in the stream; from here
  // on we touch global memory, so wait for it to complete, and let the next kernel begin its own prologue.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  const int total_units = p.tiles_m * p.n_tiles_n;
  const int kblocks = p.num_taps * p.kb_per_tap;

  if (warp >= kProducerWarp) {
    // ===================== TMA producer (one lane) =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == kProducerWarp && lane == 0) {
      for (int i = 0; i < kMaxMaps; ++i) tma_prefetch_desc(&p.amap[i]);
      tma_prefetch_desc(&p.bmap);
      int s = 0;
      uint32_t ph = 0;
      const int kb_per_tap = p.kb_per_tap, num_taps = p.num_taps;
      for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
        const TileCoord tc = decode_tile(p, unit);
        const int map0 = p.lv[tc.lvl].map0;
        for (int t = 0; t < num_taps; ++t) {
          const CUtensorMap* am = &p.amap[map0 + p.tap_map[t]];
          const int ax = tc.x0 + p.tap_dx[t], ay = tc.y0 + p.tap_dy[t];
          int kcoord = t * kb_per_tap * 64;
          for (int kc = 0; kc < kb_per_tap; ++kc, kcoord += 64) {
            mbar_wait(&empty_bar[s], ph ^ 1);         // every consumer warp has finished reading stage s
            mbar_expect_tx(&full_bar[s], kStageBytes);
            tma_load_4d(sA + (size_t)s * kABytes, am, &full_bar[s], kc * 64, ax, ay, tc.img);
            tma_load_2d(sB + (size_t)s * kBBytes, &p.bmap, &full_bar[s], kcoord, tc.n0);
            if (++s == nstages) { s = 0; ph ^= 1; }
          }
        }
      }
    } else if (warp == kEpiWarp && lane == 0 && p.epi_tma) {
      // ===================== epilogue copies (one lane): the consumers' chunk sequence, kEpiSlots chunks ahead ==========
      // Step k stores the chunk that last used slot k % kEpiSlots (once both warpgroups have written it), waits until the
      // stores have read their slots, then fills the slot for chunk k: the residual by TMA, or just a release.  Chunk 0..
      // kEpiSlots-1 of a tile are thus loaded while the consumers still run its MMAs.  kEpiSlots extra steps store the
      // last chunks.
      __shared__ int4 pend[kEpiSlots];               // chunk in each slot: {channel, x0, y0, image * 8 + level}
      for (int l = 0; l < p.num_levels; ++l) tma_prefetch_desc(&p.omap[l]);
      if (p.res_mode) tma_prefetch_desc(&p.rmap);
      int s = 0, c = 0, nchunks = 0, filled = 0;
      uint32_t ph = 0;
      int unit = blockIdx.x;
      TileCoord tc = {};
      for (int step = 0;; ++step) {
        const bool fill = unit < total_units;
        if (!fill && step >= filled + kEpiSlots) break;
        if (step >= kEpiSlots && step - kEpiSlots < filled) {
          const int4 q = pend[s];
          const LevelDesc& L = p.lv[q.w & 7];
#pragma unroll
          for (int wg = 0; wg < 2; ++wg) {
            int x, y;
            epi_box_origin(L, q.y, q.z, wg, x, y);
            mbar_wait(&epi_ready[wg * kEpiSlots + s], ph ^ 1);
            tma_store_4d(&p.omap[q.w & 7], epi_slots + (wg * kEpiSlots + s) * kEpiSlotBytes, q.x, x, y, q.w >> 3);
          }
          bulk_commit();
        }
        if (fill) {
          if (c == 0) {
            tc = decode_tile(p, unit);
            nchunks = (min(N, p.Cout - tc.n0) + 31) >> 5;
          }
          bulk_wait_read_all();                        // the store above has read the slot
#pragma unroll
          for (int wg = 0; wg < 2; ++wg) {
            uint64_t* bar = &epi_full[wg * kEpiSlots + s];
            if (p.res_mode) {
              int x, y;
              epi_box_origin(p.lv[0], tc.x0, tc.y0, wg, x, y);
              mbar_expect_tx(bar, kEpiSlotBytes);      // out-of-bounds fill counts toward the bytes
              tma_load_4d(epi_slots + (wg * kEpiSlots + s) * kEpiSlotBytes, &p.rmap, bar, tc.n0 + 32 * c, x, y, tc.img);
            } else {
              mbar_arrive(bar);
            }
          }
          pend[s] = make_int4(tc.n0 + 32 * c, tc.x0, tc.y0, tc.img * 8 + tc.lvl);
          ++filled;
          if (++c == nchunks) { c = 0; unit += gridDim.x; }
        }
        if (++s == kEpiSlots) { s = 0; ph ^= 1; }
      }
      bulk_wait_read_all();                          // the slots stay allocated until the last store has read them
    }
  } else {
    // ===================== consumers: warpgroup wg computes pixels 64*wg .. 64*wg+63 of the tile =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int wg = warp >> 2;
    const uint32_t sA0 = smem_u32(sA) + (uint32_t)wg * (64 * 128), sB0 = smem_u32(sB);
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    int s = 0, es = 0;
    uint32_t ph = 0, eph = 0;
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
      const TileCoord tc = decode_tile(p, unit);
      int prev = -1;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&full_bar[s], ph);
        wgmma_fence();
        const uint64_t adesc = make_sdesc(sA0 + (uint32_t)s * kABytes);
        const uint64_t bdesc = make_sdesc(sB0 + (uint32_t)s * kBBytes);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          // advance 16 elements (32 B) along K inside the 128-byte swizzle atom: +2 in the >>4 start field
          wgmma_f16<N>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1 : 0);
        wgmma_commit();
        wgmma_wait<1>();                             // the previous k-block's MMAs are done: release its stage
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == nstages) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs<N / 2>(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      if (p.epi_tma)
        epilogue_tma<N>(p, tc, acc, wg, warp, lane, gn_part, smem_u32(epi_slots), epi_full, epi_ready, es, eph);
      else
        epilogue<N>(p, tc, acc, wg, warp, lane, gn_part);
      if (p.gn_group) gn_flush(p, tc, gn_part, N);
    }
  }
}

// ------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

static int encode_map(CUtensorMap* m, void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                      const uint32_t* box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return SMB_ECUDA; }
  cuuint64_t d[5]; cuuint64_t s[4]; cuuint32_t b[5]; cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; es[i] = 1; }
  for (int i = 0; i < rank - 1; ++i) s[i] = strides_bytes[i];
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, base, d, s, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu] strides=[%llu,%llu,%llu] box=[%u,%u,%u,%u]",
              (int)r, rank, (unsigned long long)d[0], (unsigned long long)d[1], (unsigned long long)(rank > 2 ? d[2] : 0),
              (unsigned long long)(rank > 3 ? d[3] : 0), (unsigned long long)s[0], (unsigned long long)(rank > 2 ? s[1] : 0),
              (unsigned long long)(rank > 3 ? s[2] : 0), b[0], b[1], rank > 2 ? b[2] : 0, rank > 3 ? b[3] : 0);
    return SMB_ECUDA;
  }
  return SMB_OK;
}

// Output (or same-shape residual) of one level as seen by the shared-memory epilogue: [N, H_out, W_out, pitch] fp16, the
// first Cout channels, in boxes of one consumer warpgroup's 64 pixels x 32 channels (rows past the level's edge and
// channels past Cout are clipped on store, zero-filled on load).
static int encode_epi_map(CUtensorMap* m, const void* base, const ConvParams& p, const LevelDesc& L, int pitch) {
  const uint64_t px = (uint64_t)pitch * 2;
  const uint64_t dims[4] = {(uint64_t)p.Cout, (uint64_t)L.W_out, (uint64_t)L.H_out, (uint64_t)p.n_img};
  const uint64_t strides[3] = {px, px * L.W_out, px * L.W_out * L.H_out};
  const uint32_t box[4] = {32, (uint32_t)(L.BW < 64 ? L.BW : 64), (uint32_t)(L.BH > 1 ? L.BH / 2 : 1), 1};
  return encode_map(m, const_cast<void*>(base), 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
}

}  // namespace smb

using namespace smb;

struct smb_conv_plan {
  ConvParams p;
  int grid;
  size_t smem_bytes;
  int has_bias, has_residual, gn_stats;
};

static int g_min_tiles = 48;
extern "C" int smb_conv_set_min_tiles(int min_tiles) {
  const int prev = g_min_tiles;
  g_min_tiles = min_tiles > 0 ? min_tiles : 48;
  return prev;
}

static int num_sms() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}

// choose the BH x BW = 128 patch with the fewest tiles (ties -> wider rows, better store coalescing)
static void choose_patch(int H, int W, int* BH, int* BW) {
  const int cand[5][2] = {{1, 128}, {2, 64}, {4, 32}, {8, 16}, {16, 8}};
  long best = -1;
  for (int i = 0; i < 5; ++i) {
    const long t = (long)cdiv(H, cand[i][0]) * cdiv(W, cand[i][1]);
    if (best < 0 || t < best) { best = t; *BH = cand[i][0]; *BW = cand[i][1]; }
  }
}

static int finish_plan(smb_conv_plan* pl, int Cout, int Ktotal, const void* weight) {
  ConvParams& p = pl->p;
  // N tile (a wgmma instruction shape, so one of 256 / 128 / 64): the largest that does not exceed Cout rounded up to 64
  // and still yields >= min_tiles tiles.  Small feature maps (few M tiles) are latency-bound per tile, so they are split
  // along N to occupy more SMs.  Weight rows past Cout are TMA zero fill, their columns are not stored.
  const int cand[3] = {256, 128, 64};
  const int cmax = (Cout + 63) / 64 * 64;
  int n_tile = 64;
  for (int i = 0; i < 3; ++i) {
    if (cand[i] > cmax) continue;
    if ((long)p.tiles_m * cdiv(Cout, cand[i]) >= g_min_tiles) { n_tile = cand[i]; break; }
  }
  p.n_tile = n_tile;
  p.n_tiles_n = cdiv(Cout, n_tile);
  const size_t stage = (size_t)kABytes + (size_t)n_tile * 128;
  p.stages = ring_stages(n_tile);
  pl->smem_bytes = kEpiBytes + (size_t)p.stages * (stage + 16) + 4 * kEpiSlots * 8 + 1024;   // + barriers + alignment slack
  // Shared-memory / TMA epilogue for fp16 outputs whose rows TMA can address (16-byte aligned bases and pitch) and whose
  // residual, if any, is the same-shape tensor of a single-level plan.
  p.epi_tma = !p.out_f32 && p.out_pitch % 8 == 0 && (p.res_mode == 0 || (p.res_mode == 1 && p.num_levels == 1));
  for (int l = 0; l < p.num_levels; ++l)
    if ((uintptr_t)p.lv[l].out % 16) p.epi_tma = 0;
  for (int l = 0; l < p.num_levels && p.epi_tma; ++l) {
    const int rc = encode_epi_map(&p.omap[l], p.lv[l].out, p, p.lv[l], p.out_pitch);
    if (rc) return rc;
  }
  // weights: [Cout, Ktotal] K-major
  uint64_t dims[2] = {(uint64_t)Ktotal, (uint64_t)Cout};
  uint64_t strides[1] = {(uint64_t)Ktotal * 2};
  uint32_t box[2] = {64, (uint32_t)n_tile};
  int rc = encode_map(&p.bmap, const_cast<void*>(weight), 2, dims, strides, box);
  if (rc) return rc;
  const int units = p.tiles_m * p.n_tiles_n;
  const int sms = num_sms();
  pl->grid = units < sms ? units : sms;
  return SMB_OK;
}

extern "C" int smb_conv_plan_create_multi(const smb_conv_desc_t* d, int num_levels, const smb_conv_level_t* levels,
                                          const void* weight, smb_conv_plan_t** plan_out) {
  SMB_CHECK_ARG(d && levels && weight && plan_out, "smb_conv_plan_create: null pointer");
  SMB_CHECK_ARG(num_levels >= 1 && num_levels <= kMaxLevels, "smb_conv_plan_create: num_levels=%d outside [1,%d]", num_levels, kMaxLevels);
  SMB_CHECK_ARG(d->Cin % 64 == 0 && d->Cin > 0, "smb_conv_plan_create: Cin=%d must be a multiple of 64", d->Cin);
  SMB_CHECK_ARG(d->Cout % 16 == 0 && d->Cout > 0, "smb_conv_plan_create: Cout=%d must be a multiple of 16", d->Cout);
  SMB_CHECK_ARG((d->kh == 1 && d->kw == 1 && d->pad == 0) || (d->kh == 3 && d->kw == 3 && d->pad == 1),
                "smb_conv_plan_create: only 1x1/p0 and 3x3/p1 kernels (got %dx%d pad %d)", d->kh, d->kw, d->pad);
  SMB_CHECK_ARG(d->stride == 1 || d->stride == 2, "smb_conv_plan_create: stride %d", d->stride);
  SMB_CHECK_ARG(d->stride == 1 || num_levels == 1, "smb_conv_plan_create: strided convolutions are single-level");
  const int in_pitch = d->in_pitch ? d->in_pitch : d->Cin;
  const int out_pitch = d->out_pitch ? d->out_pitch : d->Cout;
  SMB_CHECK_ARG(in_pitch % 8 == 0 && out_pitch % 4 == 0, "smb_conv_plan_create: bad pitches");
  SMB_CHECK_ARG(((uintptr_t)weight % 16) == 0, "smb_conv_plan_create: weight must be 16-byte aligned");
  smb_conv_plan* pl = new smb_conv_plan();
  memset(&pl->p, 0, sizeof(ConvParams));
  ConvParams& p = pl->p;
  const int k = d->kh, s = d->stride;
  p.n_img = d->N;
  p.num_levels = num_levels;
  p.num_taps = k * k; p.kb_per_tap = d->Cin / 64;
  p.Cout = d->Cout;
  p.out_pitch = out_pitch; p.out_f32 = (d->out_dtype == SMB_F32);
  p.alpha = 1.0f; p.relu = d->relu;
  p.res_mode = d->has_residual ? (d->residual_upsample ? 2 : 1) : 0;
  p.res_pitch = d->Cout;
  p.gn_group = d->gn_stats ? d->Cout / 32 : 0;
  pl->has_bias = d->has_bias; pl->has_residual = d->has_residual; pl->gn_stats = d->gn_stats;
  if (d->gn_stats && !(p.gn_group == 8 || p.gn_group == 16)) {
    set_error("smb_conv_plan_create: gn_stats needs Cout/32 in {8,16}");
    delete pl;
    return SMB_EINVAL;
  }
  const uint64_t px = (uint64_t)in_pitch * 2;       // bytes per pixel
  int rc = SMB_OK;
  int tile_start = 0;
  for (int l = 0; l < num_levels && rc == SMB_OK; ++l) {
    const smb_conv_level_t& lv = levels[l];
    LevelDesc& L = p.lv[l];
    const int H = lv.H, W = lv.W;
    if (!lv.in || !lv.out || H <= 0 || W <= 0 || ((uintptr_t)lv.in % 16) || ((uintptr_t)lv.out % 16) ||
        (d->has_residual && !lv.residual) || (d->gn_stats && !lv.gn_stats)) {
      set_error("smb_conv_plan_create: level %d has a null / misaligned pointer or empty shape", l);
      rc = SMB_EINVAL;
      break;
    }
    const int Ho = (H + 2 * d->pad - k) / s + 1, Wo = (W + 2 * d->pad - k) / s + 1;
    L.H_out = Ho; L.W_out = Wo;
    choose_patch(Ho, Wo, &L.BH, &L.BW);
    L.tiles_x = cdiv(Wo, L.BW); L.tiles_y = cdiv(Ho, L.BH);
    L.tile_start = tile_start;
    tile_start += d->N * L.tiles_x * L.tiles_y;
    L.out = lv.out; L.residual = (const __half*)lv.residual; L.gn_stats = (long long*)lv.gn_stats;
    L.res_h = lv.res_h; L.res_w = lv.res_w;
    const uint32_t box[4] = {64, (uint32_t)L.BW, (uint32_t)L.BH, 1};
    if (s == 1) {
      L.map0 = l;
      uint64_t dims[4] = {(uint64_t)d->Cin, (uint64_t)W, (uint64_t)H, (uint64_t)d->N};
      uint64_t strides[3] = {px, px * W, px * W * H};
      rc = encode_map(&p.amap[l], const_cast<void*>(lv.in), 4, dims, strides, box);
    } else {
      // stride 2: input (2*oy + r - pad, 2*ox + c - pad) -> parity-split views with doubled strides
      L.map0 = 0;
      for (int py = 0; py < 2 && rc == SMB_OK; ++py)
        for (int pxp = 0; pxp < 2 && rc == SMB_OK; ++pxp) {
          const int hp = (H - py + 1) / 2, wp = (W - pxp + 1) / 2;   // rows / cols of this parity
          uint64_t dims[4] = {(uint64_t)d->Cin, (uint64_t)(wp > 0 ? wp : 1), (uint64_t)(hp > 0 ? hp : 1), (uint64_t)d->N};
          uint64_t strides[3] = {px * 2, px * W * 2, px * W * H};
          const char* base = (const char*)lv.in + ((size_t)py * W + pxp) * px;
          rc = encode_map(&p.amap[py * 2 + pxp], const_cast<char*>(base), 4, dims, strides, box);
        }
    }
  }
  if (rc == SMB_OK) {
    p.tiles_m = tile_start;
    for (int i = (s == 1 ? num_levels : 4); i < kMaxMaps; ++i) p.amap[i] = p.amap[0];
    for (int r = 0; r < k; ++r)
      for (int c = 0; c < k; ++c) {
        const int t = r * k + c;
        if (s == 1) {
          p.tap_map[t] = 0; p.tap_dx[t] = c - d->pad; p.tap_dy[t] = r - d->pad;
        } else {
          const int oy = r - d->pad, ox = c - d->pad;            // input offset relative to 2*o
          const int py = ((oy % 2) + 2) % 2, pxp = ((ox % 2) + 2) % 2;
          p.tap_map[t] = py * 2 + pxp;
          p.tap_dy[t] = (oy - py) / 2;                           // exact: oy - py is even
          p.tap_dx[t] = (ox - pxp) / 2;
        }
      }
    rc = finish_plan(pl, d->Cout, k * k * d->Cin, weight);
  }
  if (rc != SMB_OK) { delete pl; return rc; }
  *plan_out = pl;
  return SMB_OK;
}

extern "C" int smb_conv_plan_create(const smb_conv_desc_t* d, const void* in, const void* weight, void* out,
                                    smb_conv_plan_t** plan_out) {
  SMB_CHECK_ARG(d, "smb_conv_plan_create: null desc");
  // single tensor; residual / gn_stats pointers are supplied at run time (placeholders keep the level non-null)
  smb_conv_level_t lv;
  lv.in = in; lv.out = out;
  lv.residual = d->has_residual ? out : nullptr;
  lv.gn_stats = d->gn_stats ? out : nullptr;
  lv.H = d->H; lv.W = d->W; lv.res_h = d->res_h; lv.res_w = d->res_w;
  return smb_conv_plan_create_multi(d, 1, &lv, weight, plan_out);
}

// 7x7/2 stem on the SPACE-TO-DEPTH image written by smb_image_to_s2d16 / smb_preprocess_u8_s2d:
//   q [N, H/2+3, W/2+4, 16] fp16, q(Y, X, (dy*2+dx)*4 + c) = padded pixel (2Y+dy, 2X+dx) channel c.
//   out(oy, ox) = sum_{a,b<4} sum_{dy,dx,c} w[2a+dy][2b+dx][c] * q(oy+a, ox+b, (dy,dx,c)) : a 4x4 stride-1 convolution
//   over 16 channels, K = 4 filter rows x (4 cells x 16 ch = 128 contiguous bytes) = 256 instead of the 448 of a
//   pixel-window form (7 rows x 8 pixels x 8 ch) - 43 % fewer operand bytes and MMAs.
extern "C" int smb_stem_plan_create_s2d(int N, int H, int W, const void* img_s2d16, const void* weight256, void* out,
                                        smb_conv_plan_t** plan_out) {
  SMB_CHECK_ARG(img_s2d16 && weight256 && out && plan_out, "smb_stem_plan_create_s2d: null pointer");
  SMB_CHECK_ARG(H % 2 == 0 && W % 2 == 0, "smb_stem_plan_create_s2d: H, W must be even (images are padded to /32)");
  smb_conv_plan* pl = new smb_conv_plan();
  memset(&pl->p, 0, sizeof(ConvParams));
  ConvParams& p = pl->p;
  LevelDesc& L = p.lv[0];
  const int Ho = H / 2, Wo = W / 2, Hq = H / 2 + 3, Wq = W / 2 + 4;
  p.n_img = N; p.num_levels = 1;
  L.H_out = Ho; L.W_out = Wo;
  choose_patch(Ho, Wo, &L.BH, &L.BW);
  L.tiles_x = cdiv(Wo, L.BW); L.tiles_y = cdiv(Ho, L.BH);
  L.tile_start = 0; L.map0 = 0; L.out = out;
  p.tiles_m = N * L.tiles_x * L.tiles_y;
  p.num_taps = 4; p.kb_per_tap = 1;
  p.Cout = 64;
  p.out_pitch = 64; p.out_f32 = 0; p.alpha = 1.f; p.relu = 1;
  p.gn_group = 0;
  pl->has_bias = 1;
  const uint64_t rowb = (uint64_t)Wq * 32;
  const uint32_t box[4] = {64, (uint32_t)L.BW, (uint32_t)L.BH, 1};
  uint64_t dims[4] = {64, (uint64_t)Wo, (uint64_t)Hq, (uint64_t)N};
  uint64_t strides[3] = {32, rowb, rowb * Hq};          // 1-cell step along x: overlapping 4-cell (128-byte) windows
  int rc = encode_map(&p.amap[0], const_cast<void*>(img_s2d16), 4, dims, strides, box);
  for (int i = 1; i < kMaxMaps; ++i) p.amap[i] = p.amap[0];
  for (int a = 0; a < 4; ++a) { p.tap_map[a] = 0; p.tap_dy[a] = a; p.tap_dx[a] = 0; }
  if (rc == SMB_OK) rc = finish_plan(pl, 64, 256, weight256);
  if (rc != SMB_OK) { delete pl; return rc; }
  *plan_out = pl;
  return SMB_OK;
}

extern "C" void smb_conv_plan_destroy(smb_conv_plan_t* plan) { delete plan; }

// Cap the persistent grid (e.g. to half the SMs) so that two independent convolutions captured on different streams
// can run side by side and fill each other's partial waves.
extern "C" int smb_conv_plan_set_max_ctas(smb_conv_plan_t* plan, int max_ctas) {
  SMB_CHECK_ARG(plan && max_ctas >= 1, "smb_conv_plan_set_max_ctas: bad argument");
  if (max_ctas < plan->grid) plan->grid = max_ctas;
  return SMB_OK;
}

extern "C" int smb_conv_run(const smb_conv_plan_t* plan, const float* bias, const void* residual, void* gn_stats,
                            float alpha, smb_stream_t stream) {
  SMB_CHECK_ARG(plan, "smb_conv_run: null plan");
  SMB_CHECK_ARG(!plan->has_bias || bias, "smb_conv_run: plan expects a bias");
  ConvParams p = plan->p;
  p.bias = plan->has_bias ? bias : nullptr;
  // single-level plans take residual / statistics pointers at run time; multi-level plans bake them per level
  if (p.num_levels == 1) {
    if (plan->has_residual) {
      SMB_CHECK_ARG(residual, "smb_conv_run: plan expects a residual");
      p.lv[0].residual = (const __half*)residual;
      // the residual's TMA map goes into this launch's parameters (a captured graph keeps them by value); a residual
      // TMA cannot address (not 16-byte aligned) takes the register epilogue
      if (p.epi_tma && p.res_mode == 1) {
        if ((uintptr_t)residual % 16) {
          p.epi_tma = 0;
        } else {
          const int rc = encode_epi_map(&p.rmap, residual, p, p.lv[0], p.res_pitch);
          if (rc) return rc;
        }
      }
    }
    if (plan->gn_stats) {
      SMB_CHECK_ARG(gn_stats, "smb_conv_run: plan expects a gn_stats buffer");
      p.lv[0].gn_stats = (long long*)gn_stats;
    }
  }
  p.alpha = alpha;
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    SMB_CUDA_OK(cudaFuncSetAttribute(conv_gemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    SMB_CUDA_OK(cudaFuncSetAttribute(conv_gemm_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
    SMB_CUDA_OK(cudaFuncSetAttribute(conv_gemm_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget));
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(plan->grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = plan->smem_bytes;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = p.n_tile == 256 ? cudaLaunchKernelEx(&cfg, conv_gemm_kernel<256>, p)
                  : p.n_tile == 128 ? cudaLaunchKernelEx(&cfg, conv_gemm_kernel<128>, p)
                                    : cudaLaunchKernelEx(&cfg, conv_gemm_kernel<64>, p);
  if (e != cudaSuccess) {
    set_error("conv_gemm_kernel launch failed: %s (grid=%d smem=%zu n_tile=%d stages=%d tiles_m=%d n_tiles_n=%d)",
              cudaGetErrorString(e), plan->grid, plan->smem_bytes, p.n_tile, p.stages, p.tiles_m, p.n_tiles_n);
    cudaGetLastError();
    return SMB_ECUDA;
  }
  SMB_LAUNCH_OK("conv_gemm_kernel");
  return SMB_OK;
}
