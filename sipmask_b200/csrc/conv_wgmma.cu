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
#include "sm90.cuh"

namespace smb {

constexpr int kMaxTaps = 9;
constexpr int kMaxMaps = 8;
constexpr int kMaxLevels = 5;
constexpr int kConsumerWarps = 8;
// + a producer warpgroup: warp 8 issues the operand TMA loads, warp 9 the epilogue's residual loads and output stores
// (epi_tma plans), warp 10 the GroupNorm statistics' global atomics (GN plans), warp 11 exists only so that the CTA is
// whole warpgroups, which setmaxnreg needs to move registers from the producer (40 per thread) to the consumers (232
// instead of 168)
constexpr int kThreads = 32 * (kConsumerWarps + 4);
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kEpiWarp = kConsumerWarps + 1;
constexpr int kGnWarp = kConsumerWarps + 2;
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

#ifdef SMB_CONV_PHASES
// Timing build only (tools/conv_tile_phases.py compiles it; the library never does).  clock64 stamps per CTA:
//   [0, 4): globaltimer / clock64 at the first and last stamp (cycles -> ns);
//   [4, 8): warp 9: cycles blocked in bulk_wait_read, cycles blocked on epi_ready, stores committed, fills;  [8]: tiles;
//   [9, 11): warp 9: cycles from a store step's first epi_ready wait to its commit (waits included), cycles issuing fills
//   (residual TMA load or release arrival);
//   [16 + (sample * 2 + wg) * kPhaseTile, + kPhaseTile): the sample-th recorded tile of consumer warpgroup wg (every
//   phase_every-th tile of the CTA): mainloop start, last wgmma_wait<0> returned, epilogue end, cycles blocked in epi_full
//   waits, cycles in the GroupNorm statistics' shuffle reductions, cycles handing the tile's statistics to warp 10 (the
//   wait for the previous tile's flush and the arrival), and per link of the chunk chain summed over the tile's chunks:
//   slot ready -> results in registers (ldmatrix, arithmetic, GroupNorm partials), stmatrix, proxy fence, slot arrival;
//   last, the cycles staging the tile's bias before its first chunk.
constexpr int kPhaseSamples = 64;
constexpr int kPhaseTile = 11;
constexpr int kPhaseWords = 16 + kPhaseSamples * 2 * kPhaseTile;
__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define PHASE(...) __VA_ARGS__
#else
#define PHASE(...)
#endif

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
  PHASE(unsigned long long* phases; int phase_every;)
};
static_assert(sizeof(ConvParams) <= 4096, "ConvParams must fit the 4 KB kernel-parameter space");

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
// a compile-time value carried by a function argument's type (selects a template specialisation from a run-time flag)
template <typename T, T V>
struct Const { static constexpr T value = V; };

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

// GroupNorm partials of one tile: [consumer warp][group within the N tile (<= 256 / 8)][sum, sum of squares], fixed point.
// Warp 10 sums the eight warps' partials of a tile and issues one global atomic per (group, statistic): per-warp atomics
// on the same few addresses serialised in L2 when every SM ran a tower convolution.  Integer sums are exact, so the
// statistics are the same bits in any order.
typedef unsigned long long GnPart[kConsumerWarps][32][2];

// GroupNorm statistics of one 32-channel chunk of a consumer warp (pre-activation values of its 16 rows): v[2 g + s] is
// the lane's fp32 partial of group g of the chunk, statistic s (sum, sum of squares); NV = 8 for 8-channel groups (four
// per chunk), 4 for 16-channel groups (two; each already the sum of its two 8-channel blocks, in block order).  Writes
// the warp's sums to part[g][s] in 64-bit fixed point.
// A reduce-scatter: xor 16 exchanges NV / 2 values (a lane keeps the upper half when its bit 4 is set and sends the other
// half), xor 8 exchanges NV / 4, ..., and once one value is left the remaining offsets are butterfly steps; lane l ends
// with the warp's sum of value (l >> 2) & 7 (NV = 8) or (l >> 3) & 3 (NV = 4), and lanes with those bits alone convert
// it.  9 (NV = 8) or 5 (NV = 4) shuffles per chunk instead of 5 per value.  The sums are the same bits as a full
// butterfly per value: every value still goes through the pairing tree with offsets 16, 8, 4, 2, 1, step o adding the
// lane's running sum and that of lane ^ o, and fp32 addition is commutative, so each running sum is the same bits in
// every lane that holds it; so is every fixed-point partial.
template <int NV>
__device__ __forceinline__ void gn_reduce_chunk(float* v, int lane, unsigned long long (*part)[2]) {
  int n = NV;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    if (n > 1) {
      n >>= 1;
      const bool hi = lane & o;
#pragma unroll
      for (int i = 0; i < n; ++i) {
        const float send = hi ? v[i] : v[i + n];
        v[i] = (hi ? v[i + n] : v[i]) + __shfl_xor_sync(0xffffffffu, send, o);
      }
    } else {
      v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
    }
  }
  constexpr int kShift = NV == 8 ? 2 : 3;
  const int idx = (lane >> kShift) & (NV - 1);
  if ((lane & ((1 << kShift) - 1)) == 0)
    part[idx >> 1][idx & 1] = (unsigned long long)__float2ll_rn(v[0] * ((idx & 1) ? kGnSqScale : kGnSumScale));
}

// Collects one 8-channel block's statistics (s, q: the lane's sum and sum of squares over its valid rows) into the
// chunk's v[] of gn_reduce_chunk; after the chunk's last block (jj = 3) reduces them into the warp's partials of chunk c.
// group: channels per GroupNorm group, 8 or 16 (a constant where the caller is specialised on it).
__device__ __forceinline__ void gn_block(int group, float* v, int jj, float s, float q, int lane,
                                         unsigned long long (*part)[2], int c PHASE(, unsigned& shfl)) {
  if (group == 8) {
    v[2 * jj] = s; v[2 * jj + 1] = q;
  } else {                                           // 16-channel groups: blocks 2g and 2g + 1 summed in that order
    const int g = jj >> 1;
    v[2 * g] = (jj & 1) ? v[2 * g] + s : s;
    v[2 * g + 1] = (jj & 1) ? v[2 * g + 1] + q : q;
  }
  if (jj == 3) {
    PHASE(const unsigned w0 = clock();)
    if (group == 8) gn_reduce_chunk<8>(v, lane, part + 4 * c);
    else gn_reduce_chunk<4>(v, lane, part + 2 * c);
    PHASE(shfl += clock() - w0;)
  }
}

// Epilogue of one consumer warp: rows (warp%4)*16 + lane/4 + {0, 8} of its warpgroup's 64-pixel half of the tile.
// Per element: acc + bias, * alpha, + residual -> GroupNorm statistics (pre-activation) -> ReLU -> fp16 / fp32 store.
template <int N>
__device__ __forceinline__ void epilogue(const ConvParams& p, const TileCoord& tc, const float* acc, int wg, int warp, int lane,
                                         GnPart& gn_part PHASE(, unsigned& shfl)) {
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
  float gv[8];                                       // GroupNorm partials of the current 32-channel chunk (gn_block)
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
      // per-(image, group) sum / sum of squares of the conv output (pre-activation): fp32 over the warp's 16 rows, then
      // 64-bit fixed point, summed over the tile by warp 10 (integer sums: bit-reproducible whatever the tile order).
      // GroupNorm plans have Cout 256 or 512, so every 32-channel chunk is whole.
      if (p.gn_group) gn_block(p.gn_group, gv, j & 3, s, q, lane, gn_part[warp], j >> 2 PHASE(, shfl));
    }
  }
}

// The same per-element arithmetic and GroupNorm partials as epilogue(), for epi_tma plans, one 32-channel chunk at a time
// through the warpgroup's slot ring (slot es, phase eph, carried across tiles): wait until warp 9 has filled the slot
// (residual) or freed it, ldmatrix the residual, stmatrix the fp16 results over it, hand the slot to warp 9's TMA store.
// Slot layout: pixel row r (0..63, accumulator row order) at r * 64 bytes, its 16-byte channel quad q at
// ((q ^ (r >> 1) & 3) * 16): the TMA 64-byte swizzle (address bits [4,6) ^= bits [7,9)).
// Specialised on the plan's residual (RES), GroupNorm group size (GN: 0 = no statistics, 8, 16) and ReLU: the epilogue is
// bound by the consumers' instruction issue (two warps per scheduler, about 0.2 µs per chunk), and with these as run-time
// flags every chunk issued the predicated residual conversions, statistics arithmetic and ReLU of every plan.
template <int N, bool RES, int GN, bool RELU>
__device__ __forceinline__ void epilogue_tma(const ConvParams& p, const TileCoord& tc, const float* acc, int wg, int warp,
                                             int lane, GnPart& gn_part, const float* tile_bias, uint32_t slots,
                                             uint64_t* epi_full, uint64_t* epi_ready, int& es, uint32_t& eph
                                             PHASE(, long long* link, unsigned& shfl)) {
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
  // bias of 8-channel block jj of chunk cc, from the tile's copy in shared memory (tile_bias: zero past Cout): four
  // shared loads at fixed offsets per chunk, where eight predicated global loads with their bounds tests cost 0.6-0.7 µs
  // per N = 256 tile (DESIGN.md §6).  The slot wait's memory clobber keeps every load after it, so a chunk's bias is
  // read one chunk ahead, before that wait.
  auto chunk_bias = [&](int cc, float2* b) {
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) b[jj] = *reinterpret_cast<const float2*>(tile_bias + 8 * (4 * cc + jj) + cq);
  };
  float2 bnext[4];
  chunk_bias(0, bnext);
  float gv[8];                                       // GroupNorm partials of the chunk (gn_block)
#pragma unroll
  for (int c = 0; c < N / 32; ++c) {
    if (c >= nchunks) break;
    float2 bias[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) bias[jj] = bnext[jj];
    if (c + 1 < nchunks) chunk_bias(c + 1, bnext);
    PHASE(const long long w0 = clock64();)
    mbar_wait(&epi_full[wg * kEpiSlots + es], eph);
    PHASE(long long w1 = clock64(); link[0] += w1 - w0;)
    const uint32_t sa = row_addr + (uint32_t)es * kEpiSlotBytes;
    uint32_t rh[8], oh[8];                           // residual / output: block jj, row half i in register 2 jj + i
    if (RES) { ldmatrix_x4(sa + q0, rh); ldmatrix_x4(sa + q1, rh + 4); }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * c + jj;
      const float2 bb = bias[jj];                      // blocks past Cout are clipped by the TMA store
      float s = 0.f, q = 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float f0 = acc[4 * j + 2 * i] + bb.x, f1 = acc[4 * j + 2 * i + 1] + bb.y;
        if (p.alpha != 1.0f) { f0 *= p.alpha; f1 *= p.alpha; }
        if (RES) {
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(&rh[2 * jj + i]));
          f0 += r.x; f1 += r.y;
        }
        if (GN && valid[i]) { s += f0 + f1; q += f0 * f0 + f1 * f1; }
        if (RELU) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
        const __half2 h = __floats2half2_rn(f0, f1);
        oh[2 * jj + i] = *reinterpret_cast<const uint32_t*>(&h);
      }
      if (GN) gn_block(GN, gv, jj, s, q, lane, gn_part[warp], c PHASE(, shfl));   // whole chunks (Cout 256 / 512)
    }
    // timing build: the results are pinned before the stamp so that the arithmetic is counted before stmatrix
    PHASE(asm volatile("" ::"r"(oh[0]), "r"(oh[1]), "r"(oh[2]), "r"(oh[3]), "r"(oh[4]), "r"(oh[5]), "r"(oh[6]), "r"(oh[7]));
          long long w2 = clock64(); link[1] += w2 - w1;)
    stmatrix_x4(sa + q0, oh);
    stmatrix_x4(sa + q1, oh + 4);
    PHASE(w1 = clock64(); link[2] += w1 - w2;)
    fence_proxy_async_smem();
    PHASE(w2 = clock64(); link[3] += w2 - w1;)
    mbar_arrive(&epi_ready[wg * kEpiSlots + es]);
    PHASE(link[4] += clock64() - w2;)
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
  // GroupNorm plans: gn_bar[0] = a tile's partials written (every consumer thread), gn_bar[1] = summed by warp 10 (its 32
  // lanes), so the consumers may overwrite them with the next tile's
  __shared__ uint64_t gn_bar[2];
  // epi_tma plans: the bias of a tile's N channels (zero past Cout), by tile parity.  Consumer thread t loads channel t at
  // the tile's start and writes it after the mainloop; a named barrier of the 256 consumer threads publishes the tile's
  // copy, and the parity keeps it apart from the previous tile's, which a warp may still be reading.
  __shared__ float bias_s[2][256];
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
    mbar_init(&gn_bar[0], 32 * kConsumerWarps);
    mbar_init(&gn_bar[1], 32);
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
      PHASE(long long read_wait = 0, ready_wait = 0, stores = 0, store_cyc = 0, fill_cyc = 0;)
      int unit = blockIdx.x;
      TileCoord tc = {};
      for (int step = 0;; ++step) {
        const bool fill = unit < total_units;
        if (!fill && step >= filled + kEpiSlots) break;
        if (step >= kEpiSlots && step - kEpiSlots < filled) {
          const int4 q = pend[s];
          const LevelDesc& L = p.lv[q.w & 7];
          PHASE(const long long s0 = clock64();)
#pragma unroll
          for (int wg = 0; wg < 2; ++wg) {
            int x, y;
            epi_box_origin(L, q.y, q.z, wg, x, y);
            PHASE(const long long w0 = clock64();)
            mbar_wait(&epi_ready[wg * kEpiSlots + s], ph ^ 1);
            PHASE(ready_wait += clock64() - w0;)
            tma_store_4d(&p.omap[q.w & 7], epi_slots + (wg * kEpiSlots + s) * kEpiSlotBytes, q.x, x, y, q.w >> 3);
          }
          bulk_commit();
          PHASE(++stores; store_cyc += clock64() - s0;)
        }
        if (fill) {
          if (c == 0) {
            tc = decode_tile(p, unit);
            nchunks = (min(N, p.Cout - tc.n0) + 31) >> 5;
          }
          PHASE(const long long w0 = clock64();)
          bulk_wait_read_all();                        // the store above has read the slot
          PHASE(const long long f0 = clock64(); read_wait += f0 - w0;)
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
          PHASE(fill_cyc += clock64() - f0;)
          pend[s] = make_int4(tc.n0 + 32 * c, tc.x0, tc.y0, tc.img * 8 + tc.lvl);
          ++filled;
          if (++c == nchunks) { c = 0; unit += gridDim.x; }
        }
        if (++s == kEpiSlots) { s = 0; ph ^= 1; }
      }
      bulk_wait_read_all();                          // the slots stay allocated until the last store has read them
      PHASE(if (p.phases) {
              unsigned long long* r = p.phases + (size_t)blockIdx.x * kPhaseWords;
              r[4] = read_wait; r[5] = ready_wait; r[6] = stores; r[7] = filled; r[9] = store_cyc; r[10] = fill_cyc;
            })
    } else if (warp == kGnWarp && p.gn_group) {
      // ===================== GroupNorm statistics (whole warp): the consumers' tile sequence =====================
      // Once every consumer thread has written its partials of a tile: sum the eight warps' partials, one global atomic per
      // (group, statistic), then release the partials.  The consumers hand a tile over with an mbarrier arrival and go on
      // to their next mainloop: no CTA barrier on their path, and the next tile's partials are written an entire
      // mainloop later, long after this warp has read these.
      uint32_t ph = 0;
      for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
        const TileCoord tc = decode_tile(p, unit);
        const int ngl = min(N, p.Cout - tc.n0) / p.gn_group, ngroups = p.Cout / p.gn_group;
        unsigned long long* st = reinterpret_cast<unsigned long long*>(p.lv[tc.lvl].gn_stats) +
                                 ((size_t)tc.img * ngroups + tc.n0 / p.gn_group) * 2;
        mbar_wait(&gn_bar[0], ph);
        for (int e = lane; e < 2 * ngl; e += 32) {
          unsigned long long v = 0;
#pragma unroll
          for (int w = 0; w < kConsumerWarps; ++w) v += gn_part[w][e >> 1][e & 1];
          atomicAdd(st + e, v);
        }
        mbar_arrive(&gn_bar[1]);
        ph ^= 1;
      }
    }
  } else {
    // ===================== consumers: warpgroup wg computes pixels 64*wg .. 64*wg+63 of the tile =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int wg = warp >> 2;
    const uint32_t sA0 = smem_u32(sA) + (uint32_t)wg * (64 * 128), sB0 = smem_u32(sB);
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    int s = 0, es = 0, tpar = 0;
    uint32_t ph = 0, eph = 0, gph = 0;
    PHASE(unsigned long long* const rec = p.phases + (size_t)blockIdx.x * kPhaseWords;
          const bool stamp = p.phases && (threadIdx.x & 127) == 0;
          if (threadIdx.x == 0 && p.phases) { rec[0] = globaltimer(); rec[1] = clock64(); }
          int tile_i = 0;)
    for (int unit = blockIdx.x; unit < total_units; unit += gridDim.x) {
      const TileCoord tc = decode_tile(p, unit);
      PHASE(const int sample = tile_i % p.phase_every == 0 ? tile_i / p.phase_every : kPhaseSamples;
            const long long t_main = clock64(); long long link[5] = {0, 0, 0, 0, 0}, bias_cyc = 0;
            unsigned shfl = 0, hand = 0; ++tile_i;)
      // this thread's channel of the tile's bias (bias_s): loaded here, so that the load is long done when it is written
      float bias_t = 0.f;
      if (p.epi_tma && p.bias && threadIdx.x < N && tc.n0 + (int)threadIdx.x < p.Cout) bias_t = __ldg(p.bias + tc.n0 + threadIdx.x);
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
      PHASE(const long long t_mma = clock64();)
      fence_regs<N / 2>(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      PHASE(unsigned t_hand = clock();)
      if (p.gn_group) mbar_wait(&gn_bar[1], gph ^ 1);    // warp 10 has summed the previous tile's partials
      PHASE(hand = clock() - t_hand;)
      if (p.epi_tma) {
        PHASE(const long long b0 = clock64();)
        if (threadIdx.x < N) bias_s[tpar][threadIdx.x] = bias_t;
        asm volatile("bar.sync 1, %0;" ::"n"(32 * kConsumerWarps) : "memory");
        PHASE(bias_cyc = clock64() - b0;)
        // the plan's specialisation of epilogue_tma (RES, GN, RELU), chosen from the parameters of the launch
        auto run = [&](auto res, auto gn, auto relu) {
          epilogue_tma<N, decltype(res)::value, decltype(gn)::value, decltype(relu)::value>(
              p, tc, acc, wg, warp, lane, gn_part, bias_s[tpar], smem_u32(epi_slots), epi_full, epi_ready, es,
              eph PHASE(, link, shfl));
        };
        auto with_relu = [&](auto res, auto gn) {
          if (p.relu) run(res, gn, Const<bool, true>()); else run(res, gn, Const<bool, false>());
        };
        auto with_gn = [&](auto res) {
          if (p.gn_group == 8) with_relu(res, Const<int, 8>());
          else if (p.gn_group == 16) with_relu(res, Const<int, 16>());
          else with_relu(res, Const<int, 0>());
        };
        if (p.res_mode) with_gn(Const<bool, true>()); else with_gn(Const<bool, false>());
        tpar ^= 1;
      } else
        epilogue<N>(p, tc, acc, wg, warp, lane, gn_part PHASE(, shfl));
      PHASE(t_hand = clock();)
      if (p.gn_group) { mbar_arrive(&gn_bar[0]); gph ^= 1; }
      PHASE(hand += clock() - t_hand;
            if (stamp && sample < kPhaseSamples) {
              unsigned long long* r = rec + 16 + (sample * 2 + wg) * kPhaseTile;
              r[0] = t_main; r[1] = t_mma; r[2] = clock64(); r[3] = link[0]; r[4] = shfl; r[5] = hand;
              r[6] = link[1]; r[7] = link[2]; r[8] = link[3]; r[9] = link[4]; r[10] = bias_cyc;
            })
    }
    PHASE(if (threadIdx.x == 0 && p.phases) { rec[2] = globaltimer(); rec[3] = clock64(); rec[8] = tile_i; })
  }
}

// ------------------------------------------------------------------------------------------- host side
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
        (d->has_residual && (!lv.residual || (uintptr_t)lv.residual % 4)) || (d->gn_stats && !lv.gn_stats)) {
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
          // A parity with no rows (H == 1, py == 1) or no columns (W == 1, pxp == 1) is encoded with one so that its map
          // is valid, but that row / column is the next image's or lies past the tensor.  Its taps read at offset 1
          // instead: every box row / column is then at a coordinate >= 1, past the map's single one, so TMA fills zeros.
          if ((levels[0].H - py + 1) / 2 == 0) p.tap_dy[t] = 1;
          if ((levels[0].W - pxp + 1) / 2 == 0) p.tap_dx[t] = 1;
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

static_assert(SMB_CONV_MAX_LEVELS == kMaxLevels, "smb_conv_plan_info_t holds every level of a plan");

extern "C" int smb_conv_plan_info(const smb_conv_plan_t* plan, smb_conv_plan_info_t* info) {
  SMB_CHECK_ARG(plan && info, "smb_conv_plan_info: null pointer");
  const ConvParams& p = plan->p;
  memset(info, 0, sizeof(*info));
  info->num_levels = p.num_levels; info->tiles_m = p.tiles_m;
  info->n_tile = p.n_tile; info->n_tiles_n = p.n_tiles_n; info->stages = p.stages; info->epi_tma = p.epi_tma;
  info->grid = plan->grid; info->smem_bytes = (int)plan->smem_bytes;
  for (int l = 0; l < p.num_levels; ++l) {
    const LevelDesc& L = p.lv[l];
    info->H_out[l] = L.H_out; info->W_out[l] = L.W_out;
    info->BH[l] = L.BH; info->BW[l] = L.BW; info->tiles_x[l] = L.tiles_x; info->tiles_y[l] = L.tiles_y;
  }
  return SMB_OK;
}

// Cap the persistent grid (e.g. to half the SMs) so that two independent convolutions captured on different streams
// can run side by side and fill each other's partial waves.
extern "C" int smb_conv_plan_set_max_ctas(smb_conv_plan_t* plan, int max_ctas) {
  SMB_CHECK_ARG(plan && max_ctas >= 1, "smb_conv_plan_set_max_ctas: bad argument");
  if (max_ctas < plan->grid) plan->grid = max_ctas;
  return SMB_OK;
}

#ifdef SMB_CONV_PHASES
// Timing build only: launches after this call stamp into buf (kPhaseWords 64-bit words per CTA, zeroed by the caller),
// every every-th tile of each CTA; buf = null stops stamping.
static unsigned long long* g_phases = nullptr;
static int g_phase_every = 1;
extern "C" int smb_conv_phase_buffer(void* buf, int every) {
  g_phases = (unsigned long long*)buf;
  g_phase_every = every > 0 ? every : 1;
  return kPhaseWords;
}
#endif

extern "C" int smb_conv_run(const smb_conv_plan_t* plan, const float* bias, const void* residual, void* gn_stats,
                            float alpha, smb_stream_t stream) {
  SMB_CHECK_ARG(plan, "smb_conv_run: null plan");
  SMB_CHECK_ARG(!plan->has_bias || bias, "smb_conv_run: plan expects a bias");
  ConvParams p = plan->p;
  PHASE(p.phases = g_phases; p.phase_every = g_phase_every;)
  p.bias = plan->has_bias ? bias : nullptr;
  // single-level plans take residual / statistics pointers at run time; multi-level plans bake them per level
  if (p.num_levels == 1) {
    if (plan->has_residual) {
      SMB_CHECK_ARG(residual, "smb_conv_run: plan expects a residual");
      // the register epilogue reads the residual as __half2 pairs of even channels
      SMB_CHECK_ARG((uintptr_t)residual % 4 == 0, "smb_conv_run: residual must be 4-byte aligned");
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
