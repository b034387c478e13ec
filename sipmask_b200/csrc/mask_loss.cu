// SipMask's mask loss, forward and backward, fused: no [H, W, M] tensor is ever stored.
//
// Reference (SipMask-mmdetection/mmdet/, the same block in SipMask-VIS and SipMask-benchmark):
//   models/anchor_heads/sipmask_head.py:437-463     targets, Z_q = feat_mask @ cof_qᵀ, sigmoid, CropSplit, BCE, weighting
//   ops/crop/src/crop_split_cuda_kernel.cu:46-53    cell membership and cell index
//
// Per image b with M_b instances, per (pixel, instance n) with the pixel inside n's box (x1 <= w < x2, y1 <= h < y2):
//   cell = idx_h * 2 + idx_w                   (crop_split_cuda_kernel.cu:46-53, the +0.1 in double)
//   z    = sum_k X[k, h, w] * C[n, 32 * cell + k]    (fp32 fma chain, k = 0..31)
//   p    = 1 / (1 + expf(-z))                  (torch's CUDA sigmoid, IEEE fp32)
//   term = (t - 1) * max(log1p(-p), -100) - t * max(log(p), -100)   (torch's CUDA binary_cross_entropy)
//   loss[b] += term * w_n / (bw_n * bh_n * M_b)
//   dz   = ((c * (p - t)) / max((1 - p) * p, 1e-12)) * (1 - p) * p,  c = (((g_b * w_n) * (1 / M_b)) / bh_n) / bw_n
// dz is torch's BCE backward, CropSplit's backward (a copy) and sigmoid's backward in the order autograd applies them on
// the device (a division by the Python int M_b is a multiplication by its fp32 reciprocal there); a saturated p gives 0.
//
// Kernels:
//   mask_targets_kernel   gt masks -> bit planes at the mask resolution (interpolate(0.5) -> pad/crop -> gt(0.5))
//   mask_loss_pixel<GRAD> one CTA per (image, 8 x 32 pixel tile): order-preserving list of the image's instances whose
//                         box touches the tile (ballot prefix counts), then per pixel the loss partial (forward) or
//                         d feat_masks (backward, every pixel written once, NCHW)
//   mask_loss_inst        one CTA per (instance, row split): d cofs partials over the instance's box, dz recomputed by
//                         the same device function
//   mask_loss_*_reduce    d cofs = sum of the splits in split order; loss[b] = b's tile partials in a fixed tree
// Every sum has a fixed order, so the loss and both gradients are the same bits on every run.
#include "common.cuh"

namespace smb {

constexpr int kMlTh = 8, kMlTw = 32;            // pixel tile (rows x columns), one thread per pixel
constexpr int kMlThreads = kMlTh * kMlTw;
constexpr int kMlBatch = 32;                    // listed instances whose coefficients are staged at once
constexpr int kMlCofPitch = 33;                 // per cell, padded so the four cells of a warp hit different banks
constexpr int kMlSplits = 8;                    // row splits per instance in the d cofs pass: a constant, so d cofs' bits
                                                // depend on the inputs only

struct MlBox {
  float x1, y1, x2, y2, roi_w, roi_h, coef;
  int gt_row;
};

struct MaskLossParams {
  const float* feat;          // [B, 32, H, W]
  const float* cofs;          // [M, 128]
  const float* boxes;         // [M, 4]
  const int* img_offsets;     // [B + 1]
  const uint32_t* targets;    // [G, H, words]
  const int* gt_rows;         // [M]
  const float* weights;       // [M]
  const float* g;             // [B] (backward) or null (forward)
  float* d_feat;              // [B, 32, H, W]
  double* loss_part;          // [B, tiles]
  float* cof_part;            // [kMlSplits, M, 128]
  int B, M, H, W, G, words, tiles_x, tiles_y;
};

// instance range of image b, clamped so that malformed offsets cannot index outside [0, M)
__device__ __forceinline__ void image_range(const MaskLossParams& p, int b, int* n0, int* n1) {
  const int a = min(max(p.img_offsets[b], 0), p.M);
  *n0 = a;
  *n1 = min(max(p.img_offsets[b + 1], a), p.M);
}

// The per-instance constants.  Forward: coef = w / (bw * bh * M_b) for the loss; backward: coef = c of the header.
__device__ __forceinline__ MlBox load_box(const MaskLossParams& p, int n, int Mb, float gb) {
  MlBox r;
  const float* b = p.boxes + (size_t)n * 4;
  r.x1 = b[0]; r.y1 = b[1]; r.x2 = b[2]; r.y2 = b[3];
  // (roi_x2-roi_x1+0.1)/num_cell: float difference, then double (0.1 is a double literal), narrowed to float
  r.roi_w = (float)(((double)(r.x2 - r.x1) + 0.1) / 2);
  r.roi_h = (float)(((double)(r.y2 - r.y1) + 0.1) / 2);
  const float bw = r.x2 - r.x1, bh = r.y2 - r.y1;      // center_size (sipmask_head.py:16-18)
  const float w = p.weights[n];
  if (p.g) {
    const float inv_m = 1.f / (float)Mb;
    r.coef = (((gb * w) * inv_m) / bh) / bw;
  } else {
    r.coef = (float)((double)w / ((double)bw * (double)bh * (double)Mb));
  }
  const int gr = p.gt_rows[n];
  r.gt_row = (gr >= 0 && gr < p.G) ? gr : -1;          // a row outside the planes reads as an empty mask
  return r;
}

// -1 when pixel (h, w) lies outside the box, else its CropSplit cell (crop_split_cuda_kernel.cu:44-53)
__device__ __forceinline__ int cell_of(const MlBox& b, int h, int w) {
  const float hf = (float)h, wf = (float)w;
  if (!((wf >= b.x1) & (hf >= b.y1) & (wf < b.x2) & (hf < b.y2))) return -1;
  const int idx_w = (int)__fdiv_rn(wf - b.x1, b.roi_w);
  const int idx_h = (int)__fdiv_rn(hf - b.y1, b.roi_h);
  return min(max(idx_h * 2 + idx_w, 0), 3);
}

__device__ __forceinline__ float target_bit(const MaskLossParams& p, int gt_row, int h, int w) {
  if (gt_row < 0) return 0.f;
  const uint32_t word = p.targets[((size_t)gt_row * p.H + h) * p.words + (w >> 5)];
  return (float)((word >> (w & 31)) & 1u);
}

__device__ __forceinline__ float dot32(const float* x, const float* c) {
  float z = 0.f;
#pragma unroll
  for (int k = 0; k < 32; ++k) z = fmaf(x[k], c[k], z);
  return z;
}

__device__ __forceinline__ float sigmoid_ieee(float z) { return 1.f / (1.f + expf(-z)); }

__device__ __forceinline__ float bce_term(float p, float t) {
  const float l0 = fmaxf(logf(p), -100.f);
  const float l1 = fmaxf(log1pf(-p), -100.f);
  return ((t - 1.f) * l1) - (t * l0);
}

// the one place dz is computed: both backward passes call it with the same z, t and c
__device__ __forceinline__ float bce_dz(float z, float t, float c) {
  const float p = sigmoid_ieee(z);
  const float dp = (c * (p - t)) / fmaxf((1.f - p) * p, 1e-12f);
  return (dp * (1.f - p)) * p;
}

// ------------------------------------------------------------------------------------------------- pixel pass
template <bool GRAD>
__global__ void __launch_bounds__(kMlThreads) mask_loss_pixel_kernel(const __grid_constant__ MaskLossParams p) {
  __shared__ MlBox s_box[kMlBatch];
  __shared__ float s_cof[kMlBatch][4 * kMlCofPitch];
  __shared__ int s_list[kMlThreads];
  __shared__ int s_wcount[kMlThreads / 32];
  __shared__ double s_red[kMlThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const int y0 = blockIdx.y * kMlTh, x0 = blockIdx.x * kMlTw;
  const int h = y0 + warp, w = x0 + lane;
  const bool in_map = h < p.H && w < p.W;
  const size_t HW = (size_t)p.H * p.W;
  const float* xb = p.feat + (size_t)b * 32 * HW + (size_t)h * p.W + w;
  float x[32], dx[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    x[k] = in_map ? __ldg(xb + k * HW) : 0.f;
    dx[k] = 0.f;
  }
  int n_begin, n_end;
  image_range(p, b, &n_begin, &n_end);
  const int Mb = n_end - n_begin;
  const float gb = GRAD ? p.g[b] : 0.f;
  const float tx0 = (float)x0, tx1 = (float)(min(x0 + kMlTw, p.W) - 1);
  const float ty0 = (float)y0, ty1 = (float)(min(y0 + kMlTh, p.H) - 1);
  double lsum = 0.0;

  for (int c0 = n_begin; c0 < n_end; c0 += kMlThreads) {
    // ---- order-preserving list of the chunk's instances whose box touches the tile
    const int n = c0 + threadIdx.x;
    bool hit = false;
    if (n < n_end) {
      const float* bx = p.boxes + (size_t)n * 4;
      hit = (tx1 >= bx[0]) & (tx0 < bx[2]) & (ty1 >= bx[1]) & (ty0 < bx[3]);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    __syncthreads();                                    // previous chunk done with s_list / s_wcount
    if (lane == 0) s_wcount[warp] = __popc(bal);
    __syncthreads();
    int base = 0, cnt = 0;
#pragma unroll
    for (int i = 0; i < kMlThreads / 32; ++i) {
      base += i < warp ? s_wcount[i] : 0;
      cnt += s_wcount[i];
    }
    if (hit) s_list[base + __popc(bal & ((1u << lane) - 1u))] = n;
    // ---- the listed instances, kMlBatch at a time
    for (int j0 = 0; j0 < cnt; j0 += kMlBatch) {
      const int nb = min(kMlBatch, cnt - j0);
      __syncthreads();                                  // s_list written / previous batch consumed
      if (threadIdx.x < nb) s_box[threadIdx.x] = load_box(p, s_list[j0 + threadIdx.x], Mb, gb);
      for (int e = threadIdx.x; e < nb * 128; e += kMlThreads) {
        const int j = e >> 7, k = e & 127;
        s_cof[j][(k >> 5) * kMlCofPitch + (k & 31)] = __ldg(p.cofs + (size_t)s_list[j0 + j] * 128 + k);
      }
      __syncthreads();
      if (in_map) {
        for (int j = 0; j < nb; ++j) {
          const MlBox bx = s_box[j];
          const int cell = cell_of(bx, h, w);
          if (cell < 0) continue;
          const float* cf = &s_cof[j][cell * kMlCofPitch];
          const float z = dot32(x, cf);
          const float t = target_bit(p, bx.gt_row, h, w);
          if (GRAD) {
            const float dz = bce_dz(z, t, bx.coef);
#pragma unroll
            for (int k = 0; k < 32; ++k) dx[k] = fmaf(dz, cf[k], dx[k]);
          } else {
            lsum += (double)bce_term(sigmoid_ieee(z), t) * (double)bx.coef;
          }
        }
      }
    }
  }

  if (GRAD) {
    if (in_map) {
      float* db = p.d_feat + (size_t)b * 32 * HW + (size_t)h * p.W + w;
#pragma unroll
      for (int k = 0; k < 32; ++k) db[k * HW] = dx[k];
    }
  } else {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
    if (lane == 0) s_red[warp] = lsum;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int i = 0; i < kMlThreads / 32; ++i) s += s_red[i];
      p.loss_part[(size_t)b * p.tiles_x * p.tiles_y + blockIdx.y * p.tiles_x + blockIdx.x] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------------- instance pass
// CTA (n, s): rows s * per .. of the instance's box clipped to the map; for each cell q, the threads stride over the
// pixels of those rows in the cell, accumulate dz * X[k] and reduce in a fixed tree.  Writes cof_part[s][n][128].
__global__ void __launch_bounds__(kMlThreads) mask_loss_inst_kernel(const __grid_constant__ MaskLossParams p) {
  __shared__ float s_cof[128];
  __shared__ float s_red[kMlThreads / 32][32];
  __shared__ MlBox s_box;
  __shared__ int s_ok;
  const int n = blockIdx.x, split = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    int lo = 0, hi = p.B;                               // image b with img_offsets[b] <= n < img_offsets[b + 1]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (p.img_offsets[mid] <= n) lo = mid; else hi = mid;
    }
    int n0, n1;
    image_range(p, lo, &n0, &n1);
    s_ok = (n >= n0 && n < n1) ? lo : -1;
    if (s_ok >= 0) s_box = load_box(p, n, n1 - n0, p.g[lo]);
  }
  if (threadIdx.x < 128) s_cof[threadIdx.x] = __ldg(p.cofs + (size_t)n * 128 + threadIdx.x);
  __syncthreads();
  const int b = s_ok;
  float* out = p.cof_part + ((size_t)split * p.M + n) * 128;
  const MlBox bx = s_box;
  int r0 = 0, r1 = 0, c0 = 0, c1 = 0;
  if (b >= 0 && bx.x1 < bx.x2 && bx.y1 < bx.y2) {      // false for NaN boxes as well
    // a superset of the box's pixels, clipped to the map; cell_of decides membership
    const float fy1 = fminf(fmaxf(bx.y1, -1.f), (float)p.H), fy2 = fminf(fmaxf(bx.y2, -1.f), (float)p.H);
    const float fx1 = fminf(fmaxf(bx.x1, -1.f), (float)p.W), fx2 = fminf(fmaxf(bx.x2, -1.f), (float)p.W);
    const int ylo = max((int)floorf(fy1), 0), yhi = min((int)ceilf(fy2), p.H);
    c0 = max((int)floorf(fx1), 0);
    c1 = min((int)ceilf(fx2), p.W);
    if (yhi > ylo && c1 > c0) {
      const int per = (yhi - ylo + kMlSplits - 1) / kMlSplits;
      r0 = min(ylo + split * per, yhi);
      r1 = min(r0 + per, yhi);
    }
  }
  const int cols = c1 - c0;
  const int npix = (r1 > r0 && cols > 0) ? (r1 - r0) * cols : 0;
  const size_t HW = (size_t)p.H * p.W;
  const float* xb = b >= 0 ? p.feat + (size_t)b * 32 * HW : p.feat;
  for (int q = 0; q < 4; ++q) {
    float acc[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) acc[k] = 0.f;
    for (int i = threadIdx.x; i < npix; i += kMlThreads) {
      const int h = r0 + i / cols, w = c0 + i % cols;
      if (cell_of(bx, h, w) != q) continue;
      float x[32];
      const float* px = xb + (size_t)h * p.W + w;
#pragma unroll
      for (int k = 0; k < 32; ++k) x[k] = __ldg(px + k * HW);
      const float dz = bce_dz(dot32(x, s_cof + q * 32), target_bit(p, bx.gt_row, h, w), bx.coef);
#pragma unroll
      for (int k = 0; k < 32; ++k) acc[k] = fmaf(dz, x[k], acc[k]);
    }
    // fixed-order reduction: a butterfly within each warp, then the warps in order
#pragma unroll
    for (int k = 0; k < 32; ++k) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
    }
    __syncthreads();                                    // previous cell's s_red consumed
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 32; ++k) s_red[warp][k] = acc[k];
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      float s = 0.f;
      for (int i = 0; i < kMlThreads / 32; ++i) s += s_red[i][threadIdx.x];
      out[q * 32 + threadIdx.x] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------------- reductions
__global__ void mask_loss_cof_reduce_kernel(const float* __restrict__ part, int M, float* __restrict__ d_cofs) {
  const size_t total = (size_t)M * 128;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float s = part[i];
    for (int sp = 1; sp < kMlSplits; ++sp) s += part[(size_t)sp * total + i];
    d_cofs[i] = s;
  }
}

// loss[b]: image b's tile partials, thread i taking tiles i, i + 256, ... in order, then a fixed tree over the threads
__global__ void __launch_bounds__(256) mask_loss_sum_kernel(const double* __restrict__ part, int tiles,
                                                            float* __restrict__ loss) {
  __shared__ double s[256];
  const int b = blockIdx.x;
  double a = 0.0;
  for (int t = threadIdx.x; t < tiles; t += 256) a += part[(size_t)b * tiles + t];
  s[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[b] = (float)s[0];
}

// ------------------------------------------------------------------------------------------------- targets
// F.interpolate(scale_factor=0.5, bilinear, align_corners=False) samples output pixel (y, x) at source (2y + 0.5,
// 2x + 0.5): the mean of the 2 x 2 block, so on {0, 1} masks gt(0.5) <=> at least 3 of the 4 are set.  The interpolated
// size is (Hf / 2, Wf / 2) rounded down; rows and columns beyond it (the pad) are 0.
__global__ void mask_targets_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ planes, int G, int H,
                                    int W, int words, uint32_t* __restrict__ bits) {
  const size_t total = (size_t)G * H * words;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int word = (int)(i % words);
    const int y = (int)((i / words) % H);
    const int g = (int)(i / ((size_t)words * H));
    const long long off = planes[3 * g], Hf = planes[3 * g + 1], Wf = planes[3 * g + 2];
    uint32_t v = 0u;
    if (y < Hf / 2) {
      const uint8_t* r0 = src + off + (size_t)(2 * y) * Wf;
      const uint8_t* r1 = r0 + Wf;
      const int xe = (int)min((long long)W, Wf / 2);
      for (int bit = 0; bit < 32; ++bit) {
        const int x = word * 32 + bit;
        if (x >= xe) break;
        const int cnt = (r0[2 * x] != 0) + (r0[2 * x + 1] != 0) + (r1[2 * x] != 0) + (r1[2 * x + 1] != 0);
        v |= (uint32_t)(cnt >= 3) << bit;
      }
    }
    bits[i] = v;
  }
}

static unsigned grid_for(size_t n, int threads) {
  const size_t b = (n + threads - 1) / threads;
  return (unsigned)(b < 8192 ? (b > 0 ? b : 1) : 8192);
}

static size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

}  // namespace smb

using namespace smb;

extern "C" int smb_mask_targets(const void* src, const long long* planes, int G, int H, int W, uint32_t* bits,
                                smb_stream_t stream) {
  SMB_CHECK_ARG(G >= 0 && H > 0 && W > 0, "smb_mask_targets: bad shape G=%d H=%d W=%d", G, H, W);
  if (G == 0) return SMB_OK;
  SMB_CHECK_ARG(src && planes && bits, "smb_mask_targets: null pointer");
  const int words = (W + 31) / 32;
  const size_t total = (size_t)G * H * words;
  mask_targets_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)src, planes, G, H, W, words,
                                                                               bits);
  SMB_LAUNCH_OK("mask_targets_kernel");
  return SMB_OK;
}

extern "C" size_t smb_mask_loss_workspace_bytes(int B, int M, int H, int W) {
  if (B <= 0 || M < 0 || H <= 0 || W <= 0) return 0;
  const size_t tiles = (size_t)cdiv(H, kMlTh) * cdiv(W, kMlTw);
  return align256((size_t)B * tiles * sizeof(double)) + (size_t)kMlSplits * M * 128 * sizeof(float);
}

extern "C" int smb_mask_loss(const float* feat, const float* cofs, const float* boxes, const int* img_offsets,
                             const uint32_t* targets, int G, const int* gt_rows, const float* weights, const float* g,
                             int B, int M, int H, int W, float* loss, float* d_feat, float* d_cofs, void* workspace,
                             size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(B > 0 && M >= 0 && H > 0 && W > 0 && G >= 0, "smb_mask_loss: bad shape B=%d M=%d H=%d W=%d G=%d", B, M,
                H, W, G);
  SMB_CHECK_ARG((long long)B * 32 * H * W < (1ll << 31) && (long long)M * 128 * kMlSplits < (1ll << 31),
                "smb_mask_loss: tensor too large");
  SMB_CHECK_ARG(feat && img_offsets && workspace, "smb_mask_loss: null pointer");
  SMB_CHECK_ARG(M == 0 || (cofs && boxes && gt_rows && weights), "smb_mask_loss: null instance pointer");
  SMB_CHECK_ARG(G == 0 || targets, "smb_mask_loss: null targets");
  if (g) {
    SMB_CHECK_ARG(d_feat || d_cofs, "smb_mask_loss: backward needs d_feat or d_cofs");
  } else {
    SMB_CHECK_ARG(loss, "smb_mask_loss: forward needs loss");
  }
  SMB_CHECK_ARG(workspace_bytes >= smb_mask_loss_workspace_bytes(B, M, H, W), "smb_mask_loss: workspace too small");
  MaskLossParams p;
  memset(&p, 0, sizeof(p));
  p.feat = feat; p.cofs = cofs; p.boxes = boxes; p.img_offsets = img_offsets; p.targets = targets; p.gt_rows = gt_rows;
  p.weights = weights; p.g = g; p.d_feat = d_feat;
  p.B = B; p.M = M; p.H = H; p.W = W; p.G = G; p.words = (W + 31) / 32;
  p.tiles_x = cdiv(W, kMlTw); p.tiles_y = cdiv(H, kMlTh);
  const size_t tiles = (size_t)p.tiles_x * p.tiles_y;
  p.loss_part = (double*)workspace;
  p.cof_part = (float*)((char*)workspace + align256((size_t)B * tiles * sizeof(double)));
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 pgrid(p.tiles_x, p.tiles_y, B);
  if (!g) {
    mask_loss_pixel_kernel<false><<<pgrid, kMlThreads, 0, s>>>(p);
    SMB_LAUNCH_OK("mask_loss_pixel_kernel<loss>");
    mask_loss_sum_kernel<<<B, 256, 0, s>>>(p.loss_part, (int)tiles, loss);
    SMB_LAUNCH_OK("mask_loss_sum_kernel");
    return SMB_OK;
  }
  if (d_feat) {
    mask_loss_pixel_kernel<true><<<pgrid, kMlThreads, 0, s>>>(p);
    SMB_LAUNCH_OK("mask_loss_pixel_kernel<grad>");
  }
  if (d_cofs && M > 0) {
    mask_loss_inst_kernel<<<dim3(M, kMlSplits), kMlThreads, 0, s>>>(p);
    SMB_LAUNCH_OK("mask_loss_inst_kernel");
    mask_loss_cof_reduce_kernel<<<grid_for((size_t)M * 128, 256), 256, 0, s>>>(p.cof_part, M, d_cofs);
    SMB_LAUNCH_OK("mask_loss_cof_reduce_kernel");
  }
  return SMB_OK;
}
