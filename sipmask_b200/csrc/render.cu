// Detections drawn onto uint8 HWC images on the device: the mask blending and box outlines of the reference's
// show_result (SipMask-mmdetection/mmdet/apis/inference.py:119-184 for images, SipMask-VIS/mmdet/models/detectors/
// base.py:90-192 for video frames), one launch for a whole batch.
//
// CTA (band, image): rows [band * rows, band * rows + rows) of one image.
//   1. The CTA builds the image's draw list in shared memory: which detections are drawn, in the reference's order, with
//      their plane, colour and box (O(count^2) comparisons; count <= 1024, 100 for the engine's records).
//   2. The band's pixels are staged in shared memory (one contiguous span of the HWC image).
//   3. One thread per 32-pixel word of a row walks the draw list: a zero mask word is skipped, each set bit blends its
//      pixel; then the box outlines of the draw list overwrite their pixels in green.
//   4. The band is written to dst once.
// Bytes per image: the image read and written once, plus every drawn detection's mask words of the image's rows.
#include "common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kMaxRows = 8;                   // rows per CTA: about one 32-pixel word per thread, at most this many
constexpr int kPixelSmem = 48 * 1024;         // staged band bytes a CTA may use at most (one row if a row is wider)
constexpr int kBatch = 8;                     // mask words a thread loads before it blends any (loads in flight)

struct Launch {
  const smb_render_img_t* imgs;
  const uint32_t* bits;
  int max_num, cap_h, words;
  const float* det;
  const int64_t* labels;
  const int* count;
  const int32_t* obj_ids;
  const uint8_t* palette;
  int palette_rows;
  int rule;
  float score_thr;
  int boxes;
  int max_h, max_w, rows;
};

struct __align__(16) Box {
  int xa, xb, ya, yb;
};

__device__ __forceinline__ uint8_t blend(int rule, uint32_t c, uint32_t p) {
  if (rule == SMB_RENDER_IMAGES) return (uint8_t)((c + p) >> 1);        // uint8(p * 0.5 + c * 0.5), exact in float64
  // uint8(c * 0.6 + p * 0.4) in float64, each product and the sum rounded on its own (numpy has no FMA), truncated
  return (uint8_t)__double2int_rz(__dadd_rn(__dmul_rn((double)c, 0.6), __dmul_rn((double)p, 0.4)));
}

// numpy's astype(np.int32) of a float32 corner: truncation toward zero (saturating at the int32 range, NaN -> 0)
__device__ __forceinline__ int corner(float v) { return __float2int_rz(v); }

// the box colour, (0, 255, 0) in the image's channel order
__device__ __forceinline__ void green(uint8_t* p) { p[0] = 0; p[1] = 255; p[2] = 0; }

__global__ void __launch_bounds__(kThreads) render_kernel(Launch L) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int n = blockIdx.y, tid = threadIdx.x;
  const smb_render_img_t im = L.imgs[n];
  const int h = im.h, w = im.w, y0 = blockIdx.x * L.rows;
  // a row outside the launch's bounds (or an empty / filler row) is left untouched
  if (h <= 0 || w <= 0 || h > L.max_h || w > L.max_w || y0 >= h || !im.src || !im.dst) return;
  const int mx = L.max_num;
  Box* s_box = (Box*)smem;                                      // [mx] the draw list, in draw order
  int* s_plane = (int*)(s_box + mx);                            // [mx]
  uint32_t* s_col = (uint32_t*)(s_plane + mx);                  // [mx] colour, channel c in byte c
  int* s_key = (int*)(s_col + mx);                              // [mx] label (images) or object id (videos)
  float* s_score = (float*)(s_key + mx);                        // [mx]
  int* s_src = (int*)(s_score + mx);                            // [mx] the detection whose box and plane are drawn
  int* s_sel = s_src + mx;                                      // [mx] drawn or not, per detection
  uint8_t* s_px = (uint8_t*)(s_sel + mx);                       // the band's pixels, HWC
  __shared__ int s_nd;

  int cnt = L.count[n];
  cnt = cnt < 0 ? 0 : (cnt > mx ? mx : cnt);
  const float* det = L.det + (int64_t)n * mx * 5;
  for (int i = tid; i < cnt; i += kThreads) {
    s_key[i] = L.rule == SMB_RENDER_IMAGES ? (int)L.labels[(int64_t)n * mx + i] : L.obj_ids[(int64_t)n * mx + i];
    s_score[i] = det[i * 5 + 4];
  }
  if (tid == 0) s_nd = 0;
  __syncthreads();
  for (int i = tid; i < cnt; i += kThreads) {
    const int key = s_key[i];
    int src = i;
    bool sel;
    if (L.rule == SMB_RENDER_IMAGES) {
      sel = s_score[i] > L.score_thr;
    } else {
      // bbox2result_with_id is a dict: an id's entry sits where the id first appears and holds its last detection
      sel = key >= 0;
      for (int j = 0; j < i && sel; ++j) sel = s_key[j] != key;
      for (int j = i + 1; j < cnt && sel; ++j)
        if (s_key[j] == key) src = j;
      sel = sel && s_score[src] > L.score_thr;
    }
    s_src[i] = src;
    s_sel[i] = sel;
  }
  __syncthreads();
  for (int i = tid; i < cnt; i += kThreads) {
    if (!s_sel[i]) continue;
    const int key = s_key[i], src = s_src[i];
    int pos = 0;
    if (L.rule == SMB_RENDER_IMAGES) {
      // np.vstack(bbox_result): class-major, detection order kept within a class
      for (int j = 0; j < cnt; ++j) pos += s_sel[j] && (s_key[j] < key || (s_key[j] == key && j < i));
    } else {
      for (int j = 0; j < i; ++j) pos += s_sel[j];
    }
    atomicAdd(&s_nd, 1);
    const int rows = L.palette_rows;
    const uint8_t* c = L.palette + 3 * (((key % rows) + rows) % rows);
    s_col[pos] = (uint32_t)c[0] | ((uint32_t)c[1] << 8) | ((uint32_t)c[2] << 16);
    s_plane[pos] = src;
    const int xs = corner(det[src * 5 + 0]), ys = corner(det[src * 5 + 1]);
    const int xe = corner(det[src * 5 + 2]), ye = corner(det[src * 5 + 3]);
    Box b;
    b.xa = min(xs, xe); b.xb = max(xs, xe); b.ya = min(ys, ye); b.yb = max(ys, ye);
    s_box[pos] = b;
  }
  __syncthreads();
  const int nd = s_nd;
  if (nd == 0 && im.src == im.dst) return;                      // nothing drawn in place: the image stays as it is

  const int nrows = min(L.rows, h - y0);
  const int64_t pitch = 3 * (int64_t)w;
  const int64_t span = nrows * pitch;
  const uint8_t* gsrc = im.src + y0 * pitch;
  for (int64_t e = tid; e < span; e += kThreads) s_px[e] = gsrc[e];
  __syncthreads();

  if (nd > 0) {
    const int wpr = (w + 31) >> 5;
    const uint32_t* planes = L.bits + (int64_t)n * mx * L.cap_h * L.words;
    const int64_t plane_words = (int64_t)L.cap_h * L.words;
    for (int t = tid; t < nrows * wpr; t += kThreads) {
      const int r = t / wpr, wd = t - r * wpr, y = y0 + r;
      const int xlo = wd * 32, xhi = min(xlo + 32, w) - 1;
      uint8_t* px = s_px + r * pitch + 3 * xlo;
      const uint32_t valid = xhi - xlo == 31 ? 0xffffffffu : (1u << (xhi - xlo + 1)) - 1u;
      if (y < L.cap_h && wd < L.words) {
        const uint32_t* word = planes + (int64_t)y * L.words + wd;
        for (int d0 = 0; d0 < nd; d0 += kBatch) {
          uint32_t ms[kBatch];
#pragma unroll
          for (int u = 0; u < kBatch; ++u) ms[u] = d0 + u < nd ? __ldg(word + s_plane[d0 + u] * plane_words) & valid : 0u;
#pragma unroll
          for (int u = 0; u < kBatch; ++u) {
            uint32_t m = ms[u];
            if (!m) continue;
            const uint32_t c = s_col[d0 + u];
            do {
              const int b = __ffs(m) - 1;
              m &= m - 1;
              uint8_t* p = px + 3 * b;
              p[0] = blend(L.rule, c & 0xff, p[0]);
              p[1] = blend(L.rule, (c >> 8) & 0xff, p[1]);
              p[2] = blend(L.rule, (c >> 16) & 0xff, p[2]);
            } while (m);
          }
        }
      }
      if (L.boxes) {
        // cv2.rectangle(thickness=1, LINE_8): the border of the inclusive rectangle, clipped to the image
        for (int d = 0; d < nd; ++d) {
          const Box b = s_box[d];
          if (y < b.ya || y > b.yb) continue;
          if (y == b.ya || y == b.yb) {
            for (int x = max(b.xa, xlo); x <= min(b.xb, xhi); ++x) green(px + 3 * (x - xlo));
          } else {
            if (b.xa >= xlo && b.xa <= xhi) green(px + 3 * (b.xa - xlo));
            if (b.xb >= xlo && b.xb <= xhi) green(px + 3 * (b.xb - xlo));
          }
        }
      }
    }
    __syncthreads();
  }
  uint8_t* gdst = im.dst + y0 * pitch;
  for (int64_t e = tid; e < span; e += kThreads) gdst[e] = s_px[e];
}

inline size_t list_bytes(int max_num) { return (size_t)max_num * (sizeof(Box) + 6 * sizeof(int)); }

}  // namespace

extern "C" int smb_render_dev(const smb_render_img_t* imgs, int N, int max_h, int max_w, const uint32_t* mask_bits,
                              int max_num, int cap_h, int words, const float* det, const int64_t* labels, const int* count,
                              const int32_t* obj_ids, const uint8_t* palette, int palette_rows, int rule, float score_thr,
                              int boxes, smb_stream_t stream) {
  SMB_CHECK_ARG(N >= 0 && N <= 65535 && max_h >= 0 && max_w >= 0 && max_num >= 1 && max_num <= SMB_RENDER_MAX_NUM &&
                    cap_h >= 0 && words >= 0 && palette_rows >= 1,
                "smb_render_dev: bad sizes (N %d, max %dx%d, max_num %d, cap_h %d, words %d, palette_rows %d)", N, max_h,
                max_w, max_num, cap_h, words, palette_rows);
  SMB_CHECK_ARG(rule == SMB_RENDER_IMAGES || rule == SMB_RENDER_VIDEO, "smb_render_dev: unknown rule %d", rule);
  if (N == 0 || max_h == 0 || max_w == 0) return SMB_OK;
  SMB_CHECK_ARG(imgs && count && det && palette && (mask_bits || cap_h == 0 || words == 0) &&
                    (rule == SMB_RENDER_IMAGES ? labels != nullptr : obj_ids != nullptr),
                "smb_render_dev: null pointer");
  int dev = 0, optin = 0;
  SMB_CUDA_OK(cudaGetDevice(&dev));
  SMB_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t fixed = list_bytes(max_num), row = 3 * (size_t)max_w;
  int rows = kThreads / ((max_w + 31) / 32);
  rows = rows > kMaxRows ? kMaxRows : rows;
  rows = rows > (int)(kPixelSmem / row) ? (int)(kPixelSmem / row) : rows;
  rows = rows < 1 ? 1 : rows;
  const size_t smem = fixed + rows * row;
  SMB_CHECK_ARG(smem + 1024 <= (size_t)optin, "smb_render_dev: a %d-pixel row needs %zu bytes of shared memory, %d per block",
                max_w, smem, optin);
  static smb::DeviceOnce once;
  if (once.first()) SMB_CUDA_OK(cudaFuncSetAttribute(render_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - 1024));
  Launch L;
  L.imgs = imgs;
  L.bits = mask_bits; L.max_num = max_num; L.cap_h = cap_h; L.words = words;
  L.det = det; L.labels = labels; L.count = count; L.obj_ids = obj_ids;
  L.palette = palette; L.palette_rows = palette_rows;
  L.rule = rule; L.score_thr = score_thr; L.boxes = boxes != 0;
  L.max_h = max_h; L.max_w = max_w; L.rows = rows;
  const dim3 grid((unsigned)((max_h + rows - 1) / rows), (unsigned)N);
  render_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>(L);
  SMB_LAUNCH_OK("render_kernel");
  return SMB_OK;
}
