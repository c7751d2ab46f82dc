// GPU input pipeline (SURVEY 8f rank 2): the step immediately upstream of the first conv kernel.
// Replaces, for a whole batch of decoded frames in ONE launch, what the reference does per image on the CPU:
//   transform/resize/image.py:23-24 / label.py:25-31  `rescale`: cv2.resize(image, (width, height)) (INTER_LINEAR, uint8) and the
//                                                      box scaling yx *= (height / _height, width / _width)
//   transform/image.py:27-29                          BGR2RGB
// (ToTensor's 1/255 and the HWC -> network layout change are already fused into yb_conv0_u8_bn_leaky_pool_fwd.)
//
// Exactness contract: bit-identical to cv2.resize (OpenCV 4.x, 8-bit, INTER_LINEAR) -- the arithmetic lives in the
// reference's third-party dependency, so it is restated here from its published algorithm (modules/imgproc resize.cpp,
// the 8-bit fixed-point path) and pinned by fixtures generated with cv2 itself:
//   fx = float((dx + 0.5) * (src_w / dst_w) - 0.5) (double arithmetic, one rounding to float); sx = floor(fx); fx -= sx;
//   horizontally sx < 0 -> (sx, fx) = (0, 0), sx >= src_w - 1 -> (src_w - 1, 0); vertically the two rows are clamped
//   to the image but the fraction is kept; coefficients are rounded to 11-bit fixed point with round-half-even
//   (saturate_cast<short>(c * 2048)); the row pass is S[sx] * a0 + S[sx + 1] * a1 in int, the column pass
//   (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2.
#include "yb_common.h"
#include <stdint.h>

namespace yb {

struct ResizeCoef { int s0, s1, a0, a1; };

__device__ __forceinline__ ResizeCoef resize_coef(int d, int n_dst, int n_src, bool clamp_fraction) {
  const double scale = static_cast<double>(n_src) / static_cast<double>(n_dst);
  float f = static_cast<float>((static_cast<double>(d) + 0.5) * scale - 0.5);
  int s = static_cast<int>(floorf(f));
  f -= static_cast<float>(s);
  ResizeCoef c;
  if (clamp_fraction) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= n_src - 1) { f = 0.f; s = n_src - 1; }
    c.s0 = s;
    c.s1 = s + 1 < n_src ? s + 1 : n_src - 1;
  } else {
    c.s0 = s < 0 ? 0 : (s < n_src ? s : n_src - 1);
    c.s1 = s + 1 < 0 ? 0 : (s + 1 < n_src ? s + 1 : n_src - 1);
  }
  c.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  c.a1 = __float2int_rn(__fmul_rn(f, 2048.f));
  return c;
}

// one thread per output pixel (3 channels); blockIdx.y = image
__global__ void __launch_bounds__(256) resize_u8_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ src_off,
                                                        const int* __restrict__ src_hw, uint8_t* __restrict__ dst, int height, int width,
                                                        int swap_rb) {
  const int img = blockIdx.y;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= height * width) return;
  const int dy = idx / width, dx = idx - dy * width;
  const int sh = src_hw[2 * img], sw = src_hw[2 * img + 1];
  const uint8_t* s = src + src_off[img];
  const ResizeCoef cx = resize_coef(dx, width, sw, true);
  const ResizeCoef cy = resize_coef(dy, height, sh, false);
  const uint8_t* r0 = s + static_cast<long long>(cy.s0) * sw * 3;
  const uint8_t* r1 = s + static_cast<long long>(cy.s1) * sw * 3;
  uint8_t out[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = static_cast<int>(r0[cx.s0 * 3 + c]) * cx.a0 + static_cast<int>(r0[cx.s1 * 3 + c]) * cx.a1;
    const int h1 = static_cast<int>(r1[cx.s0 * 3 + c]) * cx.a0 + static_cast<int>(r1[cx.s1 * 3 + c]) * cx.a1;
    int v = (((cy.a0 * (h0 >> 4)) >> 16) + ((cy.a1 * (h1 >> 4)) >> 16) + 2) >> 2;
    v = v < 0 ? 0 : (v > 255 ? 255 : v);
    out[c] = static_cast<uint8_t>(v);
  }
  uint8_t* d = dst + (static_cast<long long>(img) * height * width + idx) * 3;
  d[0] = swap_rb ? out[2] : out[0];
  d[1] = out[1];
  d[2] = swap_rb ? out[0] : out[2];
}

// boxes [B, G, 2] (y, x): yx *= (height / src_h, width / src_w) in float32 exactly as numpy does it (label.py:27-30)
__global__ void rescale_boxes_kernel(float* __restrict__ yx_min, float* __restrict__ yx_max, const int* __restrict__ src_hw, int batch, int slots,
                                     int height, int width) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch * slots) return;
  const int img = i / slots;
  // np.array([height / _height, width / _width], np.float32): a double division rounded once more to float32
  const float sy = static_cast<float>(static_cast<double>(height) / static_cast<double>(src_hw[2 * img]));
  const float sx = static_cast<float>(static_cast<double>(width) / static_cast<double>(src_hw[2 * img + 1]));
  yx_min[2 * i] = __fmul_rn(yx_min[2 * i], sy); yx_min[2 * i + 1] = __fmul_rn(yx_min[2 * i + 1], sx);
  yx_max[2 * i] = __fmul_rn(yx_max[2 * i], sy); yx_max[2 * i + 1] = __fmul_rn(yx_max[2 * i + 1], sx);
}

// torchvision.transforms.ToTensor on a batch (transform/image.py + the `transform_tensor` step of utils/data.py:120-121):
// uint8 NHWC [B,H,W,3] -> fp32 NCHW [B,3,H,W], value / 255 (IEEE division, as `.div(255)` does).  The inference path never
// needs this (the first conv kernel reads the uint8 frames directly); the training forward and its first-layer weight
// gradient read the fp32 NCHW image the reference hands them.
__global__ void totensor_u8_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, int batch, int hw) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;     // one thread per pixel
  if (idx >= static_cast<long long>(batch) * hw) return;
  const long long img = idx / hw, pix = idx - img * hw;
  const uint8_t* s = src + idx * 3;
  float* d = dst + img * 3 * hw + pix;
#pragma unroll
  for (int c = 0; c < 3; ++c) d[static_cast<long long>(c) * hw] = __fdiv_rn(static_cast<float>(s[c]), 255.f);
}

// The configured tensor transform on a batch (transform.TensorTransform: ToTensor, then zero or more per-channel Normalize), compiled into
// a table: uint8 NHWC [B,H,W,3] -> fp32 NCHW [B,3,H,W], dst = lut[c][src].  The table holds torchvision's own result for every byte value,
// so the output is torchvision's bit for bit.
__global__ void totensor_lut_u8_kernel(const uint8_t* __restrict__ src, const float* __restrict__ lut, float* __restrict__ dst, int batch, int hw) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;     // one thread per pixel
  if (idx >= static_cast<long long>(batch) * hw) return;
  const long long img = idx / hw, pix = idx - img * hw;
  const uint8_t* s = src + idx * 3;
  float* d = dst + img * 3 * hw + pix;
#pragma unroll
  for (int c = 0; c < 3; ++c) d[static_cast<long long>(c) * hw] = __ldg(lut + c * 256 + s[c]);
}

// Augmented form (the default training resize `resize_train = transform.resize.label.RandomCrop`, config.ini:48, after the optional
// `transform.augmentation.RandomFlipHorizontally`, config.ini:47): out = cv2.resize(crop(flip(image))).  Both are pure index transforms on
// the SOURCE of the same bit-exact resize: a flipped image's column j is column (w - 1 - j) (cv2.flip(image, 1), augmentation.py:87-95),
// the crop image[y0:y1, x0:x1] (resize/label.py:73) an offset window.  crop: int[B][4] = (y0, x0, y1, x1) in the (flipped) frame or NULL;
// flip: uint8[B] or NULL.
__global__ void __launch_bounds__(256) resize_aug_u8_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ src_off,
                                                            const int* __restrict__ src_hw, const int* __restrict__ crop,
                                                            const uint8_t* __restrict__ flip, uint8_t* __restrict__ dst, int height, int width,
                                                            int swap_rb) {
  const int img = blockIdx.y;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= height * width) return;
  const int dy = idx / width, dx = idx - dy * width;
  const int sw = src_hw[2 * img + 1];
  int y0 = 0, x0 = 0, eh = src_hw[2 * img], ew = sw;
  if (crop != nullptr) { y0 = crop[4 * img]; x0 = crop[4 * img + 1]; eh = crop[4 * img + 2] - y0; ew = crop[4 * img + 3] - x0; }
  const bool fl = flip != nullptr && flip[img] != 0;
  const uint8_t* s = src + src_off[img];
  const ResizeCoef cx = resize_coef(dx, width, ew, true);
  const ResizeCoef cy = resize_coef(dy, height, eh, false);
  const uint8_t* r0 = s + static_cast<long long>(y0 + cy.s0) * sw * 3;
  const uint8_t* r1 = s + static_cast<long long>(y0 + cy.s1) * sw * 3;
  const int c0 = fl ? sw - 1 - (x0 + cx.s0) : x0 + cx.s0;
  const int c1 = fl ? sw - 1 - (x0 + cx.s1) : x0 + cx.s1;
  uint8_t out[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = static_cast<int>(r0[c0 * 3 + c]) * cx.a0 + static_cast<int>(r0[c1 * 3 + c]) * cx.a1;
    const int h1 = static_cast<int>(r1[c0 * 3 + c]) * cx.a0 + static_cast<int>(r1[c1 * 3 + c]) * cx.a1;
    int v = (((cy.a0 * (h0 >> 4)) >> 16) + ((cy.a1 * (h1 >> 4)) >> 16) + 2) >> 2;
    v = v < 0 ? 0 : (v > 255 ? 255 : v);
    out[c] = static_cast<uint8_t>(v);
  }
  uint8_t* d = dst + (static_cast<long long>(img) * height * width + idx) * 3;
  d[0] = swap_rb ? out[2] : out[0];
  d[1] = out[1];
  d[2] = swap_rb ? out[0] : out[2];
}

// boxes, in the reference's order and float32 arithmetic: flip (x' = w - x, min / max swapped; augmentation.py:91-94), crop
// (yx -= margin, the UN-truncated float32 margin; resize/label.py:74), scale by (height / crop_h, width / crop_w) (resize/label.py:27-30)
__global__ void augment_boxes_kernel(float* __restrict__ yx_min, float* __restrict__ yx_max, const int* __restrict__ src_hw, const int* __restrict__ crop,
                                     const float* __restrict__ margin, const uint8_t* __restrict__ flip, int batch, int slots, int height, int width) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch * slots) return;
  const int img = i / slots;
  float ymin = yx_min[2 * i], xmin = yx_min[2 * i + 1], ymax = yx_max[2 * i], xmax = yx_max[2 * i + 1];
  const int sw = src_hw[2 * img + 1];
  int eh = src_hw[2 * img], ew = sw;
  if (flip != nullptr && flip[img] != 0) {
    const float w = static_cast<float>(sw);
    const float t = __fsub_rn(w, xmin);
    xmin = __fsub_rn(w, xmax);
    xmax = t;
  }
  if (crop != nullptr) {
    eh = crop[4 * img + 2] - crop[4 * img]; ew = crop[4 * img + 3] - crop[4 * img + 1];
    const float my = margin[2 * img], mx = margin[2 * img + 1];
    ymin = __fsub_rn(ymin, my); xmin = __fsub_rn(xmin, mx); ymax = __fsub_rn(ymax, my); xmax = __fsub_rn(xmax, mx);
  }
  const float sy = static_cast<float>(static_cast<double>(height) / static_cast<double>(eh));
  const float sx = static_cast<float>(static_cast<double>(width) / static_cast<double>(ew));
  yx_min[2 * i] = __fmul_rn(ymin, sy); yx_min[2 * i + 1] = __fmul_rn(xmin, sx);
  yx_max[2 * i] = __fmul_rn(ymax, sy); yx_max[2 * i + 1] = __fmul_rn(xmax, sx);
}

int resize_aug_batch_u8(const void* src, const long long* src_off, const int* src_hw, const int* crop, const float* margin, const unsigned char* flip,
                        void* dst, int batch, int height, int width, int swap_rb, float* yx_min, float* yx_max, int slots, cudaStream_t stream) {
  YB_REQUIRE(src && src_off && src_hw && dst && batch > 0 && height > 0 && width > 0, "resize_aug_batch_u8: bad argument");
  YB_REQUIRE((yx_min == nullptr) == (yx_max == nullptr) && slots >= 0, "resize_aug_batch_u8: boxes come as a (yx_min, yx_max) pair");
  YB_REQUIRE(crop == nullptr || margin != nullptr || yx_min == nullptr, "resize_aug_batch_u8: cropping boxes needs the float margins");
  const int pixels = height * width;
  resize_aug_u8_kernel<<<dim3((pixels + 255) / 256, batch), 256, 0, stream>>>(static_cast<const uint8_t*>(src), src_off, src_hw, crop, flip,
                                                                              static_cast<uint8_t*>(dst), height, width, swap_rb);
  int rc = check_launch("resize_aug_u8_kernel");
  if (rc) return rc;
  if (yx_min != nullptr && slots > 0) {
    augment_boxes_kernel<<<(batch * slots + 127) / 128, 128, 0, stream>>>(yx_min, yx_max, src_hw, crop, margin, flip, batch, slots, height, width);
    rc = check_launch("augment_boxes_kernel");
  }
  return rc;
}

// ------------------------------------------------------------------------------------------------
// cv2.warpAffine(image, M, (dw, dh), flags=INTER_LINEAR, borderMode=BORDER_CONSTANT, borderValue=fill) for uint8 HWC frames, bit-exact:
// the arithmetic of the reference's `Rotator.__call__` (transform/augmentation.py:46-49, used by `random_rotate` :61-76) and of
// `transform.resize.image.fixed` (transform/resize/image.py:36-46; INTER_AREA is INTER_LINEAR inside warpAffine).  It lives in the
// reference's third-party dependency, so it is restated from OpenCV's published algorithm (imgproc imgwarp.cpp: warpAffine + remapBilinear,
// 8-bit fixed-point path) and pinned by fixtures made with cv2 itself:
//   the caller passes the INVERTED matrix (double); X0 = cvRound((m01*y + m02)*1024) + 16, adelta = cvRound(m00*x*1024) (likewise Y);
//   X = (X0 + adelta) >> 5; source pixel sx = X >> 5 with the 5-bit fraction X & 31; bilinear weights (32-fy)(32-fx)*32 ... as int16
//   (saturated to 32767, the remainder added to the last tap so they sum to 32768); out = (sum + 2^14) >> 15; taps outside the
//   frame read `fill`.
__global__ void __launch_bounds__(256) warp_affine_u8_kernel(const uint8_t* __restrict__ src, int sh, int sw, uint8_t* __restrict__ dst, int dh, int dw,
                                                             double m00, double m01, double m02, double m10, double m11, double m12, int fill0,
                                                             int fill1, int fill2) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= dh * dw) return;
  const int y = idx / dw, x = idx - y * dw;
  auto sat = [](double v) -> long long {
    const long long r = __double2ll_rn(v);
    return r < -2147483648ll ? -2147483648ll : (r > 2147483647ll ? 2147483647ll : r);
  };
  const long long X0 = sat((m01 * static_cast<double>(y) + m02) * 1024.0) + 16;
  const long long Y0 = sat((m11 * static_cast<double>(y) + m12) * 1024.0) + 16;
  const long long X = (X0 + sat(m00 * static_cast<double>(x) * 1024.0)) >> 5;
  const long long Y = (Y0 + sat(m10 * static_cast<double>(x) * 1024.0)) >> 5;
  long long sxl = X >> 5, syl = Y >> 5;
  sxl = sxl < -32768 ? -32768 : (sxl > 32767 ? 32767 : sxl);
  syl = syl < -32768 ? -32768 : (syl > 32767 ? 32767 : syl);
  const int sx = static_cast<int>(sxl), sy = static_cast<int>(syl);
  const int fx = static_cast<int>(X & 31), fy = static_cast<int>(Y & 31);
  int w[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
#pragma unroll
  for (int k = 0; k < 4; ++k) w[k] = w[k] > 32767 ? 32767 : w[k];
  w[3] += 32768 - (w[0] + w[1] + w[2] + w[3]);
  const int fill[3] = {fill0, fill1, fill2};
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int yy = sy + (k >> 1), xx = sx + (k & 1);
    const bool inside = yy >= 0 && yy < sh && xx >= 0 && xx < sw;
    const uint8_t* sp = src + (static_cast<long long>(inside ? yy : 0) * sw + (inside ? xx : 0)) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += (inside ? static_cast<int>(sp[c]) : fill[c]) * w[k];
  }
  uint8_t* d = dst + static_cast<long long>(idx) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    int v = (acc[c] + (1 << 14)) >> 15;
    d[c] = static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
}

int warp_affine_u8(const void* src, int sh, int sw, void* dst, int dh, int dw, const double* minv, const int* fill, cudaStream_t stream) {
  YB_REQUIRE(src && dst && minv && fill && sh > 0 && sw > 0 && dh > 0 && dw > 0 && static_cast<long long>(dh) * dw < (1ll << 31), "warp_affine_u8: bad argument");
  const int pixels = dh * dw;
  warp_affine_u8_kernel<<<(pixels + 255) / 256, 256, 0, stream>>>(static_cast<const uint8_t*>(src), sh, sw, static_cast<uint8_t*>(dst), dh, dw, minv[0], minv[1],
                                                                 minv[2], minv[3], minv[4], minv[5], fill[0], fill[1], fill[2]);
  return check_launch("warp_affine_u8_kernel");
}

// ------------------------------------------------------------------------------------------------
// The photometric chain of the reference's `transform/image.py` (RandomBlur, BGR2HSV, RandomHue, RandomSaturation, RandomBrightness,
// HSV2RGB, RandomGamma; config.ini `transform/image_train`) over a resized uint8 batch [B, H, W, 3], out of place, bit-exact with cv2 4.13
// (tests/photometric_oracle.py states the rules and tests/golden/photometric.npz pins them).  One launch runs one segment of the chain:
// an optional box blur, then per-pixel stages in registers.  `stages` holds 4-bit codes, first stage in the low bits.  Per image the
// parameter buffer holds {int kw, kh, 0, 0} and then one 3 x 256 lookup table per LUT stage (hue / saturation / brightness / gamma draws,
// composed on the host); it is the only thing a new draw changes, so a captured launch replays with new draws after one copy into it.
constexpr int PH_TW = 32, PH_TH = 32, PH_HALO = 2;  // output tile; halo of the largest pinned kernel, 5 x 5
constexpr int PH_MAX_STAGES = 7, PH_MAX_LUTS = 4;
enum { PH_END = 0, PH_BLUR = 1, PH_SWAP = 2, PH_BGR2HSV = 3, PH_HSV2RGB = 4, PH_LUT = 5 };

struct PhTables {
  int sdiv[256], hdiv[256];
  uint8_t lut[PH_MAX_LUTS][3][256];
};

__device__ __forceinline__ int reflect101(int i, int n) {  // BORDER_REFLECT_101 for i in [-2, n + 1]
  if (n == 1) return 0;
  i = i < 0 ? -i : i;
  i = i >= n ? 2 * n - 2 - i : i;
  return i < 0 ? -i : i;
}

// cv2 COLOR_BGR2HSV, 8-bit: OpenCV's integer rule with hsv_shift = 12
__device__ __forceinline__ void bgr2hsv_px(const PhTables& t, int& c0, int& c1, int& c2) {
  const int b = c0, g = c1, r = c2;
  const int v = max(max(b, g), r), diff = v - min(min(b, g), r);
  const int s = (diff * t.sdiv[v] + (1 << 11)) >> 12;
  const int hp = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  int h = (hp * t.hdiv[diff] + (1 << 11)) >> 12;
  c0 = h < 0 ? h + 180 : h; c1 = s; c2 = v;
}

// cv2 COLOR_HSV2RGB, 8-bit: float32 sectors with fused multiply-adds (any h, taken mod 180 through the sector); the result is truncated
// in the vector body of a row and rounded half to even in its scalar tail (`tail`: the last w mod 32 pixels)
__device__ __forceinline__ void hsv2rgb_px(bool tail, int& c0, int& c1, int& c2) {
  const float h = __fmul_rn(static_cast<float>(c0), 6.f / 180.f);
  const float s = __fmul_rn(static_cast<float>(c1), 1.f / 255.f), v = __fmul_rn(static_cast<float>(c2), 1.f / 255.f);
  const float pre = floorf(h), f = __fsub_rn(h, pre);
  const float t0 = v, t1 = __fmul_rn(v, __fsub_rn(1.f, s)), t2 = __fmul_rn(v, __fmaf_rn(-s, f, 1.f)),
              t3 = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.f, f), 1.f));
  float b, g, r;
  switch (static_cast<int>(pre) % 6) {
    case 0: b = t1; g = t3; r = t0; break;
    case 1: b = t1; g = t0; r = t2; break;
    case 2: b = t3; g = t0; r = t1; break;
    case 3: b = t0; g = t2; r = t1; break;
    case 4: b = t0; g = t1; r = t3; break;
    default: b = t2; g = t1; r = t0; break;
  }
  r = __fmul_rn(r, 255.f); g = __fmul_rn(g, 255.f); b = __fmul_rn(b, 255.f);
  c0 = min(255, tail ? __float2int_rn(r) : static_cast<int>(r));
  c1 = min(255, tail ? __float2int_rn(g) : static_cast<int>(g));
  c2 = min(255, tail ? __float2int_rn(b) : static_cast<int>(b));
}

__device__ __forceinline__ void ph_pixel(const PhTables& t, int stages, bool hsv_tail, int& c0, int& c1, int& c2) {
  int lut = 0;
#pragma unroll 1
  for (; stages != PH_END; stages >>= 4) {
    const int op = stages & 15;
    if (op == PH_SWAP) { const int x = c0; c0 = c2; c2 = x; }
    else if (op == PH_BGR2HSV) bgr2hsv_px(t, c0, c1, c2);
    else if (op == PH_HSV2RGB) hsv2rgb_px(hsv_tail, c0, c1, c2);
    else { c0 = t.lut[lut][0][c0]; c1 = t.lut[lut][1][c1]; c2 = t.lut[lut][2][c2]; ++lut; }
  }
}

// cv2.blur's window sum -> pixel (d = kw kh): copy for d = 1; the 16-bit fixed-point rule up to d = 24, whose only overflow (d = 2,
// s = 510) saturates in the 16-byte vector body of a row and wraps to 0 in its scalar tail; the exact quotient rounded half up at d = 25
__device__ __forceinline__ int blur_divide(int s, int d, int m, int delta, bool tail) {
  if (d == 1) return s;
  if (d == 25) return (2 * s + 25) / 50;
  const int v = ((s + delta) * m) >> 16;
  return v > 255 ? (tail ? v & 255 : 255) : v;
}

// one CTA = a 32 x 32 output tile of one image (blockIdx.z); 256 threads, 4 rows each.  BLUR: tile + halo into shared memory with
// REFLECT_101 indexing, integer row sums, then column sums in the epilogue.
template <bool BLUR>
__global__ void __launch_bounds__(256) photometric_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int height, int width,
                                                             const uint8_t* __restrict__ params, int stride, int stages, int nlut) {
  __shared__ PhTables t;
  constexpr int IW = PH_TW + 2 * PH_HALO, IH = PH_TH + 2 * PH_HALO;
  __shared__ uint8_t tin[BLUR ? IH * IW * 3 : 1];
  __shared__ uint16_t trow[BLUR ? IH * PH_TW * 3 : 1];
  const int tid = threadIdx.x, img = blockIdx.z;
  const int x0 = blockIdx.x * PH_TW, y0 = blockIdx.y * PH_TH;
  const uint8_t* p = params + static_cast<long long>(img) * stride;
  const uint8_t* s_img = src + static_cast<long long>(img) * height * width * 3;
  uint8_t* d_img = dst + static_cast<long long>(img) * height * width * 3;
  t.sdiv[tid] = tid ? (2 * (255 << 12) + tid) / (2 * tid) : 0;      // round((255 << 12) / i)
  t.hdiv[tid] = tid ? (2 * (180 << 12) + 6 * tid) / (12 * tid) : 0;  // round((180 << 12) / (6 i))
  for (int i = tid; i < nlut * 768; i += 256) (&t.lut[0][0][0])[i] = p[16 + i];
  int kw = 1, kh = 1, d = 1, m = 0, delta = 0;
  if (BLUR) {
    // clamped to the pinned 1..5 (the host rejects larger draws): a bad parameter block must not index outside tin / trow
    kw = min(max(reinterpret_cast<const int*>(p)[0], 1), 2 * PH_HALO + 1);
    kh = min(max(reinterpret_cast<const int*>(p)[1], 1), 2 * PH_HALO + 1);
    d = kw * kh;
    m = 65536 / d;
    if (2 * (65536 % d) < d) delta = d / 2 + 1; else { ++m; delta = d / 2; }
    for (int i = tid; i < IH * IW * 3; i += 256) {
      const int r = i / (IW * 3), rem = i - r * IW * 3, cx = rem / 3, c = rem - cx * 3;
      const int gy = reflect101(min(max(y0 - PH_HALO + r, -PH_HALO), height + 1), height);
      const int gx = reflect101(min(max(x0 - PH_HALO + cx, -PH_HALO), width + 1), width);
      tin[i] = s_img[(static_cast<long long>(gy) * width + gx) * 3 + c];
    }
    __syncthreads();
    const int xo = PH_HALO - kw / 2;
    for (int i = tid; i < IH * PH_TW * 3; i += 256) {
      const int r = i / (PH_TW * 3), rem = i - r * PH_TW * 3, x = rem / 3, c = rem - x * 3;
      const uint8_t* q = tin + (r * IW + x + xo) * 3 + c;
      int sum = 0;
      for (int j = 0; j < kw; ++j) sum += q[3 * j];
      trow[i] = static_cast<uint16_t>(sum);
    }
  }
  __syncthreads();
  const int tail_start = 3 * width - (3 * width) % 16;
  const int tx = tid & 31;
#pragma unroll 1
  for (int ty = tid >> 5; ty < PH_TH; ty += 8) {
    const int x = x0 + tx, y = y0 + ty;
    if (x >= width || y >= height) continue;
    const long long off = (static_cast<long long>(y) * width + x) * 3;
    int c[3];
    if (BLUR) {
      const uint16_t* q = trow + ((ty + PH_HALO - kh / 2) * PH_TW + tx) * 3;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        int sum = 0;
        for (int i = 0; i < kh; ++i) sum += q[i * PH_TW * 3 + k];
        c[k] = blur_divide(sum, d, m, delta, 3 * x + k >= tail_start);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) c[k] = s_img[off + k];
    }
    ph_pixel(t, stages, x >= width - width % 32, c[0], c[1], c[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) d_img[off + k] = static_cast<uint8_t>(c[k]);
  }
}

int photometric_batch_u8(const void* src, void* dst, int batch, int height, int width, const void* params, int param_stride, int stages,
                         cudaStream_t stream) {
  YB_REQUIRE(src && dst && params && batch > 0 && batch <= 65535 && height > 0 && width > 0 && src != dst, "photometric_batch_u8: bad argument");
  YB_REQUIRE(static_cast<long long>(height) * width * 3 < (1ll << 31) && stages >= 0, "photometric_batch_u8: bad argument");
  const bool blur = (stages & 15) == PH_BLUR;
  const int pixel_stages = blur ? stages >> 4 : stages;
  int n = 0, nlut = 0, rest = pixel_stages;
  for (; rest != 0; rest >>= 4, ++n) {
    const int op = rest & 15;
    YB_REQUIRE(op >= PH_SWAP && op <= PH_LUT, "photometric_batch_u8: unknown stage code, or a blur that is not the first stage");
    nlut += op == PH_LUT;
  }
  YB_REQUIRE(n + blur <= PH_MAX_STAGES && nlut <= PH_MAX_LUTS, "photometric_batch_u8: too many stages for one launch");
  YB_REQUIRE(param_stride == 16 + 768 * nlut, "photometric_batch_u8: param_stride must be 16 + 768 * (number of LUT stages)");
  const dim3 grid((width + PH_TW - 1) / PH_TW, (height + PH_TH - 1) / PH_TH, batch);
  if (blur)
    photometric_u8_kernel<true><<<grid, 256, 0, stream>>>(static_cast<const uint8_t*>(src), static_cast<uint8_t*>(dst), height, width,
                                                          static_cast<const uint8_t*>(params), param_stride, pixel_stages, nlut);
  else
    photometric_u8_kernel<false><<<grid, 256, 0, stream>>>(static_cast<const uint8_t*>(src), static_cast<uint8_t*>(dst), height, width,
                                                           static_cast<const uint8_t*>(params), param_stride, pixel_stages, nlut);
  return check_launch("photometric_u8_kernel");
}

int totensor_u8(const void* src, float* dst, int batch, int height, int width, cudaStream_t stream) {
  YB_REQUIRE(src && dst && batch > 0 && height > 0 && width > 0, "totensor_u8: bad argument");
  const long long total = static_cast<long long>(batch) * height * width;
  totensor_u8_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(static_cast<const uint8_t*>(src), dst, batch, height * width);
  return check_launch("totensor_u8_kernel");
}

int totensor_lut_u8(const void* src, const float* lut, float* dst, int batch, int height, int width, cudaStream_t stream) {
  YB_REQUIRE(src && lut && dst && batch > 0 && height > 0 && width > 0, "totensor_lut_u8: bad argument");
  const long long total = static_cast<long long>(batch) * height * width;
  totensor_lut_u8_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(static_cast<const uint8_t*>(src), lut, dst, batch,
                                                                                         height * width);
  return check_launch("totensor_lut_u8_kernel");
}

int resize_batch_u8(const void* src, const long long* src_off, const int* src_hw, void* dst, int batch, int height, int width, int swap_rb,
                    float* yx_min, float* yx_max, int slots, cudaStream_t stream) {
  YB_REQUIRE(src && src_off && src_hw && dst && batch > 0 && height > 0 && width > 0, "resize_batch_u8: bad argument");
  YB_REQUIRE((yx_min == nullptr) == (yx_max == nullptr) && slots >= 0, "resize_batch_u8: boxes come as a (yx_min, yx_max) pair");
  const int pixels = height * width;
  resize_u8_kernel<<<dim3((pixels + 255) / 256, batch), 256, 0, stream>>>(static_cast<const uint8_t*>(src), src_off, src_hw, static_cast<uint8_t*>(dst),
                                                                          height, width, swap_rb);
  int rc = check_launch("resize_u8_kernel");
  if (rc) return rc;
  if (yx_min != nullptr && slots > 0) {
    rescale_boxes_kernel<<<(batch * slots + 127) / 128, 128, 0, stream>>>(yx_min, yx_max, src_hw, batch, slots, height, width);
    rc = check_launch("rescale_boxes_kernel");
  }
  return rc;
}

}  // namespace yb
