// ImageNet minibatch augmentation on the device (loader/imagenet_loader.py): random or centre
// crop, horizontal mirror and mean subtraction of uint8 samples, in one launch.
//
// For the output row r < n (n = hdr[0], read here so the launch can be captured in a graph):
//   s           = idx ? clamp(idx[r]) : r          (dataset resident in HBM : streamed rows)
//   (y0, x0, f) = params[r]
//   xs          = x0 + (f ? cx - 1 - x : x)
//   dst[r][y][x][ch] = cvt(float(src[s][y0 + y][xs][ch]) - (mean ? mean[y0 + y][xs][ch] : 0))
// Rows r >= n are zero. The subtraction is one fp32 operation and cvt rounds to nearest even, so
// the result is bit-identical to the numpy path (fp32 transform_batch, then cast_copy).
//
// Pure data movement: the output (bf16 or fp32) is written in 8-element chunks, one 16-byte (two
// for fp32) store per thread; the 8 source bytes of a chunk are adjacent in the source row (or
// adjacent mirrored pixels), so a warp's reads cover one contiguous span of a few hundred bytes and
// the mean rows stay in L2.
#include "common.cuh"

namespace zn {

struct AugRow {
  const uint8_t* p;          // source sample, nullptr for rows >= n
  const float* m;            // mean at the crop origin (nullptr: no mean)
  int f;
};

__device__ __forceinline__ AugRow aug_row(long long r, int n, const uint8_t* src, long long src_rows,
                                          long long sample_bytes, const int* idx, const int* params,
                                          const float* mean, int sy, int sx, int C, int cy, int cx) {
  AugRow a;
  a.p = nullptr; a.m = nullptr; a.f = 0;
  if (r >= n) return a;
  long long s = idx ? (long long)idx[r] : r;
  s = s < 0 ? 0 : (s >= src_rows ? src_rows - 1 : s);
  int y0 = params[3 * r], x0 = params[3 * r + 1];
  y0 = y0 < 0 ? 0 : (y0 > sy - cy ? sy - cy : y0);
  x0 = x0 < 0 ? 0 : (x0 > sx - cx ? sx - cx : x0);
  const long long origin = ((long long)y0 * sx + x0) * C;
  a.p = src + s * sample_bytes + origin;
  if (mean) a.m = mean + origin;
  a.f = params[3 * r + 2] != 0;
  return a;
}

// output pixel (y, x) of row a -> offset of its channel 0 from the crop origin
__device__ __forceinline__ long long aug_off(const AugRow& a, int y, int x, int sx, int C, int cx) {
  return ((long long)y * sx + (a.f ? cx - 1 - x : x)) * C;
}

template <typename TD>
__global__ void __launch_bounds__(256) augment_minibatch_k(
    const uint8_t* __restrict__ src, long long src_rows, const int* __restrict__ hdr,
    const int* __restrict__ idx, const int* __restrict__ params, const float* __restrict__ mean,
    TD* __restrict__ dst, TD* __restrict__ dst_pad, const int* __restrict__ labels_src,
    int* __restrict__ labels_dst, int max_rows, int sy, int sx, int C, int cy, int cx) {
  pdl_entry();
  const int n = hdr[0];
  const long long pixels = (long long)cy * cx;                 // output pixels per sample
  const long long img = pixels * C;
  const long long total = (long long)max_rows * img;
  const long long sample_bytes = (long long)sy * sx * C;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long q = tid; q * 8 < total; q += stride) {
    const long long e0 = q * 8;
    long long r = e0 / img;
    const long long rem = e0 - r * img;
    const long long pix = rem / C;
    int ch = (int)(rem - pix * C);
    int y = (int)(pix / cx), x = (int)(pix - (long long)y * cx);
    AugRow a = aug_row(r, n, src, src_rows, sample_bytes, idx, params, mean, sy, sx, C, cy, cx);
    long long off = aug_off(a, y, x, sx, C, cx);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float val = 0.f;
      if (a.p) {
        val = (float)__ldg(a.p + off + ch);
        if (a.m) val -= __ldg(a.m + off + ch);
      }
      v[j] = val;
      if (++ch == C) {                        // next pixel, row or sample
        ch = 0;
        if (++x == cx) {
          x = 0;
          if (++y == cy) {
            y = 0;
            ++r;
            if (r < max_rows)
              a = aug_row(r, n, src, src_rows, sample_bytes, idx, params, mean, sy, sx, C, cy, cx);
          }
        }
        off = aug_off(a, y, x, sx, C, cx);
      }
    }
    if (e0 + 8 <= total) {
      st8(dst + e0, v);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (e0 + j < total) stf(dst + e0 + j, v[j]);
    }
  }
  if (dst_pad) {
    // the first conv layer's channel-padded copy [max_rows][cy][cx][8] (C < 8), zeros past C
    for (long long q = tid; q < (long long)max_rows * pixels; q += stride) {
      const long long r = q / pixels, pix = q - r * pixels;
      const int y = (int)(pix / cx), x = (int)(pix - (long long)y * cx);
      const AugRow a = aug_row(r, n, src, src_rows, sample_bytes, idx, params, mean, sy, sx, C, cy, cx);
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
      if (a.p) {
        const long long off = aug_off(a, y, x, sx, C, cx);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (j < C) {
            v[j] = (float)__ldg(a.p + off + j);
            if (a.m) v[j] -= __ldg(a.m + off + j);
          }
        }
      }
      st8(dst_pad + q * 8, v);
    }
  }
  if (labels_dst && tid < max_rows) {
    // labels gathered with the rows (resident dataset); padding rows get label 0
    long long s = idx ? (long long)idx[tid] : tid;
    s = s < 0 ? 0 : (s >= src_rows ? src_rows - 1 : s);
    labels_dst[tid] = tid < n ? labels_src[s] : 0;
  }
}

static long long g_augment_launches = 0;
long long augment_launches() { return g_augment_launches; }

void launch_augment_minibatch(const uint8_t* src, long long src_rows, const int* hdr, const int* idx,
                              const int* params, const float* mean, void* dst, void* dst_pad, bool bf16,
                              const int* labels_src, int* labels_dst, int max_rows, int sy, int sx, int C,
                              int cy, int cx, cudaStream_t st) {
  const long long chunks = ((long long)max_rows * cy * cx * C + 7) / 8;
  long long blocks = (chunks + 255) / 256;
  if (blocks > 8LL * num_sms()) blocks = 8LL * num_sms();
  if (blocks * 256 < max_rows) blocks = (max_rows + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (bf16)
    launch_k(augment_minibatch_k<__nv_bfloat16>, (int)blocks, 256, 0, st, src, src_rows, hdr, idx, params,
             mean, (__nv_bfloat16*)dst, (__nv_bfloat16*)dst_pad, labels_src, labels_dst, max_rows, sy, sx,
             C, cy, cx);
  else
    launch_k(augment_minibatch_k<float>, (int)blocks, 256, 0, st, src, src_rows, hdr, idx, params, mean,
             (float*)dst, (float*)dst_pad, labels_src, labels_dst, max_rows, sy, sx, C, cy, cx);
  ++g_augment_launches;
}

}  // namespace zn
