// Candidate shots of the localisation pipeline on the device (models/imagenet_forward/loader.py):
// for every output row r < n (n = hdr[0]) one shot of a uint8 picture [h][w][C], resident at byte
// offset pics[r].off of the picture arena, is rendered into dst[r][v][u][ch] (aperture A x A x C).
//
// The contract is render_shot's, each operation in float64 and rounded on its own, in this order
// (shot[r] = (ca, sa, scale, bw/2, bh/2, cx, cy), made on the host by loader.shot_geometry):
//   a2 = (A - 1) / 2;  ux = flip ? -(u - a2) : (u - a2);  uy = v - a2
//   bx = (ux*ca + uy*sa) / scale          by = ((-ux)*sa + uy*ca) / scale
//   px = bx + cx                          py = by + cy
//   inside = |bx| <= bw/2 && |by| <= bh/2 && 0 <= px <= w-1 && 0 <= py <= h-1
//   x0 = (int) clamp(floor(px), 0, w>1 ? w-2 : 0);  x1 = min(x0+1, w-1);  fx = clamp(px - x0, 0, 1)
//   val = (((s00*(1-fx))*(1-fy) + (s01*fx)*(1-fy)) + (s10*(1-fx))*fy) + (s11*fx)*fy
//   out = (float)((double)(m * (1.0f - a)) + val * a),  a = inside, m = mean ? mean[v][u][ch] : 0
// The explicit _rn intrinsics keep the compiler from contracting into FMAs, so the fp32 output is
// bit-identical to render_shot and bf16 is its round-to-nearest-even. The kernel evaluates no
// transcendental function: cos, sin and the scale come from the host. Rows r >= n are zero, and a
// picture that does not lie inside the arena renders as zeros instead of reading past it.
//
// One thread per output pixel (all C channels): grid.x covers the A*A pixels of a row, grid.y the
// rows, so a block reads one row's parameters and the bilinear taps of a warp fall in a few source
// rows that stay in L1.
#include "common.cuh"

namespace zn {

struct RenderPic {
  long long off, h, w, flip;       // int64 [max_rows][4] on the device
};

template <typename TD>
__global__ void __launch_bounds__(256) render_shots_k(
    const uint8_t* __restrict__ arena, long long arena_bytes, const int* __restrict__ hdr,
    const double* __restrict__ shots, const long long* __restrict__ pics, const float* __restrict__ mean,
    TD* __restrict__ dst, TD* __restrict__ dst_pad, int A, int C) {
  pdl_entry();
  const int r = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= A * A) return;
  const int v = pix / A, u = pix - v * A;
  const long long o = ((long long)r * A * A + pix) * C;
  float out[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) out[j] = 0.f;
  const RenderPic p = reinterpret_cast<const RenderPic*>(pics)[r];
  const long long h = p.h, w = p.w;
  const bool valid = r < hdr[0] && h >= 1 && w >= 1 && p.off >= 0 && p.off + h * w * C <= arena_bytes;
  if (valid) {
    const double* s = shots + 8LL * r;
    const double ca = s[0], sa = s[1], scale = s[2], hbw = s[3], hbh = s[4], cx = s[5], cy = s[6];
    const double a2 = (double)(A - 1) / 2.0;
    double ux = __dadd_rn((double)u, -a2);
    if (p.flip) ux = -ux;
    const double uy = __dadd_rn((double)v, -a2);
    const double bx = __ddiv_rn(__dadd_rn(__dmul_rn(ux, ca), __dmul_rn(uy, sa)), scale);
    const double by = __ddiv_rn(__dadd_rn(__dmul_rn(-ux, sa), __dmul_rn(uy, ca)), scale);
    const double px = __dadd_rn(bx, cx), py = __dadd_rn(by, cy);
    const double wm1 = (double)(w - 1), hm1 = (double)(h - 1);
    const bool inside = fabs(bx) <= hbw && fabs(by) <= hbh && px >= 0.0 && px <= wm1 &&
                        py >= 0.0 && py <= hm1;
    const double xhi = w > 1 ? (double)(w - 2) : 0.0, yhi = h > 1 ? (double)(h - 2) : 0.0;
    const long long x0 = (long long)fmin(fmax(floor(px), 0.0), xhi);
    const long long y0 = (long long)fmin(fmax(floor(py), 0.0), yhi);
    const long long x1 = x0 + 1 < w - 1 ? x0 + 1 : w - 1;
    const long long y1 = y0 + 1 < h - 1 ? y0 + 1 : h - 1;
    const double fx = fmin(fmax(__dadd_rn(px, -(double)x0), 0.0), 1.0);
    const double fy = fmin(fmax(__dadd_rn(py, -(double)y0), 0.0), 1.0);
    const double gx = __dadd_rn(1.0, -fx), gy = __dadd_rn(1.0, -fy);
    const uint8_t* img = arena + p.off;
    const uint8_t* t00 = img + (y0 * w + x0) * C;
    const uint8_t* t01 = img + (y0 * w + x1) * C;
    const uint8_t* t10 = img + (y1 * w + x0) * C;
    const uint8_t* t11 = img + (y1 * w + x1) * C;
    const float a = inside ? 1.0f : 0.0f;
    const float na = 1.0f - a;
    const double ad = (double)a;
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) {
      if (ch < C) {
        double val = __dmul_rn(__dmul_rn((double)__ldg(t00 + ch), gx), gy);
        val = __dadd_rn(val, __dmul_rn(__dmul_rn((double)__ldg(t01 + ch), fx), gy));
        val = __dadd_rn(val, __dmul_rn(__dmul_rn((double)__ldg(t10 + ch), gx), fy));
        val = __dadd_rn(val, __dmul_rn(__dmul_rn((double)__ldg(t11 + ch), fx), fy));
        const float m = mean ? __ldg(mean + (long long)pix * C + ch) : 0.0f;
        out[ch] = (float)__dadd_rn((double)__fmul_rn(m, na), __dmul_rn(val, ad));
      }
    }
  }
  for (int ch = 0; ch < C && ch < 8; ++ch) stf(dst + o + ch, out[ch]);
  if (dst_pad) st8(dst_pad + ((long long)r * A * A + pix) * 8, out);   // zeros past C
}

static long long g_render_launches = 0;
long long render_shots_launches() { return g_render_launches; }

void launch_render_shots(const uint8_t* arena, long long arena_bytes, const int* hdr, const double* shots,
                         const long long* pics, const float* mean, void* dst, void* dst_pad, bool bf16,
                         int max_rows, int A, int C, cudaStream_t st) {
  const dim3 grid((unsigned)cdiv((long long)A * A, 256), (unsigned)max_rows);
  if (bf16)
    launch_k(render_shots_k<__nv_bfloat16>, grid, 256, 0, st, arena, arena_bytes, hdr, shots, pics, mean,
             (__nv_bfloat16*)dst, (__nv_bfloat16*)dst_pad, A, C);
  else
    launch_k(render_shots_k<float>, grid, 256, 0, st, arena, arena_bytes, hdr, shots, pics, mean,
             (float*)dst, (float*)dst_pad, A, C);
  ++g_render_launches;
}

}  // namespace zn
