// Python bindings of the znicz_b200 sm_90a kernels (the only file that sees torch headers).
#include <torch/extension.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <vector>
#include <cstring>
#include "host_loader.h"
#include "update.h"

namespace zn {
struct ConvGeom { int N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT, PL; };
void launch_act_forward(const void*, void*, long long, int, float, bool, cudaStream_t);
void launch_act_backward(const void*, const void*, const void*, void*, long long, int, float, bool, cudaStream_t);
int err_act_colsum_slices(int rows);
void launch_err_act_colsum(void*, const void*, int, int, int, float*, int, bool, cudaStream_t);
void launch_dropout_forward(const void*, void*, void*, long long, const int*, uint32_t, float, bool, cudaStream_t);
void launch_binary(const void*, const void*, void*, long long, int, bool, cudaStream_t);
void launch_mul_backward(const void*, const void*, const void*, void*, void*, long long, bool, cudaStream_t);
void launch_axpby_2d(const void*, int, int, void*, int, int, int, int, float, float, bool, cudaStream_t);
void launch_crop_nhwc(const void*, void*, int, int, int, int, int, int, int, int, int, bool, cudaStream_t);
void launch_gather_rows(const void*, bool, const int*, void*, bool, int, int, long long, cudaStream_t);
void launch_gather_labels(const int*, const int*, int*, int, int, cudaStream_t);
void launch_gather_minibatch(const void*, bool, const int*, const int*, void*, bool, int*, int, long long, void*, int, int, cudaStream_t);
void launch_mask_mul(void*, const void*, long long, bool, cudaStream_t);
void launch_pad_channels(const void*, void*, int, int, int, bool, cudaStream_t);
void launch_cast(const void*, bool, void*, bool, long long, cudaStream_t);
void launch_scatter_offsets(const void*, const int*, void*, long long, bool, cudaStream_t);
void launch_pool_forward(const void*, void*, int*, int, int, int, int, int, int, int, int, int, int, int, const int*, bool, int, cudaStream_t);
void launch_pull_from_host(const void*, void*, long long, cudaStream_t);
int launch_fp8_quant(const void*, int, long long, int, int, int, uint8_t*, long long, float*, uint8_t*, long long, float*, cudaStream_t);
int launch_gemm_fp8_block(const void*, long long, const float*, const void*, long long, const float*, void*, int, long long, int, int, int, const float*, int, float, cudaStream_t);
long long fp8_gemm_launches();
void launch_swap01_2d(const void*, int, int, void*, int, int, int, int, int, bool, cudaStream_t);
void launch_pull_from_host_bytes(const void*, void*, int, cudaStream_t);
void launch_pool_backward(const void*, const int*, void*, int, int, int, int, int, int, int, int, int, int, int, bool, const void*, int, const void*, int, cudaStream_t);
void launch_lrn_forward(const void*, void*, long long, int, int, float, float, float, bool, cudaStream_t);
void launch_lrn_backward(const void*, const void*, void*, long long, int, int, float, float, float, bool, int, cudaStream_t);
void launch_softmax_rows(const void*, bool, float*, int*, int, int, cudaStream_t);
void launch_evaluate_softmax(const float*, const int*, const int*, void*, bool, const float*, int, int, int*, int*, float*, cudaStream_t);
void launch_evaluate_mse(const void*, const void*, bool, void*, bool, const float*, int, int, const float*, int, float*, float*, cudaStream_t);
void launch_mse_find_closest(const void*, bool, const float*, const int*, const float*, int, int, int, int*, cudaStream_t);
void launch_fused_update(const TensorDesc&, const float* const*, int, uint32_t* const*, uint32_t*, int, int, cudaStream_t);
void launch_col_sums(const float*, float*, int, int, int, cudaStream_t);
void launch_rbm_sample(const void*, void*, long long, long long, const int*, bool, cudaStream_t);
void launch_rbm_apply(float*, const float*, float*, const float*, float*, const float*, int, int, float, cudaStream_t);
void launch_lstm_cell_fwd(const float*, const float*, float*, float*, void*, long long, void*, long long, int, int, bool, cudaStream_t);
void launch_lstm_cell_bwd(const void*, long long, const void*, long long, const float*, const float*, const float*, const float*, float*, void*, int, int, bool, cudaStream_t);
int fc_small_max_out();
void launch_fc_small_forward(const void*, bool, const float*, const float*, void*, float*, int*, int, int, int, int, int, const int*, void*, int, const float*, int*, int*, float*, cudaStream_t);
void launch_fc_small_backward(void*, const void*, const void*, bool, const float*, void*, float*, float*, int, int, int, int, float, float, int, cudaStream_t);
int launch_gemm_pair(const void*, long long, const void*, long long, void*, int, long long, int, int, int,
                     const float*, int, float, cudaStream_t);
long long im2col_tma_launches();
long long conv_pair_launches();
long long conv_halo_launches();
long long augment_launches();
void launch_augment_minibatch(const uint8_t*, long long, const int*, const int*, const int*, const float*, void*, void*, bool, const int*, int*, int, int, int, int, int, int, cudaStream_t);
long long render_shots_launches();
void launch_render_shots(const uint8_t*, long long, const int*, const double*, const long long*, const float*, void*, void*, bool, int, int, int, cudaStream_t);
int launch_fc_wgrad_pair(const void*, long long, const void*, long long, float*, long long, int, int, int,
                         cudaStream_t);
void set_dp_gradient_scale(float);
float get_dp_gradient_scale();
int multi_update_pack(TensorDesc&, int, long long);
void launch_multi_update(const void*, int, int, int, int, uint32_t* const*, uint32_t*, int, unsigned*, float* const*, long long, int, float* const*, float*, float*, int, int, cudaStream_t);
void launch_refresh_shadows(const float*, long long, int, int, __nv_bfloat16*, int, __nv_bfloat16*, int, int, int, int, cudaStream_t);
void launch_gemm_simt(const void*, bool, long long, int, const void*, bool, long long, int, void*, bool, long long, int, int, int, int, const float*, int, float, float, int, long long, cudaStream_t);
struct ConvGeomS { int N, H, W, C, OH, OW, F, KY, KX, SY, SX, PT, PL; };
int umma_pick_splits(int, int, int, int);
void launch_som_winners(const float*, const float*, int*, int*, int, int, int, int, cudaStream_t);
void launch_som_update(const float*, float*, const float*, const int*, int, int, int, float, float, cudaStream_t);
int launch_gemm_umma(const void*, long long, int, const void*, long long, int, void*, int, long long, int, int, int, int, const float*, int, float, float, int, long long, cudaStream_t);
int launch_conv_fprop_umma(const void*, const void*, long long, const float*, void*, int, int, int, int, int, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
int launch_conv_dgrad_umma(const void*, const void*, long long, void*, int, int, int, int, int, int, int, int, int, int, int, int, int, int, float, float, const void*, int, cudaStream_t);
int launch_conv_wgrad_umma(const void*, const void*, float*, int, int, int, int, int, int, int, int, int, int, int, int, int, int, float*, cudaStream_t);
}  // namespace zn

// The SIMT conv launchers take a struct by value; redeclare with the real layout.
namespace zn {
struct ConvGeom2 { int N, H, W, C; int OH, OW, F; int KY, KX, SY, SX; int PT, PL; };
void launch_conv_fprop_simt_raw(const void*, bool, const float*, long long, int, const float*, void*, bool, const int*, int, cudaStream_t);
void launch_conv_dgrad_simt_raw(const void*, bool, const float*, long long, int, void*, bool, const int*, float, float, cudaStream_t);
void launch_conv_wgrad_simt_raw(const void*, bool, const void*, bool, float*, int, const int*, int, cudaStream_t);
}

using torch::Tensor;
static inline cudaStream_t cur() { return c10::cuda::getCurrentCUDAStream().stream(); }
static inline bool is_bf16(const Tensor& t) { return t.scalar_type() == torch::kBFloat16; }
static inline void chk(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
  TORCH_CHECK(t.scalar_type() == torch::kFloat32 || t.scalar_type() == torch::kBFloat16 ||
                  t.scalar_type() == torch::kInt32,
              name, ": unsupported dtype");
}
static inline void same_dt(const Tensor& a, const Tensor& b) {
  TORCH_CHECK(a.scalar_type() == b.scalar_type(), "dtype mismatch");
}
static inline const float* fptr_or_null(const c10::optional<Tensor>& t) {
  if (!t.has_value() || !t->defined() || t->numel() == 0) return nullptr;
  TORCH_CHECK(t->scalar_type() == torch::kFloat32 && t->is_cuda());
  return t->data_ptr<float>();
}
static void kcheck() {
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "znicz_b200 kernel launch failed: ", cudaGetErrorString(e));
}

void act_forward(Tensor x, Tensor y, int64_t act, double factor) {
  chk(x, "x"); chk(y, "y"); same_dt(x, y);
  zn::launch_act_forward(x.data_ptr(), y.data_ptr(), x.numel(), (int)act, (float)factor, is_bf16(x), cur());
  kcheck();
}
void act_backward(Tensor err_y, c10::optional<Tensor> x, c10::optional<Tensor> y, Tensor err_x,
                  int64_t act, double factor) {
  chk(err_y, "err_y"); chk(err_x, "err_x"); same_dt(err_y, err_x);
  const void* xp = (x.has_value() && x->defined()) ? x->data_ptr() : nullptr;
  const void* yp = (y.has_value() && y->defined()) ? y->data_ptr() : nullptr;
  if (xp) same_dt(*x, err_y);
  if (yp) same_dt(*y, err_y);
  zn::launch_act_backward(err_y.data_ptr(), xp, yp, err_x.data_ptr(), err_y.numel(), (int)act,
                          (float)factor, is_bf16(err_y), cur());
  kcheck();
}
int64_t colsum_slices(int64_t rows) { return zn::err_act_colsum_slices((int)rows); }
// err_y *= f'(y) in place; partial[slices, cols] receives per-slice column sums
void err_act_colsum(Tensor err_y, c10::optional<Tensor> y, int64_t rows, int64_t cols, int64_t act,
                    c10::optional<Tensor> partial) {
  chk(err_y, "err_y");
  const void* yp = nullptr;
  if (y.has_value() && y->defined()) { same_dt(*y, err_y); yp = y->data_ptr(); }
  float* pp = nullptr; int slices = zn::err_act_colsum_slices((int)rows);
  if (partial.has_value() && partial->defined()) {
    TORCH_CHECK(partial->scalar_type() == torch::kFloat32 && partial->numel() >= slices * cols);
    pp = partial->data_ptr<float>();
  }
  TORCH_CHECK(act == 0 || yp, "activation derivative needs y");
  zn::launch_err_act_colsum(err_y.data_ptr(), yp, (int)rows, (int)cols, (int)act, pp, slices,
                            is_bf16(err_y), cur());
  kcheck();
}
void dropout_forward(Tensor x, Tensor y, Tensor mask, Tensor rng, int64_t threshold, double scale) {
  chk(x, "x"); same_dt(x, y); same_dt(x, mask);
  zn::launch_dropout_forward(x.data_ptr(), y.data_ptr(), mask.data_ptr(), x.numel(), rng.data_ptr<int>(),
                             (uint32_t)threshold, (float)scale, is_bf16(x), cur());
  kcheck();
}
void binary_op(Tensor a, Tensor b, Tensor o, int64_t op) {
  chk(a, "a"); same_dt(a, b); same_dt(a, o);
  zn::launch_binary(a.data_ptr(), b.data_ptr(), o.data_ptr(), a.numel(), (int)op, is_bf16(a), cur());
  kcheck();
}
void mul_backward(Tensor x, Tensor y, Tensor e, Tensor ex, Tensor ey) {
  chk(x, "x"); same_dt(x, y); same_dt(x, e); same_dt(x, ex); same_dt(x, ey);
  zn::launch_mul_backward(x.data_ptr(), y.data_ptr(), e.data_ptr(), ex.data_ptr(), ey.data_ptr(),
                          x.numel(), is_bf16(x), cur());
  kcheck();
}
void axpby_2d(Tensor src, int64_t soff, Tensor dst, int64_t doff, int64_t len, double alpha, double beta) {
  chk(src, "src"); same_dt(src, dst);
  int rows = (int)src.size(0);
  zn::launch_axpby_2d(src.data_ptr(), (int)(src.numel() / rows), (int)soff, dst.data_ptr(),
                      (int)(dst.numel() / rows), (int)doff, rows, (int)len, (float)alpha, (float)beta,
                      is_bf16(src), cur());
  kcheck();
}
// dst[(j * A + i)][doff + c] = src[(i * Bn + j)][soff + c]; row pitches given explicitly
void swap01_2d(Tensor src, int64_t src_ld, int64_t soff, Tensor dst, int64_t dst_ld, int64_t doff,
               int64_t A, int64_t Bn, int64_t len) {
  chk(src, "src"); same_dt(src, dst);
  TORCH_CHECK(soff + len <= src_ld && doff + len <= dst_ld && src.numel() >= A * Bn * src_ld - (src_ld - soff - len)
              && dst.numel() >= A * Bn * dst_ld - (dst_ld - doff - len), "swap01_2d: out of range");
  zn::launch_swap01_2d(src.data_ptr(), (int)src_ld, (int)soff, dst.data_ptr(), (int)dst_ld, (int)doff,
                       (int)A, (int)Bn, (int)len, is_bf16(src), cur());
  kcheck();
}
void crop_nhwc(Tensor in, Tensor out, int64_t top, int64_t left, bool backward) {
  chk(in, "in"); same_dt(in, out);
  const Tensor& big = backward ? out : in;
  const Tensor& small = backward ? in : out;
  zn::launch_crop_nhwc(in.data_ptr(), out.data_ptr(), (int)big.size(0), (int)big.size(1), (int)big.size(2),
                       (int)big.size(3), (int)small.size(1), (int)small.size(2), (int)top, (int)left,
                       backward ? 1 : 0, is_bf16(in), cur());
  kcheck();
}
void gather_rows(Tensor src, Tensor idx, Tensor dst, int64_t count) {
  chk(src, "src"); chk(dst, "dst");
  long long row = src.numel() / src.size(0);
  zn::launch_gather_rows(src.data_ptr(), is_bf16(src), idx.data_ptr<int>(), dst.data_ptr(), is_bf16(dst),
                         (int)count, (int)dst.size(0), row, cur());
  kcheck();
}
void gather_labels(Tensor src, Tensor idx, Tensor dst, int64_t count) {
  zn::launch_gather_labels(src.data_ptr<int>(), idx.data_ptr<int>(), dst.data_ptr<int>(), (int)count,
                           (int)dst.size(0), cur());
  kcheck();
}
void gather_minibatch(Tensor src, c10::optional<Tensor> labels_src, Tensor hdr, Tensor dst,
                      c10::optional<Tensor> labels_dst, c10::optional<Tensor> dst_pad, int64_t C) {
  chk(src, "src"); chk(dst, "dst");
  long long row = src.numel() / src.size(0);
  void* pad = nullptr;
  if (dst_pad.has_value() && dst_pad->defined()) {
    same_dt(dst, *dst_pad);
    TORCH_CHECK(C >= 1 && C < 8 && row % C == 0 && dst_pad->numel() == dst.size(0) * (row / C) * 8,
                "padded minibatch must be [rows][pixels][8]");
    pad = dst_pad->data_ptr();
  }
  TORCH_CHECK(row % 8 == 0, "gather_minibatch needs row % 8 == 0");
  const int* ls = (labels_src.has_value() && labels_src->defined()) ? labels_src->data_ptr<int>() : nullptr;
  int* ld = (labels_dst.has_value() && labels_dst->defined()) ? labels_dst->data_ptr<int>() : nullptr;
  zn::launch_gather_minibatch(src.data_ptr(), is_bf16(src), ls, hdr.data_ptr<int>(), dst.data_ptr(),
                              is_bf16(dst), ld, (int)dst.size(0), row, pad, (int)C, 8, cur());
  kcheck();
}
// ImageNet augmentation (csrc/augment.cu): crop at params[r] = (y0, x0, flip), mirror, subtract the
// mean, convert; rows >= hdr[0] zero. src = uint8 [rows][sy][sx][C] gathered through idx (a dataset
// resident in HBM) or read in order (streamed rows); labels only with idx.
void augment_minibatch(Tensor src, Tensor hdr, c10::optional<Tensor> idx, Tensor params,
                       c10::optional<Tensor> mean, Tensor dst, c10::optional<Tensor> labels_src,
                       c10::optional<Tensor> labels_dst, c10::optional<Tensor> dst_pad) {
  TORCH_CHECK(src.is_cuda() && src.is_contiguous() && src.scalar_type() == torch::kUInt8 && src.dim() == 4,
              "augment_minibatch: src must be a contiguous uint8 [rows][sy][sx][C] device tensor");
  chk(dst, "dst");
  TORCH_CHECK(dst.scalar_type() != torch::kInt32 && dst.dim() == 4, "dst must be fp32 or bf16 [n][cy][cx][C]");
  const int max_rows = (int)dst.size(0), cy = (int)dst.size(1), cx = (int)dst.size(2), C = (int)dst.size(3);
  const int sy = (int)src.size(1), sx = (int)src.size(2);
  TORCH_CHECK(src.size(3) == C && cy <= sy && cx <= sx && cy >= 1 && cx >= 1, "augment_minibatch: crop ",
              cy, "x", cx, "x", C, " does not fit the samples ", sy, "x", sx, "x", src.size(3));
  chk(hdr, "hdr"); chk(params, "params");
  TORCH_CHECK(hdr.scalar_type() == torch::kInt32 && hdr.numel() >= 1, "hdr must be int32");
  TORCH_CHECK(params.scalar_type() == torch::kInt32 && params.numel() >= 3LL * max_rows, "params must be int32 [n][3]");
  const int* ip = nullptr;
  if (idx.has_value() && idx->defined()) {
    chk(*idx, "idx");
    TORCH_CHECK(idx->scalar_type() == torch::kInt32 && idx->numel() >= max_rows, "idx must be int32 [n]");
    ip = idx->data_ptr<int>();
  } else {
    TORCH_CHECK(src.size(0) >= max_rows, "streamed rows: src must hold one row per output row");
  }
  const float* mp = nullptr;
  if (mean.has_value() && mean->defined()) {
    chk(*mean, "mean");
    TORCH_CHECK(mean->scalar_type() == torch::kFloat32 && mean->numel() == (int64_t)sy * sx * C,
                "mean must be fp32 [sy][sx][C]");
    mp = mean->data_ptr<float>();
  }
  const bool has_ls = labels_src.has_value() && labels_src->defined();
  const bool has_ld = labels_dst.has_value() && labels_dst->defined();
  TORCH_CHECK(has_ls == has_ld && (!has_ld || ip), "labels need labels_src, labels_dst and idx");
  if (has_ld) {
    chk(*labels_src, "labels_src"); chk(*labels_dst, "labels_dst");
    TORCH_CHECK(labels_src->scalar_type() == torch::kInt32 && labels_src->numel() >= src.size(0) &&
                labels_dst->scalar_type() == torch::kInt32 && labels_dst->numel() >= max_rows, "labels: int32");
  }
  void* pad = nullptr;
  if (dst_pad.has_value() && dst_pad->defined()) {
    chk(*dst_pad, "dst_pad"); same_dt(dst, *dst_pad);
    TORCH_CHECK(C < 8 && dst_pad->numel() == (int64_t)max_rows * cy * cx * 8, "padded minibatch must be [n][cy][cx][8]");
    pad = dst_pad->data_ptr();
  }
  zn::launch_augment_minibatch(src.data_ptr<uint8_t>(), src.size(0), hdr.data_ptr<int>(), ip,
                               params.data_ptr<int>(), mp, dst.data_ptr(), pad, is_bf16(dst),
                               has_ls ? labels_src->data_ptr<int>() : nullptr,
                               has_ld ? labels_dst->data_ptr<int>() : nullptr, max_rows, sy, sx, C, cy, cx, cur());
  kcheck();
}
// Localisation shots (csrc/render.cu): row r < hdr[0] renders the uint8 picture [h][w][C] at byte
// offset pics[r] = (off, h, w, flip) of arena with shots[r] = (ca, sa, scale, bw/2, bh/2, cx, cy, -);
// rows >= hdr[0] are zero.
void render_shots(Tensor arena, Tensor hdr, Tensor shots, Tensor pics, c10::optional<Tensor> mean,
                  Tensor dst, c10::optional<Tensor> dst_pad) {
  auto dev_tensor = [](const Tensor& t, const char* name, c10::ScalarType dt) {
    TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.scalar_type() == dt, "render_shots: ", name,
                " must be a contiguous ", c10::toString(dt), " CUDA tensor");
  };
  dev_tensor(arena, "arena", torch::kUInt8);
  chk(dst, "dst");
  TORCH_CHECK((dst.scalar_type() == torch::kFloat32 || is_bf16(dst)) && dst.dim() == 4 && dst.size(1) == dst.size(2),
              "render_shots: dst must be fp32 or bf16 [n][A][A][C]");
  const int max_rows = (int)dst.size(0), A = (int)dst.size(1), C = (int)dst.size(3);
  TORCH_CHECK(max_rows >= 1 && max_rows <= 65535 && A >= 1 && C >= 1 && C <= 8,
              "render_shots: needs 1..65535 rows and 1..8 channels, got ", max_rows, " and ", C);
  dev_tensor(hdr, "hdr", torch::kInt32);
  dev_tensor(shots, "shots", torch::kFloat64);
  dev_tensor(pics, "pics", torch::kInt64);
  TORCH_CHECK(hdr.numel() >= 1, "hdr must hold n");
  TORCH_CHECK(shots.numel() == 8LL * max_rows, "shots must be float64 [n][8]");
  TORCH_CHECK(pics.numel() == 4LL * max_rows, "pics must be int64 [n][4]");
  const float* mp = nullptr;
  if (mean.has_value() && mean->defined()) {
    chk(*mean, "mean");
    TORCH_CHECK(mean->scalar_type() == torch::kFloat32 && mean->numel() == (int64_t)A * A * C,
                "mean must be fp32 [A][A][C]");
    mp = mean->data_ptr<float>();
  }
  void* pad = nullptr;
  if (dst_pad.has_value() && dst_pad->defined()) {
    chk(*dst_pad, "dst_pad"); same_dt(dst, *dst_pad);
    TORCH_CHECK(C < 8 && dst_pad->numel() == (int64_t)max_rows * A * A * 8, "padded minibatch must be [n][A][A][8]");
    pad = dst_pad->data_ptr();
  }
  zn::launch_render_shots(arena.data_ptr<uint8_t>(), arena.numel(), hdr.data_ptr<int>(), shots.data_ptr<double>(),
                          (const long long*)pics.data_ptr<int64_t>(), mp, dst.data_ptr(), pad, is_bf16(dst),
                          max_rows, A, C, cur());
  kcheck();
}
// dst (device) <- src (pinned host tensor), by a kernel that reads the host memory (see
// launch_pull_from_host). Both 16-byte aligned; sizes in bytes must match.
void pull_from_host(Tensor src, Tensor dst) {
  TORCH_CHECK(!src.is_cuda() && src.is_pinned() && src.is_contiguous(), "src must be pinned host memory");
  TORCH_CHECK(dst.is_cuda() && dst.is_contiguous(), "dst must be a device tensor");
  const long long nbytes = (long long)src.numel() * src.element_size();
  TORCH_CHECK(nbytes == (long long)dst.numel() * dst.element_size(), "size mismatch");
  void* alias = nullptr;
  cudaError_t e = cudaHostGetDevicePointer(&alias, src.data_ptr(), 0);
  TORCH_CHECK(e == cudaSuccess, "cudaHostGetDevicePointer: ", cudaGetErrorString(e));
  TORCH_CHECK(((uintptr_t)alias & 15) == 0 && ((uintptr_t)dst.data_ptr() & 15) == 0, "16-byte alignment");
  zn::launch_pull_from_host(alias, dst.data_ptr(), nbytes, cur());
  kcheck();
}
// ---- streaming-loader step in ONE call ------------------------------------------------------------
// The per-step sequence "wait until the staging buffer was consumed -> pull the pinned slot on the
// copy stream -> events -> main stream waits -> device-to-device copy -> event" was 8 torch calls
// (~58 us of host time per 195 us step, host-bound end to end). The ring keeps its CUDA events here
// and issues the whole sequence with raw runtime calls (~6 us).
namespace {
struct StreamRing {
  std::vector<cudaEvent_t> stage_evt, pull_evt, slot_evt;
  std::vector<char> stage_used, slot_used;
  int k = 0;
};
std::vector<StreamRing*> g_rings;
StreamRing& ring_at(int64_t id) {
  TORCH_CHECK(id >= 0 && id < (int64_t)g_rings.size() && g_rings[id] != nullptr, "bad stream ring id");
  return *g_rings[id];
}
}  // namespace
int64_t stream_ring_create(int64_t n_stage, int64_t n_slots) {
  TORCH_CHECK(n_stage >= 1 && n_slots >= 1);
  auto* r = new StreamRing();
  auto mk = [](std::vector<cudaEvent_t>& v, int64_t n) {
    v.resize(n);
    for (auto& e : v) TORCH_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming) == cudaSuccess);
  };
  mk(r->stage_evt, n_stage); mk(r->pull_evt, n_stage); mk(r->slot_evt, n_slots);
  r->stage_used.assign(n_stage, 0); r->slot_used.assign(n_slots, 0);
  g_rings.push_back(r);
  return (int64_t)g_rings.size() - 1;
}
void stream_ring_destroy(int64_t id) {
  StreamRing& r = ring_at(id);
  for (auto* v : {&r.stage_evt, &r.pull_evt, &r.slot_evt})
    for (auto e : *v) cudaEventDestroy(e);
  delete g_rings[id];
  g_rings[id] = nullptr;
}
// pinned slot `slot` -> stage[k] on `side_stream` -> dev on the current stream
void stream_ring_step(int64_t id, Tensor pin, int64_t slot, std::vector<Tensor> stage, Tensor dev,
                      int64_t side_stream) {
  StreamRing& r = ring_at(id);
  TORCH_CHECK(stage.size() == r.stage_evt.size() && slot >= 0 && slot < (int64_t)r.slot_evt.size());
  TORCH_CHECK(!pin.is_cuda() && pin.is_pinned() && pin.is_contiguous() && dev.is_cuda() && dev.is_contiguous());
  const long long nbytes = (long long)pin.numel() * pin.element_size();
  const int k = r.k;
  r.k = (k + 1) % (int)stage.size();
  Tensor& st = stage[k];
  TORCH_CHECK(st.is_cuda() && st.is_contiguous() && (long long)st.numel() * st.element_size() == nbytes &&
              (long long)dev.numel() * dev.element_size() == nbytes, "size mismatch");
  void* alias = nullptr;
  TORCH_CHECK(cudaHostGetDevicePointer(&alias, pin.data_ptr(), 0) == cudaSuccess, "cudaHostGetDevicePointer");
  TORCH_CHECK((((uintptr_t)alias | (uintptr_t)st.data_ptr() | (uintptr_t)dev.data_ptr()) & 15) == 0, "16-byte alignment");
  cudaStream_t side = reinterpret_cast<cudaStream_t>(side_stream);
  cudaStream_t main = cur();
  if (r.stage_used[k]) cudaStreamWaitEvent(side, r.stage_evt[k], 0);   // its previous contents were copied out
  zn::launch_pull_from_host(alias, st.data_ptr(), nbytes, side);
  cudaEventRecord(r.pull_evt[k], side);
  cudaEventRecord(r.slot_evt[slot], side);                             // pinned slot free once the pull is done
  r.slot_used[slot] = 1;
  cudaStreamWaitEvent(main, r.pull_evt[k], 0);
  zn::launch_pull_from_host(st.data_ptr(), dev.data_ptr(), nbytes, main);
  cudaEventRecord(r.stage_evt[k], main);
  r.stage_used[k] = 1;
  kcheck();
}
bool stream_ring_slot_done(int64_t id, int64_t slot) {
  StreamRing& r = ring_at(id);
  if (!r.slot_used[slot]) return true;
  return cudaEventQuery(r.slot_evt[slot]) == cudaSuccess;
}
void stream_ring_slot_sync(int64_t id, int64_t slot) {
  StreamRing& r = ring_at(id);
  if (r.slot_used[slot]) {
    pybind11::gil_scoped_release nogil;
    cudaEventSynchronize(r.slot_evt[slot]);
  }
}
// dst (pinned host tensor) <- src (device): the same kernel storing straight into mapped host
// memory (per-step result read-back without a copy-engine operation in the stream).
void push_to_host(Tensor src, Tensor dst) {
  TORCH_CHECK(!dst.is_cuda() && dst.is_pinned() && dst.is_contiguous(), "dst must be pinned host memory");
  TORCH_CHECK(src.is_cuda() && src.is_contiguous(), "src must be a device tensor");
  const long long nbytes = (long long)src.numel() * src.element_size();
  TORCH_CHECK(nbytes == (long long)dst.numel() * dst.element_size(), "size mismatch");
  void* alias = nullptr;
  cudaError_t e = cudaHostGetDevicePointer(&alias, dst.data_ptr(), 0);
  TORCH_CHECK(e == cudaSuccess, "cudaHostGetDevicePointer: ", cudaGetErrorString(e));
  if ((((uintptr_t)alias | (uintptr_t)src.data_ptr()) & 15) == 0) {
    zn::launch_pull_from_host(src.data_ptr(), alias, nbytes, cur());
  } else {      // unaligned (tiny) payloads: byte tail path only
    TORCH_CHECK(nbytes <= 256, "unaligned push_to_host is limited to 256 bytes");
    zn::launch_pull_from_host_bytes(src.data_ptr(), alias, (int)nbytes, cur());
  }
  kcheck();
}
// device -> device byte copy by the same SM kernel (no copy-engine operation in the stream)
void device_copy(Tensor src, Tensor dst) {
  TORCH_CHECK(src.is_cuda() && dst.is_cuda() && src.is_contiguous() && dst.is_contiguous());
  const long long nbytes = (long long)src.numel() * src.element_size();
  TORCH_CHECK(nbytes == (long long)dst.numel() * dst.element_size(), "size mismatch");
  TORCH_CHECK((((uintptr_t)src.data_ptr() | (uintptr_t)dst.data_ptr()) & 15) == 0, "16-byte alignment");
  zn::launch_pull_from_host(src.data_ptr(), dst.data_ptr(), nbytes, cur());
  kcheck();
}
// ---- block-scaled fp8 (compute_type "fp8"): quantisers of fp8.cu + the fp8 mode of gemm_pair.cu
static uint8_t* codes_or_null(const c10::optional<Tensor>& t, long long* ld) {
  if (!t.has_value() || !t->defined()) return nullptr;
  TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->dim() == 2 && t->element_size() == 1,
              "fp8 codes: contiguous 2-D 1-byte tensor");
  *ld = t->size(1);
  return reinterpret_cast<uint8_t*>(t->data_ptr());
}
static float* scales_or_null(const c10::optional<Tensor>& t, long long need) {
  if (!t.has_value() || !t->defined()) return nullptr;
  TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->scalar_type() == torch::kFloat32 && t->numel() >= need,
              "fp8 scales: contiguous fp32 tensor of ", need, " elements");
  return t->data_ptr<float>();
}
// x [rows][cols] (bf16, or fp32 with tile = 1) -> row-block codes q [rows][ldq] + scales
// sq [ceil(cols / 128)][round_up(rows, 128)] and / or transposed codes qt [cols][ldqt] + scales
// sqt [ceil(rows / 128)][round_up(cols, 128)]; tile = 1: one scale per 128 x 128 tile
int64_t fp8_quant(Tensor x, int64_t rows, int64_t cols, int64_t tile, c10::optional<Tensor> q,
                  c10::optional<Tensor> sq, c10::optional<Tensor> qt, c10::optional<Tensor> sqt) {
  chk(x, "x");
  TORCH_CHECK(x.numel() == rows * cols, "x: rows x cols elements");
  const long long rp = (rows + 127) / 128 * 128, cp = (cols + 127) / 128 * 128;
  long long ldq = 0, ldqt = 0;
  uint8_t* qp = codes_or_null(q, &ldq);
  uint8_t* qtp = codes_or_null(qt, &ldqt);
  if (qp) TORCH_CHECK(q->size(0) == rows, "q: [rows][ldq]");
  if (qtp) TORCH_CHECK(qt->size(0) == cols, "qt: [cols][ldqt]");
  float* sqp = qp ? scales_or_null(sq, cp / 128 * rp) : nullptr;
  float* sqtp = qtp ? scales_or_null(sqt, rp / 128 * cp) : nullptr;
  int r = zn::launch_fp8_quant(x.data_ptr(), is_bf16(x) ? 0 : 1, cols, (int)rows, (int)cols, (int)tile,
                               qp, ldq, sqp, qtp, ldqt, sqtp, cur());
  if (r == 0) kcheck();
  return r;
}
// out[M][N] = act(alpha * sum_kb sa[kb][m] sb[kb][n] (a_kb . b_kb^T) + bias): a [M][lda], b [N][ldb]
// e4m3 codes, scales as written by fp8_quant. Returns 0, or non-zero when refused.
int64_t fp8_gemm(Tensor a, Tensor sa, Tensor b, Tensor sb, Tensor out, int64_t M, int64_t N, int64_t K,
                 c10::optional<Tensor> bias, int64_t act, double alpha) {
  long long lda = 0, ldb = 0;
  const uint8_t* ap = codes_or_null(a, &lda);
  const uint8_t* bp = codes_or_null(b, &ldb);
  TORCH_CHECK(ap && bp && a.size(0) >= M && b.size(0) >= N, "fp8 operands [M][lda], [N][ldb]");
  const long long kb = (K + 127) / 128;
  const float* sap = scales_or_null(sa, kb * ((M + 127) / 128 * 128));
  const float* sbp = scales_or_null(sb, kb * ((N + 127) / 128 * 128));
  chk(out, "out");
  TORCH_CHECK(out.numel() == M * N, "out: M x N elements");
  int r = zn::launch_gemm_fp8_block(ap, lda, sap, bp, ldb, sbp, out.data_ptr(), is_bf16(out) ? 0 : 1, N,
                                    (int)M, (int)N, (int)K, fptr_or_null(bias), (int)act, (float)alpha, cur());
  if (r == 0) kcheck();
  return r;
}
void pad_channels(Tensor x, Tensor y, int64_t C, int64_t CP) {
  chk(x, "x"); same_dt(x, y);
  zn::launch_pad_channels(x.data_ptr(), y.data_ptr(), (int)(x.numel() / C), (int)C, (int)CP, is_bf16(x), cur());
  kcheck();
}
void mask_mul(Tensor w, Tensor mask) {
  chk(w, "w"); same_dt(w, mask);
  zn::launch_mask_mul(w.data_ptr(), mask.data_ptr(), w.numel(), is_bf16(w), cur());
  kcheck();
}
void cast_copy(Tensor s, Tensor d) {
  chk(s, "s"); chk(d, "d");
  TORCH_CHECK(s.numel() == d.numel());
  zn::launch_cast(s.data_ptr(), is_bf16(s), d.data_ptr(), is_bf16(d), s.numel(), cur());
  kcheck();
}
void scatter_offsets(Tensor in, Tensor offs, Tensor out) {
  chk(in, "in"); same_dt(in, out);
  cudaMemsetAsync(out.data_ptr(), 0, out.numel() * out.element_size(), cur());
  zn::launch_scatter_offsets(in.data_ptr(), offs.data_ptr<int>(), out.data_ptr(), in.numel(), is_bf16(in), cur());
  kcheck();
}
void pool_forward(Tensor in, c10::optional<Tensor> out, c10::optional<Tensor> offs, int64_t OH, int64_t OW,
                  int64_t KY, int64_t KX, int64_t SY, int64_t SX, int64_t mode, c10::optional<Tensor> rng,
                  int64_t act) {
  chk(in, "in");
  TORCH_CHECK(act >= 0 && act <= 4 && (act == 0 || mode <= 2), "fused activation: max/maxabs/avg pooling only");
  void* op = (out.has_value() && out->defined()) ? out->data_ptr() : nullptr;
  int* fp = (offs.has_value() && offs->defined()) ? offs->data_ptr<int>() : nullptr;
  const int* rp = (rng.has_value() && rng->defined()) ? rng->data_ptr<int>() : nullptr;
  TORCH_CHECK(mode == 2 || fp, "offsets required");
  TORCH_CHECK(mode < 3 || rp, "rng required for stochastic pooling");
  zn::launch_pool_forward(in.data_ptr(), op, fp, (int)in.size(0), (int)in.size(1), (int)in.size(2),
                          (int)in.size(3), (int)OH, (int)OW, (int)KY, (int)KX, (int)SY, (int)SX, (int)mode,
                          rp, is_bf16(in), (int)act, cur());
  kcheck();
}
void pool_backward(Tensor err_out, c10::optional<Tensor> offs, Tensor err_in, int64_t OH, int64_t OW,
                   int64_t KY, int64_t KX, int64_t SY, int64_t SX, bool is_avg, c10::optional<Tensor> yact,
                   int64_t act, c10::optional<Tensor> xin, int64_t in_act) {
  chk(err_out, "err_out"); same_dt(err_out, err_in);
  const void* xp = nullptr;
  if (in_act != 0) {      // err_input *= f'(pooling input): the producer's activation derivative
    TORCH_CHECK(in_act >= 1 && in_act <= 4 && xin.has_value() && xin->defined(), "input derivative needs the input");
    same_dt(err_in, *xin);
    TORCH_CHECK(xin->numel() == err_in.numel());
    xp = xin->data_ptr();
  }
  const void* yp = nullptr;
  if (act != 0) {
    TORCH_CHECK(act >= 1 && act <= 4 && yact.has_value() && yact->defined(), "fused activation needs the output");
    same_dt(err_out, *yact);
    TORCH_CHECK(yact->numel() == err_out.numel());
    yp = yact->data_ptr();
  }
  const int* fp = (offs.has_value() && offs->defined()) ? offs->data_ptr<int>() : nullptr;
  TORCH_CHECK(is_avg || fp, "offsets required");
  zn::launch_pool_backward(err_out.data_ptr(), fp, err_in.data_ptr(), (int)err_in.size(0), (int)err_in.size(1),
                           (int)err_in.size(2), (int)err_in.size(3), (int)OH, (int)OW, (int)KY, (int)KX,
                           (int)SY, (int)SX, is_avg ? 1 : 0, is_bf16(err_out), yp, (int)act, xp, (int)in_act, cur());
  kcheck();
}
void lrn_forward(Tensor x, Tensor y, int64_t n, double alpha, double beta, double k) {
  chk(x, "x"); same_dt(x, y);
  int C = (int)x.size(-1);
  zn::launch_lrn_forward(x.data_ptr(), y.data_ptr(), x.numel() / C, C, (int)n, (float)alpha, (float)beta,
                         (float)k, is_bf16(x), cur());
  kcheck();
}
void lrn_backward(Tensor ey, Tensor x, Tensor eh, int64_t n, double alpha, double beta, double k,
                  int64_t in_act) {
  chk(x, "x"); same_dt(x, ey); same_dt(x, eh);
  TORCH_CHECK(in_act >= 0 && in_act <= 4, "producer derivative: tanh / softplus / relu / sigmoid only");
  int C = (int)x.size(-1);
  zn::launch_lrn_backward(ey.data_ptr(), x.data_ptr(), eh.data_ptr(), x.numel() / C, C, (int)n,
                          (float)alpha, (float)beta, (float)k, is_bf16(x), (int)in_act, cur());
  kcheck();
}
void softmax_rows(Tensor in, Tensor out, Tensor max_idx) {
  chk(in, "in");
  TORCH_CHECK(out.scalar_type() == torch::kFloat32);
  int rows = (int)in.size(0); int cols = (int)(in.numel() / rows);
  zn::launch_softmax_rows(in.data_ptr(), is_bf16(in), out.data_ptr<float>(), max_idx.data_ptr<int>(), rows,
                          cols, cur());
  kcheck();
}
void evaluate_softmax(Tensor y, Tensor max_idx, Tensor labels, Tensor err, Tensor bp, Tensor n_err,
                      c10::optional<Tensor> confusion, Tensor max_err_sum) {
  TORCH_CHECK(y.scalar_type() == torch::kFloat32);
  int rows = (int)y.size(0); int cols = (int)(y.numel() / rows);
  int* cp = (confusion.has_value() && confusion->defined() && confusion->numel()) ? confusion->data_ptr<int>() : nullptr;
  zn::launch_evaluate_softmax(y.data_ptr<float>(), max_idx.data_ptr<int>(), labels.data_ptr<int>(),
                              err.data_ptr(), is_bf16(err), bp.data_ptr<float>(), rows, cols,
                              n_err.data_ptr<int>(), cp, max_err_sum.data_ptr<float>(), cur());
  kcheck();
}
void evaluate_mse(Tensor y, Tensor target, Tensor err, Tensor bp, c10::optional<Tensor> denorm_mul,
                  bool root, Tensor metrics, Tensor mse) {
  chk(y, "y"); same_dt(y, target);
  int rows = (int)y.size(0); int cols = (int)(y.numel() / rows);
  zn::launch_evaluate_mse(y.data_ptr(), target.data_ptr(), is_bf16(y), err.data_ptr(), is_bf16(err),
                          bp.data_ptr<float>(), rows, cols, fptr_or_null(denorm_mul), root ? 1 : 0,
                          metrics.data_ptr<float>(), mse.data_ptr<float>(), cur());
  kcheck();
}
void mse_find_closest(Tensor y, Tensor class_targets, Tensor labels, Tensor bp, Tensor n_err) {
  chk(y, "y");
  int rows = (int)y.size(0); int cols = (int)(y.numel() / rows);
  zn::launch_mse_find_closest(y.data_ptr(), is_bf16(y), class_targets.data_ptr<float>(),
                              labels.data_ptr<int>(), bp.data_ptr<float>(), rows, cols,
                              (int)class_targets.size(0), n_err.data_ptr<int>(), cur());
  kcheck();
}

static __nv_bfloat16* bptr_or_null(const c10::optional<Tensor>& t) {
  if (!t.has_value() || !t->defined() || t->numel() == 0) return nullptr;
  TORCH_CHECK(t->scalar_type() == torch::kBFloat16 && t->is_cuda());
  return reinterpret_cast<__nv_bfloat16*>(t->data_ptr());
}
static float* mfptr_or_null(const c10::optional<Tensor>& t) {
  if (!t.has_value() || !t->defined() || t->numel() == 0) return nullptr;
  TORCH_CHECK(t->scalar_type() == torch::kFloat32 && t->is_cuda());
  return t->data_ptr<float>();
}

// One parameter update (kernels/api.py::UpdateDesc), read by attribute name: a missing attribute
// raises. Every check of the update's inputs is here, for both update kernels.
static zn::TensorDesc parse_desc(const py::handle& desc) {
  // a buffer: None or an empty tensor is absent (null)
  auto buf = [&](const char* name, torch::ScalarType dt) -> Tensor {
    const py::object o = desc.attr(name);
    const Tensor t = o.is_none() ? Tensor() : o.cast<Tensor>();
    if (!t.defined() || t.numel() == 0) return Tensor();
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == dt, "update descriptor: ", name, " must be a CUDA ",
                dt == torch::kFloat32 ? "float32" : "bfloat16", " tensor");
    return t;
  };
  auto f32 = [&](const char* name) {
    const Tensor t = buf(name, torch::kFloat32);
    return t.defined() ? t.data_ptr<float>() : nullptr;
  };
  auto bf16 = [&](const char* name) {
    const Tensor t = buf(name, torch::kBFloat16);
    return t.defined() ? reinterpret_cast<__nv_bfloat16*>(t.data_ptr()) : nullptr;
  };
  auto num = [&](const char* name) { return desc.attr(name).cast<int64_t>(); };
  const Tensor w = desc.attr("w").cast<Tensor>();
  TORCH_CHECK(w.scalar_type() == torch::kFloat32 && w.is_cuda() && w.is_contiguous(),
              "update descriptor: w must be a contiguous CUDA float32 tensor");
  zn::TensorDesc d{};
  d.w = w.data_ptr<float>();
  d.size = w.numel();
  d.grad = f32("grad");
  TORCH_CHECK(d.grad, "update descriptor: no gradient");
  d.grad_out = f32("grad_out"); d.acc = f32("acc"); d.vel = f32("vel"); d.col_sums = f32("col_sums");
  d.sh.lp = bf16("lp"); d.sh.lp_conv = bf16("lp_conv");
  d.part_stride = num("part_stride");
  d.nparts = (int)num("nparts"); d.g_cpad = (int)num("g_cpad"); d.flags = (int)num("flags");
  d.is_bias = (int)num("is_bias"); d.rows = (int)num("rows"); d.cols = (int)num("cols");
  d.lanes = (int)num("lanes");
  d.sh.ld = (int)num("ld"); d.sh.lp_cpad = (int)num("lp_cpad"); d.sh.taps = (int)num("taps");
  d.sh.C = (int)num("c"); d.sh.c_pad = (int)num("c_pad");
  // solver state (update.cu::step_elem): s0 adagrad h / adadelta E[dx^2] / RProp lrs,
  // s1 adadelta E[g^2], s2 fast f; each one element per weight
  auto state = [&](const char* name) {
    const Tensor t = buf(name, torch::kFloat32);
    TORCH_CHECK(!t.defined() || t.numel() == d.size, "update descriptor: solver state must match the weights");
    return t.defined() ? t.data_ptr<float>() : nullptr;
  };
  d.s0 = state("s0"); d.s1 = state("s1"); d.s2 = state("s2");
  const int fl = d.flags;
  TORCH_CHECK(!(fl & 256) || (d.grad_out && d.s0), "update descriptor: RProp needs grad_out (previous gradient) and the rates");
  TORCH_CHECK(!(fl & (32 | 64)) || d.s0, "update descriptor: adagrad / adadelta need s0");
  TORCH_CHECK(!(fl & 64) || d.s1, "update descriptor: adadelta needs s1");
  TORCH_CHECK(!(fl & 128) || d.s2, "update descriptor: fast needs s2");
  const Tensor hyper = desc.attr("hyper").cast<Tensor>();
  TORCH_CHECK(hyper.is_cuda() && hyper.scalar_type() == torch::kFloat32 &&
              hyper.numel() >= ((fl & (32 | 64 | 128 | 256)) ? 21 : 13),
              "update descriptor: the hyper vector is too short (solver slots 13-20)");
  d.hyper = hyper.data_ptr<float>();
  return d;
}

// The per-tensor step. grad_ptrs: every rank's split-K partials (int64 device addresses, rank
// order) when data-parallel; empty: the descriptor's local gradient.
void fused_update(py::handle desc, std::vector<int64_t> grad_ptrs, std::vector<int64_t> peer_flags,
                  int64_t epoch_ptr, int64_t rank, int64_t blocks) {
  const zn::TensorDesc d = parse_desc(desc);
  TORCH_CHECK(grad_ptrs.size() <= 8);
  const float* gp[8] = {d.grad}; uint32_t* fl[8];
  for (size_t i = 0; i < grad_ptrs.size(); ++i) gp[i] = reinterpret_cast<const float*>(grad_ptrs[i]);
  const int nranks = grad_ptrs.empty() ? 1 : (int)grad_ptrs.size();
  const bool multi = (int)peer_flags.size() == nranks && nranks > 1;
  if (multi) for (size_t i = 0; i < peer_flags.size(); ++i) fl[i] = reinterpret_cast<uint32_t*>(peer_flags[i]);
  zn::launch_fused_update(d, gp, nranks, multi ? fl : nullptr, reinterpret_cast<uint32_t*>(epoch_ptr),
                          (int)rank, (int)blocks, cur());
  kcheck();
}

// Whole-network step table: one descriptor per tensor, enabled[i] = tensor i is stepped this time.
// Returns (packed CPU uint8 tensor [n * sizeof(TensorDesc)], total_tiles, end of the reduction
// buffer, whether a tensor has the ortho regulariser: the kernel's column-sum phase).
std::tuple<Tensor, int64_t, int64_t, bool> multi_update_table(std::vector<py::object> descs,
                                                              std::vector<bool> enabled, int64_t red_base) {
  TORCH_CHECK(descs.size() <= (size_t)zn::MU_MAX_TENSORS,
              "multi_update handles at most ", zn::MU_MAX_TENSORS, " tensors per launch");
  TORCH_CHECK(enabled.size() == descs.size(), "multi_update_table: one enabled flag per descriptor");
  const size_t ds = sizeof(zn::TensorDesc);
  Tensor out = torch::zeros({(int64_t)(descs.size() * ds)}, torch::dtype(torch::kUInt8));
  int tiles = 0;
  long long red = red_base;
  bool has_ortho = false;
  for (size_t i = 0; i < descs.size(); ++i) {
    zn::TensorDesc d = parse_desc(descs[i]);
    d.enabled = enabled[i] ? 1 : 0;
    has_ortho |= (d.flags & 8) && d.col_sums && !d.is_bias;
    tiles += zn::multi_update_pack(d, tiles, red);
    std::memcpy(out.data_ptr<uint8_t>() + i * ds, &d, ds);
    // one fp32 slot per element in the cross-GPU reduction buffer; every tensor starts on a
    // 16-byte boundary (the 4-elements-per-thread tile path uses float4 accesses)
    red += (d.size + 3) / 4 * 4;
  }
  return std::make_tuple(out, (int64_t)tiles, (int64_t)red, has_ortho);
}
void multi_update(Tensor table, int64_t n, int64_t total_tiles, bool has_ortho,
                  std::vector<int64_t> peer_flags, int64_t epoch_ptr, int64_t rank, Tensor gridsync,
                  std::vector<int64_t> red_ptrs, int64_t red_half, int64_t chunks,
                  std::vector<int64_t> sum_ptrs, int64_t mc_red, int64_t mc_sum, int64_t algo,
                  int64_t max_blocks) {
  TORCH_CHECK(table.is_cuda() && table.scalar_type() == torch::kUInt8);
  TORCH_CHECK(gridsync.is_cuda() && gridsync.scalar_type() == torch::kInt32 && gridsync.numel() >= 2);
  uint32_t* fl[8];
  const int nranks = peer_flags.size() > 1 ? (int)peer_flags.size() : 1;
  TORCH_CHECK(nranks <= 8);
  for (int i = 0; i < nranks && peer_flags.size() > 1; ++i) fl[i] = reinterpret_cast<uint32_t*>(peer_flags[i]);
  float* rp[8] = {nullptr};
  if (nranks > 1) {
    TORCH_CHECK((int)red_ptrs.size() == nranks, "data-parallel multi_update needs the reduction buffers");
    for (int i = 0; i < nranks; ++i) rp[i] = reinterpret_cast<float*>(red_ptrs[i]);
  }
  float* sp[8] = {nullptr};
  TORCH_CHECK(algo >= 0 && algo <= 2, "multi_update: unknown algo");
  if (nranks > 1 && algo == 1) {
    TORCH_CHECK((int)sum_ptrs.size() == nranks, "two-shot multi_update needs the sum buffers");
    for (int i = 0; i < nranks; ++i) sp[i] = reinterpret_cast<float*>(sum_ptrs[i]);
    TORCH_CHECK((mc_red == 0) == (mc_sum == 0), "two-shot: both multicast mappings or none");
  }
  if (nranks > 1 && algo == 2) TORCH_CHECK(mc_red != 0, "one-shot NVLS needs the multicast mapping");
  zn::launch_multi_update(table.data_ptr(), (int)n, (int)total_tiles, has_ortho ? 1 : 0, nranks,
                          nranks > 1 ? fl : nullptr, reinterpret_cast<uint32_t*>(epoch_ptr), (int)rank,
                          reinterpret_cast<unsigned*>(gridsync.data_ptr<int32_t>()), nranks > 1 ? rp : nullptr, (long long)red_half, (int)chunks,
                          (nranks > 1 && algo == 1) ? sp : nullptr, reinterpret_cast<float*>(mc_red),
                          reinterpret_cast<float*>(mc_sum), (int)algo, (int)max_blocks, cur());
  kcheck();
}
void col_sums(Tensor w, Tensor out, int64_t rows, int64_t cols, bool transposed) {
  zn::launch_col_sums(w.data_ptr<float>(), out.data_ptr<float>(), (int)rows, (int)cols, transposed ? 1 : 0, cur());
  kcheck();
}
// RBM Gibbs sample: out = Bernoulli(in) on the first batch_size rows, a copy of in on the rest
void rbm_sample(Tensor in, Tensor out, int64_t batch_size, Tensor rng) {
  chk(in, "in"); chk(out, "out"); same_dt(in, out);
  TORCH_CHECK(in.scalar_type() != torch::kInt32 && in.numel() == out.numel() && in.dim() >= 1, "rbm_sample: operands");
  TORCH_CHECK(rng.is_cuda() && rng.scalar_type() == torch::kInt32 && rng.numel() >= 2, "rbm_sample: rng");
  const int64_t rows = in.size(0), cols = rows ? in.numel() / rows : 0;
  TORCH_CHECK(batch_size >= 0 && batch_size <= rows, "rbm_sample: batch_size out of range");
  zn::launch_rbm_sample(in.data_ptr(), out.data_ptr(), batch_size * cols, in.numel(), rng.data_ptr<int>(),
                        is_bf16(in), cur());
  kcheck();
}
// RBM update: w[H][V] += lr * g[V][H]^T, hbias[H] += lr * hgrad, vbias[V] += lr * vgrad (all fp32)
void rbm_apply(Tensor w, Tensor g, Tensor hbias, Tensor hgrad, Tensor vbias, Tensor vgrad, double lr) {
  for (const Tensor* t : {&w, &g, &hbias, &hgrad, &vbias, &vgrad}) {
    chk(*t, "rbm_apply operand");
    TORCH_CHECK(t->scalar_type() == torch::kFloat32, "rbm_apply: fp32 operands");
  }
  TORCH_CHECK(w.dim() == 2, "rbm_apply: w must be [H][V]");
  const int64_t H = w.size(0), V = w.size(1);
  TORCH_CHECK(g.numel() == H * V && hbias.numel() == H && hgrad.numel() == H && vbias.numel() == V &&
              vgrad.numel() == V, "rbm_apply: shapes");
  zn::launch_rbm_apply(w.data_ptr<float>(), g.data_ptr<float>(), hbias.data_ptr<float>(), hgrad.data_ptr<float>(),
                       vbias.data_ptr<float>(), vgrad.data_ptr<float>(), (int)H, (int)V, (float)lr, cur());
  kcheck();
}
void refresh_shadows(Tensor w, int64_t rows, int64_t cols, c10::optional<Tensor> lp, int64_t ld,
                     c10::optional<Tensor> lp_conv, int64_t taps, int64_t C, int64_t c_pad, int64_t lp_cpad) {
  zn::launch_refresh_shadows(w.data_ptr<float>(), w.numel(), (int)rows, (int)cols, bptr_or_null(lp), (int)ld,
                             bptr_or_null(lp_conv), (int)taps, (int)C, (int)c_pad, (int)lp_cpad, cur());
  kcheck();
}

// LSTM sequence cell (ops/lstm_seq.py). Strided destinations are given as base tensor + element
// offset + leading dimension.
static inline size_t esz(const Tensor& t) { return (size_t)t.element_size(); }
void lstm_cell_fwd(Tensor z, c10::optional<Tensor> c_prev, Tensor c, Tensor gates, Tensor h_out,
                   int64_t h_off, int64_t ldh, c10::optional<Tensor> h_next, int64_t n_off, int64_t ldn,
                   int64_t batch, int64_t H) {
  TORCH_CHECK(z.scalar_type() == torch::kFloat32 && c.scalar_type() == torch::kFloat32 &&
              gates.scalar_type() == torch::kFloat32 && z.is_cuda());
  TORCH_CHECK(z.numel() >= batch * 4 * H && gates.numel() >= batch * 4 * H && c.numel() >= batch * H);
  chk(h_out, "h_out");
  void* hn = nullptr;
  if (h_next.has_value() && h_next->defined()) {
    same_dt(h_out, *h_next);
    hn = static_cast<char*>(h_next->data_ptr()) + n_off * esz(*h_next);
  }
  zn::launch_lstm_cell_fwd(z.data_ptr<float>(), fptr_or_null(c_prev), c.data_ptr<float>(),
                           gates.data_ptr<float>(), static_cast<char*>(h_out.data_ptr()) + h_off * esz(h_out),
                           ldh, hn, ldn, (int)batch, (int)H, is_bf16(h_out), cur());
  kcheck();
}
void lstm_cell_bwd(c10::optional<Tensor> err_h, int64_t e_off, int64_t lde, c10::optional<Tensor> dh_rec,
                   int64_t r_off, int64_t ldr, c10::optional<Tensor> dc_next, Tensor gates, Tensor c,
                   c10::optional<Tensor> c_prev, Tensor dc_prev, Tensor dz, int64_t batch, int64_t H) {
  chk(dz, "dz");
  TORCH_CHECK(gates.scalar_type() == torch::kFloat32 && c.scalar_type() == torch::kFloat32 &&
              dc_prev.scalar_type() == torch::kFloat32);
  const void* ep = nullptr; const void* rp = nullptr;
  if (err_h.has_value() && err_h->defined()) {
    same_dt(dz, *err_h);
    ep = static_cast<const char*>(err_h->data_ptr()) + e_off * esz(*err_h);
  }
  if (dh_rec.has_value() && dh_rec->defined()) {
    same_dt(dz, *dh_rec);
    rp = static_cast<const char*>(dh_rec->data_ptr()) + r_off * esz(*dh_rec);
  }
  zn::launch_lstm_cell_bwd(ep, lde, rp, ldr, fptr_or_null(dc_next), gates.data_ptr<float>(),
                           c.data_ptr<float>(), fptr_or_null(c_prev), dc_prev.data_ptr<float>(),
                           dz.data_ptr(), (int)batch, (int)H, is_bf16(dz), cur());
  kcheck();
}

// FC layers with n_out <= fc_small_max_out(): see csrc/fc_small.cu
int64_t fc_small_max_out() { return zn::fc_small_max_out(); }
// ev = [labels(int32), err_output, batch_dev(float[2]), n_err(int32[2]), max_err_sum(float[1]),
//       confusion(int32, optional)] - the fused softmax evaluator (see fc_small.cu::EvalArgs)
void fc_small_forward(Tensor x, Tensor w, c10::optional<Tensor> bias, Tensor out, c10::optional<Tensor> max_idx,
                      int64_t batch, int64_t n_in, int64_t n_out, int64_t act, bool softmax,
                      std::vector<Tensor> ev) {
  chk(x, "x"); chk(out, "out");
  TORCH_CHECK(w.scalar_type() == torch::kFloat32 && w.is_cuda() && w.is_contiguous(), "weights must be fp32");
  TORCH_CHECK(n_out <= zn::fc_small_max_out() && w.numel() == n_out * n_in);
  TORCH_CHECK(x.numel() >= batch * n_in && out.numel() >= batch * n_out);
  const bool out_f32 = out.scalar_type() == torch::kFloat32;
  TORCH_CHECK(out_f32 || out.scalar_type() == x.scalar_type(), "output dtype must be fp32 or match the input");
  int* mi = nullptr;
  if (max_idx.has_value() && max_idx->defined()) {
    TORCH_CHECK(max_idx->scalar_type() == torch::kInt32 && max_idx->numel() >= batch);
    mi = max_idx->data_ptr<int>();
  }
  const bool xb = is_bf16(x);
  // fp32 output of a bf16 input goes through out_f; same-dtype output through out_t
  void* out_t = (out_f32 && xb) ? nullptr : out.data_ptr();
  float* out_f = (out_f32 && xb) ? out.data_ptr<float>() : nullptr;
  if (!xb) { out_t = out.data_ptr(); out_f = nullptr; }
  const int* ev_labels = nullptr; void* ev_err = nullptr; int ev_bf16 = 0; const float* ev_bp = nullptr;
  int* ev_n_err = nullptr; int* ev_conf = nullptr; float* ev_max = nullptr;
  if (!ev.empty()) {
    TORCH_CHECK(softmax && mi && ev.size() >= 5, "fused evaluator needs the softmax + arg-max path");
    TORCH_CHECK(ev[0].scalar_type() == torch::kInt32 && ev[0].numel() >= batch, "labels");
    chk(ev[1], "err_output");
    TORCH_CHECK(ev[1].numel() >= batch * n_out, "err_output size");
    TORCH_CHECK(ev[2].scalar_type() == torch::kFloat32 && ev[2].numel() >= 2, "batch scalars");
    TORCH_CHECK(ev[3].scalar_type() == torch::kInt32 && ev[3].numel() >= 2, "n_err");
    TORCH_CHECK(ev[4].scalar_type() == torch::kFloat32 && ev[4].numel() >= 1, "max_err_sum");
    ev_labels = ev[0].data_ptr<int>(); ev_err = ev[1].data_ptr(); ev_bf16 = is_bf16(ev[1]) ? 1 : 0;
    ev_bp = ev[2].data_ptr<float>(); ev_n_err = ev[3].data_ptr<int>(); ev_max = ev[4].data_ptr<float>();
    if (ev.size() > 5) {
      TORCH_CHECK(ev[5].scalar_type() == torch::kInt32 && ev[5].numel() >= n_out * n_out, "confusion");
      ev_conf = ev[5].data_ptr<int>();
    }
  }
  zn::launch_fc_small_forward(x.data_ptr(), xb, w.data_ptr<float>(), fptr_or_null(bias), out_t, out_f, mi,
                              (int)batch, (int)n_in, (int)n_out, (int)act, softmax ? 1 : 0, ev_labels,
                              ev_err, ev_bf16, ev_bp, ev_n_err, ev_conf, ev_max, cur());
  kcheck();
}
void fc_small_backward(Tensor err, c10::optional<Tensor> y, Tensor x, Tensor w, c10::optional<Tensor> err_in,
                       c10::optional<Tensor> gw_parts, c10::optional<Tensor> gb_parts, int64_t batch,
                       int64_t n_in, int64_t n_out, int64_t act, double alpha, double beta, int64_t bsplit) {
  chk(err, "err"); chk(x, "x");
  same_dt(err, x);
  TORCH_CHECK(w.scalar_type() == torch::kFloat32 && w.is_cuda() && w.is_contiguous());
  TORCH_CHECK(n_out <= zn::fc_small_max_out() && bsplit >= 1);
  TORCH_CHECK(act >= 0 && act <= 4, "fc_small_backward supports linear/tanh/relu/strict relu/sigmoid");
  const void* yp = nullptr;
  if (act != 0) {
    TORCH_CHECK(y.has_value() && y->defined(), "activation derivative needs the output");
    same_dt(err, *y);
    yp = y->data_ptr();
  }
  void* eip = nullptr;
  if (err_in.has_value() && err_in->defined()) { same_dt(err, *err_in); eip = err_in->data_ptr(); }
  float* gw = nullptr; float* gb = nullptr;
  if (gw_parts.has_value() && gw_parts->defined()) {
    TORCH_CHECK(gw_parts->scalar_type() == torch::kFloat32 && gw_parts->numel() >= bsplit * n_out * n_in);
    gw = gw_parts->data_ptr<float>();
  }
  if (gb_parts.has_value() && gb_parts->defined()) {
    TORCH_CHECK(gb_parts->scalar_type() == torch::kFloat32 && gb_parts->numel() >= bsplit * n_out);
    gb = gb_parts->data_ptr<float>();
  }
  zn::launch_fc_small_backward(err.data_ptr(), yp, x.data_ptr(), is_bf16(err), w.data_ptr<float>(), eip, gw, gb,
                               (int)batch, (int)n_in, (int)n_out, (int)act, (float)alpha, (float)beta,
                               (int)bsplit, cur());
  kcheck();
}

// generic GEMM: out[M,N] = act(alpha * opA(a) opB(b) + bias) + beta*out ; engine: 0 simt, 1 umma
// transa: A stored [K][lda]; transb: B stored [N][ldb] (i.e. "NT" when transb = 1)
int64_t gemm(Tensor a, int64_t lda, bool transa, Tensor b, int64_t ldb, bool transb, Tensor out,
             int64_t ldo, bool out_trans, int64_t M, int64_t N, int64_t K, c10::optional<Tensor> bias,
             int64_t act, double alpha, double beta, int64_t splits, int64_t split_stride, int64_t engine) {
  chk(a, "a"); chk(b, "b"); chk(out, "out");
  if (engine == 1) {
    TORCH_CHECK(is_bf16(a) && is_bf16(b), "wgmma path needs bf16 operands");
    int r = zn::launch_gemm_umma(a.data_ptr(), lda, transa ? 1 : 0, b.data_ptr(), ldb, transb ? 0 : 1,
                                 out.data_ptr(), is_bf16(out) ? 1 : 0, ldo, out_trans ? 1 : 0, (int)M,
                                 (int)N, (int)K, fptr_or_null(bias), (int)act, (float)alpha, (float)beta,
                                 (int)splits, split_stride, cur());
    if (r == 0) kcheck();
    return r;
  }
  zn::launch_gemm_simt(a.data_ptr(), is_bf16(a), lda, transa ? 1 : 0, b.data_ptr(), is_bf16(b), ldb,
                       transb ? 1 : 0, out.data_ptr(), is_bf16(out), ldo, out_trans ? 1 : 0, (int)M, (int)N,
                       (int)K, fptr_or_null(bias), (int)act, (float)alpha, (float)beta,
                       (int)(splits < 1 ? 1 : splits), split_stride, cur());
  kcheck();
  return 0;
}
// persistent warp-specialised wgmma GEMM (gemm_pair.cu): out[M][N] = act(alpha * a[M][K] . b[N][K]^T + bias)
int64_t gemm_pair(Tensor a, Tensor b, Tensor out, c10::optional<Tensor> bias, int64_t act, double alpha) {
  chk(a, "a"); chk(b, "b"); chk(out, "out");
  TORCH_CHECK(is_bf16(a) && is_bf16(b) && a.dim() == 2 && b.dim() == 2 && out.dim() == 2);
  TORCH_CHECK(a.size(1) == b.size(1) && out.size(0) == a.size(0) && out.size(1) == b.size(0));
  TORCH_CHECK(is_bf16(out) || out.scalar_type() == torch::kFloat32);
  int r = zn::launch_gemm_pair(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(),
                               is_bf16(out) ? 0 : 1, out.stride(0), (int)a.size(0), (int)b.size(0),
                               (int)a.size(1), fptr_or_null(bias), (int)act, (float)alpha, cur());
  if (r == 0) kcheck();
  return r;
}
// FC weight gradient on the persistent kernel: out[n_out][n_in] fp32 = err[batch][n_out]^T . x[batch][n_in]
int64_t fc_wgrad_pair(Tensor err, Tensor x, Tensor out) {
  chk(err, "err"); chk(x, "x"); chk(out, "out");
  TORCH_CHECK(is_bf16(err) && is_bf16(x) && out.scalar_type() == torch::kFloat32);
  TORCH_CHECK(err.dim() == 2 && x.dim() == 2 && err.size(0) == x.size(0));
  TORCH_CHECK(out.numel() == err.size(1) * x.size(1));
  int r = zn::launch_fc_wgrad_pair(err.data_ptr(), err.size(1), x.data_ptr(), x.size(1),
                                   out.data_ptr<float>(), x.size(1), (int)err.size(1), (int)x.size(1),
                                   (int)err.size(0), cur());
  if (r == 0) kcheck();
  return r;
}
int64_t pick_splits(int64_t M, int64_t N, int64_t K, int64_t max_splits) {
  return zn::umma_pick_splits((int)M, (int)N, (int)K, (int)max_splits);
}

// geometry vector: [N,H,W,C,OH,OW,F,KY,KX,SY,SX,PT,PL]
int64_t conv_fprop(Tensor x, Tensor w, int64_t ldw, bool w_trans, c10::optional<Tensor> bias, Tensor out,
                   std::vector<int64_t> g, int64_t act, int64_t engine) {
  TORCH_CHECK(g.size() == 13);
  int gi[13]; for (int i = 0; i < 13; ++i) gi[i] = (int)g[i];
  if (engine == 1) {
    TORCH_CHECK(is_bf16(x) && is_bf16(w));
    int r = zn::launch_conv_fprop_umma(x.data_ptr(), w.data_ptr(), ldw, fptr_or_null(bias), out.data_ptr(),
                                       is_bf16(out) ? 1 : 0, gi[0], gi[1], gi[2], gi[3], gi[4], gi[5], gi[6],
                                       gi[7], gi[8], gi[9], gi[10], gi[11], gi[12], (int)act, cur());
    if (r == 0) kcheck();
    return r;
  }
  TORCH_CHECK(w.scalar_type() == torch::kFloat32);
  zn::launch_conv_fprop_simt_raw(x.data_ptr(), is_bf16(x), w.data_ptr<float>(), ldw, w_trans ? 1 : 0,
                                 fptr_or_null(bias), out.data_ptr(), is_bf16(out), gi, (int)act, cur());
  kcheck();
  return 0;
}
// dmul / dact (engine 1 only): err_in *= f'(dmul), dmul = the layer's input (the producer's output)
int64_t conv_dgrad(Tensor err_out, Tensor w, int64_t ldw, bool w_trans, Tensor err_in,
                   std::vector<int64_t> g, double alpha, double beta, int64_t engine,
                   c10::optional<Tensor> dmul, int64_t dact) {
  TORCH_CHECK(g.size() == 13);
  int gi[13]; for (int i = 0; i < 13; ++i) gi[i] = (int)g[i];
  const void* dm = nullptr;
  if (dmul.has_value() && dmul->defined() && dact != 0) {
    TORCH_CHECK(engine == 1 && dact >= 1 && dact <= 4 && is_bf16(*dmul) && dmul->is_cuda() &&
                dmul->is_contiguous() && dmul->numel() == err_in.numel(), "dgrad derivative operand");
    dm = dmul->data_ptr();
  }
  if (engine == 1) {
    TORCH_CHECK(is_bf16(err_out) && is_bf16(w));
    int r = zn::launch_conv_dgrad_umma(err_out.data_ptr(), w.data_ptr(), ldw, err_in.data_ptr(),
                                       is_bf16(err_in) ? 1 : 0, gi[0], gi[1], gi[2], gi[3], gi[4], gi[5],
                                       gi[6], gi[7], gi[8], gi[9], gi[10], gi[11], gi[12], (float)alpha,
                                       (float)beta, dm, (int)dact, cur());
    if (r == 0) kcheck();
    return r;
  }
  TORCH_CHECK(w.scalar_type() == torch::kFloat32);
  zn::launch_conv_dgrad_simt_raw(err_out.data_ptr(), is_bf16(err_out), w.data_ptr<float>(), ldw,
                                 w_trans ? 1 : 0, err_in.data_ptr(), is_bf16(err_in), gi, (float)alpha,
                                 (float)beta, cur());
  kcheck();
  return 0;
}
int64_t conv_wgrad(Tensor err_out, Tensor x, Tensor partials, int64_t splits, std::vector<int64_t> g,
                   bool out_trans, int64_t engine, c10::optional<Tensor> bias_parts) {
  TORCH_CHECK(g.size() == 13 && partials.scalar_type() == torch::kFloat32);
  int gi[13]; for (int i = 0; i < 13; ++i) gi[i] = (int)g[i];
  if (engine == 1) {
    TORCH_CHECK(is_bf16(err_out) && is_bf16(x) && !out_trans);
    float* bp = nullptr;
    if (bias_parts.has_value() && bias_parts->defined()) {
      TORCH_CHECK(bias_parts->scalar_type() == torch::kFloat32 && bias_parts->numel() >= splits * gi[6]);
      bp = bias_parts->data_ptr<float>();
    }
    int r = zn::launch_conv_wgrad_umma(err_out.data_ptr(), x.data_ptr(), partials.data_ptr<float>(),
                                       (int)splits, gi[0], gi[1], gi[2], gi[3], gi[4], gi[5], gi[6], gi[7],
                                       gi[8], gi[9], gi[10], gi[11], gi[12], bp, cur());
    if (r == 0 || r == 1) kcheck();
    return r;
  }
  zn::launch_conv_wgrad_simt_raw(err_out.data_ptr(), is_bf16(err_out), x.data_ptr(), is_bf16(x),
                                 partials.data_ptr<float>(), (int)splits, gi, out_trans ? 1 : 0, cur());
  kcheck();
  return 0;
}

namespace zn {
void launch_som_split(const float*, __nv_bfloat16*, int, int, int, long long, long long, int, float*, cudaStream_t);
void launch_som_argmin(const float*, const float*, int*, int*, int, int, cudaStream_t);
void launch_som_gravity_split(const float*, const int*, __nv_bfloat16*, float*, int, int, int, float, cudaStream_t);
void launch_som_apply(float*, const float*, const float*, int, int, float, cudaStream_t);
}
// fp32 [rows][len] -> bf16 hi/lo parts (see som.cu); stack_rows: parts stacked along the rows of
// dst ([3 * rows_pad][ld]) instead of concatenated along its columns ([rows][3 * kp])
void som_split(Tensor src, Tensor dst, int64_t rows, int64_t len, int64_t kp, int64_t ld,
               int64_t part_stride, int64_t pattern, c10::optional<Tensor> norm_out) {
  TORCH_CHECK(src.scalar_type() == torch::kFloat32 && is_bf16(dst) && src.is_cuda() && dst.is_cuda());
  TORCH_CHECK(src.numel() >= rows * len && dst.numel() >= 2 * part_stride + (rows - 1) * ld + kp);
  zn::launch_som_split(src.data_ptr<float>(), reinterpret_cast<__nv_bfloat16*>(dst.data_ptr()), (int)rows,
                       (int)len, (int)kp, ld, part_stride, (int)pattern, mfptr_or_null(norm_out), cur());
  kcheck();
}
namespace zn {
int launch_lstm_fwd_persist(void*, const void*, long long, const float*, void*, int, int, int, int, long long*,
                            cudaStream_t);
int launch_lstm_bwd_persist(const void*, long long, int, const void*, void*, void*, const void*, long long, void*,
                            int, int, int, int, cudaStream_t);
void launch_lstm_unpack_state(const void*, float*, float*, int, int, int, cudaStream_t);
long long lstm_persist_state_elems(int, int, int, int);
long long lstm_persist_part_elems(int, int);
long long lstm_persist_launches();
}
// whole LSTM time loop in one cluster launch (lstm_persist.cu); != 0: shape outside its range.
// `state` (lstm_state_floats() fp32 words) carries gates / cells to the backward kernel; h_t is written into
// the [x | h] operand xh[t + 1][:, I:].
int64_t lstm_fwd_persist(Tensor xh, Tensor w_lp, c10::optional<Tensor> bias, Tensor state, int64_t hidden,
                         c10::optional<Tensor> dbg) {
  chk(xh, "xh"); chk(w_lp, "w_lp"); chk(state, "state");
  TORCH_CHECK(is_bf16(xh) && is_bf16(w_lp) && xh.dim() == 3 && state.scalar_type() == torch::kFloat32);
  const int T = (int)xh.size(0) - 1, B = (int)xh.size(1), H = (int)hidden;
  const int I = (int)xh.size(2) - H;
  TORCH_CHECK(T >= 1 && I > 0 && w_lp.size(0) == 4 * H && w_lp.size(1) >= I + H);
  const long long need = zn::lstm_persist_state_elems(T, B, I, H);
  if (need == 0) return -3;
  TORCH_CHECK(state.numel() >= need * 4, "lstm state buffer too small");
  int r = zn::launch_lstm_fwd_persist(xh.data_ptr(), w_lp.data_ptr(), w_lp.size(1), fptr_or_null(bias),
                                      state.data_ptr(), T, B, I, H,
                                      (dbg.has_value() && dbg->defined()) ? (long long*)dbg->data_ptr<int64_t>() : nullptr,
                                      cur());
  if (r == 0) kcheck();
  return r;
}
int64_t lstm_bwd_persist(Tensor err, bool seq, Tensor state, Tensor part, Tensor dz, Tensor w_lp, Tensor whp,
                         int64_t n_in) {
  chk(err, "err"); chk(state, "state"); chk(part, "part"); chk(dz, "dz"); chk(w_lp, "w_lp"); chk(whp, "whp");
  TORCH_CHECK(is_bf16(err) && is_bf16(dz) && is_bf16(w_lp) && is_bf16(whp) && dz.dim() == 3);
  TORCH_CHECK(state.scalar_type() == torch::kFloat32 && part.scalar_type() == torch::kFloat32);
  const int T = (int)dz.size(0), B = (int)dz.size(1), H = (int)dz.size(2) / 4;
  const long long need = zn::lstm_persist_state_elems(T, B, (int)n_in, H);
  if (need == 0) return -3;
  TORCH_CHECK(state.numel() >= need * 4 && whp.numel() >= (int64_t)4 * H * H);
  TORCH_CHECK(part.numel() >= zn::lstm_persist_part_elems(B, H) * 4, "lstm partial-sum buffer too small");
  TORCH_CHECK(err.numel() == (int64_t)B * H * (seq ? T : 1) && w_lp.size(0) == 4 * H && w_lp.size(1) >= n_in + H);
  int r = zn::launch_lstm_bwd_persist(err.data_ptr(), seq ? (long long)T * H : (long long)H, seq ? 1 : 0,
                                      state.data_ptr(), part.data_ptr(), dz.data_ptr(), w_lp.data_ptr(),
                                      w_lp.size(1), whp.data_ptr(), T, B, (int)n_in, H, cur());
  if (r == 0) kcheck();
  return r;
}
int64_t lstm_state_floats(int64_t T, int64_t B, int64_t I, int64_t H) {
  return 4 * zn::lstm_persist_state_elems((int)T, (int)B, (int)I, (int)H);
}
int64_t lstm_part_floats(int64_t B, int64_t H) { return 4 * zn::lstm_persist_part_elems((int)B, (int)H); }
void lstm_unpack_state(Tensor state, Tensor gates, Tensor cells) {
  chk(state, "state"); chk(gates, "gates"); chk(cells, "cells");
  TORCH_CHECK(gates.scalar_type() == torch::kFloat32 && cells.scalar_type() == torch::kFloat32 && gates.dim() == 3);
  const int T = (int)gates.size(0), B = (int)gates.size(1), H = (int)gates.size(2) / 4;
  zn::launch_lstm_unpack_state(state.data_ptr(), gates.data_ptr<float>(), cells.data_ptr<float>(), T, B, H, cur());
  kcheck();
}
namespace zn {
void launch_space_to_depth(const void*, bool, void*, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
void launch_s2d_pack_weights(const float*, void*, int, int, int, int, int, int, int, int, cudaStream_t);
void launch_s2d_unpack_grad(const float*, float*, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
}
// space-to-depth form of a strided first-layer convolution (s2d.cu)
void space_to_depth(Tensor x, Tensor xs, int64_t s, int64_t pad_t, int64_t pad_l) {
  chk(x, "x"); chk(xs, "xs");
  TORCH_CHECK(x.dim() == 4 && xs.dim() == 4 && is_bf16(xs) && xs.size(0) == x.size(0));
  TORCH_CHECK(xs.size(3) >= s * s * x.size(3));
  zn::launch_space_to_depth(x.data_ptr(), is_bf16(x), xs.data_ptr(), (int)x.size(0), (int)x.size(1),
                            (int)x.size(2), (int)x.size(3), (int)s, (int)pad_t, (int)pad_l, (int)xs.size(1),
                            (int)xs.size(2), (int)xs.size(3), cur());
  kcheck();
}
void s2d_pack_weights(Tensor w, Tensor ws, int64_t F, int64_t ky, int64_t kx, int64_t C, int64_t s, int64_t kyp,
                      int64_t kxp, int64_t Cp) {
  chk(w, "w"); chk(ws, "ws");
  TORCH_CHECK(w.scalar_type() == torch::kFloat32 && is_bf16(ws) && w.numel() >= F * ky * kx * C &&
              ws.numel() >= F * kyp * kxp * Cp && Cp >= s * s * C);
  zn::launch_s2d_pack_weights(w.data_ptr<float>(), ws.data_ptr(), (int)F, (int)ky, (int)kx, (int)C, (int)s, (int)kyp,
                              (int)kxp, (int)Cp, cur());
  kcheck();
}
void s2d_unpack_grad(Tensor gs, Tensor g, int64_t parts, int64_t F, int64_t Fr, int64_t ky, int64_t kx, int64_t C,
                     int64_t s, int64_t kyp, int64_t kxp, int64_t Cp) {
  chk(gs, "gs"); chk(g, "g");
  TORCH_CHECK(gs.scalar_type() == torch::kFloat32 && g.scalar_type() == torch::kFloat32);
  TORCH_CHECK(gs.numel() >= parts * Fr * kyp * kxp * Cp && g.numel() >= parts * F * ky * kx * C && Fr >= F);
  zn::launch_s2d_unpack_grad(gs.data_ptr<float>(), g.data_ptr<float>(), (int)parts, (int)F, (int)Fr, (int)ky, (int)kx,
                             (int)C, (int)s, (int)kyp, (int)kxp, (int)Cp, cur());
  kcheck();
}
namespace zn {
void launch_metric_reduce(const double* const*, int, int, uint32_t* const*, uint32_t*, double*, int, int, int, cudaStream_t);
}
// epoch-end metrics: sum the first n_sum and take the maximum of the next n_max doubles of every rank's
// symmetric slot (src_ptrs / flag_ptrs: one address per rank, epoch_ptr: this rank's counter)
void metric_reduce(std::vector<int64_t> src_ptrs, std::vector<int64_t> flag_ptrs, int64_t epoch_ptr, int64_t rank,
                   Tensor out, int64_t n_sum, int64_t n_max, int64_t slot) {
  const int n = (int)src_ptrs.size();
  TORCH_CHECK(n >= 1 && n <= 8 && (int)flag_ptrs.size() == n && rank >= 0 && rank < n);
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == torch::kFloat64 && out.numel() >= n_sum + n_max);
  const double* src[8]; uint32_t* flags[8];
  for (int r = 0; r < n; ++r) {
    src[r] = reinterpret_cast<const double*>(src_ptrs[r]);
    flags[r] = reinterpret_cast<uint32_t*>(flag_ptrs[r]);
  }
  zn::launch_metric_reduce(src, n, (int)rank, flags, reinterpret_cast<uint32_t*>(epoch_ptr), out.data_ptr<double>(),
                           (int)n_sum, (int)n_max, (int)slot, cur());
  kcheck();
}
namespace zn {
void launch_split_parts(const float*, long long, int, __nv_bfloat16*, long long, long long, int, int, int,
                        __nv_bfloat16*, long long, long long, int, int, int, cudaStream_t);
void launch_split_conv_wt(const float*, __nv_bfloat16*, int, int, int, int, int, int, int, cudaStream_t);
}
// fp32 [rows][len] -> bf16 hi/lo parts (split.cu). Each destination is described by
// [ld, part_stride, kp, nparts, pattern]; the second one is optional.
void split_parts(Tensor src, int64_t rows, int64_t len, Tensor a, std::vector<int64_t> da,
                 c10::optional<Tensor> b, std::vector<int64_t> db) {
  TORCH_CHECK(src.scalar_type() == torch::kFloat32 && src.is_cuda() && src.is_contiguous());
  TORCH_CHECK(src.numel() >= rows * len && is_bf16(a) && a.is_cuda() && da.size() == 5);
  TORCH_CHECK(da[3] >= 1 && da[3] <= 4 && da[2] >= len);
  TORCH_CHECK(a.numel() >= (da[3] - 1) * da[1] + (rows - 1) * da[0] + da[2], "split_parts: dst a too small");
  __nv_bfloat16* bp = nullptr;
  if (b.has_value() && b->defined()) {
    TORCH_CHECK(is_bf16(*b) && b->is_cuda() && db.size() == 5 && db[3] >= 1 && db[3] <= 4 && db[2] >= len);
    TORCH_CHECK(b->numel() >= (db[3] - 1) * db[1] + (rows - 1) * db[0] + db[2], "split_parts: dst b too small");
    bp = reinterpret_cast<__nv_bfloat16*>(b->data_ptr());
  } else {
    db = {0, 0, 0, 0, 0};
  }
  zn::launch_split_parts(src.data_ptr<float>(), rows, (int)len, reinterpret_cast<__nv_bfloat16*>(a.data_ptr()),
                         da[0], da[1], (int)da[2], (int)da[3], (int)da[4], bp, db[0], db[1], (int)db[2],
                         (int)db[3], (int)db[4], cur());
  kcheck();
}
void split_conv_wt(Tensor w, Tensor dst, int64_t F, int64_t taps, int64_t C, int64_t Fp, int64_t Cp,
                   int64_t nparts, int64_t pattern) {
  TORCH_CHECK(w.scalar_type() == torch::kFloat32 && w.is_cuda() && w.is_contiguous() && is_bf16(dst));
  TORCH_CHECK(w.numel() >= F * taps * C && dst.numel() >= taps * nparts * Fp * Cp && Fp >= F && Cp >= C);
  zn::launch_split_conv_wt(w.data_ptr<float>(), reinterpret_cast<__nv_bfloat16*>(dst.data_ptr()), (int)F,
                           (int)taps, (int)C, (int)Fp, (int)Cp, (int)nparts, (int)pattern, cur());
  kcheck();
}
void som_argmin(Tensor dots, Tensor wnorm, Tensor argmins, c10::optional<Tensor> winners) {
  TORCH_CHECK(dots.scalar_type() == torch::kFloat32 && wnorm.scalar_type() == torch::kFloat32 && dots.dim() == 2);
  int* wp = (winners.has_value() && winners->defined()) ? winners->data_ptr<int>() : nullptr;
  zn::launch_som_argmin(dots.data_ptr<float>(), wnorm.data_ptr<float>(), argmins.data_ptr<int>(), wp,
                        (int)dots.size(0), (int)dots.size(1), cur());
  kcheck();
}
void som_gravity_split(Tensor coords, Tensor argmins, Tensor dst, Tensor rowsum, int64_t batch, int64_t bp,
                       double sigma) {
  TORCH_CHECK(is_bf16(dst) && rowsum.scalar_type() == torch::kFloat32);
  const int neurons = (int)rowsum.numel();
  TORCH_CHECK(dst.numel() >= (int64_t)neurons * 3 * bp);
  zn::launch_som_gravity_split(coords.data_ptr<float>(), argmins.data_ptr<int>(),
                               reinterpret_cast<__nv_bfloat16*>(dst.data_ptr()), rowsum.data_ptr<float>(),
                               neurons, (int)batch, (int)bp, (float)sigma, cur());
  kcheck();
}
void som_apply(Tensor w, Tensor m, Tensor rowsum, double gmult) {
  TORCH_CHECK(w.scalar_type() == torch::kFloat32 && m.scalar_type() == torch::kFloat32 && w.numel() == m.numel());
  const int neurons = (int)rowsum.numel();
  zn::launch_som_apply(w.data_ptr<float>(), m.data_ptr<float>(), rowsum.data_ptr<float>(), neurons,
                       (int)(w.numel() / neurons), (float)gmult, cur());
  kcheck();
}
void som_winners(Tensor x, Tensor w, Tensor argmins, c10::optional<Tensor> winners) {
  TORCH_CHECK(x.scalar_type() == torch::kFloat32 && w.scalar_type() == torch::kFloat32);
  int batch = (int)x.size(0), neurons = (int)w.size(0), len = (int)(w.numel() / w.size(0));
  int* wp = (winners.has_value() && winners->defined()) ? winners->data_ptr<int>() : nullptr;
  zn::launch_som_winners(x.data_ptr<float>(), w.data_ptr<float>(), argmins.data_ptr<int>(), wp, batch,
                         neurons, len, wp ? 1 : 0, cur());
  kcheck();
}
void som_update(Tensor x, Tensor w, Tensor coords, Tensor argmins, double sigma, double gmult) {
  int batch = (int)x.size(0), neurons = (int)w.size(0), len = (int)(w.numel() / w.size(0));
  zn::launch_som_update(x.data_ptr<float>(), w.data_ptr<float>(), coords.data_ptr<float>(),
                        argmins.data_ptr<int>(), batch, neurons, len, (float)sigma, (float)gmult, cur());
  kcheck();
}

// ---------------------------------------------------------------------------- host-side loader
// (host_loader.h) Streaming loaders: the minibatch is assembled straight into the pinned staging
// slot the H2D copy reads - converted to bf16 on the fly when the device-side minibatch is bf16,
// so only half the bytes cross PCIe and no cast kernel runs - synchronously or one step ahead on
// the prefetch pool.
// A uint8 src with a uint8 dst is the raw-bytes mode: rows are copied as they are.
static znhost::GatherJob make_gather_job(const Tensor& src, const Tensor& idx, const Tensor& dst, int64_t n) {
  TORCH_CHECK(!src.is_cuda() && !idx.is_cuda() && !dst.is_cuda(), "host tensors expected");
  TORCH_CHECK(src.is_contiguous() && dst.is_contiguous() && idx.is_contiguous());
  TORCH_CHECK(idx.scalar_type() == torch::kInt32, "idx must be int32");
  const bool raw = src.scalar_type() == torch::kUInt8;
  const bool to_bf16 = dst.scalar_type() == torch::kBFloat16;
  TORCH_CHECK(raw ? dst.scalar_type() == torch::kUInt8
                  : src.scalar_type() == torch::kFloat32 && (to_bf16 || dst.scalar_type() == torch::kFloat32),
              "src must be fp32 (dst fp32 or bf16) or uint8 (dst uint8)");
  TORCH_CHECK(src.dim() >= 1 && dst.dim() >= 1, "src and dst need a row dimension");
  znhost::GatherJob j;
  j.rows = src.size(0); j.row = src.numel() / std::max<int64_t>(j.rows, 1);
  j.cap = dst.size(0); j.n = n;
  TORCH_CHECK(n >= 0 && n <= j.cap && n <= idx.numel() && dst.numel() == j.cap * j.row, "shape mismatch");
  TORCH_CHECK(n == 0 || j.rows > 0, "empty src");
  j.src = src.data_ptr(); j.idx = idx.data_ptr<int>(); j.dst = dst.data_ptr(); j.to_bf16 = to_bf16; j.raw = raw;
  return j;
}
void host_gather_rows(Tensor src, Tensor idx, Tensor dst, int64_t n) {
  znhost::GatherJob j = make_gather_job(src, idx, dst, n);
  znhost::gather_range(j, 0, j.cap);
}
// The caller keeps src / dst alive until host_prefetch_wait(ticket) returned.
int64_t host_prefetch_submit(Tensor src, Tensor idx, Tensor dst, int64_t n) {
  return (int64_t)znhost::HostPrefetcher::get().submit(make_gather_job(src, idx, dst, n));
}
void host_prefetch_wait(int64_t ticket) { znhost::HostPrefetcher::get().wait((uint64_t)ticket); }

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("som_winners", &som_winners); m.def("som_update", &som_update);
  m.doc() = "znicz_b200 sm_90a kernels";
  m.def("act_forward", &act_forward); m.def("act_backward", &act_backward);
  m.def("colsum_slices", &colsum_slices); m.def("err_act_colsum", &err_act_colsum);
  m.def("dropout_forward", &dropout_forward); m.def("binary_op", &binary_op);
  m.def("mul_backward", &mul_backward); m.def("axpby_2d", &axpby_2d); m.def("crop_nhwc", &crop_nhwc);
  m.def("gather_rows", &gather_rows); m.def("gather_labels", &gather_labels);
  m.def("gather_minibatch", &gather_minibatch);
  m.def("augment_minibatch", &augment_minibatch);
  m.def("augment_launches", []() { return (int64_t)zn::augment_launches(); });
  m.def("render_shots", &render_shots);
  m.def("render_shots_launches", []() { return (int64_t)zn::render_shots_launches(); });
  m.def("swap01_2d", &swap01_2d); m.def("device_copy", &device_copy); m.def("metric_reduce", &metric_reduce);
  m.def("space_to_depth", &space_to_depth); m.def("s2d_pack_weights", &s2d_pack_weights); m.def("s2d_unpack_grad", &s2d_unpack_grad);
  m.def("stream_ring_create", &stream_ring_create); m.def("stream_ring_destroy", &stream_ring_destroy);
  m.def("stream_ring_step", &stream_ring_step); m.def("stream_ring_slot_done", &stream_ring_slot_done);
  m.def("stream_ring_slot_sync", &stream_ring_slot_sync);
  m.def("fp8_quant", &fp8_quant); m.def("fp8_gemm", &fp8_gemm);
  m.def("fp8_gemm_launches", []() { return (int64_t)zn::fp8_gemm_launches(); });
  m.def("pull_from_host", &pull_from_host); m.def("push_to_host", &push_to_host);
  m.def("host_gather_rows", &host_gather_rows);
  m.def("host_prefetch_submit", &host_prefetch_submit);
  m.def("host_prefetch_wait", &host_prefetch_wait, py::call_guard<py::gil_scoped_release>());
  m.def("mask_mul", &mask_mul); m.def("pad_channels", &pad_channels); m.def("cast_copy", &cast_copy); m.def("scatter_offsets", &scatter_offsets);
  m.def("pool_forward", &pool_forward); m.def("pool_backward", &pool_backward);
  m.def("lrn_forward", &lrn_forward); m.def("lrn_backward", &lrn_backward);
  m.def("softmax_rows", &softmax_rows); m.def("evaluate_softmax", &evaluate_softmax);
  m.def("evaluate_mse", &evaluate_mse); m.def("mse_find_closest", &mse_find_closest);
  m.def("fused_update", &fused_update);
  m.def("som_split", &som_split); m.def("split_parts", &split_parts); m.def("split_conv_wt", &split_conv_wt); m.def("som_argmin", &som_argmin);
  m.def("som_gravity_split", &som_gravity_split); m.def("som_apply", &som_apply);
  m.def("multi_update_table", &multi_update_table);
  m.def("set_dp_gradient_scale", [](double s) { zn::set_dp_gradient_scale((float)s); });
  m.def("get_dp_gradient_scale", []() { return (double)zn::get_dp_gradient_scale(); });
  m.def("multi_update_max_tensors", []() { return (int64_t)zn::MU_MAX_TENSORS; }); m.def("multi_update", &multi_update);
  m.def("col_sums", &col_sums); m.def("refresh_shadows", &refresh_shadows);
  m.def("rbm_sample", &rbm_sample); m.def("rbm_apply", &rbm_apply);
  m.def("lstm_fwd_persist", &lstm_fwd_persist); m.def("lstm_bwd_persist", &lstm_bwd_persist);
  m.def("lstm_state_floats", &lstm_state_floats); m.def("lstm_part_floats", &lstm_part_floats); m.def("lstm_unpack_state", &lstm_unpack_state);
  m.def("lstm_persist_launches", []() { return (int64_t)zn::lstm_persist_launches(); });
  m.def("lstm_cell_fwd", &lstm_cell_fwd); m.def("lstm_cell_bwd", &lstm_cell_bwd);
  m.def("fc_small_max_out", &fc_small_max_out); m.def("fc_small_forward", &fc_small_forward);
  m.def("fc_small_backward", &fc_small_backward);
  m.def("fc_wgrad_pair", &fc_wgrad_pair);
  m.def("conv_pair_launches", []() { return (int64_t)zn::conv_pair_launches(); });
  m.def("im2col_tma_launches", []() { return (int64_t)zn::im2col_tma_launches(); });
  m.def("conv_halo_launches", []() { return (int64_t)zn::conv_halo_launches(); });
  m.def("gemm", &gemm); m.def("pick_splits", &pick_splits); m.def("gemm_pair", &gemm_pair);
  m.def("conv_fprop", &conv_fprop); m.def("conv_dgrad", &conv_dgrad); m.def("conv_wgrad", &conv_wgrad);
}
