// The parameter-update descriptor shared by update.cu (both update kernels) and ext.cpp (which
// fills it from kernels/api.py::UpdateDesc). Plain data: compiled by nvcc and the host compiler.
#pragma once
#include <cuda_bf16.h>

namespace zn {

struct ShadowSpec {
  __nv_bfloat16* lp;       // [rows][ld] bf16 copy of w (row-major as w), may be null
  int ld;
  int lp_cpad;             // > 0: lp rows are [tap][lp_cpad] channel-padded
  __nv_bfloat16* lp_conv;  // conv dgrad operand [tap][f_pad = roundup(rows, 8)][c_pad], may be null
  int taps, C, c_pad;
};

struct TensorDesc {
  float* w; float* grad_out; float* acc; float* vel;
  const float* hyper; float* col_sums;
  const float* grad;          // this rank's split-K partials, part_stride elements apart
  long long part_stride, size;
  int nparts, g_cpad, flags, is_bias, rows, cols, lanes, enabled;
  ShadowSpec sh;
  // set by multi_update_pack (whole-network kernel only)
  int tile_begin, n_tiles;
  int ept;                    // elements per thread (lanes == 1 only): 4 for large tensors
  int vec4;                   // ept == 4 and every array / stride is 16-byte aligned: float4 path
  long long red_off;          // offset of this tensor in the cross-GPU reduction buffer
  float* s0; float* s1; float* s2;   // solver state (step_elem), null when unused
};

constexpr int MU_MAX_TENSORS = 48;          // descriptors per multi_update_k launch (shared memory)

}  // namespace zn
