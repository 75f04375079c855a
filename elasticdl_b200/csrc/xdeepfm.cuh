// What the xDeepFM tower's two files share (include/b200_deepfm.h: b200_deepfm_xdeepfm_*): the flat parameter
// layout of its CIN, the scratch buffer's layout, and the Wide & Deep tile kernel's xDeepFM instance, which
// deepfm_tower2.cu launches for xdeepfm_cin.cu.
#pragma once
#include "tile_tower.cuh"

namespace deepfm {

constexpr int CIN_H = 128;            // channels of each CIN layer (layer_size = (128, 128))
constexpr int CIN_HALF = CIN_H / 2;   // split_half: layer 0's next hidden state, H_1 = 64
constexpr int CIN_P = CIN_HALF + CIN_H;  // p = [direct_0 64 | direct_1 128]
constexpr float CIN_L2 = 1e-5f;       // the CIN filters' l2_reg

// The flat layout: Wide & Deep's (deepfm_common.cuh Layout, DeepFM's), then
//   [ W_0 128 x G^2 | b_0 128 | W_1 128 x 64G | b_1 128 | w_ex 192 | b_ex 1 ]
// filter row h contiguous over K = i H_k + j.
struct CinLayout {
  Layout l;  // l.total = the whole buffer
  int o_w0, o_b0, o_w1, o_b1, o_wex, o_bex;
};
__host__ __device__ inline CinLayout cin_layout(int G) {
  CinLayout c;
  c.l = layout(G);
  c.o_w0 = c.l.total;
  c.o_b0 = c.o_w0 + CIN_H * G * G;
  c.o_w1 = c.o_b0 + CIN_H;
  c.o_b1 = c.o_w1 + CIN_H * CIN_HALF * G;
  c.o_wex = c.o_b1 + CIN_H;
  c.o_bex = c.o_wex + CIN_P;
  c.l.total = c.o_bex + 1;
  return c;
}

// The kernels' K: layer 0 runs K = i Hp0 + j with j padded to Hp0 = G rounded up to the mma step (8), so that a
// k-step never straddles two i; layer 1 needs no padding (H_1 = 64).  The data pass's A operand (W^T) is padded
// to whole m16 tiles.
struct CinShape {
  int hp0, k0, k1, k0b;  // Hp0, padded K of layer 0, K of layer 1, k0 rounded up to 16
};
__host__ __device__ inline CinShape cin_shape(int G) {
  CinShape s;
  s.hp0 = (G + 7) / 8 * 8;
  s.k0 = G * s.hp0;
  s.k1 = CIN_HALF * G;
  s.k0b = (s.k0 + 15) / 16 * 16;
  return s;
}

// The scratch buffer (floats; B-dependent):
//   W1x [NCOL][16] | tile counter (16)     the Wide & Deep tile kernel's (deepfm_tower2.cu), first
//   cin_logit [Bp] | dz [Bp]               written by the CIN forward / the tile kernel, Bp = B rounded up to 4
//   counters (16)                          the CIN forward's and data pass's dynamic tile counters
//   Wf0 [128 k0] | Wf1 [128 k1]            W_k as the forward's A operand, in fragment order
//   Wb0 [128 k0b] | Wb1 [128 k1]           W_k^T as the data pass's A operand, direct channels scaled by w_ex
//   p [B][192] | masks [B][64] | X_1 [B][64][8] | dC_0 first half [B][64][8]
struct CinScratch {
  long long o_logit, o_dz, o_cnt, o_wf0, o_wf1, o_wb0, o_wb1, o_p, o_mask, o_x1, o_dc0, total;
};
__host__ __device__ inline CinScratch cin_scratch(int G, long long B) {
  const CinShape s = cin_shape(G);
  const long long bp = (B + 3) / 4 * 4;
  CinScratch c;
  c.o_logit = (long long)NCOL * H1 + 16;
  c.o_dz = c.o_logit + bp;
  c.o_cnt = c.o_dz + bp;
  c.o_wf0 = c.o_cnt + 16;
  c.o_wf1 = c.o_wf0 + (long long)CIN_H * s.k0;
  c.o_wb0 = c.o_wf1 + (long long)CIN_H * s.k1;
  c.o_wb1 = c.o_wb0 + (long long)CIN_H * s.k0b;
  c.o_p = c.o_wb1 + (long long)CIN_H * s.k1;
  c.o_mask = c.o_p + CIN_P * B;
  c.o_x1 = c.o_mask + 64 * B;
  c.o_dc0 = c.o_x1 + (long long)CIN_HALF * D * B;
  c.total = c.o_dc0 + (long long)CIN_HALF * D * B;
  return c;
}

// The Wide & Deep prep and tile kernel with the CIN logit added to z and dz stored (deepfm_tower2.cu), as
// launch_tile_tower runs them (what: 1 prep, 2 tile kernel, 3 both), counted on `launches`.
template <bool BACKWARD>
int launch_xdeepfm_tile(const b200_deepfm_args_t* args, void* stream, int what, entry::LaunchCount& launches);

}  // namespace deepfm
