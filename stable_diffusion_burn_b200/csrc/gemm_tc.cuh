// gemm_tc.cuh — descriptor of one wgmma implicit-GEMM launch (conv3x3 / conv1x1 / Linear).
#pragma once
#include "common.cuh"

namespace sdb {

// A operand = fp16 activation tensor viewed as 5-D [n][phase][h][w][c] (c innermost), loaded by TMA
// boxes {64 c, TW, TH, 1, TN} at tap-shifted coordinates (zero fill outside = conv padding).
// B operand = packed fp16 weights [N][K] (K-major), K index = tap * Cin_total + c.
// D (fp32, registers of two consumer warpgroups) [128 rows = TN*TH*TW output pixels][BN output channels].
struct GemmMaps {
  CUtensorMap a[4][2];  // [source][hi/lo]: 0/1 = channel-concatenated operands of every tap; 2/3 = "extra K" operands read at
                        // the centre tap only, appended after the taps (the ResBlock's 1x1 skip conv folded into conv_out)
  CUtensorMap bx[2];    // weights of the extra-K segment [N][xK]
  CUtensorMap b[2];     // [hi/lo]  box {64, BN}
};

struct GemmParams {
  int nimg, H, W;  // output pixel grid (per phase plane for stride-2 inputs)
  int TN, TH, TW;
  int tiles_n, tiles_h, tiles_w;
  int N;               // GEMM N (packed weight rows)
  int kc;              // 64-wide channel chunks per tap (both sources)
  int kc0;             // chunks taken from source 0
  int num_taps;
  int xkc, xkc0;       // extra-K chunks appended after the taps (total, and those from source 2)
  int8_t tap_dh[9], tap_dw[9], tap_ph[9];
  int split_k;
  int up2, gn_phase_slots; // up2 = 1: folded nearest-2x upsample conv, grid.z = the 4 output phases (weights packed [4][N][K], taps
                           // / output pixel shifted by the phase); gn_phase_slots = GroupNorm partial slots one phase writes
  // epilogue
  float* out_f32;          // [M][ldc] or null
  __half* out_f16;         // [M][ldc16] or null (hi part)
  __half* out_f16_lo;      // residual part for multi-pass consumers, or null
  const float* bias;       // [N] or null
  const float* residual;   // [M][ldc] or null
  int ldc;                 // row stride of out_f32 / residual (elements)
  int ldc16;               // row stride of out_f16
  int geglu;               // 1: columns are (x|gate) interleaved per tile, output width N/2
  long long* dbg;          // SDB_GEMM_DBG: 8 clock64 stamps of CTA (0,0,0) (entry, prologue done, first TMA issued, first
                           // operands landed, last MMA issued, accumulator ready, epilogue stores done, exit)
  int act;                 // 1: QuickGELU x*sigmoid(1.702x) on the result (CLIP MLP, clip/mod.rs:224-226)
  // GroupNorm statistics of the OUTPUT tensor, produced here so that the consuming GroupNorm needs neither a statistics pass over
  // the tensor nor a grid rendezvous: per (image, slot, channel bucket) partial (sum, sum of squares) of the final fp32 values,
  // slot = gn_slot0 + (tile_in_image * split_k + z). Layout [nimg][gn_cap][N / gn_bucket][2] floats. Null = not requested.
  float* gn_part;
  int gn_cap, gn_bucket, gn_slot0;
  int gn_rpi, gn_nimg;     // flattened [rows][C] outputs (1x1 conv / Linear over tokens): rows per image (a multiple or a divisor
                           // of 128) and the image count; gn_rpi = 0: images follow the tile geometry (nimg, TN)
  // LayerNorm folded into the GEMMs around it (no LayerNorm launch): the producer of the normalised tensor leaves per-row partial
  // (sum, sum of squares) — ln_out [rows][ln_slots][2], slot = N tile * 2 + chunk share — and the consumer, whose weights carry
  // gamma, applies out = rstd * (acc - mean * ln_u[c]) + bias[c] from ln_in [rows][ln_in_slots][2]
  float* ln_out;
  int ln_slots;
  const float* ln_in;
  int ln_in_slots, ln_C;
  float ln_eps;
  const float* ln_u;       // [N] column sums of the folded fp16 weights that this launch multiplies (hi, or hi + lo)
  // residual kept as an fp16 hi + lo pair (row stride ldc16) instead of fp32: the transformer's residual stream
  const __half* res_hi;
  const __half* res_lo;
  float* ws;               // split-K workspace [split][M][N]
  unsigned int* tickets;   // split-K: one counter per output tile, all zero between launches (self-cleaning)
  // output pixel mapping: out row = ((n*OH + h*os + oa)*OW + w*os + ob)
  int OH, OW, os, oa, ob;
};

void gemm_tc_launch(const GemmMaps& maps, const GemmParams& p, int BN, int passes, cudaStream_t stream);
// pipeline stages of the (BN, passes) kernel instance: the depth of its shared-memory operand ring
int gemm_tc_stages(int BN, int passes);

}  // namespace sdb
