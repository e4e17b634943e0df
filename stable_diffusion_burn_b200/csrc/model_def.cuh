// model_def.cuh — weight tree of the hot path. Tensor names are the reference's dump-dir paths
// (src/model/unet/load.rs:213-306, src/model/autoencoder/load.rs:16-198).
#pragma once
#include <map>
#include <memory>

#include "runtime.cuh"

namespace sdb {

struct ConvW {
  int cin = 0, cout = 0, k = 0;
  int wi = -1, bi = -1;     // registry indices (weight, bias)
  WeightOp packed;          // [cout][k*k*cin] fp16 hi/lo (or 4 folded-upsample phases)
  float* bias = nullptr;    // device pointer into the master arena
  float* w_small = nullptr; // fp32 [cout][9][cin] for Cout <= 4
  int passes = 1;
};
struct LinW {
  int in = 0, out = 0;
  int wi = -1, bi = -1;
  WeightOp packed;  // [out][in]
  float* bias = nullptr;
  int passes = 1;
};
struct NormW {
  int c = 0;
  int gi = -1, bi = -1;
  float* gamma = nullptr;
  float* beta = nullptr;
  float eps = 1e-5f;  // a dump-dir's eps.npy overrides it (load_group_norm / load_layer_norm)
};
struct ResBlockW {
  int cin = 0, cout = 0;
  NormW norm_in, norm_out;
  ConvW conv_in, conv_out, skip;
  LinW lin_embed;
  bool has_skip = false;
  float* bias_merged = nullptr;  // conv_out.bias + skip_connection.bias (skip conv folded into conv_out's K loop)
  int emb_off = 0;  // offset of this block's row in the fused time-embedding GEMV output
  int passes = 1;
};
struct AttnW {
  LinW query, key, value, out;
};
struct SpatialTransformerW {
  int c = 0, heads = 8, d = 0, dpad = 0;
  NormW norm, ln1, ln2, ln3;
  ConvW proj_in, proj_out;
  AttnW attn1, attn2;
  LinW geglu, ff;
  // fused / re-laid-out projections
  WeightOp w_qkv1;     // [3*heads*dpad][c]   self-attention q|k|v, head-padded (V is consumed MN-major by the attention kernel)
  WeightOp w_q2;       // [heads*dpad][c]     cross-attention q
  WeightOp w_kv2;      // [2*heads*dpad][768] cross-attention k|v (context), head-padded
  WeightOp w_o1, w_o2; // [c][heads*d] out projections (un-padded input)
  WeightOp w_geglu;    // [8c][c] tile-interleaved x|gate
  float* geglu_bias = nullptr;  // packed order
  // LayerNorm folded into the consuming GEMMs (w_qkv1 <- ln1, w_q2 <- ln2, w_geglu <- ln3: gamma is inside the packed weights):
  // u = column sums of the packed fp16 weights (hi / hi + lo), v = beta^T W (+ bias)
  float *u_qkv_hi = nullptr, *u_qkv_full = nullptr, *v_qkv = nullptr;
  float *u_q2_hi = nullptr, *u_q2_full = nullptr, *v_q2 = nullptr;
  float *u_geglu_hi = nullptr, *u_geglu_full = nullptr, *v_geglu = nullptr;
  int passes = 1;
};
enum BlockKind : int { BK_CONV = 0, BK_DOWN, BK_R, BK_RT, BK_RU, BK_RTU };
struct UNetBlockW {
  int kind = BK_R, cin = 0, cout = 0;
  ConvW conv;  // BK_CONV / BK_DOWN / upsample conv
  ResBlockW res;
  SpatialTransformerW st;
  int level = 0;  // 0: H, 1: H/2, 2: H/4, 3: H/8 (resolution at which the block's ResBlock runs)
};
struct ResnetW {
  int cin = 0, cout = 0;
  NormW norm1, norm2;
  ConvW conv1, conv2, nin;
  bool has_nin = false;
  float* bias_merged = nullptr;  // conv2.bias + nin_shortcut.bias
  int passes = 1;
};
struct VaeAttnW {
  NormW norm;
  ConvW q, k, v, proj_out;
  int passes = 1;
};
struct DecoderBlockW {
  ResnetW res[3];
  bool has_up = false;
  ConvW up;
};

struct EncoderBlockW {  // autoencoder/mod.rs:249-266
  ResnetW res[2];
  bool has_down = false;
  ConvW down;  // PaddedConv2d(0,1,0,1) stride 2
};
struct EncoderW {       // autoencoder/mod.rs:122-145 + quant_conv (:60-66)
  ConvW conv_in, conv_out, quant;
  float* conv_in_w4 = nullptr;  // conv_in weights padded to 4 input channels (the Cin = 4 CUDA-core conv kernel)
  EncoderBlockW blocks[4];
  ResnetW mid_block1, mid_block2;
  VaeAttnW mid_attn;
  NormW norm_out;
};

struct ClipBlockW {  // src/model/clip/mod.rs:77-115
  NormW attn_ln, mlp_ln;
  LinW query, key, value, out, fc1, fc2;
  WeightOp w_qk;             // [2*768][768] fused q|k
  float* bias_qk = nullptr;  // [1536]
  float* bias_out = nullptr; // out.bias + value.bias @ W_out  (the v bias commutes with the softmax average)
};
struct ClipW {
  int tok_i = -1, pos_i = -1;
  std::vector<ClipBlockW> blocks;
  NormW ln_final;
};

// One packing unit of model_finalize: what sdb_lora_apply re-packs, in place, when one of its weights changes (DESIGN §7 f8).
// off0 / off1: the packed arena offsets at the unit's start and end, recorded by the last finalize.
enum PackUnitKind : int { U_RES = 0, U_ST, U_CONV, U_UP, U_EMB, U_CLIP };
struct PackUnit {
  int kind = U_RES;
  ResBlockW* res = nullptr;
  SpatialTransformerW* st = nullptr;
  ConvW* conv = nullptr;
  ClipBlockW* clip = nullptr;
  int passes = 0;  // U_CONV / U_UP: the conv's pass count (0 = left as it is)
  size_t off0 = 0, off1 = 0;
};

// LoRA adapters of a context (DESIGN §7 f8). Factors and effective weights live in their own device allocations, outside the
// master, packed and work arenas.
struct LoraTerm {
  int tensor = -1, rank = 0;
  float* down = nullptr;  // device [rank][fan-in]
  float* up = nullptr;    // device [out][rank]
  double alpha = 0.0;
  uint64_t serial = 0;    // unique per added term: a removed and re-added term counts as a change
};
struct LoraAdapter {
  double multiplier = 1.0;
  std::vector<LoraTerm> terms;  // in the order they were added
};
struct LoraState {
  std::map<int, LoraAdapter> adapters;               // ascending id = accumulation order
  std::unordered_map<int, float*> buf;               // tensor -> W_eff buffer (device), while any term targets the tensor
  std::unordered_map<int, float*> eff;               // tensor -> its buf, for tensors with an active term as of the last merge
  std::unordered_map<int, std::vector<std::pair<uint64_t, float>>> applied;  // tensor -> (term serial, scale) merged into eff
  uint64_t next_serial = 1;
  bool pending = false;  // an add / scale / remove since the last apply or finalize (model_lora_pending settles it)
  ~LoraState() {
    for (auto& a : adapters)
      for (LoraTerm& t : a.second.terms) cudaFree(t.down), cudaFree(t.up);
    for (auto& e : buf) cudaFree(e.second);
  }
};

struct Model {
  ClipW clip;
  EncoderW enc;
  // UNet
  LinW lin1_time, lin2_time;
  std::vector<UNetBlockW> in_blocks, out_blocks;
  ResBlockW mid_res1, mid_res2;
  SpatialTransformerW mid_st;
  NormW norm_out;
  ConvW conv_out;
  std::vector<ResBlockW*> resblocks;     // all 22, in execution order
  std::vector<SpatialTransformerW*> sts; // all 16, in execution order
  float* emb_w_all = nullptr;            // fp32 [1280][emb_total]: every lin_embed side by side
  float* emb_b_all = nullptr;            // fp32 [emb_total]: lin_embed bias + conv_in bias
  int emb_total = 0;
  // VAE decoder
  ConvW post_quant, vae_conv_in, vae_conv_out;
  ResnetW mid_block1, mid_block2;
  VaeAttnW mid_attn;
  DecoderBlockW dec[4];
  NormW vae_norm_out;
  // sampler
  int alphas_i = -1;
  std::vector<float> alphas_host;
  // captured UNet step passes of the sampler loop (model.cu: step_graph), keyed by shape and matched on the addresses they bake in
  struct GraphEntry {
    long long key = 0;
    cudaGraphExec_t exec = nullptr;
    int64_t launches = 0;         // kernel launches one replay stands for
    const float* xb = nullptr;    // the step's UNet input and output
    const float* eps = nullptr;
    const void* kv = nullptr;     // the context K/V of the first transformer
    size_t work_mark = 0;         // the step's own temporaries start here in the work arena
    const float* cond = nullptr;  // the UNet's extra input channels (io slot kIoUNetCond) or null
  };
  std::vector<GraphEntry> graphs;
  // packing units in finalize order: the UNet blocks, then the time-embedding table (unit_emb), then the CLIP blocks
  std::vector<PackUnit> units;
  int unit_emb = -1;
  std::unordered_map<int, int> lora_target;  // LoRA target tensor -> index of the unit that packs it
  LoraState lora;
};

}  // namespace sdb
