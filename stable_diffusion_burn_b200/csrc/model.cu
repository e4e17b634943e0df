// model.cu — the sampling graph: weight packing, UNet::forward, Autoencoder::decode_latent, DDIM sampler.
//
// Reference call stacks reproduced here (SURVEY §3):
//   StableDiffusion::sample_image / sample_latent / forward_diffuser  src/model/stablediffusion/mod.rs:51-192
//   UNet::forward                                                     src/model/unet/mod.rs:109-142
//   ResBlock / SpatialTransformer / TransformerBlock / MLP / MHA      src/model/unet/mod.rs:461-481,521-527,551-592,641-653,712-734
//   Autoencoder::decode_latent / Decoder / ResnetBlock / attention    src/model/autoencoder/mod.rs:68-71,204-217,307-324,513-528,562-608
// Activations are NHWC fp32 (residual stream); GEMM operands are staged as fp16 hi(/lo) tensors.
#include "model.cuh"

#include "../../include/sdb200.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>

#include "model_def.cuh"

namespace sdb {

static Model& M(Ctx& c) { return *reinterpret_cast<Model*>(c.model); }
static const Model& M(const Ctx& c) { return *reinterpret_cast<const Model*>(c.model); }
static int round_up(int x, int m) { return (x + m - 1) / m * m; }

// tensor-core passes per product as a function of the UNet resolution level (0 = full latent resolution).
// Budgeted with the oracle's operand-rounding emulation (DESIGN.md "precision"): the two highest-resolution
// levels carry ~85 % of the fp16 rounding error of a UNet step, so they run the 3-term split product.
static int g_level_passes[4] = {3, 3, 1, 1};
// VAE decoder (same emulation study, per block): the latent-resolution stage (mid blocks, attention, first
// DecoderBlock) and the three upsample convs inject ~63 % of the fp16 rounding error for ~20 % of the FLOPs
// -> split product there, single pass on the 128^2..512^2 ResnetBlocks.
static int g_vae_passes_lowres = 3, g_vae_passes_up = 3, g_vae_passes_highres = 1;

// ================================================================================ packing
static Half2Ptr alloc_half2(Arena& a, size_t count) {
  Half2Ptr p;
  p.hi = a.get<__half>(count);
  p.lo = a.get<__half>(count);
  return p;
}
static float* mptr(Ctx& c, int idx) {
  return idx < 0 ? nullptr : reinterpret_cast<float*>(c.master.base) + c.tensors[idx].offset;
}
// the weight a packer reads: the LoRA-merged W_eff of a tensor with an active adapter term, else the master copy. Packing only:
// every run-time read goes through mptr and sees the base weights.
static float* wsrc(Ctx& c, int idx) {
  if (idx >= 0) {
    const auto& eff = M(c).lora.eff;
    auto it = eff.find(idx);
    if (it != eff.end()) return it->second;
  }
  return mptr(c, idx);
}

// An OIHW conv weight `src` packed into `a` for the kernel that runs the conv: the implicit GEMM ([Cout][k*k*Cin], or with up2 the
// nearest-2x upsample folded in, [4][Cout][4*Cin]) when Cin is a multiple of 64 and Cout of 32; otherwise a CUDA-core conv, which
// reads fp32 [Cout][9][Cin] for a 3x3 conv with Cout <= 8 and the master weights for the rest
static void pack_conv_weight(Ctx& c, ConvW& w, const float* src, Arena& a, bool up2) {
  if (w.cin % 64 != 0 || w.cout % 32 != 0) {
    if (w.cout <= 8 && w.k == 3 && w.cin % 4 == 0) {
      w.w_small = a.get<float>((size_t)w.cout * 9 * w.cin);
      pack_small_cout_launch(src, w.cout, w.cin, w.w_small, c.stream);
    }
    return;
  }
  if (up2) {
    w.packed.p = alloc_half2(a, (size_t)16 * w.cout * w.cin);
    w.packed.N = w.cout, w.packed.K = 4 * w.cin;
    pack_conv_up2_launch(src, w.cout, w.cin, w.packed.p, c.stream);
  } else {
    w.packed.p = alloc_half2(a, (size_t)w.cout * w.k * w.k * w.cin);
    w.packed.N = w.cout, w.packed.K = w.k * w.k * w.cin;
    pack_conv_launch(src, w.cout, w.cin, w.k, w.packed.p, c.stream);
  }
}
static void pack_conv(Ctx& c, ConvW& w, bool up2 = false) {
  w.bias = mptr(c, w.bi);
  pack_conv_weight(c, w, wsrc(c, w.wi), c.packed, up2);
}
static void pack_lin(Ctx& c, LinW& w) {
  w.bias = mptr(c, w.bi);
  w.packed.p = alloc_half2(c.packed, (size_t)w.out * w.in);
  w.packed.N = w.out, w.packed.K = w.in;
  pack_linear_launch(wsrc(c, w.wi), w.in, w.out, w.packed.p, 0, c.stream);
}
static void pack_norm(Ctx& c, NormW& n) {
  n.gamma = mptr(c, n.gi), n.beta = mptr(c, n.bi);
  const std::string& g = c.tensors[n.gi].name;
  auto it = c.norm_eps.find(g.substr(0, g.rfind('/')));
  n.eps = it == c.norm_eps.end() ? 1e-5f : it->second;
}

// [rows = heads*dpad][in]: head h occupies rows h*dpad .. h*dpad+d (pad rows stay zero)
static void pack_heads(Ctx& c, const LinW& src, int heads, int d, int dpad, Half2Ptr dst, int row_offset,
                       const float* in_scale = nullptr) {
  for (int h = 0; h < heads; ++h)
    pack_linear_launch(wsrc(c, src.wi), src.in, d, dst, row_offset + h * dpad, c.stream, src.out, h * d, in_scale);
}

static void pack_resblock(Ctx& c, ResBlockW& r, int passes) {
  r.passes = passes;
  pack_norm(c, r.norm_in), pack_norm(c, r.norm_out);
  pack_conv(c, r.conv_in), pack_conv(c, r.conv_out);
  if (r.has_skip) {
    pack_conv(c, r.skip);
    r.bias_merged = c.packed.get<float>(r.cout);
    add_vec_launch(r.conv_out.bias, r.skip.bias, r.cout, r.bias_merged, c.stream);
  }
  r.lin_embed.bias = mptr(c, r.lin_embed.bi);
}
// The LayerNorms of the TransformerBlock (unet/mod.rs:523-525) have no launch: gamma is folded into the weights of the GEMM that
// consumes the normalised tensor (W' = diag(gamma) W), u = row sums of the packed W' (the exact fp16 values the tensor cores
// multiply), v = beta^T W; the GEMM reads the raw tensor and applies rstd * (acc - mean * u) + v + bias. pack(dst, scale) packs the
// consumer's [N][K] weights with input feature i multiplied by scale[i]: w.p with gamma, then `scratch` (N * K pairs at least) with
// beta, whose hi + lo hold 22 bits of beta * W. u_hi, u_full and v ([N] each) come from arena `a`; the caller adds its bias to v.
static void ln_fold(Ctx& c, Arena& a, Half2Ptr scratch, WeightOp& w, float*& u_hi, float*& u_full, float*& v,
                    const std::function<void(Half2Ptr, const float*)>& pack, const NormW& ln) {
  pack(w.p, ln.gamma);
  u_hi = a.get<float>(w.N), u_full = a.get<float>(w.N), v = a.get<float>(w.N);
  rowsum_f16_launch(w.p, w.N, w.K, u_hi, u_full, c.stream);
  SDB_CUDA(cudaMemsetAsync(scratch.hi, 0, (size_t)w.N * w.K * 2, c.stream));  // head-pad rows stay zero
  SDB_CUDA(cudaMemsetAsync(scratch.lo, 0, (size_t)w.N * w.K * 2, c.stream));
  pack(scratch, ln.beta);
  rowsum_f16_launch(scratch, w.N, w.K, nullptr, v, c.stream);
}
static void pack_st(Ctx& c, SpatialTransformerW& s, int passes) {
  s.passes = passes;
  pack_norm(c, s.norm), pack_norm(c, s.ln1), pack_norm(c, s.ln2), pack_norm(c, s.ln3);
  pack_conv(c, s.proj_in), pack_conv(c, s.proj_out);
  const int hd = s.heads * s.dpad;
  Half2Ptr scratch = alloc_half2(c.work, (size_t)8 * s.c * s.c);
  s.w_qkv1.p = alloc_half2(c.packed, (size_t)3 * hd * s.c), s.w_qkv1.N = 3 * hd, s.w_qkv1.K = s.c;
  ln_fold(c, c.packed, scratch, s.w_qkv1, s.u_qkv_hi, s.u_qkv_full, s.v_qkv, [&](Half2Ptr dst, const float* sc) {
    pack_heads(c, s.attn1.query, s.heads, s.d, s.dpad, dst, 0, sc);
    pack_heads(c, s.attn1.key, s.heads, s.d, s.dpad, dst, hd, sc);
    pack_heads(c, s.attn1.value, s.heads, s.d, s.dpad, dst, 2 * hd, sc);
  }, s.ln1);
  pack_lin(c, s.attn1.out), s.w_o1 = s.attn1.out.packed;
  s.w_q2.p = alloc_half2(c.packed, (size_t)hd * s.c), s.w_q2.N = hd, s.w_q2.K = s.c;
  ln_fold(c, c.packed, scratch, s.w_q2, s.u_q2_hi, s.u_q2_full, s.v_q2,
          [&](Half2Ptr dst, const float* sc) { pack_heads(c, s.attn2.query, s.heads, s.d, s.dpad, dst, 0, sc); }, s.ln2);
  s.w_kv2.p = alloc_half2(c.packed, (size_t)2 * hd * 768), s.w_kv2.N = 2 * hd, s.w_kv2.K = 768;
  pack_heads(c, s.attn2.key, s.heads, s.d, s.dpad, s.w_kv2.p, 0);
  pack_heads(c, s.attn2.value, s.heads, s.d, s.dpad, s.w_kv2.p, hd);
  pack_lin(c, s.attn2.out), s.w_o2 = s.attn2.out.packed;
  s.w_geglu.p = alloc_half2(c.packed, (size_t)8 * s.c * s.c), s.w_geglu.N = 8 * s.c, s.w_geglu.K = s.c;
  s.geglu_bias = c.packed.get<float>((size_t)8 * s.c);
  ln_fold(c, c.packed, scratch, s.w_geglu, s.u_geglu_hi, s.u_geglu_full, s.v_geglu, [&](Half2Ptr dst, const float* sc) {
    pack_geglu_launch(wsrc(c, s.geglu.wi), mptr(c, s.geglu.bi), s.c, 4 * s.c, 64, dst, dst.hi == s.w_geglu.p.hi ? s.geglu_bias : nullptr,
                      c.stream, sc);
  }, s.ln3);
  add_vec_launch(s.v_geglu, s.geglu_bias, 8 * s.c, s.v_geglu, c.stream);  // v = beta^T W + b (packed order)
  pack_lin(c, s.ff);
  SDB_CUDA(cudaStreamSynchronize(c.stream));  // the scratch packing lives in the work arena
  c.work.reset();
}
static void pack_resnet(Ctx& c, ResnetW& r, int passes) {
  r.passes = passes;
  pack_norm(c, r.norm1), pack_norm(c, r.norm2);
  pack_conv(c, r.conv1), pack_conv(c, r.conv2);
  if (r.has_nin) {
    pack_conv(c, r.nin);
    r.bias_merged = c.packed.get<float>(r.cout);
    add_vec_launch(r.conv2.bias, r.nin.bias, r.cout, r.bias_merged, c.stream);
  }
}

// fused time-embedding projection: every lin_embed side by side, bias = lin bias + conv_in bias
static void pack_emb(Ctx& c) {
  Model& m = M(c);
  m.emb_total = 0;
  for (ResBlockW* r : m.resblocks) r->emb_off = m.emb_total, m.emb_total += r->cout;
  m.emb_w_all = c.packed.get<float>((size_t)1280 * m.emb_total);
  m.emb_b_all = c.packed.get<float>(m.emb_total);
  std::vector<float> hb(m.emb_total), t1, t2;
  for (ResBlockW* r : m.resblocks) {
    SDB_CUDA(cudaMemcpy2DAsync(m.emb_w_all + r->emb_off, (size_t)m.emb_total * 4, wsrc(c, r->lin_embed.wi),
                               (size_t)r->cout * 4, (size_t)r->cout * 4, 1280, cudaMemcpyDeviceToDevice, c.stream));
    t1.resize(r->cout), t2.resize(r->cout);
    SDB_CUDA(cudaMemcpyAsync(t1.data(), mptr(c, r->lin_embed.bi), r->cout * 4, cudaMemcpyDeviceToHost, c.stream));
    SDB_CUDA(cudaMemcpyAsync(t2.data(), mptr(c, r->conv_in.bi), r->cout * 4, cudaMemcpyDeviceToHost, c.stream));
    SDB_CUDA(cudaStreamSynchronize(c.stream));
    for (int i = 0; i < r->cout; ++i) hb[r->emb_off + i] = t1[i] + t2[i];
  }
  SDB_CUDA(cudaMemcpyAsync(m.emb_b_all, hb.data(), hb.size() * 4, cudaMemcpyHostToDevice, c.stream));
}
static void pack_clip_block(Ctx& c, ClipBlockW& cb) {
  pack_norm(c, cb.attn_ln), pack_norm(c, cb.mlp_ln);
  cb.w_qk.p = alloc_half2(c.packed, (size_t)2 * 768 * 768), cb.w_qk.N = 1536, cb.w_qk.K = 768;
  pack_linear_launch(wsrc(c, cb.query.wi), 768, 768, cb.w_qk.p, 0, c.stream);
  pack_linear_launch(wsrc(c, cb.key.wi), 768, 768, cb.w_qk.p, 768, c.stream);
  cb.bias_qk = c.packed.get<float>(1536);
  SDB_CUDA(cudaMemcpyAsync(cb.bias_qk, mptr(c, cb.query.bi), 768 * 4, cudaMemcpyDeviceToDevice, c.stream));
  SDB_CUDA(cudaMemcpyAsync(cb.bias_qk + 768, mptr(c, cb.key.bi), 768 * 4, cudaMemcpyDeviceToDevice, c.stream));
  pack_lin(c, cb.value), pack_lin(c, cb.out), pack_lin(c, cb.fc1), pack_lin(c, cb.fc2);
  // softmax rows sum to one, so P.(V + 1 b_v^T) = P.V + b_v^T: fold the value bias into the out-projection bias
  cb.bias_out = c.packed.get<float>(768);
  gemv_launch(mptr(c, cb.value.bi), wsrc(c, cb.out.wi), mptr(c, cb.out.bi), 768, 768, cb.bias_out, c.stream);
}

static void pack_unit(Ctx& c, PackUnit& u) {
  switch (u.kind) {
    case U_RES:
      pack_resblock(c, *u.res, u.passes);
      break;
    case U_ST:
      pack_st(c, *u.st, u.passes);
      break;
    case U_CONV:
    case U_UP:
      pack_conv(c, *u.conv, /*up2=*/u.kind == U_UP);
      if (u.passes) u.conv->passes = u.passes;
      break;
    case U_EMB:
      pack_emb(c);
      break;
    case U_CLIP:
      pack_clip_block(c, *u.clip);
      break;
  }
}

// The packing units in finalize order and the LoRA target -> unit map (DESIGN §7 f8), built once from the weight tree.
static void build_units(Model& m) {
  if (!m.units.empty()) return;
  auto add = [&](PackUnit u, std::initializer_list<int> targets) {
    for (int t : targets)
      if (t >= 0) m.lora_target[t] = (int)m.units.size();
    m.units.push_back(u);
  };
  auto res = [&](ResBlockW& r, int p) {
    PackUnit u;
    u.kind = U_RES, u.res = &r, u.passes = p;
    add(u, {r.conv_in.wi, r.conv_out.wi, r.has_skip ? r.skip.wi : -1});
  };
  auto st = [&](SpatialTransformerW& s, int p) {
    PackUnit u;
    u.kind = U_ST, u.st = &s, u.passes = p;
    add(u, {s.proj_in.wi, s.proj_out.wi, s.attn1.query.wi, s.attn1.key.wi, s.attn1.value.wi, s.attn1.out.wi, s.attn2.query.wi,
            s.attn2.key.wi, s.attn2.value.wi, s.attn2.out.wi, s.geglu.wi, s.ff.wi});
  };
  auto block = [&](UNetBlockW& b) {
    const int p = g_level_passes[std::min(b.level, 3)];
    PackUnit u;
    u.conv = &b.conv;
    switch (b.kind) {
      case BK_CONV:  // unet/input_blocks/conv runs on CUDA cores from the master arena: no packed copy, not a target
        u.kind = U_CONV;
        add(u, {});
        break;
      case BK_DOWN:
        u.kind = U_CONV, u.passes = p;
        add(u, {b.conv.wi});
        break;
      case BK_R:
        res(b.res, p);
        break;
      case BK_RT:
        res(b.res, p), st(b.st, p);
        break;
      case BK_RU:
      case BK_RTU:
        res(b.res, p);
        if (b.kind == BK_RTU) st(b.st, p);
        u.kind = U_UP, u.passes = g_level_passes[std::max(b.level - 1, 0)];  // the conv runs at the upsampled resolution
        add(u, {b.conv.wi});
        break;
    }
  };
  for (auto& b : m.in_blocks) block(b);
  res(m.mid_res1, g_level_passes[3]), st(m.mid_st, g_level_passes[3]), res(m.mid_res2, g_level_passes[3]);
  for (auto& b : m.out_blocks) block(b);
  m.unit_emb = (int)m.units.size();
  PackUnit e;
  e.kind = U_EMB;
  m.units.push_back(e);
  for (ResBlockW* r : m.resblocks) m.lora_target[r->lin_embed.wi] = m.unit_emb;
  for (ClipBlockW& cb : m.clip.blocks) {
    PackUnit u;
    u.kind = U_CLIP, u.clip = &cb;
    add(u, {cb.query.wi, cb.key.wi, cb.value.wi, cb.out.wi, cb.fc1.wi, cb.fc2.wi});
  }
}

static void run_unit(Ctx& c, PackUnit& u) {
  u.off0 = c.packed.off;
  pack_unit(c, u);
  u.off1 = c.packed.off;
}

static void lora_merge_all(Ctx& c);

void model_finalize(Ctx& c) {
  Model& m = M(c);
  model_invalidate_graphs(c);
  build_units(m);
  lora_merge_all(c);  // W_eff of every tensor with an active adapter term, on the current base
  c.packed.reset();
  SDB_CUDA(cudaMemsetAsync(c.packed.base, 0, c.packed.cap, c.stream));  // head-pad rows must be zero
  // ---- UNet
  m.lin1_time.bias = mptr(c, m.lin1_time.bi), m.lin2_time.bias = mptr(c, m.lin2_time.bi);
  for (int i = 0; i < m.unit_emb; ++i) run_unit(c, m.units[i]);
  pack_norm(c, m.norm_out);
  pack_conv(c, m.conv_out);
  run_unit(c, m.units[m.unit_emb]);
  // ---- VAE decoder
  pack_conv(c, m.post_quant), pack_conv(c, m.vae_conv_in), pack_conv(c, m.vae_conv_out);
  pack_resnet(c, m.mid_block1, g_vae_passes_lowres), pack_resnet(c, m.mid_block2, g_vae_passes_lowres);
  pack_norm(c, m.mid_attn.norm);
  pack_conv(c, m.mid_attn.q), pack_conv(c, m.mid_attn.k), pack_conv(c, m.mid_attn.v), pack_conv(c, m.mid_attn.proj_out);
  m.mid_attn.passes = g_vae_passes_lowres;
  for (int i = 0; i < 4; ++i) {
    for (int j = 0; j < 3; ++j) pack_resnet(c, m.dec[i].res[j], i == 0 ? g_vae_passes_lowres : g_vae_passes_highres);
    if (m.dec[i].has_up) pack_conv(c, m.dec[i].up, /*up2=*/true), m.dec[i].up.passes = g_vae_passes_up;
  }
  pack_norm(c, m.vae_norm_out);
  // ---- VAE encoder (row f4): every GEMM 3-term split-fp16 (runs once per image; no accuracy budget spent here)
  {
    EncoderW& e = m.enc;
    pack_conv(c, e.conv_in), pack_conv(c, e.conv_out), pack_conv(c, e.quant);
    // conv_in has 3 input channels: the Cin = 4 CUDA-core kernel gets weights padded with a zero fourth channel
    e.conv_in_w4 = c.packed.get<float>((size_t)128 * 36);
    SDB_CUDA(cudaMemsetAsync(e.conv_in_w4, 0, (size_t)128 * 36 * 4, c.stream));
    SDB_CUDA(cudaMemcpy2DAsync(e.conv_in_w4, 36 * 4, mptr(c, e.conv_in.wi), 27 * 4, 27 * 4, 128, cudaMemcpyDeviceToDevice, c.stream));
    for (int i = 0; i < 4; ++i) {
      pack_resnet(c, e.blocks[i].res[0], 3), pack_resnet(c, e.blocks[i].res[1], 3);
      if (e.blocks[i].has_down) pack_conv(c, e.blocks[i].down), e.blocks[i].down.passes = 3;
    }
    pack_resnet(c, e.mid_block1, 3), pack_resnet(c, e.mid_block2, 3);
    pack_norm(c, e.mid_attn.norm);
    pack_conv(c, e.mid_attn.q), pack_conv(c, e.mid_attn.k), pack_conv(c, e.mid_attn.v), pack_conv(c, e.mid_attn.proj_out);
    e.mid_attn.passes = 3;
    pack_norm(c, e.norm_out);
  }
  // ---- CLIP text encoder
  for (size_t i = m.unit_emb + 1; i < m.units.size(); ++i) run_unit(c, m.units[i]);
  pack_norm(c, m.clip.ln_final);
  // ---- schedule
  m.alphas_host.resize(1000);
  SDB_CUDA(cudaMemcpyAsync(m.alphas_host.data(), mptr(c, m.alphas_i), 4000, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  // a context filled through sdb_set_tensor without the schedule tensor would divide by sqrt(0) in every DDIM step
  for (float a : m.alphas_host)
    SDB_CHECK(a > 0.f && a <= 1.f, "alpha_cumulative_products must lie in (0, 1]: set the schedule tensor before sdb_finalize_weights");
}

void model_invalidate_graphs(Ctx& c) {
  Model& m = M(c);
  for (auto& g : m.graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  m.graphs.clear();
}

// ================================================================================ LoRA adapters (DESIGN §7 f8)
struct ActiveTerm {
  const LoraTerm* t;
  float s;
};
using ActiveMap = std::unordered_map<int, std::vector<ActiveTerm>>;
// tensor -> its active terms in accumulation order (adapters by ascending id, terms in the order they were added)
static ActiveMap lora_active(const Model& m) {
  ActiveMap out;
  for (const auto& a : m.lora.adapters) {
    if (a.second.multiplier == 0.0) continue;
    for (const LoraTerm& t : a.second.terms) out[t.tensor].push_back({&t, (float)(a.second.multiplier * t.alpha / t.rank)});
  }
  return out;
}
static std::vector<std::pair<uint64_t, float>> lora_sig(const ActiveMap& act, int tensor) {
  std::vector<std::pair<uint64_t, float>> s;
  auto it = act.find(tensor);
  if (it != act.end())
    for (const ActiveTerm& a : it->second) s.push_back({a.t->serial, a.s});
  return s;
}
// out (rows, cols) of a target weight as stored, and its fan-in
static void lora_geometry(const TensorInfo& t, int& rows, int& cols, int& out, int& fan_in, bool& lin) {
  lin = t.kind == K_LIN_W;
  rows = (int)t.dims[0], cols = (int)(t.count / t.dims[0]);
  out = lin ? cols : rows, fan_in = lin ? rows : cols;
}

// Tensors whose active terms differ from what was last merged (a term added, removed or rescaled), ascending.
static std::vector<int> lora_changed(const LoraState& L, const ActiveMap& act) {
  std::vector<int> cand;
  for (auto& a : act) cand.push_back(a.first);
  for (auto& a : L.applied)
    if (!act.count(a.first)) cand.push_back(a.first);
  std::sort(cand.begin(), cand.end());
  std::vector<int> changed;
  for (int t : cand) {
    auto ap = L.applied.find(t);
    if (ap == L.applied.end() || ap->second != lora_sig(act, t)) changed.push_back(t);
  }
  return changed;
}

// Writes W_eff of `tensors` in one lora_merge_launch into their buffers (allocated by lora_add, so nothing is allocated here) and
// returns after the device has finished; only then are the merged tensors pointed at their W_eff. A tensor without an active term
// drops its W_eff: the packers then read the base. The caller records `applied` once the packing has been updated too.
static void lora_merge(Ctx& c, const std::vector<int>& tensors, const ActiveMap& act) {
  LoraState& L = M(c).lora;
  std::vector<LoraTensorDesc> td;
  std::vector<LoraTermDesc> tt;
  std::vector<int> merged;
  long long tiles = 0;
  for (int idx : tensors) {
    auto it = act.find(idx);
    if (it == act.end()) continue;
    const TensorInfo& ti = c.tensors[idx];
    LoraTensorDesc d;
    int o, f;
    bool lin;
    lora_geometry(ti, d.rows, d.cols, o, f, lin);
    d.base = mptr(c, idx), d.out = L.buf.at(idx), d.transposed = lin;
    d.term0 = (int)tt.size(), d.nterms = (int)it->second.size();
    d.tiles_c = (d.cols + 63) / 64;
    d.tile0 = tiles;
    tiles += (long long)((d.rows + 63) / 64) * d.tiles_c;
    for (const ActiveTerm& a : it->second) tt.push_back({a.t->down, a.t->up, a.t->rank, a.s});
    td.push_back(d);
    merged.push_back(idx);
  }
  if (!td.empty()) {
    SDB_CUDA(cudaStreamSynchronize(c.stream));  // the tables live in the work arena
    c.work.reset();
    LoraTensorDesc* d_td = c.work.get<LoraTensorDesc>(td.size());
    LoraTermDesc* d_tt = c.work.get<LoraTermDesc>(tt.size());
    SDB_CUDA(cudaMemcpyAsync(d_td, td.data(), td.size() * sizeof(LoraTensorDesc), cudaMemcpyHostToDevice, c.stream));
    SDB_CUDA(cudaMemcpyAsync(d_tt, tt.data(), tt.size() * sizeof(LoraTermDesc), cudaMemcpyHostToDevice, c.stream));
    lora_merge_launch(d_td, (int)td.size(), d_tt, tiles, c.stream);
    SDB_CUDA(cudaStreamSynchronize(c.stream));
    c.work.reset();
  }
  for (int idx : tensors) L.eff.erase(idx);
  for (int idx : merged) L.eff[idx] = L.buf.at(idx);
}
static void lora_record(LoraState& L, const std::vector<int>& tensors, const ActiveMap& act) {
  for (int idx : tensors) {
    auto s = lora_sig(act, idx);
    if (s.empty())
      L.applied.erase(idx);
    else
      L.applied[idx] = std::move(s);
  }
}

static void lora_merge_all(Ctx& c) {
  LoraState& L = M(c).lora;
  const ActiveMap act = lora_active(M(c));
  std::vector<int> ts;
  for (auto& a : act) ts.push_back(a.first);
  for (auto& e : L.eff)
    if (!act.count(e.first)) ts.push_back(e.first);
  for (auto& a : L.applied)
    if (!act.count(a.first)) ts.push_back(a.first);
  std::sort(ts.begin(), ts.end());
  ts.erase(std::unique(ts.begin(), ts.end()), ts.end());
  lora_merge(c, ts, act);
  lora_record(L, ts, act);
  L.pending = false;
}

// `pending` is set by every add / scale / remove; whether anything really differs from what was merged is settled here, so an add
// undone by a remove leaves nothing pending.
bool model_lora_pending(Ctx& c) {
  LoraState& L = M(c).lora;
  if (L.pending && lora_changed(L, lora_active(M(c))).empty()) L.pending = false;
  return L.pending;
}

void model_lora_add(Ctx& c, int adapter, const char* tensor, int rank, const float* down, const float* up, double alpha) {
  Model& m = M(c);
  build_units(m);
  char msg[512];
  snprintf(msg, sizeof(msg), "lora_add: adapter %d must be >= 0", adapter);
  SDB_CHECK(adapter >= 0, msg);
  SDB_CHECK(tensor, "lora_add: tensor is NULL");
  auto it = c.index.find(tensor);
  snprintf(msg, sizeof(msg), "lora_add: unknown tensor '%s'", tensor);
  SDB_CHECK(it != c.index.end(), msg);
  const int idx = it->second;
  snprintf(msg, sizeof(msg),
           "lora_add: tensor '%s' is not a LoRA target (targets: the packed UNet ResBlock, SpatialTransformer and resample "
           "weights and the CLIP attention / MLP weights; not norms, biases, embeddings, the VAE, unet/input_blocks/conv, "
           "unet/lin{1,2}_time_embed or unet/conv_out)", tensor);
  SDB_CHECK(m.lora_target.count(idx), msg);
  snprintf(msg, sizeof(msg), "lora_add: rank %d must be >= 1", rank);
  SDB_CHECK(rank >= 1, msg);
  SDB_CHECK(down, "lora_add: down is NULL");
  SDB_CHECK(up, "lora_add: up is NULL");
  snprintf(msg, sizeof(msg), "lora_add: alpha %.17g must be finite and > 0", alpha);
  SDB_CHECK(std::isfinite(alpha) && alpha > 0.0, msg);
  auto ad = m.lora.adapters.find(adapter);
  if (ad != m.lora.adapters.end())
    for (const LoraTerm& t : ad->second.terms) {
      snprintf(msg, sizeof(msg), "lora_add: adapter %d already has a term for '%s'", adapter, tensor);
      SDB_CHECK(t.tensor != idx, msg);
    }
  int rows, cols, out, fan_in;
  bool lin;
  lora_geometry(c.tensors[idx], rows, cols, out, fan_in, lin);
  LoraTerm t;
  t.tensor = idx, t.rank = rank, t.alpha = alpha;
  // the tensor's W_eff buffer is allocated with its first term and kept until no term targets it, so that neither an apply
  // nor a scale to 0 and back allocates or frees device memory (each cudaMalloc / cudaFree synchronises the device)
  float* wbuf = nullptr;
  const bool new_buf = !m.lora.buf.count(idx);
  try {
    SDB_CUDA(cudaMalloc(&t.down, (size_t)rank * fan_in * sizeof(float)));
    SDB_CUDA(cudaMalloc(&t.up, (size_t)out * rank * sizeof(float)));
    if (new_buf) SDB_CUDA(cudaMalloc(&wbuf, c.tensors[idx].count * sizeof(float)));
    SDB_CUDA(cudaMemcpy(t.down, down, (size_t)rank * fan_in * sizeof(float), cudaMemcpyHostToDevice));
    SDB_CUDA(cudaMemcpy(t.up, up, (size_t)out * rank * sizeof(float), cudaMemcpyHostToDevice));
  } catch (...) {
    cudaFree(t.down), cudaFree(t.up), cudaFree(wbuf);
    throw;
  }
  if (new_buf) m.lora.buf[idx] = wbuf;
  t.serial = m.lora.next_serial++;
  m.lora.adapters[adapter].terms.push_back(t);
  m.lora.pending = true;
}

void model_lora_scale(Ctx& c, int adapter, double multiplier) {
  LoraState& L = M(c).lora;
  char msg[160];
  auto it = L.adapters.find(adapter);
  snprintf(msg, sizeof(msg), "lora_scale: no adapter %d", adapter);
  SDB_CHECK(it != L.adapters.end(), msg);
  snprintf(msg, sizeof(msg), "lora_scale: multiplier %.17g must be finite", multiplier);
  SDB_CHECK(std::isfinite(multiplier), msg);
  it->second.multiplier = multiplier;
  L.pending = true;
}

void model_lora_remove(Ctx& c, int adapter) {
  LoraState& L = M(c).lora;
  char msg[160];
  snprintf(msg, sizeof(msg), "lora_remove: no adapter %d (-1 removes all)", adapter);
  SDB_CHECK(adapter == -1 || L.adapters.count(adapter), msg);
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  for (auto it = L.adapters.begin(); it != L.adapters.end();) {
    if (adapter != -1 && it->first != adapter) {
      ++it;
      continue;
    }
    for (LoraTerm& t : it->second.terms) cudaFree(t.down), cudaFree(t.up);
    it = L.adapters.erase(it);
  }
  std::unordered_set<int> targeted;
  for (const auto& a : L.adapters)
    for (const LoraTerm& t : a.second.terms) targeted.insert(t.tensor);
  for (auto it = L.buf.begin(); it != L.buf.end();) {
    if (targeted.count(it->first)) {
      ++it;
      continue;
    }
    L.eff.erase(it->first);  // its packing is re-made from the base by the next apply or finalize
    cudaFree(it->second);
    it = L.buf.erase(it);
  }
  L.pending = true;
}

void model_lora_apply(Ctx& c) {
  Model& m = M(c);
  build_units(m);
  SDB_CUDA(cudaStreamSynchronize(c.stream));  // nothing queued may still read the packed weights about to be rewritten
  const ActiveMap act = lora_active(m);
  const std::vector<int> changed = lora_changed(m.lora, act);
  lora_merge(c, changed, act);
  if (c.finalized) {
    // re-run the packing unit of every changed tensor into its own packed addresses; the step graphs captured those addresses
    // and stay valid. Head-pad rows are never written by the packers and stay zero.
    std::vector<int> units;
    for (int t : changed) units.push_back(m.lora_target.at(t));
    std::sort(units.begin(), units.end());
    units.erase(std::unique(units.begin(), units.end()), units.end());
    const size_t off = c.packed.off;
    for (int ui : units) {
      PackUnit& u = m.units[ui];
      c.packed.off = u.off0;
      pack_unit(c, u);
      SDB_CHECK(c.packed.off == u.off1, "lora_apply: a re-packed unit did not end where finalize left it");
    }
    c.packed.off = off;
    SDB_CUDA(cudaStreamSynchronize(c.stream));
    c.work.reset();
  }
  lora_record(m.lora, changed, act);  // only now: a failure above leaves these tensors changed for the next apply
  m.lora.pending = false;
}

void model_get_merged_tensor(Ctx& c, const char* tensor, float* host, int64_t count) {
  SDB_CHECK(tensor && host, "get_merged_tensor: null argument");
  const TensorInfo& t = c.info(tensor);
  SDB_CHECK(count == t.count, "get_merged_tensor: element count mismatch");
  SDB_CHECK(!model_lora_pending(c), "get_merged_tensor: adapter changes are pending: call sdb_lora_apply first");
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  SDB_CUDA(cudaMemcpy(host, wsrc(c, c.index.at(tensor)), t.count * sizeof(float), cudaMemcpyDeviceToHost));
}

// ================================================================================ forward helpers
struct Act {
  float* p = nullptr;
  Half2Ptr raw16;  // optional fp16 hi/lo copy of the same values, written by the producing epilogue for consumers that
                   // read this tensor as a raw GEMM operand (skip 1x1 convs, upsample convs): no staging launch
  int n = 0, H = 0, W = 0, C = 0;
  GnPart gn;       // GroupNorm statistics left by the producing GEMM (gn.slots > 0 once a producer filled them)
  size_t count() const { return (size_t)n * H * W * C; }
};
// channel bucket of the producer-side GroupNorm statistics: must divide the group size of every GroupNorm that reads the tensor,
// alone or concatenated: 10 for the UNet widths (320/640/960/1280/1920/2560 -> groups of 10..80), C/32 for the VAE (128/256/512)
static int gn_bucket_of(int C) { return C % 320 == 0 ? 10 : (C % 32 == 0 ? C / 32 : 0); }

struct Fwd {
  Ctx& c;
  Model& m;
  int nb;
  double* gn_sums = nullptr;  // [slots][nb][32][2]
  unsigned int* gn_tickets = nullptr;  // [slots][nb]
  int gn_slot = 0, gn_slots = 0;
  Fwd(Ctx& c_, int nb_) : c(c_), m(M(c_)), nb(nb_) {}
  void init_sums(int slots) {
    gn_slots = slots;
    gn_sums = c.work.get<double>((size_t)slots * nb * 64);
    gn_tickets = c.work.get<unsigned int>((size_t)slots * nb * 2);  // one ticket counter per (slot, image); the second half is spare
    SDB_CUDA(cudaMemsetAsync(gn_tickets, 0, sizeof(unsigned int) * slots * nb * 2, c.stream));
  }
  // GroupNorm statistics of one tensor as [nb][32][2] sums (for the fused GroupNorm + SiLU + small-Cout convs): from the
  // producer's partials when it left any, else by reading the tensor
  double* stats(const Act& x) {
    SDB_CHECK(gn_slot < gn_slots, "GroupNorm statistics slots exhausted");
    double* sums = gn_sums + (size_t)gn_slot * nb * 64;
    unsigned int* tk = gn_tickets + (size_t)gn_slot * nb * 2;
    gn_slot++;
    const int HW = x.H * x.W;
    if (x.gn.slots > 0) {
      if (c.trace_on) c.trace.push_back({TRACE_GN, {x.gn.slots > 128 ? GN_PATH_SUMS_FOLD : GN_PATH_SUMS_PARTIALS}});
      const GnSrc s = partials(x);
      const int nbk = x.C / x.gn.bucket;
      KernelScope ks(c, KC_GN_STATS, 0, (double)nb * s.slots * nbk * 8.0);
      gn_sums_from_partials_launch(s.part, s.cap, s.slots, nbk, x.C, x.gn.bucket, nb, sums, c.stream);
      return sums;
    }
    if (c.trace_on) c.trace.push_back({TRACE_GN, {GN_PATH_SUMS_STATS}});
    float* part = c.work.get<float>(gn_stats_partial_floats(nb, HW));
    KernelScope ks(c, KC_GN_STATS, 0, (double)nb * HW * x.C * 4.0);
    gn_stats_launch(x.p, x.C, nb, HW, sums, part, tk, c.stream);
    return sums;
  }
  // x with its producer's partials, pre-folded 64:1 above 128 slots: keeps the fold each consumer CTA repeats short
  GnSrc partials(const Act& x) {
    GnSrc s;
    s.x = x.p, s.C = x.C, s.part = x.gn.buf, s.cap = x.gn.cap, s.slots = x.gn.slots;
    if (x.gn.slots > 128) {
      const int nbk = x.C / x.gn.bucket, s2 = gn_fold_slots(x.gn.slots);
      float* folded = c.work.get<float>((size_t)nb * s2 * nbk * 2);
      KernelScope ks(c, KC_GN_STATS, 0, (double)nb * x.gn.slots * nbk * 8.0);
      gn_fold_launch(x.gn.buf, x.gn.cap, x.gn.slots, nbk, nb, folded, c.stream);
      s.part = folded, s.cap = s2, s.slots = s2;
    }
    return s;
  }
  Act act16(int H, int W, int C) {
    Act a = act(H, W, C);
    if (c.opt_raw16) a.raw16 = half2(a.count(), true);
    return a;
  }
  ActOp raw16_operand(const Act& x) {
    ActOp a;
    a.n = nb, a.H = x.H, a.W = x.W, a.C = x.C, a.p = x.raw16;
    return a;
  }
  Act act(int H, int W, int C) {
    Act a;
    a.n = nb, a.H = H, a.W = W, a.C = C;
    a.p = c.work.get<float>(a.count());
    a.gn.bucket = gn_bucket_of(C);
    if (a.gn.bucket && c.opt_gn_epilogue) {
      a.gn.cap = std::max(3 * ((H * W + 127) / 128), 160);
      a.gn.buf = c.work.get<float>((size_t)nb * a.gn.cap * (C / a.gn.bucket) * 2);
    }
    return a;
  }
  Half2Ptr half2(size_t count, bool lo) {
    Half2Ptr p;
    p.hi = c.work.get<__half>(count);
    if (lo) p.lo = c.work.get<__half>(count);
    return p;
  }
  // GroupNorm(+SiLU) of cat(x0,x1) staged as an fp16 operand
  ActOp gn_operand(const Act& x0, const Act* x1, const NormW& nw, bool silu, bool lo) {
    const int C = x0.C + (x1 ? x1->C : 0);
    ActOp a;
    a.n = nb, a.H = x0.H, a.W = x0.W, a.C = C;
    a.p = half2((size_t)nb * x0.H * x0.W * C, lo);
    const int HW = x0.H * x0.W;
    if (x0.gn.slots > 0 && (!x1 || (x1->gn.slots > 0 && x1->gn.bucket == x0.gn.bucket)) && (C / 32) % x0.gn.bucket == 0) {
      const GnSrc s0 = partials(x0), s1 = x1 ? partials(*x1) : GnSrc{};
      if (c.trace_on)
        c.trace.push_back({TRACE_GN, {x0.gn.slots > 128 || (x1 && x1->gn.slots > 128) ? GN_PATH_APPLY_FOLD : GN_PATH_APPLY}});
      KernelScope ks(c, KC_PREP, 0, (double)nb * HW * C * (4.0 + 2.0 + (lo ? 2.0 : 0.0)));
      gn_apply_launch(s0, s1, x0.gn.bucket, nb, x0.H, x0.W, silu ? 1 : 0, nw.gamma, nw.beta, nw.eps, a.p, c.stream);
      return a;
    }
    SDB_CHECK(gn_slot < gn_slots, "GroupNorm statistics slots exhausted");
    unsigned int* tk = gn_tickets + (size_t)gn_slot * nb * 2;
    gn_slot++;
    float* part = c.work.get<float>(gn_fused_partial_floats(nb, HW));
    if (c.trace_on) c.trace.push_back({TRACE_GN, {GN_PATH_FUSED}});
    KernelScope ks(c, KC_PREP, 0, (double)nb * HW * C * (8.0 + 2.0 + (lo ? 2.0 : 0.0)));
    gn_fused_launch(x0.p, x0.C, x1 ? x1->p : nullptr, x1 ? x1->C : 0, nb, x0.H, x0.W, silu ? 1 : 0, nw.gamma, nw.beta, nw.eps,
                    a.p, part, tk, c.stream);
    return a;
  }
  // raw (un-normalised) fp16 staging; phase2: the four stride-2 phase planes a stride-2 conv reads
  ActOp raw_operand(const Act& x0, const Act* x1, bool phase2, bool lo) {
    const int C = x0.C + (x1 ? x1->C : 0);
    ActOp a;
    a.n = nb, a.C = C;
    if (phase2)
      a.P = 4, a.H = x0.H / 2, a.W = x0.W / 2;
    else
      a.H = x0.H, a.W = x0.W;
    a.p = half2((size_t)nb * x0.H * x0.W * C, lo);
    KernelScope ks(c, KC_PREP, 0, (double)x0.n * x0.H * x0.W * C * (4.0 + 2.0 + (lo ? 2.0 : 0.0)));
    prep_operand_launch(x0.p, x0.C, x1 ? x1->p : nullptr, x1 ? x1->C : 0, nb, x0.H, x0.W, phase2, a.p, c.stream);
    return a;
  }
  ActOp rows_operand(Half2Ptr p, long long rows, int C) {
    ActOp a;
    a.p = p, a.n = 1, a.H = 1, a.W = (int)rows, a.C = C;
    return a;
  }
};

// reference unet/mod.rs:712-734 (emb_bias = conv_in.bias + lin_embed(silu(emb)); nullptr for the VAE ResnetBlock)
static void run_resblock(Fwd& f, const NormW& n1, const ConvW& c1, const NormW& n2, const ConvW& c2, const ConvW* skip,
                         const float* bias_merged, int passes, const Act& x0, const Act* x1, const float* emb_bias, Act& out) {
  Ctx& c = f.c;
  const size_t mark = c.work.off;
  const bool lo = passes >= 2 || c.opt_precision >= 2;
  ActOp a = f.gn_operand(x0, x1, n1, true, lo);
  ActOp raw, raw1;
  const bool have16 = x0.raw16.hi && (!lo || x0.raw16.lo) && (!x1 || (x1->raw16.hi && (!lo || x1->raw16.lo)));
  if (skip) {
    if (have16) {
      raw = f.raw16_operand(x0);
      if (x1) raw1 = f.raw16_operand(*x1);
    } else {
      raw = f.raw_operand(x0, x1, false, lo);
    }
  }
  Act h = f.act(x0.H, x0.W, c1.cout);
  {
    Epilogue ep;
    ep.out_f32 = h.p, ep.gn = &h.gn;
    ep.bias = emb_bias ? emb_bias : c1.bias;
    run_gemm(c, G_CONV3, a, nullptr, c1.packed, passes, ep);
  }
  ActOp b = f.gn_operand(h, nullptr, n2, true, lo);
  // the 1x1 skip conv rides in conv_out's K loop when its inputs already exist as fp16 operands
  const bool merge = skip && have16 && bias_merged && c.opt_skip_merge;
  if (skip && !merge) {
    Epilogue ep;
    ep.out_f32 = out.p;
    ep.bias = skip->bias;
    run_gemm(c, G_CONV1, raw, (have16 && x1) ? &raw1 : nullptr, skip->packed, passes, ep);
  }
  {
    Epilogue ep;
    ep.out_f32 = out.p, ep.out_f16 = out.raw16, ep.gn = &out.gn;
    ExtraK xk;
    if (merge) {
      xk.x0 = raw, xk.has_x1 = x1 != nullptr, xk.w = skip->packed;
      if (x1) xk.x1 = raw1;
      ep.bias = bias_merged;
    } else {
      ep.bias = c2.bias;
      ep.residual = skip ? out.p : x0.p;  // in-place accumulate onto the skip-conv result, or + x
    }
    run_gemm(c, G_CONV3, b, nullptr, c2.packed, passes, ep, merge ? &xk : nullptr);
  }
  c.work.off = mark;  // temporaries are dead once the block's kernels are queued (stream order)
}

// per-layer K / V^T of the context tokens (constant over the DDIM steps)
struct CtxKV {
  __half* kv = nullptr;     // [nb*Lpad][2*heads*dpad]: K | V of the context tokens, head-padded
  __half* kv_lo = nullptr;  // lo halves (the split QK^T of the 3-pass levels reads K as a hi + lo pair)
};
struct CtxState {
  Half2Ptr ctx16;  // [nb*Lpad][768]
  int Lpad = 0;
  int* kvlen = nullptr;  // device [nb]
  std::vector<CtxKV> kv; // one per SpatialTransformer in execution order
};

// device copies of the block's intermediate state (sdb_test_spatial_transformer), taken in stream order before the next stage
// rewrites it: y [Mt][C] as hi + lo after proj_in, attn1, attn2 and the MLP, and the LayerNorm row statistics [Mt][ln_slots(C)][2]
// that norm1 / norm2 / norm3 read
struct StTaps {
  Half2Ptr y[4];
  float* ln[3];
};

// reference unet/mod.rs:461-481 + 521-527 + 641-653 + 551-592
// The block's residual stream y lives as an fp16 hi + lo pair (22 significant bits; no fp32 copy): every GEMM that reads it as
// an operand takes the pair as it is, every GEMM that adds to it reads and rewrites the pair in place. The three LayerNorms have
// no launch (see pack_st): the producers of y leave row statistics, the consumers normalise in their epilogue.
static void run_spatial_transformer(Fwd& f, SpatialTransformerW& s, const CtxState& cs, const CtxKV& kv, const Act& x,
                                    Act& out, const StTaps* taps = nullptr) {
  Ctx& c = f.c;
  const size_t mark = c.work.off;
  const int P = s.passes;
  const bool lo = P >= 2 || c.opt_precision >= 2;
  const int HW = x.H * x.W;
  const long long Mt = (long long)f.nb * HW;
  const int C = s.c, hd = s.heads * s.dpad;
  const int ls = ln_slots(C);
  // GroupNorm (no activation) -> proj_in (1x1 conv == GEMM over tokens)
  ActOp a = f.gn_operand(x, nullptr, s.norm, false, lo);
  Half2Ptr y16 = f.half2((size_t)Mt * C, true);
  float* st1 = c.work.get<float>((size_t)Mt * ls * 2);
  float* st2 = c.work.get<float>((size_t)Mt * ls * 2);
  float* st3 = c.work.get<float>((size_t)Mt * ls * 2);
  // taps: y after stage i and the LayerNorm statistics it left (none after the MLP)
  auto tap = [&](int i, const float* st) {
    if (!taps) return;
    SDB_CUDA(cudaMemcpyAsync(taps->y[i].hi, y16.hi, (size_t)Mt * C * 2, cudaMemcpyDeviceToDevice, c.stream));
    SDB_CUDA(cudaMemcpyAsync(taps->y[i].lo, y16.lo, (size_t)Mt * C * 2, cudaMemcpyDeviceToDevice, c.stream));
    if (st) SDB_CUDA(cudaMemcpyAsync(taps->ln[i], st, (size_t)Mt * ls * 2 * 4, cudaMemcpyDeviceToDevice, c.stream));
  };
  {
    Epilogue ep;
    ep.out_f16 = y16, ep.bias = s.proj_in.bias, ep.ln_out = st1;
    run_gemm(c, G_CONV1, a, nullptr, s.proj_in.packed, P, ep);
  }
  tap(0, st1);
  Half2Ptr o16 = f.half2((size_t)Mt * C, lo);
  auto ln_consume = [&](Epilogue& ep, const float* stats, const NormW& nw, const float* u_hi, const float* u_full, const float* v) {
    ep.ln_in = stats, ep.ln_in_slots = ls, ep.ln_C = C, ep.ln_eps = nw.eps, ep.ln_u_hi = u_hi, ep.ln_u_full = u_full, ep.bias = v;
  };
  // ---- self attention: x += out(attn(q,k,v = LN1(x))); one GEMM for q | k | v (head-padded columns), the attention kernel
  // takes V as it is written here (MN-major operand)
  // on the 3-pass levels q and k also get their lo halves: the attention kernel forms the logits as a 3-term split product
  const bool qk_split = lo && c.opt_attn_split && attention_supports_qk3(s.dpad);
  __half* qkv = c.work.get<__half>((size_t)Mt * 3 * hd);
  __half* qkv_lo = qk_split ? c.work.get<__half>((size_t)Mt * 3 * hd) : nullptr;
  {
    Epilogue ep;
    ep.out_f16.hi = qkv, ep.out_f16.lo = qkv_lo;
    ln_consume(ep, st1, s.ln1, s.u_qkv_hi, s.u_qkv_full, s.v_qkv);
    run_gemm(c, G_LINEAR, f.rows_operand(y16, Mt, C), nullptr, s.w_qkv1, P, ep);
  }
  {
    AttnOp at;
    at.q = qkv, at.ldq = 3 * hd, at.q_col0 = 0, at.q_rows = HW;
    at.k = qkv, at.ldk = 3 * hd, at.k_col0 = hd, at.k_rows = HW;
    at.vT = qkv, at.ldv = 3 * hd, at.v_mn = 1, at.v_col0 = 2 * hd;
    at.q_lo = qkv_lo, at.k_lo = qkv_lo;
    at.nb = f.nb, at.heads = s.heads, at.d = s.d, at.dpad = s.dpad, at.Nq = HW, at.Nk = HW;
    at.out = o16, at.ldo = C;
    run_attention(c, at);
  }
  {
    Epilogue ep;
    ep.out_f16 = y16, ep.residual16 = y16, ep.bias = s.attn1.out.bias, ep.ln_out = st2;
    run_gemm(c, G_LINEAR, f.rows_operand(o16, Mt, C), nullptr, s.w_o1, P, ep);
  }
  tap(1, st2);
  // ---- cross attention: x += out(attn(q = LN2(x), k,v = context))
  __half* q2 = c.work.get<__half>((size_t)Mt * hd);
  __half* q2_lo = qk_split ? c.work.get<__half>((size_t)Mt * hd) : nullptr;
  {
    Epilogue ep;
    ep.out_f16.hi = q2, ep.out_f16.lo = q2_lo;
    ln_consume(ep, st2, s.ln2, s.u_q2_hi, s.u_q2_full, s.v_q2);
    run_gemm(c, G_LINEAR, f.rows_operand(y16, Mt, C), nullptr, s.w_q2, P, ep);
  }
  {
    AttnOp at;
    at.q = q2, at.ldq = hd, at.q_col0 = 0, at.q_rows = HW;
    at.k = kv.kv, at.ldk = 2 * hd, at.k_col0 = 0, at.k_rows = cs.Lpad;
    at.vT = kv.kv, at.ldv = 2 * hd, at.v_mn = 1, at.v_col0 = hd;
    at.q_lo = q2_lo, at.k_lo = kv.kv_lo;
    at.nb = f.nb, at.heads = s.heads, at.d = s.d, at.dpad = s.dpad, at.Nq = HW, at.Nk = cs.Lpad;
    at.kvlen = cs.kvlen;
    at.out = o16, at.ldo = C;
    run_attention(c, at);
  }
  {
    Epilogue ep;
    ep.out_f16 = y16, ep.residual16 = y16, ep.bias = s.attn2.out.bias, ep.ln_out = st3;
    run_gemm(c, G_LINEAR, f.rows_operand(o16, Mt, C), nullptr, s.w_o2, P, ep);
  }
  tap(2, st3);
  // ---- GEGLU MLP: x += lin(x_a * gelu(gate)), LN3 folded into the GEGLU projection
  Half2Ptr g16 = f.half2((size_t)Mt * 4 * C, lo);
  {
    Epilogue ep;
    ep.geglu = 1, ep.out_f16 = g16;
    ln_consume(ep, st3, s.ln3, s.u_geglu_hi, s.u_geglu_full, s.v_geglu);
    run_gemm(c, G_LINEAR, f.rows_operand(y16, Mt, C), nullptr, s.w_geglu, P, ep);
  }
  {
    Epilogue ep;
    ep.out_f16 = y16, ep.residual16 = y16, ep.bias = s.ff.bias;
    run_gemm(c, G_LINEAR, f.rows_operand(g16, Mt, 4 * C), nullptr, s.ff.packed, P, ep);
  }
  tap(3, nullptr);
  // ---- proj_out + residual with the block input
  {
    Epilogue ep;
    ep.out_f32 = out.p, ep.out_f16 = out.raw16, ep.residual = x.p, ep.bias = s.proj_out.bias, ep.gn = &out.gn, ep.gn_rpi = HW;
    run_gemm(c, G_LINEAR, f.rows_operand(y16, Mt, C), nullptr, s.proj_out.packed, P, ep);
  }
  c.work.off = mark;
}

// context tokens -> fp16 + per-layer K / V^T (reference unet/mod.rs:646-647 with context = Some(..))
static void prepare_context(Fwd& f, const float* d_ctx /*[nb][Lpad][768] zero padded*/, int Lpad, int* d_kvlen,
                            CtxState& cs) {
  Ctx& c = f.c;
  Model& m = f.m;
  cs.Lpad = Lpad;
  cs.kvlen = d_kvlen;
  const long long rows = (long long)f.nb * Lpad;
  cs.ctx16 = f.half2((size_t)rows * 768, true);
  {
    KernelScope ks(c, KC_ELEMENTWISE);
    convert_f16_launch(d_ctx, rows * 768, cs.ctx16, c.stream);
  }
  cs.kv.resize(m.sts.size());
  for (size_t i = 0; i < m.sts.size(); ++i) {
    SpatialTransformerW& s = *m.sts[i];
    const int hd = s.heads * s.dpad;
    CtxKV& kv = cs.kv[i];
    kv.kv = c.work.get<__half>((size_t)rows * 2 * hd);
    kv.kv_lo = c.work.get<__half>((size_t)rows * 2 * hd);
    {
      Epilogue ep;
      ep.out_f16.hi = kv.kv, ep.out_f16.lo = kv.kv_lo;
      run_gemm(c, G_LINEAR, f.rows_operand(cs.ctx16, rows, 768), nullptr, s.w_kv2, 3, ep);
    }
  }
}

// ================================================================================ UNet::forward
struct UNetIO {
  const float* x;      // [nb,4,H,W] NCHW (sample stride x_stride)
  const int* t_dev;    // device scalar timestep
  float* out;          // [nb,4,H,W] NCHW
  int H, W;
  const float* emb_all = nullptr;  // [1000][emb_total] rows precomputed per timestep value (sample_latent), or null
  const float* tf_dev = nullptr;   // device real timestep (DESIGN §7 f15): the per-step embedding reads it instead of t_dev
  // 9- / 8-channel conv_in (DESIGN §7 f9, f10): input channels 4.. of sample i at cond + (i % cond_mod) * cond_stride
  long long x_stride = 0;
  const float* cond = nullptr;
  long long cond_stride = 0;
  int cond_mod = 1;
};

// The conditioned UNets' extra input channels (unet_pass): a 9-channel UNet reads d_x [nb,4,H,W] and d_cond [nb/2,5,H,W] (both
// CFG halves of a step share it), an 8-channel one d_x [nb,4,H,W] and d_cond [nb,4,H,W] (each guidance group has its own); with
// d_cond null either reads d_x [nb,cin,H,W].
static void unet_cond_io(const Ctx& c, int nb, const float* d_x, const float* d_cond, UNetIO& io) {
  const long long hw = (long long)io.H * io.W;
  const int cin = c.unet_cin;
  if (cin != 4) {
    if (d_cond)
      io.x_stride = 4 * hw, io.cond = d_cond, io.cond_stride = (cin - 4) * hw, io.cond_mod = cin == 9 ? nb / 2 : nb;
    else
      io.x_stride = cin * hw, io.cond = d_x + 4 * hw, io.cond_stride = cin * hw, io.cond_mod = nb;
  }
}

// conv_in (unet/mod.rs:124-127, first input block): 3x3 Cin 4 / 8 / 9 -> 320 on CUDA cores, with the fp16 copy the first
// ResBlock's skip reads
static void unet_conv_in(Fwd& f, const UNetBlockW& b, const UNetIO& io, const Act& o) {
  Ctx& c = f.c;
  KernelScope ks(c, KC_SMALLCONV, 2.0 * f.nb * io.H * io.W * 9.0 * b.cin * b.cout);
  if (b.cin != 4) {
    conv3x3_cin_cond_launch(b.cin, io.x, io.x_stride, io.cond, io.cond_stride, io.cond_mod, f.nb, io.H, io.W, mptr(c, b.conv.wi),
                            b.conv.bias, b.cout, o.p, o.raw16, c.stream);
    if (c.trace_on) c.trace.push_back({TRACE_COND, {io.cond_mod}});
  } else {
    conv3x3_cin4_launch(io.x, f.nb, io.H, io.W, mptr(c, b.conv.wi), b.conv.bias, b.cout, nullptr, nullptr, 1.f, o.p, o.raw16,
                        c.stream);
  }
}

// GroupNorm + SiLU + 3x3 conv to cout <= 8 channels, fused, fp32 on CUDA cores, NCHW result y [nb,cout,H,W]: the UNet's out
// (unet/mod.rs:138-140, 320 -> 4), the decoder's norm_out + conv_out (autoencoder/mod.rs:215-216, 128 -> 3) and the encoder's
// (512 -> 8)
static void norm_conv_out(Fwd& f, const Act& x, const NormW& norm, const ConvW& conv, int cout, float* y) {
  Ctx& c = f.c;
  double* sums = f.stats(x);
  KernelScope ks(c, KC_SMALLCONV, 2.0 * f.nb * x.H * x.W * 9.0 * x.C * cout);
  const SmallCoutVariant v = conv3x3_small_cout_launch(x.p, f.nb, x.H, x.W, x.C, sums, norm.gamma, norm.beta, norm.eps,
                                                       conv.w_small, conv.bias, cout, y, c.stream);
  if (c.trace_on) c.trace.push_back({TRACE_CONV, {v.th, v.ck, v.ks}});
}

static void unet_forward(Fwd& f, const UNetIO& io, const CtxState& cs) {
  Ctx& c = f.c;
  Model& m = f.m;
  const size_t mark0 = c.work.off;
  f.gn_slot = 0;
  f.init_sums(64);
  // ---- time embedding (unet/mod.rs:19-30, 115-118) and all 22 lin_embed rows in one GEMV (:718-722)
  float* emb_hidden = c.work.get<float>(1280);
  float* emb_silu = c.work.get<float>(1280);
  float* emb_rows = c.work.get<float>(m.emb_total);
  if (io.emb_all) {
    // the rows of this timestep were computed before the step loop (model_sample_dev): one copy instead of three GEMVs
    KernelScope ks(c, KC_ELEMENTWISE, 0.0, 8.0 * m.emb_total);
    emb_select_launch(io.emb_all, io.t_dev, m.emb_total, emb_rows, c.stream);
  } else {
    {
      KernelScope ks(c, KC_ELEMENTWISE);
      if (io.tf_dev)
        time_embed_launch(io.tf_dev, mptr(c, m.lin1_time.wi), m.lin1_time.bias, mptr(c, m.lin2_time.wi), m.lin2_time.bias,
                          emb_hidden, emb_silu, c.stream);
      else
        time_embed_launch(io.t_dev, mptr(c, m.lin1_time.wi), m.lin1_time.bias, mptr(c, m.lin2_time.wi), m.lin2_time.bias,
                          emb_hidden, emb_silu, c.stream);
    }
    {
      KernelScope ks(c, KC_ELEMENTWISE, 2.0 * 1280 * m.emb_total, 4.0 * 1280 * m.emb_total);
      gemv_launch(emb_silu, m.emb_w_all, m.emb_b_all, 1280, m.emb_total, emb_rows, c.stream);
    }
  }
  int st_index = 0;
  std::vector<Act> saved;
  Act x;
  int H = io.H, W = io.W;
  auto do_res = [&](ResBlockW& r, const Act& x0, const Act* x1, Act& o) {
    run_resblock(f, r.norm_in, r.conv_in, r.norm_out, r.conv_out, r.has_skip ? &r.skip : nullptr, r.bias_merged, r.passes, x0, x1,
                 emb_rows + r.emb_off, o);
  };
  auto do_block = [&](UNetBlockW& b, const Act& x0, const Act* x1) -> Act {
    Act o;
    switch (b.kind) {
      case BK_CONV:
        o = f.act16(H, W, b.cout);
        unet_conv_in(f, b, io, o);
        break;
      case BK_DOWN: {  // unet/mod.rs:412-427: 3x3 stride 2 pad 1
        o = f.act16(H / 2, W / 2, b.cout);
        const size_t mk = c.work.off;
        const bool lo = b.conv.passes >= 2 || c.opt_precision >= 2;
        ActOp a = f.raw_operand(x0, nullptr, true, lo);
        Epilogue ep;
        ep.out_f32 = o.p, ep.out_f16 = o.raw16, ep.bias = b.conv.bias, ep.gn = &o.gn;
        run_gemm(c, G_CONV3_S2, a, nullptr, b.conv.packed, b.conv.passes, ep);
        c.work.off = mk;
        H /= 2, W /= 2;
        break;
      }
      case BK_R:
        o = f.act16(H, W, b.cout);
        do_res(b.res, x0, x1, o);
        break;
      case BK_RT: {
        o = f.act16(H, W, b.cout);
        Act r = f.act(H, W, b.cout);
        do_res(b.res, x0, x1, r);
        run_spatial_transformer(f, b.st, cs, cs.kv[st_index++], r, o);
        break;
      }
      case BK_RU:
      case BK_RTU: {
        o = f.act16(2 * H, 2 * W, b.cout);
        const size_t mk = c.work.off;
        // the tensor the upsample conv reads (resblock or transformer output) gets its fp16 copy from its producer
        Act r = b.kind == BK_RTU ? f.act(H, W, b.cout) : f.act16(H, W, b.cout);
        do_res(b.res, x0, x1, r);
        Act u = r;
        if (b.kind == BK_RTU) {
          u = f.act16(H, W, b.cout);
          run_spatial_transformer(f, b.st, cs, cs.kv[st_index++], r, u);
        }
        // unet/mod.rs:390-398: nearest 2x + conv3x3, folded into four 2x2-tap phase convolutions
        const bool lo = b.conv.passes >= 2 || c.opt_precision >= 2;
        ActOp a = u.raw16.hi ? f.raw16_operand(u) : f.raw_operand(u, nullptr, false, lo);
        Epilogue ep;
        ep.out_f32 = o.p, ep.out_f16 = o.raw16, ep.bias = b.conv.bias, ep.gn = &o.gn;
        run_gemm(c, G_CONV3_UP2, a, nullptr, b.conv.packed, b.conv.passes, ep);
        // `o` was allocated before mk, so releasing the temporaries keeps it alive
        c.work.off = mk;
        H *= 2, W *= 2;
        break;
      }
    }
    return o;
  };
  // input blocks (unet/mod.rs:124-127)
  for (auto& b : m.in_blocks) {
    x = do_block(b, x, nullptr);
    saved.push_back(x);
  }
  // middle block (:130)
  {
    Act r1 = f.act(H, W, 1280), t = f.act(H, W, 1280), r2 = f.act16(H, W, 1280);
    do_res(m.mid_res1, x, nullptr, r1);
    run_spatial_transformer(f, m.mid_st, cs, cs.kv[st_index++], r1, t);
    do_res(m.mid_res2, t, nullptr, r2);
    x = r2;
  }
  // output blocks: x = cat([x, saved.pop()], 1) (:133-136) — the concat is never materialised in fp32
  for (auto& b : m.out_blocks) {
    Act skip = saved.back();
    saved.pop_back();
    x = do_block(b, x, &skip);
  }
  // out: GroupNorm + SiLU + conv 320 -> 4 (:138-140)
  norm_conv_out(f, x, m.norm_out, m.conv_out, 4, io.out);
  c.work.off = mark0;
}

// ================================================================================ VAE decoder
static void run_resnet(Fwd& f, ResnetW& r, const Act& x, Act& out) {
  run_resblock(f, r.norm1, r.conv1, r.norm2, r.conv2, r.has_nin ? &r.nin : nullptr, r.bias_merged, r.passes, x, nullptr, nullptr,
               out);
}

// reference autoencoder/mod.rs:562-608: 1 head, d = C = 512, N = H*W tokens. S is materialised per image
// (64 MB at 64x64) because the op runs once per image; q/k/v/proj are the same wgmma GEMMs.
// o_tap (sdb_test_vae_stage): caller-allocated hi + lo storage [nb*HW][C] that receives the attention output before proj_out; its lo
// is cleared when the policy keeps no lo half
static void run_vae_attention(Fwd& f, VaeAttnW& a, const Act& x, Act& out, Half2Ptr* o_tap = nullptr) {
  Ctx& c = f.c;
  const size_t mark = c.work.off;
  const int P = a.passes;
  const bool lo = P >= 2 || c.opt_precision >= 2;
  const int HW = x.H * x.W, C = x.C;
  const long long Mt = (long long)f.nb * HW;
  ActOp h = f.gn_operand(x, nullptr, a.norm, false, lo);
  const int Mp = round_up((int)Mt, 32);
  Half2Ptr q16 = f.half2((size_t)Mt * C, lo), k16 = f.half2((size_t)Mt * C, lo), vT = f.half2((size_t)C * Mp, lo);
  Half2Ptr o16;
  if (o_tap) {
    if (!lo) o_tap->lo = nullptr;
    o16 = *o_tap;
  } else {
    o16 = f.half2((size_t)Mt * C, lo);
  }
  {
    Epilogue ep;
    ep.out_f16 = q16, ep.bias = a.q.bias;
    run_gemm(c, G_CONV1, h, nullptr, a.q.packed, P, ep);
  }
  {
    Epilogue ep;
    ep.out_f16 = k16, ep.bias = a.k.bias;
    run_gemm(c, G_CONV1, h, nullptr, a.k.packed, P, ep);
  }
  {
    // V^T = Wv . h^T ; the v bias is added after P.V (softmax rows sum to one)
    WeightOp tok;
    tok.p = h.p, tok.N = Mp, tok.rows = (int)Mt, tok.K = C;
    Epilogue ep;
    ep.out_f16 = vT;
    run_gemm(c, G_LINEAR, f.rows_operand(a.v.packed.p, C, C), nullptr, tok, P, ep);
  }
  float* S = c.work.get<float>((size_t)HW * HW);
  Half2Ptr p16 = f.half2((size_t)HW * HW, lo);
  const float scale = (float)(1.0 / std::sqrt((double)C));
  for (int s = 0; s < f.nb; ++s) {
    Half2Ptr qs{q16.hi + (size_t)s * HW * C, q16.lo ? q16.lo + (size_t)s * HW * C : nullptr};
    WeightOp ks_;
    ks_.p.hi = k16.hi + (size_t)s * HW * C, ks_.p.lo = k16.lo ? k16.lo + (size_t)s * HW * C : nullptr;
    ks_.N = HW, ks_.K = C;
    {
      Epilogue ep;
      ep.out_f32 = S;
      run_gemm(c, G_LINEAR, f.rows_operand(qs, HW, C), nullptr, ks_, P, ep);
    }
    {
      KernelScope ks(c, KC_ELEMENTWISE, 0, (double)HW * HW * 6.0);
      const int per = softmax_rows_launch(S, HW, HW, scale, p16, c.stream);
      if (c.trace_on) c.trace.push_back({TRACE_SOFTMAX, {per}});
    }
    WeightOp vs;
    vs.p.hi = vT.hi + (size_t)s * HW, vs.p.lo = vT.lo ? vT.lo + (size_t)s * HW : nullptr;
    vs.N = C, vs.K = HW, vs.ld = Mp;
    Epilogue ep;
    ep.out_f16.hi = o16.hi + (size_t)s * HW * C, ep.out_f16.lo = o16.lo ? o16.lo + (size_t)s * HW * C : nullptr;
    ep.bias = a.v.bias;
    run_gemm(c, G_LINEAR, f.rows_operand(p16, HW, HW), nullptr, vs, P, ep);
  }
  {
    Epilogue ep;
    ep.out_f32 = out.p, ep.residual = x.p, ep.bias = a.proj_out.bias, ep.gn = &out.gn, ep.gn_rpi = HW;
    run_gemm(c, G_LINEAR, f.rows_operand(o16, Mt, C), nullptr, a.proj_out.packed, P, ep);
  }
  c.work.off = mark;
}

// decoder conv_in 4 -> 512 with post_quant_conv (1x1, 4->4) and the latent's pre-scale folded into its input gather
// (autoencoder/mod.rs:68-71, 205): latent [nb,4,H,W] NCHW -> x
static void vae_dec_conv_in(Fwd& f, const float* d_latent, float pre_scale, const Act& x) {
  Ctx& c = f.c;
  Model& m = f.m;
  KernelScope ks(c, KC_SMALLCONV, 2.0 * f.nb * x.H * x.W * 36.0 * 512);
  conv3x3_cin4_launch(d_latent, f.nb, x.H, x.W, mptr(c, m.vae_conv_in.wi), m.vae_conv_in.bias, 512, mptr(c, m.post_quant.wi),
                      m.post_quant.bias, pre_scale, x.p, Half2Ptr{}, c.stream);
}

// latent [nb,4,H,W] NCHW (already divided by 0.18215 when called from latent_to_image) -> img [nb,3,8H,8W] NCHW
static void vae_decode(Fwd& f, const float* d_latent, int H, int W, float pre_scale, float* d_img) {
  Ctx& c = f.c;
  Model& m = f.m;
  const size_t mark0 = c.work.off;
  f.gn_slot = 0;
  f.init_sums(40);
  Act x = f.act(H, W, 512);
  vae_dec_conv_in(f, d_latent, pre_scale, x);
  // Mid (autoencoder/mod.rs:456-463)
  {
    Act a = f.act(H, W, 512), b = f.act(H, W, 512), d = f.act(H, W, 512);
    run_resnet(f, m.mid_block1, x, a);
    run_vae_attention(f, m.mid_attn, a, b);
    run_resnet(f, m.mid_block2, b, d);
    x = d;
  }
  // DecoderBlocks (autoencoder/mod.rs:307-324)
  for (int i = 0; i < 4; ++i) {
    DecoderBlockW& db = m.dec[i];
    for (int j = 0; j < 3; ++j) {
      // the tensor the upsampler reads gets its fp16 hi/lo copy from the producing epilogue
      Act o = (j == 2 && db.has_up) ? f.act16(H, W, db.res[j].cout) : f.act(H, W, db.res[j].cout);
      run_resnet(f, db.res[j], x, o);
      x = o;
    }
    if (db.has_up) {
      Act o = f.act16(2 * H, 2 * W, db.up.cout);  // read raw by the next block's nin_shortcut
      const size_t mk = c.work.off;
      const bool lo = db.up.passes >= 2 || c.opt_precision >= 2;
      ActOp a = x.raw16.hi ? f.raw16_operand(x) : f.raw_operand(x, nullptr, false, lo);
      Epilogue ep;
      ep.out_f32 = o.p, ep.out_f16 = o.raw16, ep.bias = db.up.bias, ep.gn = &o.gn;
      run_gemm(c, G_CONV3_UP2, a, nullptr, db.up.packed, db.up.passes, ep);
      c.work.off = mk;
      x = o;
      H *= 2, W *= 2;
    }
  }
  // norm_out + SiLU + conv_out 128 -> 3 (autoencoder/mod.rs:215-216)
  norm_conv_out(f, x, m.vae_norm_out, m.vae_conv_out, 3, d_img);
  c.work.off = mark0;
}

// ================================================================================ VAE encoder (SURVEY §8f row f4)
// Autoencoder::encode_image (autoencoder/mod.rs:60-66): Encoder::forward (:133-145) -> quant_conv -> channels [0,4).
// d_img4: the image with a zero fourth plane [nb][4][H][W]; d_latent [nb][4][H/8][W/8], or with out_stride > 0 sample i at
// d_latent + i * out_stride, scaled by out_scale (the inpainting conditioning tensor).
// conv_in 3 -> 128 (:138) on the Cin = 4 kernel: d_img4 [nb,4,H,W] with weights padded by a zero fourth input channel
static void vae_enc_conv_in(Fwd& f, const float* d_img4, const Act& x) {
  Ctx& c = f.c;
  EncoderW& e = f.m.enc;
  KernelScope ks(c, KC_SMALLCONV, 2.0 * f.nb * x.H * x.W * 27.0 * 128);
  conv3x3_cin4_launch(d_img4, f.nb, x.H, x.W, e.conv_in_w4, e.conv_in.bias, 128, nullptr, nullptr, 1.f, x.p, Half2Ptr{}, c.stream);
}

// an EncoderBlock's downsampler (:255-265): 3x3 stride 2, padded bottom/right only, with the GroupNorm partials the next
// ResnetBlock's norm1 reads. x [nb,H,W,C] -> o [nb,H/2,W/2,C] (o allocated by the caller)
static void vae_enc_down(Fwd& f, const ConvW& down, const Act& x, Act& o) {
  Ctx& c = f.c;
  SDB_CHECK(x.H % 2 == 0 && x.W % 2 == 0, "encode_image: image height and width must be multiples of 8");
  const size_t mk = c.work.off;
  ActOp a = f.raw_operand(x, nullptr, true, true);
  Epilogue ep;
  ep.out_f32 = o.p, ep.bias = down.bias, ep.gn = &o.gn;
  run_gemm(c, G_CONV3_S2_PAD01, a, nullptr, down.packed, down.passes, ep);
  c.work.off = mk;
}

// quant_conv 8 -> 8 and the slice [0,4) (:60-66): y8 [nb,8,HW] -> d_latent [nb,4,HW], or with out_stride > 0 sample i at
// d_latent + i * out_stride, scaled by out_scale
static void vae_enc_quant(Fwd& f, const float* y8, int HW, float* d_latent, long long out_stride, float out_scale) {
  Ctx& c = f.c;
  EncoderW& e = f.m.enc;
  KernelScope ks(c, KC_ELEMENTWISE);
  if (out_stride)
    quant_conv_slice_scaled_launch(y8, mptr(c, e.quant.wi), e.quant.bias, f.nb, HW, out_stride, out_scale, d_latent, c.stream);
  else
    quant_conv_slice_launch(y8, mptr(c, e.quant.wi), e.quant.bias, f.nb, HW, d_latent, c.stream);
}

static void vae_encode(Fwd& f, const float* d_img4, int H, int W, float* d_latent, long long out_stride = 0, float out_scale = 1.f) {
  Ctx& c = f.c;
  EncoderW& e = f.m.enc;
  const size_t mark0 = c.work.off;
  f.gn_slot = 0;
  f.init_sums(40);
  Act x = f.act(H, W, 128);
  vae_enc_conv_in(f, d_img4, x);
  // EncoderBlocks (:255-265): two ResnetBlocks, then the stride-2 conv padded bottom/right only
  for (int i = 0; i < 4; ++i) {
    EncoderBlockW& eb = e.blocks[i];
    for (int j = 0; j < 2; ++j) {
      Act o = f.act(H, W, eb.res[j].cout);
      run_resnet(f, eb.res[j], x, o);
      x = o;
    }
    if (eb.has_down) {
      SDB_CHECK(H % 2 == 0 && W % 2 == 0, "encode_image: image height and width must be multiples of 8");
      Act o = f.act(H / 2, W / 2, eb.down.cout);
      vae_enc_down(f, eb.down, x, o);
      x = o;
      H /= 2, W /= 2;
    }
  }
  // Mid (:456-463)
  {
    Act a = f.act(H, W, 512), b = f.act(H, W, 512), d = f.act(H, W, 512);
    run_resnet(f, e.mid_block1, x, a);
    run_vae_attention(f, e.mid_attn, a, b);
    run_resnet(f, e.mid_block2, b, d);
    x = d;
  }
  // norm_out + SiLU + conv_out 512 -> 8 (fp32 CUDA cores, NCHW), then quant_conv 8 -> 8 and the slice [0,4)
  float* y8 = c.work.get<float>((size_t)f.nb * 8 * H * W);
  norm_conv_out(f, x, e.norm_out, e.conv_out, 8, y8);
  vae_enc_quant(f, y8, H * W, d_latent, out_stride, out_scale);
  c.work.off = mark0;
}

// ================================================================================ public entry points
namespace {
struct StreamJoin {  // run on c.stream ordered after / before the caller's stream
  Ctx& c;
  cudaStream_t caller;
  cudaEvent_t ev = nullptr;
  StreamJoin(Ctx& c_, cudaStream_t s) : c(c_), caller(s) {
    if (caller != c.stream) {
      SDB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
      SDB_CUDA(cudaEventRecord(ev, caller));
      SDB_CUDA(cudaStreamWaitEvent(c.stream, ev, 0));
    }
  }
  ~StreamJoin() {
    if (ev) {
      cudaEventRecord(ev, c.stream);
      cudaStreamWaitEvent(caller, ev, 0);
      cudaEventDestroy(ev);
    }
  }
};
}  // namespace

// UNet pass over nb samples with per-sample context lengths. d_ctx_padded [nb][Lpad][768]. d_x / d_cond: see unet_cond_io.
// d_tf: a real timestep the time embedding reads instead of d_t (emb_all null).
static void unet_pass(Ctx& c, int nb, const float* d_x, const int* d_t, const float* d_ctx_padded, int Lpad, int* d_kvlen,
                      int H, int W, float* d_out, const CtxState* shared_cs, const float* emb_all = nullptr,
                      const float* d_cond = nullptr, const float* d_tf = nullptr) {
  Fwd f(c, nb);
  const size_t mark = c.work.off;
  CtxState local;
  const CtxState* cs = shared_cs;
  if (!cs) {
    prepare_context(f, d_ctx_padded, Lpad, d_kvlen, local);
    cs = &local;
  }
  UNetIO io{d_x, d_t, d_out, H, W};
  io.emb_all = emb_all, io.tf_dev = d_tf;
  unet_cond_io(c, nb, d_x, d_cond, io);
  unet_forward(f, io, *cs);
  c.work.off = mark;
}

// The timestep of a single UNet pass: the integer t of sdb_unet_forward, or the real t of sdb_unet_forward_at, rounded once to f32
struct PassTime {
  int t = 0;
  bool real = false;
  float tf = 0.f;
};

static void unet_forward_dev(Ctx& c, const float* d_x, PassTime pt, const float* d_context, int n, int H, int W, int L,
                             float* d_out, cudaStream_t caller) {
  SDB_CHECK(n >= 1 && H % 8 == 0 && W % 8 == 0 && L >= 1, "unet_forward arguments");
  // the deepest level has (H/8)*(W/8) tokens per sample; TMA tile origins inside the V^T matrix are
  // per-sample column offsets and must stay 16-byte aligned
  SDB_CHECK(((H / 8) * (W / 8)) % 8 == 0, "unsupported latent size: (H/8)*(W/8) must be a multiple of 8");
  StreamJoin join(c, caller);
  c.work.reset();
  const int Lpad = round_up(L, 32);
  float* ctxp = c.work.get<float>((size_t)n * Lpad * 768);
  int* d_t = c.work.get<int>(1);
  int* d_len = c.work.get<int>(n);
  std::vector<int> lens(n, L);
  SDB_CUDA(cudaMemsetAsync(ctxp, 0, (size_t)n * Lpad * 768 * 4, c.stream));
  SDB_CUDA(cudaMemcpy2DAsync(ctxp, (size_t)Lpad * 768 * 4, d_context, (size_t)L * 768 * 4, (size_t)L * 768 * 4, n,
                             cudaMemcpyDeviceToDevice, c.stream));
  if (pt.real)
    SDB_CUDA(cudaMemcpyAsync(d_t, &pt.tf, 4, cudaMemcpyHostToDevice, c.stream));
  else
    SDB_CUDA(cudaMemcpyAsync(d_t, &pt.t, 4, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaMemcpyAsync(d_len, lens.data(), 4 * n, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));  // host staging buffers (t, lens) must outlive the copies
  unet_pass(c, n, d_x, d_t, ctxp, Lpad, d_len, H, W, d_out, nullptr, nullptr, nullptr, pt.real ? (const float*)d_t : nullptr);
}

void model_unet_forward_dev(Ctx& c, const float* d_x, int t, const float* d_context, int n, int H, int W, int L,
                            float* d_out, cudaStream_t caller) {
  PassTime pt;
  pt.t = t;
  unet_forward_dev(c, d_x, pt, d_context, n, H, W, L, d_out, caller);
}

static void unet_forward_host(Ctx& c, const float* x, PassTime pt, const float* context, int n, int H, int W, int L, float* out) {
  const size_t xe = (size_t)n * 4 * H * W, ie = (size_t)n * c.unet_cin * H * W, ce = (size_t)n * L * 768;
  float* d_x = (float*)c.io(0, ie * 4);
  float* d_c = (float*)c.io(1, ce * 4);
  float* d_o = (float*)c.io(2, xe * 4);
  SDB_CUDA(cudaMemcpyAsync(d_x, x, ie * 4, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaMemcpyAsync(d_c, context, ce * 4, cudaMemcpyHostToDevice, c.stream));
  unet_forward_dev(c, d_x, pt, d_c, n, H, W, L, d_o, c.stream);
  SDB_CUDA(cudaMemcpyAsync(out, d_o, xe * 4, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

void model_unet_forward_host(Ctx& c, const float* x, int t, const float* context, int n, int H, int W, int L, float* out) {
  PassTime pt;
  pt.t = t;
  unet_forward_host(c, x, pt, context, n, H, W, L, out);
}

// sdb_unet_forward at a real timestep (DESIGN §7 f15): t finite in [0, 999], rounded once to f32; the time embedding takes the
// float path, which at an integer t gives sdb_unet_forward's rows, hence its output, bit for bit
void model_unet_forward_at_host(Ctx& c, const float* x, double t, const float* context, int n, int H, int W, int L, float* out) {
  char msg[160];
  snprintf(msg, sizeof(msg), "unet_forward_at: t = %.17g must be finite and in [0, 999]", t);
  SDB_CHECK(std::isfinite(t) && t >= 0.0 && t <= 999.0, msg);
  PassTime pt;
  pt.real = true, pt.tf = (float)t;
  unet_forward_host(c, x, pt, context, n, H, W, L, out);
}

// The autoencoder's mid attention (run_vae_attention) takes the latent's H * W positions as one row of S and of P: the row
// softmax holds at most kSoftmaxRowsMax = 9216 = 96 x 96 of them (a 768 x 768 px image); the S GEMM has N = HW (a multiple of 32)
// and the P.V GEMM reads P [HW][HW] as an operand of HW channels (a multiple of 64). Every entry that decodes or encodes refuses
// other latents here, before it launches anything.
static void check_vae_latent(int H, int W, const std::string& what) {
  char msg[320];
  snprintf(msg, sizeof(msg), "%s: unsupported latent size %dx%d: the autoencoder's attention needs H*W a multiple of 64",
           what.c_str(), H, W);
  SDB_CHECK(H >= 1 && W >= 1 && ((long long)H * W) % 64 == 0, msg);
  snprintf(msg, sizeof(msg),
           "%s: a %dx%d latent (%dx%d px) is too large for the autoencoder's attention, which takes at most %d latent positions "
           "(H*W): the largest supported image is 768x768 px (a 96x96 latent)",
           what.c_str(), H, W, 8 * H, 8 * W, kSoftmaxRowsMax);
  SDB_CHECK((long long)H * W <= kSoftmaxRowsMax, msg);
}

static void decode_chunked(Ctx& c, const float* d_latent, int n, int H, int W, float pre_scale, float* d_img) {
  // bounded working set: at most 4 images of 128-channel 8Hx8W activations at a time
  const int chunk = 4;
  for (int i = 0; i < n; i += chunk) {
    const int nb = std::min(chunk, n - i);
    Fwd f(c, nb);
    vae_decode(f, d_latent + (size_t)i * 4 * H * W, H, W, pre_scale, d_img + (size_t)i * 3 * 64 * H * W);
  }
}

void model_decode_dev(Ctx& c, const float* d_latent, int n, int H, int W, float* d_img, cudaStream_t caller) {
  check_vae_latent(H, W, "decode_latent");
  StreamJoin join(c, caller);
  c.work.reset();
  decode_chunked(c, d_latent, n, H, W, 1.0f, d_img);
}

void model_decode_host(Ctx& c, const float* latent, int n, int H, int W, float* img) {
  const size_t le = (size_t)n * 4 * H * W, ie = (size_t)n * 3 * 64 * H * W;
  float* d_l = (float*)c.io(0, le * 4);
  float* d_i = (float*)c.io(1, ie * 4);
  SDB_CUDA(cudaMemcpyAsync(d_l, latent, le * 4, cudaMemcpyHostToDevice, c.stream));
  model_decode_dev(c, d_l, n, H, W, d_i, c.stream);
  SDB_CUDA(cudaMemcpyAsync(img, d_i, ie * 4, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

void model_encode_dev(Ctx& c, const float* d_img, int n, int H, int W, float* d_latent, cudaStream_t caller) {
  SDB_CHECK(n >= 1 && H >= 64 && W >= 64 && H % 8 == 0 && W % 8 == 0 && ((H / 8) * (W / 8)) % 8 == 0,
            "encode_image: height and width must be multiples of 8, at least 64, with (H/8)*(W/8) a multiple of 8");
  check_vae_latent(H / 8, W / 8, "encode_image");
  StreamJoin join(c, caller);
  c.work.reset();
  const size_t plane = (size_t)H * W;
  for (int i0 = 0; i0 < n; i0 += 4) {  // chunks of 4 images bound the work arena like decode_chunked
    const int nb = std::min(4, n - i0);
    const size_t mark = c.work.off;
    float* img4 = c.work.get<float>((size_t)nb * 4 * plane);
    SDB_CUDA(cudaMemsetAsync(img4, 0, (size_t)nb * 4 * plane * 4, c.stream));
    SDB_CUDA(cudaMemcpy2DAsync(img4, 4 * plane * 4, d_img + (size_t)i0 * 3 * plane, 3 * plane * 4, 3 * plane * 4, nb,
                               cudaMemcpyDeviceToDevice, c.stream));
    Fwd f(c, nb);
    vae_encode(f, img4, H, W, d_latent + (size_t)i0 * 4 * (plane / 64));
    c.work.off = mark;
  }
}

void model_encode_host(Ctx& c, const float* img, int n, int H, int W, float* latent) {
  const size_t ie = (size_t)n * 3 * H * W, le = (size_t)n * 4 * (H / 8) * (W / 8);
  float* d_i = (float*)c.io(0, ie * 4);
  float* d_l = (float*)c.io(1, le * 4);
  SDB_CUDA(cudaMemcpyAsync(d_i, img, ie * 4, cudaMemcpyHostToDevice, c.stream));
  model_encode_dev(c, d_i, n, H, W, d_l, c.stream);
  SDB_CUDA(cudaMemcpyAsync(latent, d_l, le * 4, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

// latent_to_image (stablediffusion/mod.rs:69-100)
static void latent_to_image_dev(Ctx& c, const float* d_latent, int n, int H, int W, uint8_t* d_rgb) {
  check_vae_latent(H, W, "latent_to_image");
  float* d_img = c.work.get<float>((size_t)n * 3 * 64 * H * W);
  // `latent * (1.0 / 0.18215)`: the scalar is rounded to f32 before the multiply, as burn's mul_scalar does
  decode_chunked(c, d_latent, n, H, W, (float)(1.0 / 0.18215), d_img);
  KernelScope ks(c, KC_ELEMENTWISE);
  to_rgb8_launch(d_img, n, 8 * H, 8 * W, d_rgb, c.stream);
}

void model_latent_to_image_host(Ctx& c, const float* latent, int n, int H, int W, uint8_t* rgb) {
  const size_t le = (size_t)n * 4 * H * W, re = (size_t)n * 3 * 64 * H * W;
  float* d_l = (float*)c.io(0, le * 4);
  uint8_t* d_r = (uint8_t*)c.io(1, re);
  c.work.reset();
  SDB_CUDA(cudaMemcpyAsync(d_l, latent, le * 4, cudaMemcpyHostToDevice, c.stream));
  latent_to_image_dev(c, d_l, n, H, W, d_r);
  SDB_CUDA(cudaMemcpyAsync(rgb, d_r, re, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

// an 8-channel InstructPix2Pix UNet (sdb_create_pix2pix) reads an image latent and runs three-way guidance: only sdb_edit_image
// (and the single-pass sdb_unet_forward) drive it
static void check_not_pix2pix(const Ctx& c, const char* what) {
  SDB_CHECK(c.unet_cin != 8, std::string(what) + ": this context runs an 8-channel InstructPix2Pix UNet (sdb_create_pix2pix), "
                                                 "which needs an input image and image guidance; call sdb_edit_image");
}

// timesteps (stablediffusion/mod.rs:111,123): (0..1000).rev().step_by(1000 / n_steps)
static std::vector<int> ddim_timesteps(int n_steps) {
  std::vector<int> ts;
  for (int t = 999; t >= 0; t -= 1000 / n_steps) ts.push_back(t);
  return ts;
}

// The Karras et al. 2022 sigma grid (DESIGN §7 f15; k-diffusion's get_sigmas_karras at rho = 7 and sigma_to_t). The sigma table
// sigma_j = sqrt((1 - abar_j) / abar_j), abar read as f32 and widened, needs every abar_j finite, in (0, 1) and strictly
// decreasing in j: checked on every call, since a load can replace the schedule.
static double karras_sigma(const std::vector<float>& alphas, int j) {
  const double a = (double)alphas[j];
  return std::sqrt((1.0 - a) / a);
}

static std::vector<double> karras_log_sigmas(const std::vector<float>& alphas) {
  std::vector<double> ls(alphas.size());
  for (size_t j = 0; j < alphas.size(); ++j) {
    const double a = (double)alphas[j];
    char msg[240];
    snprintf(msg, sizeof(msg),
             "Karras schedule: alpha_cumulative_products[%d] = %.9g: every value must be finite, in (0, 1) and below the one "
             "before it",
             (int)j, a);
    SDB_CHECK(std::isfinite(a) && a > 0.0 && a < 1.0 && (j == 0 || a < (double)alphas[j - 1]), msg);
    ls[j] = std::log(karras_sigma(alphas, (int)j));
  }
  return ls;
}

// k-diffusion's sigma_to_t: linear in log sigma between the table neighbours; the low index is the largest j with
// log sigma_j <= log sigma, clamped to [0, 998], and w is clamped to [0, 1]
static double karras_sigma_to_t(const std::vector<double>& ls, double sigma) {
  const double l = std::log(sigma);
  int lo = 0;
  for (int j = 0; j < (int)ls.size(); ++j)
    if (ls[j] <= l) lo = j;
  lo = std::min(lo, (int)ls.size() - 2);
  const double w = std::min(1.0, std::max(0.0, (ls[lo] - l) / (ls[lo] - ls[lo + 1])));
  return (1.0 - w) * lo + w * (lo + 1);
}

// The steps a sampling call walks (DESIGN §7 f6, f15): step i runs at abar[i] toward abar[i + 1]; abar[N] = 1.
//   DDIM grid (the reference's): ts[i] = 999 - i (1000 / n_steps), abar[i] = alphas[ts[i]] widened from f32.
//   Karras grid: sigma_i = (sigma_max^(1/7) + i / (N - 1) (sigma_min^(1/7) - sigma_max^(1/7)))^7 with sigma_max = sigma_999 and
//   sigma_min = sigma_0 (the ends exactly; N = 1: sigma_max alone), abar[i] = 1 / (1 + sigma_i^2), tf[i] = sigma_to_t(sigma_i)
//   rounded once to f32.
struct Grid {
  std::vector<int> ts;       // DDIM grid: the timestep values
  std::vector<float> tf;     // Karras grid: the real timesteps (empty on the DDIM grid)
  std::vector<double> abar;  // [N + 1]
  int n() const { return (int)abar.size() - 1; }
  bool karras() const { return !tf.empty(); }
};

static Grid sample_grid(const Ctx& c, const std::vector<float>& alphas, int n_steps) {
  Grid g;
  if (c.sampler_schedule == SDB_SCHEDULE_KARRAS) {
    const std::vector<double> ls = karras_log_sigmas(alphas);
    const double smax = karras_sigma(alphas, 999), smin = karras_sigma(alphas, 0);
    const double rmax = std::pow(smax, 1.0 / 7.0), rmin = std::pow(smin, 1.0 / 7.0);
    for (int i = 0; i < n_steps; ++i) {
      double sig = i == 0 ? smax : (i == n_steps - 1 ? smin : std::pow(rmax + (double)i / (n_steps - 1) * (rmin - rmax), 7.0));
      g.tf.push_back((float)karras_sigma_to_t(ls, sig));
      g.abar.push_back(1.0 / (1.0 + sig * sig));
    }
  } else {
    g.ts = ddim_timesteps(n_steps);
    for (int t : g.ts) g.abar.push_back((double)alphas[t]);  // read as f32, widened (stablediffusion/mod.rs:124-140)
  }
  g.abar.push_back(1.0);
  return g;
}

// The schedule index img2img starts from (DESIGN §7 f5): k = floor(strength * N) of the N timesteps run, the last k of them.
static int img2img_first(double strength, int N) {
  SDB_CHECK(std::isfinite(strength) && strength > 0.0 && strength <= 1.0, "img2img: strength must be finite and in (0, 1]");
  const int k = (int)std::floor(strength * (double)N);
  char msg[160];
  snprintf(msg, sizeof(msg), "img2img: strength %.17g runs none of the %d timesteps; the smallest valid strength is 1/%d = %.17g",
           strength, N, N, 1.0 / N);
  SDB_CHECK(k >= 1, msg);
  return N - k;
}

// Rejects a request before anything is staged. The context kind comes first, so a call on the wrong context names the right
// entry whatever its pointers are; then the batch descriptor (naming the field, the sample and the value), the shape and step
// arguments, the pointers, the strength and the scales. host: a NULL start is drawn from the seed(s). Returns the schedule index
// the call starts from.
static int sample_n(const SampleRequest& r) { return r.batch ? r.batch->n : r.n; }

static int check_request(const Ctx& c, const SampleRequest& r, bool host) {
  const bool txt2img = r.kind == SAMPLE_TXT2IMG, img2img = r.kind == SAMPLE_IMG2IMG, edit = r.kind == SAMPLE_EDIT;
  char msg[240];
  if (edit) {
    snprintf(msg, sizeof(msg),
             "edit_image: this context's UNet takes %d input channels; InstructPix2Pix needs the 8-channel UNet of a context from "
             "sdb_create_pix2pix",
             c.unet_cin);
    SDB_CHECK(c.unet_cin == 8, msg);
  } else {
    // a 9-channel UNet (sdb_create_inpaint) reads a mask and a masked-image latent that text-to-image does not have
    SDB_CHECK(!txt2img || c.unet_cin != 9,
              "sample: this context runs a 9-channel inpainting UNet (sdb_create_inpaint), which needs a mask and an image; for "
              "text-to-image call sdb_img2img with an all-255 mask at strength 1");
    check_not_pix2pix(c, txt2img ? "sample" : "img2img");
  }
  const sdb_batch* b = r.batch;
  if (r.batched) {
    SDB_CHECK(b, "batch: null descriptor");
    snprintf(msg, sizeof(msg), "batch: n = %d must be >= 1", b->n);
    SDB_CHECK(b->n >= 1, msg);
    snprintf(msg, sizeof(msg), "batch: the row strides L = %d and Lu = %d must be >= 1", b->L, b->Lu);
    SDB_CHECK(b->L >= 1 && b->Lu >= 1, msg);
    SDB_CHECK(b->context, "batch: context is NULL");
    SDB_CHECK(b->uncond, "batch: uncond is NULL");
    SDB_CHECK(b->guidance_scale, "batch: guidance_scale is NULL");
    SDB_CHECK(b->seed || r.start, "batch: seed is NULL and no init latent / noise is given");
    for (int i = 0; i < b->n; ++i) {
      const int l = b->context_len ? b->context_len[i] : b->L, lu = b->uncond_len ? b->uncond_len[i] : b->Lu;
      snprintf(msg, sizeof(msg), "batch: context_len[%d] = %d is outside [1, L = %d]", i, l, b->L);
      SDB_CHECK(l >= 1 && l <= b->L, msg);
      snprintf(msg, sizeof(msg), "batch: uncond_len[%d] = %d is outside [1, Lu = %d]", i, lu, b->Lu);
      SDB_CHECK(lu >= 1 && lu <= b->Lu, msg);
      snprintf(msg, sizeof(msg), "batch: guidance_scale[%d] = %.17g is not finite", i, b->guidance_scale[i]);
      SDB_CHECK(std::isfinite(b->guidance_scale[i]), msg);
    }
  }
  const int L = b ? b->L : r.L, Lu = b ? b->Lu : r.Lu;
  SDB_CHECK(sample_n(r) >= 1 && L >= 1 && Lu >= 1, "sample arguments");
  SDB_CHECK(r.n_steps >= 1 && r.n_steps <= 1000, "n_steps must be in [1,1000] (step_by(0) panics in the reference)");
  SDB_CHECK(r.H % 8 == 0 && r.W % 8 == 0, "latent size must be a multiple of 8");
  SDB_CHECK(((r.H / 8) * (r.W / 8)) % 8 == 0, "unsupported latent size: (H/8)*(W/8) must be a multiple of 8");
  const std::string what = img2img ? "img2img" : (edit ? "edit_image" : (b ? "sample_batch" : "sample"));
  // the autoencoder runs when the request encodes an image or asks for RGB: refuse a latent it cannot take before any UNet step
  if (!txt2img || r.rgb) check_vae_latent(r.H, r.W, what);
  if (!txt2img) {
    SDB_CHECK(r.image && (b ? b->context : r.context) && (b ? b->uncond : r.uncond), what + ": null image, context or uncond");
    SDB_CHECK(edit || r.mask || c.unet_cin == 4,
              "img2img: the mask is NULL; a 9-channel inpainting UNet (sdb_create_inpaint) needs one");
  }
  if (!txt2img || b) SDB_CHECK(r.latent_out || r.rgb, what + ": request the latent, the image or both");
  if (!txt2img && !host && !b) SDB_CHECK(r.start, what + (img2img ? ": the device entry needs the noise latent"
                                                                  : ": the device entry needs the start latent"));
  if (edit) {
    snprintf(msg, sizeof(msg), "edit_image: text_scale = %.17g is not finite", r.scale);
    SDB_CHECK(std::isfinite(r.scale), msg);
    snprintf(msg, sizeof(msg), "edit_image: image_scale = %.17g is not finite", r.image_scale);
    SDB_CHECK(std::isfinite(r.image_scale), msg);
  }
  // the active schedule's grid: N, and on the Karras grid the check of the schedule tensor
  const int N = sample_grid(c, M(c).alphas_host, r.n_steps).n();
  return img2img ? img2img_first(r.strength, N) : 0;
}

namespace {
// The n requests of a sampling call (DESIGN §7 f7). The single-request entries describe a uniform batch: every sample reads the L
// prompt rows and the one broadcast negative, under one scale, and eta noise runs over the call's flat latent. The batch entries
// give each sample its own prompt length, negative, scale and noise seed.
struct Batch {
  int n = 0;
  const float* cond = nullptr;    // device [n][L][768]
  int L = 0;
  const float* uncond = nullptr;  // device [n][Lu][768] (ustride = Lu * 768) or [Lu][768] broadcast (ustride = 0)
  int Lu = 0;
  long long ustride = 0;
  std::vector<int> len, ulen;     // [n] prompt / negative rows sample i reads
  double scale = 0.0;             // uniform guidance scale (d_scale null)
  const float* d_scale = nullptr;          // device [n]: per-sample scales; selects the per-sample fused step
  const uint64_t* d_noise_seed = nullptr;  // device [n]: eta noise seeds of the per-sample step
};

struct BatchTab {  // the per-sample tables of a batch call on the device (io slot kIoBatchTab)
  const uint64_t* seed = nullptr;
  const uint64_t* noise_seed = nullptr;
  const float* scale = nullptr;
};

// What the sampler loop starts from and conditions on, resolved from a request by sample_run
struct StepCond {
  int groups = 2;                 // 3: InstructPix2Pix (DESIGN §7 f10), groups e_U | e_I | e_T
  const float* start = nullptr;   // txt2img, edit: [n,4,H,W] copied into every group
  float* z0 = nullptr;            // img2img (start from img2img_prep): [n,4,H,W] encoder output, scaled by 0.18215 in place
  const float* eps = nullptr;     // img2img: [n,4,H,W] the noise
  const uint8_t* mask = nullptr;  // masked img2img: [n,8H,8W]
  float* w = nullptr;             // masked img2img: [n,H,W] latent mask, written by img2img_prep; selects the blend
  float sa = 0.f, sb = 0.f;       // img2img: sqrt(abar[t0]), sqrt(1 - abar[t0])
  // the UNet's extra input channels (io slot kIoUNetCond) or null: [n,5,H,W] latent mask | z_m (9-channel inpainting, DESIGN §7
  // f9), [3n,4,H,W] 0 | c_I | c_I (InstructPix2Pix, one block per guidance group)
  const float* cond = nullptr;
  double image_scale = 0.0;       // s_I of an edit; the Batch's scale is s_T
};
}  // namespace

// u8 HWC images [n][8H][8W][3] (or, d_image null, encoder inputs [n][4][8H][8W] already staged) -> the encoder in chunks of 4 (the
// work arena bound of decode_chunked) -> sample i's latent at dst + i * stride, times scale (stride 0: [n,4,H,W], unscaled)
static void encode_images(Ctx& c, const uint8_t* d_image, const float* d_enc_in, int n, int H, int W, float* dst,
                          long long stride = 0, float scale = 1.f) {
  const int Hp = 8 * H, Wp = 8 * W;
  const size_t plane = (size_t)Hp * Wp;
  for (int i0 = 0; i0 < n; i0 += 4) {
    const int nb = std::min(4, n - i0);
    const size_t mark = c.work.off;
    const float* in = d_enc_in + (size_t)i0 * 4 * plane;
    if (d_image) {
      float* img4 = c.work.get<float>((size_t)nb * 4 * plane);
      KernelScope ks(c, KC_ELEMENTWISE);
      u8_to_enc_input_launch(d_image + (size_t)i0 * 3 * plane, nb, Hp, Wp, img4, c.stream);
      in = img4;
    }
    Fwd f(c, nb);
    vae_encode(f, in, Hp, Wp, dst + i0 * (stride ? stride : 4ll * H * W), stride, scale);
    c.work.off = mark;
  }
}

// The fused step's per-step scalars for a step from abar a_t to a_prev (DESIGN §7 f6, f15): computed in double, rounded once to
// f32. last: the final step (a_prev = 1); key: the step's noise key (Grid). h_prev: DPM++'s h of the previous step this call ran;
// has_prev: the step has one (second order).
static void step_scalars(const Ctx& c, int kind, double a_t, double a_prev, bool last, int key, bool has_prev, double& h_prev,
                         CfgStepArgs& a) {
  double dir = std::sqrt(1.0 - a_prev);
  SamplerStep& s = a.s;
  if (kind != STEP_DDIM) {
    s.ka = (float)std::sqrt(a_prev), s.kb = (float)dir;
    if (kind == STEP_DDIM_ETA) {  // Song et al. 2021 eq. 16; s = 0 on the final step (a_prev = 1)
      const double sig = c.sampler_eta * std::sqrt((1.0 - a_prev) / (1.0 - a_t)) * std::sqrt(1.0 - a_t / a_prev);
      dir = std::sqrt(std::max(0.0, 1.0 - a_prev - sig * sig));
      s.s = (float)sig;
      step_noise_keys(c.sampler_noise_seed, key, &s.k0, &s.k1);
    } else if (last) {  // DPM++ final step: sigma' = 0, h = inf: first order, x' = x0
      s.cx = 0.f, s.cd = 1.f;
    } else {  // DPM-Solver++(2M) (Lu et al. 2022), data prediction, lambda = ln(alpha / sigma)
      const double lam = std::log(std::sqrt(a_t) / std::sqrt(1.0 - a_t));
      const double lam_next = std::log(std::sqrt(a_prev) / std::sqrt(1.0 - a_prev));
      const double h = lam_next - lam;
      s.cx = (float)(std::sqrt(1.0 - a_prev) / std::sqrt(1.0 - a_t));
      s.cd = (float)(-std::sqrt(a_prev) * std::expm1(-h));
      if (has_prev) {  // second order: the first step a call runs has no history
        const double c2 = 1.0 / (2.0 * (h_prev / h));
        s.second = 1, s.c1 = (float)(1.0 + c2), s.c2 = (float)c2;
      }
      h_prev = h;
    }
  }
  s.t = key;
  a.sqrt_1m_at = (float)std::sqrt(1.0 - a_t), a.sqrt_at = (float)std::sqrt(a_t), a.sqrt_aprev = (float)std::sqrt(a_prev);
  a.dir_coef = (float)dir;
}

// The cached CUDA graph of the step's UNet pass (`pass`), captured on first use. A graph bakes in the addresses of xb, eps, the
// context K/V, the step's temporaries (work_mark on) and cond, an io slot that can grow and move between calls, so those are
// matched beside the shape key; txt2img, img2img and batch calls of one shape share their graphs.
template <class Pass>
static Model::GraphEntry step_graph(Ctx& c, Model::GraphEntry want, int* d_tcur, const int* d_t, const Pass& pass) {
  Model& m = M(c);
  for (const Model::GraphEntry& g : m.graphs)
    if (g.key == want.key && g.xb == want.xb && g.eps == want.eps && g.kv == want.kv && g.work_mark == want.work_mark &&
        g.cond == want.cond)
      return g;
  // warm-up pass outside capture (sets kernel attributes), then capture
  SDB_CUDA(cudaMemcpyAsync(d_tcur, d_t, 4, cudaMemcpyDeviceToDevice, c.stream));
  pass();
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  const int64_t before = c.launches;
  cudaGraph_t graph;
  SDB_CUDA(cudaStreamBeginCapture(c.stream, cudaStreamCaptureModeThreadLocal));
  try {
    pass();
  } catch (...) {
    cudaGraph_t g2;
    cudaStreamEndCapture(c.stream, &g2);
    throw;
  }
  SDB_CUDA(cudaStreamEndCapture(c.stream, &graph));
  want.launches = c.launches - before;
  c.launches = before;
  SDB_CUDA(cudaGraphInstantiate(&want.exec, graph, 0));
  cudaGraphDestroy(graph);
  m.graphs.push_back(want);
  return want;
}

// sample_latent + latent_to_image (stablediffusion/mod.rs:51-160) from schedule index `first` on. The guidance groups of a step
// (forward_diffuser :162-192) run as ONE batch-(groups n) UNet pass: weights stream from HBM once. Two groups: unconditional |
// prompt. Three (an edit): negative without the image, negative with it, prompt with it, and k.cond holds each group's image
// channels. Runs on c.stream; the caller joins the streams.
static void sample_loop(Ctx& c, const Batch& b, const Grid& grid, int first, const StepCond& k, int H, int W, float* d_latent_out,
                        uint8_t* d_rgb) {
  Model& m = M(c);
  c.work.reset();
  const int n = b.n;
  const int groups = k.groups;
  const int nb = groups * n;
  // padded to the longest row count any sample reads, not to the caller's strides: the step graph is keyed on Lpad
  int lmax = 1;
  for (int i = 0; i < n; ++i) lmax = std::max(lmax, std::max(b.len[i], b.ulen[i]));
  const int Lpad = round_up(lmax, 32);
  const size_t le = (size_t)n * 4 * H * W;
  // batch layout: samples [0,n) = unconditional context, [n,2n) = prompt context; an edit: [0,2n) negative, [2n,3n) prompt
  float* ctxp = c.work.get<float>((size_t)nb * Lpad * 768);
  float* xb = c.work.get<float>(groups * le);
  float* eps = c.work.get<float>(groups * le);
  int* d_t = c.work.get<int>(1024);
  int* d_len = c.work.get<int>(nb);
  std::vector<int> lens(nb);
  const int nu = (groups - 1) * n;  // samples that read the negative
  for (int i = 0; i < nb; ++i) lens[i] = i < nu ? b.ulen[i % n] : b.len[i - nu];
  SDB_CUDA(cudaMemcpyAsync(d_len, lens.data(), nb * 4, cudaMemcpyHostToDevice, c.stream));
  {
    KernelScope ks(c, KC_ELEMENTWISE);
    stage_cfg_context_launch(b.cond, b.L, b.uncond, b.ustride, d_len, n, Lpad, ctxp, c.stream, groups);
  }
  if (k.z0) {
    KernelScope ks(c, KC_ELEMENTWISE);
    img2img_prep_launch(k.z0, k.eps, xb, (long long)le, k.sa, k.sb, k.mask, k.w, H, W, c.stream);
  } else {
    for (int g = 0; g < groups; ++g)
      SDB_CUDA(cudaMemcpyAsync(xb + g * le, k.start, le * 4, cudaMemcpyDeviceToDevice, c.stream));
  }
  // img2img runs the last k steps only. d_t holds, per step the call runs, the word the step graph reads at d_tcur: the timestep
  // value on the DDIM grid; on the Karras grid (DESIGN §7 f15) the grid index i, which is the step's emb_all row, or with
  // emb_hoist off the f32 bits of its real timestep, which the per-step embedding reads
  const int N = grid.n(), rows = N - first;
  const bool karras = grid.karras(), real_t = karras && !c.opt_emb_hoist;
  std::vector<int> words(rows);
  for (int i = first; i < N; ++i) {
    int& w = words[i - first];
    if (!karras)
      w = grid.ts[i];
    else if (real_t)
      memcpy(&w, &grid.tf[i], 4);
    else
      w = i;
  }
  SDB_CUDA(cudaMemcpyAsync(d_t, words.data(), rows * 4, cudaMemcpyHostToDevice, c.stream));
  // the Karras grid's real timesteps, for the hoisted embedding rows (an io slot: the work arena's layout is the DDIM grid's)
  float* d_tf = karras && c.opt_emb_hoist ? (float*)c.io(kIoSchedule, 1000 * 4) : nullptr;
  if (d_tf) SDB_CUDA(cudaMemcpyAsync(d_tf, grid.tf.data() + first, rows * 4, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));  // host staging buffers (words, tf, lens) must outlive the copies

  // time-embedding rows of every timestep of the schedule, once per call (unet/mod.rs:19-30, 115-118, 718-722 depend on t alone).
  // Fixed-size table indexed by the timestep value (DDIM grid) or the grid index (Karras grid): the addresses of everything
  // allocated after it do not depend on n_steps or on the grid, which the cached step graphs rely on.
  float* emb_all = nullptr;
  if (c.opt_emb_hoist) {
    emb_all = c.work.get<float>((size_t)1000 * m.emb_total);
    const size_t mk = c.work.off;
    float* hid = c.work.get<float>((size_t)rows * 1280);
    float* sil = c.work.get<float>((size_t)rows * 1280);
    {
      KernelScope ks(c, KC_ELEMENTWISE, 2.0 * 1280 * m.emb_total * rows, 4.0 * 1280 * m.emb_total * ((rows + 4) / 5));
      if (d_tf)
        time_embed_rows_launch(d_tf, d_t, rows, mptr(c, m.lin1_time.wi), m.lin1_time.bias, mptr(c, m.lin2_time.wi),
                               m.lin2_time.bias, m.emb_w_all, m.emb_b_all, m.emb_total, hid, sil, emb_all, c.stream);
      else
        time_embed_rows_launch(d_t, rows, mptr(c, m.lin1_time.wi), m.lin1_time.bias, mptr(c, m.lin2_time.wi),
                               m.lin2_time.bias, m.emb_w_all, m.emb_b_all, m.emb_total, hid, sil, emb_all, c.stream);
    }
    c.launches += 2;  // three launches under one scope
    c.work.off = mk;  // stream order: the temporaries are dead before anything else is written there
  }

  Fwd f(c, nb);
  CtxState cs;
  prepare_context(f, ctxp, Lpad, d_len, cs);  // context K/V: once per image, not once per step

  int* d_tcur = c.work.get<int>(1);
  auto pass = [&] {
    unet_pass(c, nb, xb, d_tcur, nullptr, Lpad, d_len, H, W, eps, &cs, emb_all, k.cond, real_t ? (const float*)d_tcur : nullptr);
  };
  // one CUDA graph of the UNet step per (nb,H,W,Lpad); replayed with a different timestep slot each step. The hoisted embedding
  // reads an emb_all row on either grid, so a Karras call replays the DDIM graph of its shape; the per-step embedding of a real
  // timestep is another graph (bit 2 of the key), so neither kind of graph replays the other
  Model::GraphEntry graph;
  graph.key = ((long long)nb << 48) ^ ((long long)H << 36) ^ ((long long)W << 24) ^ ((long long)Lpad << 8) ^
              (long long)(c.opt_precision & 3) ^ (real_t ? 4ll : 0ll);
  graph.xb = xb, graph.eps = eps, graph.kv = cs.kv[0].kv, graph.work_mark = c.work.off, graph.cond = k.cond;
  if (c.opt_graphs && !c.profiling) graph = step_graph(c, graph, d_tcur, d_t, pass);
  // the sampler (DESIGN §7 f6): DDIM with eta = 0 is sample_latent's own step
  const bool dpm = c.sampler_kind == SDB_SAMPLER_DPMPP_2M;
  CfgStepArgs call;
  call.kind = dpm ? STEP_DPMPP_2M : (c.sampler_eta != 0.0 ? STEP_DDIM_ETA : STEP_DDIM);
  call.groups = groups;
  call.eu = eps, call.ec = eps + le, call.lat = xb, call.count = (long long)le, call.plane = H * W;
  call.scale = (float)b.scale, call.scale_i = (float)k.image_scale;
  if (k.w) call.z0 = k.z0, call.e0 = k.eps, call.w = k.w;
  call.s.hist = dpm ? (float*)c.io(kIoSamplerHist, le * 4) : nullptr;
  call.s.scales = b.d_scale, call.s.noise_seeds = b.d_noise_seed;  // per-sample step (batch entries) when set
  double h_prev = 0.0;  // DPM++: h of the previous step this call ran (none before the first)
  for (int i = 0; i < rows; ++i) {
    SDB_CUDA(cudaMemcpyAsync(d_tcur, d_t + i, 4, cudaMemcpyDeviceToDevice, c.stream));
    if (graph.exec) {
      SDB_CUDA(cudaGraphLaunch(graph.exec, c.stream));
      c.launches += graph.launches;
    } else {
      c.work.off = graph.work_mark;
      pass();
    }
    KernelScope ks(c, KC_ELEMENTWISE);
    CfgStepArgs a = call;
    const int gi = first + i;  // the step's index in the grid: Karras noise is keyed by it, DDIM noise by the timestep value
    step_scalars(c, a.kind, grid.abar[gi], grid.abar[gi + 1], gi + 1 == N, karras ? gi : grid.ts[gi], i > 0, h_prev, a);
    cfg_step_launch(a, c.stream);
  }
  c.work.off = graph.work_mark;
  if (d_latent_out) SDB_CUDA(cudaMemcpyAsync(d_latent_out, xb, le * 4, cudaMemcpyDeviceToDevice, c.stream));
  if (d_rgb) latent_to_image_dev(c, xb, n, H, W, d_rgb);
}

// Scales are cast to float as the single-request entries cast theirs; a NULL noise_seed array means the context's noise seed
// (sdb_set_sampler) for every sample.
static BatchTab upload_batch_tab(Ctx& c, const sdb_batch& b) {
  const int n = b.n;
  std::vector<uint64_t> u(2 * n);
  std::vector<float> f(n);
  for (int i = 0; i < n; ++i) {
    u[i] = b.seed ? b.seed[i] : 0;
    u[n + i] = b.noise_seed ? b.noise_seed[i] : c.sampler_noise_seed;
    f[i] = (float)b.guidance_scale[i];
  }
  char* d = (char*)c.io(kIoBatchTab, (size_t)n * 20);
  SDB_CUDA(cudaMemcpyAsync(d, u.data(), (size_t)n * 16, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaMemcpyAsync(d + (size_t)n * 16, f.data(), (size_t)n * 4, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));  // the host tables must outlive the copies
  return {(const uint64_t*)d, (const uint64_t*)d + n, (const float*)(d + (size_t)n * 16)};
}

// The Batch of a request whose context and uncond are device pointers
static Batch batch_of(const SampleRequest& r, const BatchTab& tab) {
  Batch b;
  if (!r.batch) {  // uniform
    b.n = r.n, b.cond = r.context, b.L = r.L, b.uncond = r.uncond, b.Lu = r.Lu, b.scale = r.scale;
    b.len.assign(r.n, r.L), b.ulen.assign(r.n, r.Lu);
    return b;
  }
  const sdb_batch& sb = *r.batch;
  b.n = sb.n, b.cond = sb.context, b.L = sb.L, b.uncond = sb.uncond, b.Lu = sb.Lu, b.ustride = (long long)sb.Lu * 768;
  for (int i = 0; i < sb.n; ++i) {
    b.len.push_back(sb.context_len ? sb.context_len[i] : sb.L);
    b.ulen.push_back(sb.uncond_len ? sb.uncond_len[i] : sb.Lu);
  }
  b.d_scale = tab.scale, b.d_noise_seed = tab.noise_seed;
  return b;
}

// One checked request with device pointers, on c.stream. A batch's NULL start is drawn per sample into io slot kIoStart: sample i is
// the latent the single-request entries draw for seed[i] at n = 1.
// img2img: the encoder writes z0 into an io slot, then the sampler loop runs from t0 = ts[first]. z0 and the latent mask live in
// io slots, not in the work arena: the arena prefix up to the loop's work_mark is laid out exactly as txt2img lays it out, so no
// cached step graph can see img2img data where it expects its own temporaries. A 9-channel UNet (DESIGN §7 f9) gets no blend:
// inpaint_prep writes the masked image's encoder input and the latent mask, and a second encoder pass writes z_m, so the
// conditioning tensor [n,5,H,W] (io slot kIoUNetCond) holds m_lat | z_m for conv_in.
// edit: the encoder writes c_I, unscaled, into group 1 of the conditioning tensor [3n,4,H,W] (io slot kIoUNetCond); group 2 is a
// copy and group 0 zero. Then the sampler loop from t = 999 over the full schedule with three guidance groups.
static void sample_run(Ctx& c, const SampleRequest& r, int first) {
  Model& m = M(c);
  BatchTab tab;
  if (r.batch) tab = upload_batch_tab(c, *r.batch);
  const Batch b = batch_of(r, tab);
  const int n = b.n, H = r.H, W = r.W;
  const size_t le = (size_t)n * 4 * H * W;
  const float* start = r.start;
  if (!start && r.batch) {
    float* d = (float*)c.io(kIoStart, le * 4);
    KernelScope ks(c, KC_ELEMENTWISE);
    randn_seeds_launch(d, n, 4ll * H * W, tab.seed, c.stream);
    start = d;
  }
  const Grid grid = sample_grid(c, m.alphas_host, r.n_steps);
  StepCond k;
  if (r.kind == SAMPLE_IMG2IMG) {
    const double abar = grid.abar[first];
    k.sa = (float)std::sqrt(abar), k.sb = (float)std::sqrt(1.0 - abar);
    const bool inpaint = c.unet_cin == 9;
    k.eps = start, k.mask = inpaint ? nullptr : r.mask;
    k.z0 = (float*)c.io(kIoImg2ImgZ0, le * 4);
    if (k.mask) k.w = (float*)c.io(kIoImg2ImgW, (size_t)n * H * W * 4);
    float* cond = inpaint ? (float*)c.io(kIoUNetCond, (size_t)n * 5 * H * W * 4) : nullptr;
    c.work.reset();
    encode_images(c, r.image, nullptr, n, H, W, k.z0);
    if (inpaint) {
      float* enc_in = c.work.get<float>((size_t)n * 4 * 64 * H * W);
      {
        KernelScope ks(c, KC_ELEMENTWISE);
        inpaint_prep_launch(r.image, r.mask, n, 8 * H, 8 * W, enc_in, cond, c.stream);
      }
      encode_images(c, nullptr, enc_in, n, H, W, cond + (size_t)H * W, 5ll * H * W, 0.18215f);
      k.cond = cond;
    }
  } else if (r.kind == SAMPLE_EDIT) {
    float* cond = (float*)c.io(kIoUNetCond, 3 * le * 4);
    c.work.reset();
    SDB_CUDA(cudaMemsetAsync(cond, 0, le * 4, c.stream));
    encode_images(c, r.image, nullptr, n, H, W, cond + le);
    SDB_CUDA(cudaMemcpyAsync(cond + 2 * le, cond + le, le * 4, cudaMemcpyDeviceToDevice, c.stream));
    k.groups = 3, k.start = start, k.cond = cond, k.image_scale = r.image_scale;
  } else {
    k.start = start;
  }
  sample_loop(c, b, grid, first, k, H, W, r.latent_out, r.rgb);
}

void model_sample_dev(Ctx& c, const SampleRequest& r, cudaStream_t caller) {
  const int first = check_request(c, r, false);
  StreamJoin join(c, caller);
  sample_run(c, r, first);
}

// Copies a host request's inputs into the staging io slots, runs it on c.stream, copies the requested outputs back and
// synchronises. A NULL start of a single request is the latent randn_launch draws for its seed (uncounted, as txt2img has always
// drawn it); a batch draws its own per-sample seeds in sample_run.
void model_sample_host(Ctx& c, const SampleRequest& r) {
  const int first = check_request(c, r, true);
  const int n = sample_n(r);
  const size_t le = (size_t)n * 4 * r.H * r.W, re = (size_t)n * 3 * 64 * r.H * r.W, me = (size_t)n * 64 * r.H * r.W;
  auto upload = [&](int slot, const void* host, size_t bytes) {
    void* d = c.io(slot, bytes);
    SDB_CUDA(cudaMemcpyAsync(d, host, bytes, cudaMemcpyHostToDevice, c.stream));
    return d;
  };
  SampleRequest d = r;
  sdb_batch db;
  if (r.batch) {
    db = *r.batch;
    db.context = (const float*)upload(kIoContext, db.context, (size_t)n * db.L * 768 * 4);
    db.uncond = (const float*)upload(kIoUncond, db.uncond, (size_t)n * db.Lu * 768 * 4);
    d.batch = &db;
  } else {
    d.context = (const float*)upload(kIoContext, r.context, (size_t)n * r.L * 768 * 4);
    d.uncond = (const float*)upload(kIoUncond, r.uncond, (size_t)r.Lu * 768 * 4);
  }
  if (r.image) d.image = (const uint8_t*)upload(kIoImage, r.image, re);
  if (r.mask) d.mask = (const uint8_t*)upload(kIoMask, r.mask, me);
  if (r.start) {
    d.start = (const float*)upload(kIoStart, r.start, le * 4);
  } else if (!r.batch) {
    float* s = (float*)c.io(kIoStart, le * 4);
    randn_launch(s, (long long)le, r.seed, c.stream);
    d.start = s;
  }
  d.latent_out = r.latent_out ? (float*)c.io(kIoLatentOut, le * 4) : nullptr;
  d.rgb = r.rgb ? (uint8_t*)c.io(kIoRgb, re) : nullptr;
  sample_run(c, d, first);
  if (r.latent_out) SDB_CUDA(cudaMemcpyAsync(r.latent_out, d.latent_out, le * 4, cudaMemcpyDeviceToHost, c.stream));
  if (r.rgb) SDB_CUDA(cudaMemcpyAsync(r.rgb, d.rgb, re, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

// forward_diffuser (stablediffusion/mod.rs:162-192): the two UNet evaluations of one guidance step as ONE batch-2n pass (the
// same pass sample_latent replays as a CUDA graph, its context staged by the same kernel), then pred = u + (c - u) * scale.
// d_u / d_c may be null.
void model_forward_diffuser_dev(Ctx& c, const float* d_latent, int t, const float* d_context, int n, int L, const float* d_uncond,
                                int Lu, double scale, int H, int W, float* d_pred, float* d_u, float* d_c, cudaStream_t caller) {
  check_not_pix2pix(c, "forward_diffuser (two-way guidance)");
  SDB_CHECK(n >= 1 && L >= 1 && Lu >= 1 && t >= 0 && t < 1000, "forward_diffuser arguments");
  SDB_CHECK(H % 8 == 0 && W % 8 == 0 && ((H / 8) * (W / 8)) % 8 == 0, "unsupported latent size");
  StreamJoin join(c, caller);
  c.work.reset();
  const int nb = 2 * n;
  const int Lpad = round_up(std::max(L, Lu), 32);
  const size_t le = (size_t)n * 4 * H * W, li = (size_t)n * c.unet_cin * H * W;  // output / input latent elements
  float* ctxp = c.work.get<float>((size_t)nb * Lpad * 768);
  float* xb = c.work.get<float>(2 * li);
  float* eps = c.work.get<float>(2 * le);
  int* d_t = c.work.get<int>(1);
  int* d_len = c.work.get<int>(nb);
  std::vector<int> lens(nb);
  for (int i = 0; i < nb; ++i) lens[i] = i < n ? Lu : L;
  SDB_CUDA(cudaMemcpyAsync(d_t, &t, 4, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaMemcpyAsync(d_len, lens.data(), nb * 4, cudaMemcpyHostToDevice, c.stream));
  {
    KernelScope ks(c, KC_ELEMENTWISE);
    stage_cfg_context_launch(d_context, L, d_uncond, 0, d_len, n, Lpad, ctxp, c.stream);
  }
  SDB_CUDA(cudaMemcpyAsync(xb, d_latent, li * 4, cudaMemcpyDeviceToDevice, c.stream));
  SDB_CUDA(cudaMemcpyAsync(xb + li, d_latent, li * 4, cudaMemcpyDeviceToDevice, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  unet_pass(c, nb, xb, d_t, ctxp, Lpad, d_len, H, W, eps, nullptr);
  if (d_u) SDB_CUDA(cudaMemcpyAsync(d_u, eps, le * 4, cudaMemcpyDeviceToDevice, c.stream));
  if (d_c) SDB_CUDA(cudaMemcpyAsync(d_c, eps + le, le * 4, cudaMemcpyDeviceToDevice, c.stream));
  if (d_pred) {
    KernelScope ks(c, KC_ELEMENTWISE);
    cfg_combine_launch(eps, eps + le, (long long)le, (float)scale, d_pred, c.stream);
  }
}

void model_forward_diffuser_host(Ctx& c, const float* latent, int t, const float* context, int n, int L, const float* uncond,
                                 int Lu, double scale, int H, int W, float* pred, float* out_u, float* out_c) {
  const size_t le = (size_t)n * 4 * H * W, li = (size_t)n * c.unet_cin * H * W, ce = (size_t)n * L * 768, ue = (size_t)Lu * 768;
  float* d_l = (float*)c.io(0, li * 4);
  float* d_c = (float*)c.io(1, ce * 4);
  float* d_u = (float*)c.io(2, ue * 4);
  float* d_o = (float*)c.io(3, 3 * le * 4);
  SDB_CUDA(cudaMemcpyAsync(d_l, latent, li * 4, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaMemcpyAsync(d_c, context, ce * 4, cudaMemcpyHostToDevice, c.stream));
  SDB_CUDA(cudaMemcpyAsync(d_u, uncond, ue * 4, cudaMemcpyHostToDevice, c.stream));
  model_forward_diffuser_dev(c, d_l, t, d_c, n, L, d_u, Lu, scale, H, W, d_o, d_o + le, d_o + 2 * le, c.stream);
  if (pred) SDB_CUDA(cudaMemcpyAsync(pred, d_o, le * 4, cudaMemcpyDeviceToHost, c.stream));
  if (out_u) SDB_CUDA(cudaMemcpyAsync(out_u, d_o + le, le * 4, cudaMemcpyDeviceToHost, c.stream));
  if (out_c) SDB_CUDA(cudaMemcpyAsync(out_c, d_o + 2 * le, le * 4, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

// ================================================================================ CLIP text encoder
// The encoder's working set for n samples of L tokens. Rows are laid out at the per-sample pitch Lp = round_up(L, 8), which keeps
// every TMA tile origin 16-byte aligned; the rows l >= L of a sample are padding.
struct ClipBufs {
  int n = 0, L = 0, Lp = 0, Mr = 0, Mp = 0;
  float* x = nullptr;  // residual stream [Mr][768] fp32, updated in place by each block
  Half2Ptr l16, o16, h16;  // LayerNorm output, attention output [Mr][768], QuickGELU(fc1) [Mr][3072]: fp16 hi + lo
  __half* qk = nullptr;  // q | k [Mr][1536], single fp16 values
  __half* vT = nullptr;  // V^T [768][Mp], sample s at columns s*Lp; the GEMM that writes it is Mp = round_up(Mr, 32) wide
};
static ClipBufs clip_bufs(Fwd& f, int n, int L) {
  Ctx& c = f.c;
  const int D = 768;
  ClipBufs b;
  b.n = n, b.L = L, b.Lp = round_up(L, 8), b.Mr = n * b.Lp, b.Mp = round_up(b.Mr, 32);
  b.x = c.work.get<float>((size_t)b.Mr * D);
  b.l16 = f.half2((size_t)b.Mr * D, true), b.o16 = f.half2((size_t)b.Mr * D, true), b.h16 = f.half2((size_t)b.Mr * 4 * D, true);
  b.qk = c.work.get<__half>((size_t)b.Mr * 2 * D);
  b.vT = c.work.get<__half>((size_t)D * b.Mp);
  // pad rows (l >= L) never reach a real row (causal mask, row-wise ops) but must stay finite: 0 * NaN would poison P.V
  SDB_CUDA(cudaMemsetAsync(b.o16.hi, 0, (size_t)b.Mr * D * 2, c.stream));
  SDB_CUDA(cudaMemsetAsync(b.o16.lo, 0, (size_t)b.Mr * D * 2, c.stream));
  return b;
}

static void clip_layernorm(Ctx& c, const ClipBufs& b, const NormW& nw, Half2Ptr o, float* o32) {
  KernelScope ks(c, KC_LAYERNORM);
  layernorm_launch(b.x, b.Mr, 768, nw.gamma, nw.beta, nw.eps, o, o32, c.stream);
}

// device copies of one block's intermediate state (sdb_test_clip_block), taken in stream order before the next step rewrites the
// buffer: LN1 and LN2 (hi + lo), q | k, V^T, the attention output (hi + lo), x after the attention, QuickGELU(fc1) (hi + lo)
struct ClipTaps {
  Half2Ptr ln1, ln2, o, h;
  __half* qk = nullptr;
  __half* vT = nullptr;
  float* x_attn = nullptr;
};

// reference src/model/clip/mod.rs:109-115 (block), :158-180 (attention with the causal mask of src/backend.rs:130-139), :204-227
// (MLP with QuickGELU)
static void run_clip_block(Fwd& f, const ClipBlockW& cb, const ClipBufs& b, const ClipTaps* taps = nullptr) {
  Ctx& c = f.c;
  const int D = 768, heads = 12, Mr = b.Mr;
  auto copy = [&](void* dst, const void* src, size_t bytes) {
    SDB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, c.stream));
  };
  auto tap16 = [&](Half2Ptr dst, Half2Ptr src, size_t count) { copy(dst.hi, src.hi, count * 2), copy(dst.lo, src.lo, count * 2); };
  clip_layernorm(c, b, cb.attn_ln, b.l16, nullptr);
  if (taps) tap16(taps->ln1, b.l16, (size_t)Mr * D);
  {
    Epilogue ep;
    ep.out_f16.hi = b.qk, ep.bias = cb.bias_qk;
    run_gemm(c, G_LINEAR, f.rows_operand(b.l16, Mr, D), nullptr, cb.w_qk, 3, ep);
  }
  {
    WeightOp tok;
    tok.p = b.l16, tok.N = b.Mp, tok.rows = Mr, tok.K = D;
    Epilogue ep;
    ep.out_f16.hi = b.vT;
    run_gemm(c, G_LINEAR, f.rows_operand(cb.value.packed.p, D, D), nullptr, tok, 3, ep);
  }
  if (taps) copy(taps->qk, b.qk, (size_t)Mr * 2 * D * 2), copy(taps->vT, b.vT, (size_t)D * b.Mp * 2);
  {
    AttnOp at;
    at.q = b.qk, at.ldq = 2 * D, at.q_col0 = 0, at.q_rows = b.Lp;
    at.k = b.qk, at.ldk = 2 * D, at.k_col0 = D, at.k_rows = b.Lp;
    at.vT = b.vT, at.ldv = b.Mp;
    at.nb = b.n, at.heads = heads, at.d = 64, at.dpad = 64, at.Nq = b.L, at.Nk = b.L;
    at.causal = 1;
    at.out = b.o16, at.ldo = D;
    run_attention(c, at);
  }
  if (taps) tap16(taps->o, b.o16, (size_t)Mr * D);
  {
    Epilogue ep;
    ep.out_f32 = b.x, ep.residual = b.x, ep.bias = cb.bias_out;
    run_gemm(c, G_LINEAR, f.rows_operand(b.o16, Mr, D), nullptr, cb.out.packed, 3, ep);
  }
  if (taps) copy(taps->x_attn, b.x, (size_t)Mr * D * 4);
  clip_layernorm(c, b, cb.mlp_ln, b.l16, nullptr);
  if (taps) tap16(taps->ln2, b.l16, (size_t)Mr * D);
  {
    Epilogue ep;
    ep.out_f16 = b.h16, ep.bias = cb.fc1.bias, ep.act = 1;
    run_gemm(c, G_LINEAR, f.rows_operand(b.l16, Mr, D), nullptr, cb.fc1.packed, 3, ep);
  }
  if (taps) tap16(taps->h, b.h16, (size_t)Mr * 4 * D);
  {
    Epilogue ep;
    ep.out_f32 = b.x, ep.residual = b.x, ep.bias = cb.fc2.bias;
    run_gemm(c, G_LINEAR, f.rows_operand(b.h16, Mr, 4 * D), nullptr, cb.fc2.packed, 3, ep);
  }
}

// reference src/model/clip/mod.rs:56-75 (CLIP::forward). tokens [n][L] int32 -> out [n][L][768]. SURVEY §8f row f1.
void model_clip_forward_dev(Ctx& c, const int* d_tok, int n, int L, float* d_out, cudaStream_t caller) {
  Model& m = M(c);
  SDB_CHECK(n >= 1 && L >= 1 && L <= 77, "clip_forward: 1 <= L <= 77 (position table), n >= 1");
  StreamJoin join(c, caller);
  c.work.reset();
  Fwd f(c, n);
  const int D = 768;
  const ClipBufs b = clip_bufs(f, n, L);
  const int Lp = b.Lp;
  float* y = c.work.get<float>((size_t)b.Mr * D);
  {
    KernelScope ks(c, KC_ELEMENTWISE);
    embed_tokens_launch(d_tok, mptr(c, m.clip.tok_i), mptr(c, m.clip.pos_i), n, L, Lp, D, 49408, b.x, c.stream);
  }
  for (const ClipBlockW& cb : m.clip.blocks) run_clip_block(f, cb, b);
  clip_layernorm(c, b, m.clip.ln_final, Half2Ptr{}, y);
  SDB_CUDA(cudaMemcpy2DAsync(d_out, (size_t)L * D * 4, y, (size_t)Lp * D * 4, (size_t)L * D * 4, n, cudaMemcpyDeviceToDevice,
                             c.stream));
}

void model_clip_forward_host(Ctx& c, const int* tokens, int n, int L, float* out) {
  SDB_CHECK(n >= 1 && L >= 1 && L <= 77, "clip_forward: 1 <= L <= 77 (position table), n >= 1");
  // the reference's embedding lookup panics on an id outside the table; the host entry rejects it (the *_dev entry,
  // which cannot see the ids without a sync, clamps instead)
  for (long long i = 0; i < (long long)n * L; ++i)
    SDB_CHECK(tokens[i] >= 0 && tokens[i] < 49408, "clip_forward: token id outside the 49408-entry vocabulary");
  int* d_t = (int*)c.io(0, (size_t)n * L * 4);
  float* d_o = (float*)c.io(1, (size_t)n * L * 768 * 4);
  SDB_CUDA(cudaMemcpyAsync(d_t, tokens, (size_t)n * L * 4, cudaMemcpyHostToDevice, c.stream));
  model_clip_forward_dev(c, d_t, n, L, d_o, c.stream);
  SDB_CUDA(cudaMemcpyAsync(out, d_o, (size_t)n * L * 768 * 4, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

// ================================================================================ test-entry launch records and staging
void TraceScope::write() const {
  if (!out) return;
  static_assert(sizeof(TraceRecord) == 16 * sizeof(int32_t), "sdb200.h documents 16-int records");
  constexpr size_t kMax = (SDB_TRACE_INTS - 1) / 16;
  SDB_CHECK(c.trace.size() <= kMax, "launch trace: " + std::to_string(c.trace.size()) + " records do not fit SDB_TRACE_INTS (" +
                                        std::to_string(kMax) + " records)");
  std::fill(out, out + SDB_TRACE_INTS, 0);
  out[0] = (int)c.trace.size();
  std::memcpy(out + 1, c.trace.data(), c.trace.size() * sizeof(TraceRecord));
}

void fetch_pair(Ctx& c, Half2Ptr p, size_t count, float* out, bool planes) {
  std::vector<__half> hi(p.hi ? count : 0), lo(p.lo ? count : 0);
  if (p.hi) SDB_CUDA(cudaMemcpyAsync(hi.data(), p.hi, count * 2, cudaMemcpyDeviceToHost, c.stream));
  if (p.lo) SDB_CUDA(cudaMemcpyAsync(lo.data(), p.lo, count * 2, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  for (size_t i = 0; i < count; ++i) {
    const float h = p.hi ? __half2float(hi[i]) : 0.f, l = p.lo ? __half2float(lo[i]) : 0.f;
    if (planes)
      out[i] = h, out[count + i] = l;
    else
      out[i] = h + l;
  }
}

void fetch_half2(Ctx& c, Half2Ptr p, int n, int C, int H, int W, float* out) {
  const size_t hw = (size_t)H * W;
  std::vector<float> v((size_t)n * hw * C);
  fetch_pair(c, p, v.size(), v.data());
  for (int s = 0; s < n; ++s)
    for (size_t i = 0; i < hw; ++i)
      for (int ch = 0; ch < C; ++ch) out[((size_t)s * C + ch) * hw + i] = v[((size_t)s * hw + i) * C + ch];
}

// NCHW host output of an NHWC fp32 activation
static void fetch_act(Ctx& c, const Act& a, float* out) {
  float* d = c.work.get<float>(a.count());
  nhwc_to_nchw_launch(a.p, a.n, a.C, a.H, a.W, d, c.stream);
  SDB_CUDA(cudaMemcpyAsync(out, d, a.count() * 4, cudaMemcpyDeviceToHost, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

// ================================================================================ attention unit-test entry
// V transposed (flags & 2): stages q / k / V^T exactly as model_clip_forward_dev does
static void test_attention_vt(Ctx& c, const float* q, const float* k, const float* v, int n, int L, int C, int heads,
                              const int* lens, bool causal, float* out) {
  const int d = C / heads;
  SDB_CHECK(d % 16 == 0, "test_attention: V transposed needs a head dim that is a multiple of 16");
  const int Lp = round_up(L, 8), Mr = n * Lp, Mp = round_up(Mr, 32);
  // q | k in one [n*Lp][2C] matrix (single fp16 values), V^T [C][Mp] with sample s at columns s*Lp; pad rows / columns zero
  std::vector<__half> hqk((size_t)Mr * 2 * C, __float2half(0.f)), hvT((size_t)C * Mp, __float2half(0.f));
  for (int s = 0; s < n; ++s)
    for (int i = 0; i < L; ++i)
      for (int j = 0; j < C; ++j) {
        const size_t src = ((size_t)s * L + i) * C + j, row = (size_t)s * Lp + i;
        hqk[row * 2 * C + j] = __float2half(q[src]);
        hqk[row * 2 * C + C + j] = __float2half(k[src]);
        hvT[(size_t)j * Mp + row] = __float2half(v[src]);
      }
  const __half* dqk = upload(c, hqk.data(), hqk.size());
  Half2Ptr o16;
  o16.hi = c.work.get<__half>((size_t)Mr * C);
  o16.lo = c.work.get<__half>((size_t)Mr * C);
  AttnOp at;
  at.q = dqk, at.ldq = 2 * C, at.q_col0 = 0, at.q_rows = Lp;
  at.k = dqk, at.ldk = 2 * C, at.k_col0 = C, at.k_rows = Lp;
  at.vT = upload(c, hvT.data(), hvT.size()), at.ldv = Mp;
  at.nb = n, at.heads = heads, at.d = d, at.dpad = d, at.Nq = L, at.Nk = L;
  at.kvlen = upload(c, lens, n);
  at.causal = causal ? 1 : 0;
  at.out = o16, at.ldo = C;
  run_attention(c, at);
  std::vector<float> o((size_t)Mr * C);
  fetch_pair(c, o16, o.size(), o.data());
  for (int s = 0; s < n; ++s)
    for (int i = 0; i < L; ++i) std::copy_n(&o[((size_t)s * Lp + i) * C], C, out + ((size_t)s * L + i) * C);
}

void model_test_attention(Ctx& c, const float* q, const float* k, const float* v, int n, int Nq, int Nk, int C, int heads,
                          const int32_t* kvlen, int flags, float* out) {
  SDB_CHECK(n >= 1 && Nq >= 1 && Nk >= 1 && heads >= 1 && C % heads == 0, "test_attention: shapes");
  SDB_CHECK((flags & ~3) == 0, "test_attention: flags are 1 (causal) | 2 (V transposed)");
  // the kernel clamps a device-side length into [1, Nk] (it cannot report an error); this entry rejects it instead
  std::vector<int> lens(n, Nk);
  if (kvlen)
    for (int s = 0; s < n; ++s) {
      SDB_CHECK(kvlen[s] >= 1 && kvlen[s] <= Nk, "test_attention: every kvlen must be in [1, Nk]");
      lens[s] = kvlen[s];
    }
  if (flags & 2) {
    SDB_CHECK(Nq == Nk, "test_attention: V transposed stages q and k in one matrix (CLIP layout): Nq must equal Nk");
    return test_attention_vt(c, q, k, v, n, Nk, C, heads, kvlen ? lens.data() : nullptr, flags & 1, out);
  }
  // stages q / k|v exactly as the SpatialTransformer does: head-padded rows, V row-major beside K (consumed MN-major)
  const int d = C / heads, dpad = (d % 16 == 0) ? d : (d + 15) / 16 * 16, hd = heads * dpad;
  const int Nkp = round_up(Nk, 8);
  std::vector<__half> hq((size_t)n * Nq * hd, __float2half(0.f)), hkv((size_t)n * Nkp * 2 * hd, __float2half(0.f));
  std::vector<__half> hq_lo(hq.size(), __float2half(0.f)), hkv_lo(hkv.size(), __float2half(0.f));
  auto split = [](float v, __half& hi, __half& lo) {
    hi = __float2half(v);
    lo = __float2half(v - __half2float(hi));
  };
  for (int s = 0; s < n; ++s)
    for (int i = 0; i < Nq; ++i)
      for (int h = 0; h < heads; ++h)
        for (int j = 0; j < d; ++j)
          split(q[((size_t)s * Nq + i) * C + h * d + j], hq[((size_t)s * Nq + i) * hd + h * dpad + j], hq_lo[((size_t)s * Nq + i) * hd + h * dpad + j]);
  for (int s = 0; s < n; ++s)
    for (int i = 0; i < Nk; ++i)
      for (int h = 0; h < heads; ++h)
        for (int j = 0; j < d; ++j) {
          split(k[((size_t)s * Nk + i) * C + h * d + j], hkv[((size_t)s * Nkp + i) * 2 * hd + h * dpad + j], hkv_lo[((size_t)s * Nkp + i) * 2 * hd + h * dpad + j]);
          hkv[((size_t)s * Nkp + i) * 2 * hd + hd + h * dpad + j] = __float2half(v[((size_t)s * Nk + i) * C + h * d + j]);
        }
  const __half* dkv = upload(c, hkv.data(), hkv.size());
  Half2Ptr o16;
  o16.hi = c.work.get<__half>((size_t)n * Nq * C);
  o16.lo = c.work.get<__half>((size_t)n * Nq * C);
  AttnOp at;
  at.q = upload(c, hq.data(), hq.size()), at.ldq = hd, at.q_rows = Nq;
  at.k = dkv, at.ldk = 2 * hd, at.k_rows = Nkp;
  at.vT = dkv, at.ldv = 2 * hd, at.v_mn = 1, at.v_col0 = hd;
  // used by the head dims that have the split-product kernel (40, 80) unless attn_split = 0
  at.q_lo = upload(c, hq_lo.data(), hq_lo.size()), at.k_lo = upload(c, hkv_lo.data(), hkv_lo.size());
  at.nb = n, at.heads = heads, at.d = d, at.dpad = dpad, at.Nq = Nq, at.Nk = Nkp;
  at.kvlen = upload(c, lens.data(), n);  // always set: the key matrix is padded to Nkp rows per sample
  at.causal = flags & 1;
  at.out = o16, at.ldo = C;
  run_attention(c, at);
  fetch_pair(c, o16, (size_t)n * Nq * C, out);
}

// ================================================================================ GEMM, conv and LayerNorm-fold test entries
void model_test_gemm_ex(Ctx& c, const float* a, const float* w, const float* bias, const float* residual, int M, int K, int N,
                        int passes, int flags, const float* xa, const float* xw, int XK, float* out, int32_t* trace) {
  TraceScope ts(c, trace);
  const bool geglu = flags & 1, from_f16 = flags & 4, planes = flags & 8;
  SDB_CHECK(!planes || from_f16, "gemm_ex test: the separate fp16 planes (flag 8) need the fp16 outputs (flag 4)");
  SDB_CHECK(!geglu || (N % 128 == 0 && !residual && !xa), "GEGLU test: N (= 2 * hidden) must be a multiple of 128, no residual / extra K");
  const int Nout = geglu ? N / 2 : N;
  float* d_a = upload(c, a, (size_t)M * K);
  float* d_w = upload(c, w, (size_t)K * N);
  float* d_b = upload(c, bias, N);
  float* d_r = upload(c, residual, (size_t)M * N);
  float* d_c = c.work.get<float>((size_t)M * Nout);
  ActOp A;
  A.p = alloc_half2(c.work, (size_t)M * K);
  A.W = M, A.C = K;
  convert_f16_launch(d_a, (long long)M * K, A.p, c.stream);
  WeightOp Wp;
  Wp.p = alloc_half2(c.work, (size_t)N * K);
  Wp.N = N, Wp.K = K;
  float* d_bp = d_b;
  if (geglu) {
    SDB_CHECK(bias, "GEGLU test needs a bias");
    d_bp = c.work.get<float>(N);
    pack_geglu_launch(d_w, d_b, K, N / 2, 64, Wp.p, d_bp, c.stream);
  } else {
    pack_linear_launch(d_w, K, N, Wp.p, 0, c.stream);
  }
  ExtraK xk;
  if (xa) {
    SDB_CHECK(xw && XK % 64 == 0, "extra-K test operands");
    float* d_xa = upload(c, xa, (size_t)M * XK);
    float* d_xw = upload(c, xw, (size_t)XK * N);
    xk.x0.p = alloc_half2(c.work, (size_t)M * XK);
    xk.x0.W = M, xk.x0.C = XK;
    convert_f16_launch(d_xa, (long long)M * XK, xk.x0.p, c.stream);
    xk.w.p = alloc_half2(c.work, (size_t)N * XK);
    xk.w.N = N, xk.w.K = XK;
    pack_linear_launch(d_xw, XK, N, xk.w.p, 0, c.stream);
  }
  Epilogue ep;
  Half2Ptr o16;
  if (geglu || from_f16) o16 = alloc_half2(c.work, (size_t)M * Nout);
  ep.out_f32 = geglu ? nullptr : d_c;
  ep.out_f16 = o16;
  ep.bias = d_bp, ep.residual = d_r, ep.geglu = geglu ? 1 : 0;
  run_gemm(c, G_LINEAR, A, nullptr, Wp, passes, ep, xa ? &xk : nullptr);
  if (geglu || from_f16) {
    fetch_pair(c, o16, (size_t)M * Nout, out, planes);
  } else {
    SDB_CUDA(cudaMemcpyAsync(out, d_c, sizeof(float) * M * Nout, cudaMemcpyDeviceToHost, c.stream));
    SDB_CUDA(cudaStreamSynchronize(c.stream));
  }
  ts.write();
}

// A test conv's OIHW weights (device) packed into the work arena by the model's packer; only the implicit-GEMM layouts
static ConvW test_conv_weights(Ctx& c, const float* w, float* b, int cin, int cout, int k, bool up2 = false) {
  SDB_CHECK(cin % 64 == 0 && cout % 32 == 0, "test conv: channels must be multiples of 64 (in) and 32 (out)");
  ConvW cw;
  cw.cin = cin, cw.cout = cout, cw.k = k;
  pack_conv_weight(c, cw, w, c.work, up2);
  cw.bias = b;
  return cw;
}

// A conv on a host NCHW tensor the way the model runs its GEMM convs: the input staged by Fwd::raw_operand, the weights by
// pack_conv_weight, the output an activation from Fwd::act. 1x1 (G_CONV1), 3x3 pad 1 (G_CONV3), 3x3 stride 2 on the four phase
// planes (G_CONV3_S2, the UNet downsample), 3x3 after a nearest-2x upsample folded into the weights (G_CONV3_UP2). gn: the epilogue
// also writes the output's GroupNorm partials into the buffer Fwd::act gave it (none with the gn_epilogue option off)
static Act test_conv(Fwd& f, const float* x, const float* w, const float* bias, int cin, int H, int W, int cout, int k, int stride,
                     int upsample, int passes, bool gn) {
  Ctx& c = f.c;
  SDB_CHECK(k == 1 || k == 3, "ksize");
  SDB_CHECK((stride == 1 && (upsample == 0 || (upsample == 1 && k == 3))) || (stride == 2 && k == 3 && !upsample),
            "stride / upsample");
  Act xh;
  xh.n = f.nb, xh.H = H, xh.W = W, xh.C = cin;
  xh.p = c.work.get<float>(xh.count());
  nchw_to_nhwc_launch(upload(c, x, xh.count()), f.nb, cin, H, W, xh.p, c.stream);
  const ActOp a = f.raw_operand(xh, nullptr, stride == 2, true);
  const ConvW cw = test_conv_weights(c, upload(c, w, (size_t)cout * cin * k * k), upload(c, bias, cout), cin, cout, k, upsample);
  const int kind = k == 1 ? G_CONV1 : stride == 2 ? G_CONV3_S2 : upsample ? G_CONV3_UP2 : G_CONV3;
  Act o = f.act(upsample ? 2 * H : H / stride, upsample ? 2 * W : W / stride, cout);
  Epilogue ep;
  ep.out_f32 = o.p, ep.bias = cw.bias;
  if (gn) ep.gn = &o.gn;
  run_gemm(c, kind, a, nullptr, cw.packed, passes, ep);
  return o;
}

void model_test_conv2d(Ctx& c, const float* x, const float* w, const float* bias, int n, int cin, int H, int W, int cout, int k,
                       int stride, int upsample, int passes, float* y, int32_t* trace) {
  Fwd f(c, n);
  TraceScope ts(c, trace);
  fetch_act(c, test_conv(f, x, w, bias, cin, H, W, cout, k, stride, upsample, passes, false), y);
  ts.write();
}

void model_test_conv_groupnorm(Ctx& c, const float* x, const float* w, const float* bias, const float* gamma, const float* beta,
                               int n, int cin, int H, int W, int cout, int k, int stride, int upsample, int passes, int silu,
                               float* y, int* slots, int32_t* trace) {
  Fwd f(c, n);
  TraceScope ts(c, trace);
  const Act o = test_conv(f, x, w, bias, cin, H, W, cout, k, stride, upsample, passes, true);
  if (slots) *slots = o.gn.slots;
  SDB_CHECK(o.gn.slots > 0, "the GEMM did not produce GroupNorm statistics for this shape");
  Half2Ptr o16 = alloc_half2(c.work, o.count());
  GnSrc s0, s1;
  s0.x = o.p, s0.C = cout, s0.part = o.gn.buf, s0.cap = o.gn.cap, s0.slots = o.gn.slots;
  gn_apply_launch(s0, s1, o.gn.bucket, n, o.H, o.W, silu, upload(c, gamma, cout), upload(c, beta, cout), 1e-5f, o16, c.stream);
  fetch_half2(c, o16, n, cout, o.H, o.W, y);
  ts.write();
}

void model_test_ln_fold(Ctx& c, const float* a, const float* a2, const float* w0, const float* b0, const float* gamma,
                        const float* beta, const float* w1, const float* b1, int M, int K0, int C, int N, int passes, int geglu,
                        float* out, int32_t* trace) {
  TraceScope ts(c, trace);
  SDB_CHECK(C % 160 == 0 && K0 % 64 == 0 && (!geglu || (N % 128 == 0 && b1)), "ln_fold test shapes");
  float *d_w0 = upload(c, w0, (size_t)K0 * C), *d_b0 = upload(c, b0, C), *d_w1 = upload(c, w1, (size_t)C * N),
        *d_b1 = upload(c, b1, N);
  NormW ln;
  ln.c = C, ln.gamma = upload(c, gamma, C), ln.beta = upload(c, beta, C);
  WeightOp W0;
  W0.p = alloc_half2(c.work, (size_t)C * K0), W0.N = C, W0.K = K0;
  pack_linear_launch(d_w0, K0, C, W0.p, 0, c.stream);
  // the consumer's weights with the LayerNorm folded in, as pack_st folds it
  WeightOp W1;
  W1.p = alloc_half2(c.work, (size_t)N * C), W1.N = N, W1.K = C;
  float* bp = geglu ? c.work.get<float>(N) : nullptr;
  float *u_hi, *u_full, *v;
  ln_fold(c, c.work, alloc_half2(c.work, (size_t)N * C), W1, u_hi, u_full, v, [&](Half2Ptr dst, const float* sc) {
    if (geglu)
      pack_geglu_launch(d_w1, d_b1, C, N / 2, 64, dst, dst.hi == W1.p.hi ? bp : nullptr, c.stream, sc);
    else
      pack_linear_launch(d_w1, C, N, dst, 0, c.stream, 0, 0, sc);
  }, ln);
  if (geglu) add_vec_launch(v, bp, N, v, c.stream);
  else if (d_b1) add_vec_launch(v, d_b1, N, v, c.stream);
  // producer(s): y = a w0 + b0 (+ a2 w0 + b0 accumulated in place onto the fp16 pair), leaving row statistics
  Half2Ptr y16 = alloc_half2(c.work, (size_t)M * C);
  const int ls = ln_slots(C);
  float* st = c.work.get<float>((size_t)M * ls * 2);
  for (int pass = 0; pass < (a2 ? 2 : 1); ++pass) {
    float* d_a = upload(c, pass ? a2 : a, (size_t)M * K0);
    ActOp A;
    A.p = alloc_half2(c.work, (size_t)M * K0), A.W = M, A.C = K0;
    convert_f16_launch(d_a, (long long)M * K0, A.p, c.stream);
    Epilogue ep;
    ep.out_f16 = y16, ep.bias = d_b0, ep.ln_out = st;
    if (pass) ep.residual16 = y16;
    run_gemm(c, G_LINEAR, A, nullptr, W0, 3, ep);
  }
  const int Nout = geglu ? N / 2 : N;
  Half2Ptr o16 = alloc_half2(c.work, (size_t)M * Nout);
  {
    ActOp Y;
    Y.p = y16, Y.W = M, Y.C = C;
    Epilogue ep;
    ep.out_f16 = o16, ep.geglu = geglu ? 1 : 0;
    ep.ln_in = st, ep.ln_in_slots = ls, ep.ln_C = C, ep.ln_eps = 1e-5f, ep.ln_u_hi = u_hi, ep.ln_u_full = u_full, ep.bias = v;
    run_gemm(c, G_LINEAR, Y, nullptr, W1, passes, ep);
  }
  fetch_pair(c, o16, (size_t)M * Nout, out);
  ts.write();
}

// ================================================================================ ResBlock / GroupNorm unit-test entries
// An NCHW host tensor staged as a model activation. stats = true: written by a 3-pass identity 3x3 conv with the epilogue a
// ResBlock output gets (fp32, fp16 hi/lo copy, GroupNorm partials); the 3-pass product returns hi + lo of the input (22 bits,
// exact in fp32). stats = false: the fp32 tensor and its fp16 copy without statistics, as the UNet's conv_in leaves it.
static Act stage_activation(Fwd& f, const float* h, int C, int H, int W, bool stats) {
  Ctx& c = f.c;
  Act a = f.act16(H, W, C);
  float* d = upload(c, h, a.count());
  if (!stats) {
    nchw_to_nhwc_launch(d, f.nb, C, H, W, a.p, c.stream);
    if (a.raw16.hi) convert_f16_launch(a.p, (long long)a.count(), a.raw16, c.stream);
    return a;
  }
  float* xh = c.work.get<float>(a.count());
  nchw_to_nhwc_launch(d, f.nb, C, H, W, xh, c.stream);
  ActOp A;
  A.n = f.nb, A.H = H, A.W = W, A.C = C;
  A.p = f.half2(a.count(), true);
  convert_f16_launch(xh, (long long)a.count(), A.p, c.stream);
  // identity weights [C][C][3][3]: a one at the centre tap of (i, i)
  float* id = c.work.get<float>((size_t)C * C * 9);
  SDB_CUDA(cudaMemsetAsync(id, 0, (size_t)C * C * 9 * 4, c.stream));
  const std::vector<float> ones(C, 1.f);
  SDB_CUDA(cudaMemcpy2DAsync(id + 4, (size_t)(C + 1) * 9 * 4, ones.data(), 4, 4, C, cudaMemcpyHostToDevice, c.stream));
  const ConvW wid = test_conv_weights(c, id, nullptr, C, C, 3);
  Epilogue ep;
  ep.out_f32 = a.p, ep.out_f16 = a.raw16, ep.gn = &a.gn;
  // 3 passes whatever the precision option forces on the block under test: the staging must hand on hi + lo of the input
  const int prec = c.opt_precision;
  c.opt_precision = 0;
  try {
    run_gemm(c, G_CONV3, A, nullptr, wid.packed, 3, ep);
  } catch (...) {
    c.opt_precision = prec;
    throw;
  }
  c.opt_precision = prec;
  return a;
}


void model_test_resblock(Ctx& c, const float* x0, const float* x1, int n, int C0, int C1, int H, int W, int Cout,
                         const float* n1g, const float* n1b, const float* w1, const float* b1, const float* n2g, const float* n2b,
                         const float* w2, const float* b2, const float* wsk, const float* bsk, const float* emb_bias, int passes,
                         int flags, float* out, float* out16, float* outn, int32_t* trace) {
  SDB_CHECK(n >= 1 && H >= 1 && W >= 1 && C0 > 0 && C1 >= 0 && (C1 > 0) == (x1 != nullptr), "test_resblock: shapes");
  SDB_CHECK(b1 && b2 && (!wsk || bsk) && (wsk || (!x1 && C0 == Cout)), "test_resblock: biases / skip (a block without one adds x0)");
  SDB_CHECK((flags & ~3) == 0, "test_resblock: flags are 1 (x0 with producer statistics) | 2 (x1 with producer statistics)");
  const int Cin = C0 + C1;
  Fwd f(c, n);
  f.init_sums(4);
  NormW nw1, nw2;
  nw1.c = Cin, nw1.gamma = upload(c, n1g, Cin), nw1.beta = upload(c, n1b, Cin);
  nw2.c = Cout, nw2.gamma = upload(c, n2g, Cout), nw2.beta = upload(c, n2b, Cout);
  const ConvW cw1 = test_conv_weights(c, upload(c, w1, (size_t)Cout * Cin * 9), upload(c, b1, Cout), Cin, Cout, 3);
  const ConvW cw2 = test_conv_weights(c, upload(c, w2, (size_t)Cout * Cout * 9), upload(c, b2, Cout), Cout, Cout, 3);
  ConvW sk;
  float* bias_merged = nullptr;
  if (wsk) {  // packed as pack_resblock / pack_resnet do
    sk = test_conv_weights(c, upload(c, wsk, (size_t)Cout * Cin), upload(c, bsk, Cout), Cin, Cout, 1);
    bias_merged = c.work.get<float>(Cout);
    add_vec_launch(cw2.bias, sk.bias, Cout, bias_merged, c.stream);
  }
  const float* d_emb = upload(c, emb_bias, Cout);
  const Act a0 = stage_activation(f, x0, C0, H, W, flags & 1);
  Act a1;
  if (x1) a1 = stage_activation(f, x1, C1, H, W, flags & 2);
  Act o = f.act16(H, W, Cout);
  ActOp g;
  {
    TraceScope ts(c, trace);
    run_resblock(f, nw1, cw1, nw2, cw2, wsk ? &sk : nullptr, bias_merged, passes, a0, x1 ? &a1 : nullptr, d_emb, o);
    g = f.gn_operand(o, nullptr, nw2, true, true);  // a consumer of the output: reads the partials conv_out left
    ts.write();
  }
  float* d = c.work.get<float>(o.count());
  nhwc_to_nchw_launch(o.p, n, Cout, H, W, d, c.stream);
  SDB_CUDA(cudaMemcpyAsync(out, d, o.count() * 4, cudaMemcpyDeviceToHost, c.stream));
  fetch_half2(c, o.raw16, n, Cout, H, W, out16);
  fetch_half2(c, g.p, n, Cout, H, W, outn);
}

void model_test_groupnorm_cat(Ctx& c, const float* x0, const float* x1, int n, int C0, int C1, int H, int W, const float* gamma,
                              const float* beta, int silu, int mode, float* y, int32_t* trace) {
  SDB_CHECK(n >= 1 && H >= 1 && W >= 1 && C0 > 0 && C1 >= 0 && (C1 > 0) == (x1 != nullptr), "test_groupnorm_cat: shapes");
  SDB_CHECK(mode == 1 || mode == 2, "test_groupnorm_cat: mode is 1 (fused statistics + apply) or 2 (apply from producer partials)");
  const int C = C0 + C1;
  Fwd f(c, n);
  f.init_sums(1);
  NormW nw;
  nw.c = C, nw.gamma = upload(c, gamma, C), nw.beta = upload(c, beta, C);
  const Act a0 = stage_activation(f, x0, C0, H, W, mode == 2);
  Act a1;
  if (x1) a1 = stage_activation(f, x1, C1, H, W, mode == 2);
  TraceScope ts(c, trace);
  const ActOp g = f.gn_operand(a0, x1 ? &a1 : nullptr, nw, silu != 0, true);
  ts.write();
  fetch_half2(c, g.p, n, C, H, W, y);
}

// ================================================================================ SpatialTransformer unit-test entry
void model_test_spatial_transformer(Ctx& c, int index, const float* x, int n, int Cx, int H, int W, const float* context, int Lmax,
                                    const int32_t* lens, int flags, float* out, float* out16, float* out_norm, float* taps_y,
                                    float* taps_ln, int32_t* trace) {
  Model& m = M(c);
  SDB_CHECK(index >= 0 && index < (int)m.sts.size(), "test_spatial_transformer: index is the execution-order position 0..15");
  SDB_CHECK(n >= 1 && H >= 1 && W >= 1 && Lmax >= 1 && x && context && lens, "test_spatial_transformer: arguments");
  SDB_CHECK((H * W) % 8 == 0, "unsupported latent size: H*W must be a multiple of 8");  // the UNet's (H/8)*(W/8) rule
  SDB_CHECK((flags & ~1) == 0, "test_spatial_transformer: flags are 1 (the output carries an fp16 hi + lo copy)");
  for (int s = 0; s < n; ++s) SDB_CHECK(lens[s] >= 1 && lens[s] <= Lmax, "test_spatial_transformer: lengths must lie in [1, Lmax]");
  SpatialTransformerW& st = *m.sts[index];
  SDB_CHECK(Cx == st.c, "test_spatial_transformer: x must have the block's channel count (" + std::to_string(st.c) + ")");
  const int C = st.c, HW = H * W, ls = ln_slots(C);
  const long long Mt = (long long)n * HW;
  Fwd f(c, n);
  f.init_sums(4);
  // context [n][Lpad][768], zero padded, per-sample lengths: as model_unet_forward_dev / the sampling entries stage it
  const int Lpad = round_up(Lmax, 32);
  float* ctxp = c.work.get<float>((size_t)n * Lpad * 768);
  SDB_CUDA(cudaMemsetAsync(ctxp, 0, (size_t)n * Lpad * 768 * 4, c.stream));
  SDB_CUDA(cudaMemcpy2DAsync(ctxp, (size_t)Lpad * 768 * 4, context, (size_t)Lmax * 768 * 4, (size_t)Lmax * 768 * 4, n,
                             cudaMemcpyHostToDevice, c.stream));
  int* d_len = upload(c, lens, n);
  CtxState cs;
  prepare_context(f, ctxp, Lpad, d_len, cs);
  const Act a = stage_activation(f, x, C, H, W, true);
  Act o = (flags & 1) ? f.act16(H, W, C) : f.act(H, W, C);
  StTaps taps;
  for (Half2Ptr& y : taps.y) y = f.half2((size_t)Mt * C, true);
  for (float*& l : taps.ln) l = c.work.get<float>((size_t)Mt * ls * 2);
  ActOp g;
  {
    TraceScope ts(c, trace);
    run_spatial_transformer(f, st, cs, cs.kv[index], a, o, &taps);
    g = f.gn_operand(o, nullptr, st.norm, true, true);  // a consumer of the output, as the next ResBlock's norm_in stages it
    ts.write();
  }
  float* d = c.work.get<float>(o.count());
  nhwc_to_nchw_launch(o.p, n, C, H, W, d, c.stream);
  SDB_CUDA(cudaMemcpyAsync(out, d, o.count() * 4, cudaMemcpyDeviceToHost, c.stream));
  fetch_half2(c, o.raw16, n, C, H, W, out16);
  fetch_half2(c, g.p, n, C, H, W, out_norm);
  // taps: y as [Mt][C] hi + lo, the statistics folded over their slots in index order (as the consuming epilogue adds them)
  for (int i = 0; i < 4; ++i) fetch_pair(c, taps.y[i], (size_t)Mt * C, taps_y + i * Mt * C);
  std::vector<float> sl((size_t)Mt * ls * 2);
  for (int i = 0; i < 3; ++i) {
    SDB_CUDA(cudaMemcpyAsync(sl.data(), taps.ln[i], sl.size() * 4, cudaMemcpyDeviceToHost, c.stream));
    SDB_CUDA(cudaStreamSynchronize(c.stream));
    for (long long r = 0; r < Mt; ++r) {
      float sm = 0.f, sq = 0.f;
      for (int k = 0; k < ls; ++k) sm += sl[(r * ls + k) * 2], sq += sl[(r * ls + k) * 2 + 1];
      taps_ln[(i * Mt + r) * 2] = sm, taps_ln[(i * Mt + r) * 2 + 1] = sq;
    }
  }
}

// ================================================================================ autoencoder stage test entry

void model_test_vae_stage(Ctx& c, int stage, const float* x, const float* cond, int n, int Cx, int H, int W, float scale, int flags,
                          float* out, float* out16, float* tap, float* out_norm, int32_t* trace) {
  Model& m = M(c);
  EncoderW& e = m.enc;
  SDB_CHECK(stage >= SDB_VAE_DEC_IN && stage <= SDB_VAE_ENC_DOWN2, "test_vae_stage: stage is one of SDB_VAE_*");
  SDB_CHECK(n >= 1 && H >= 1 && W >= 1 && x && out, "test_vae_stage: arguments");
  SDB_CHECK((flags & ~3) == 0 && (!(flags & 2) || stage == SDB_VAE_ENC_OUT),
            "test_vae_stage: flags are 1 (x with producer GroupNorm partials) | 2 (SDB_VAE_ENC_OUT: strided, scaled quant slice)");
  const bool attn = stage == SDB_VAE_DEC_ATTN || stage == SDB_VAE_ENC_ATTN;
  const bool down = stage >= SDB_VAE_ENC_DOWN0;
  const int di = stage - SDB_VAE_ENC_DOWN0;
  int cin = 4, cout = 0;
  switch (stage) {
    case SDB_VAE_DEC_IN: cout = 512; break;
    case SDB_VAE_DEC_ATTN: case SDB_VAE_ENC_ATTN: cin = cout = 512; break;
    case SDB_VAE_DEC_OUT: cin = 128, cout = 3; break;
    case SDB_VAE_UNET_OUT: cin = 320, cout = 4; break;
    case SDB_VAE_ENC_OUT: cin = 512, cout = 8; break;
    case SDB_VAE_ENC_IN: cout = 128; break;
    case SDB_VAE_UNET_IN: cout = 320; break;
    default: cin = cout = e.blocks[di].down.cout; break;
  }
  SDB_CHECK(Cx == cin, "test_vae_stage: x must have " + std::to_string(cin) + " channels for this stage");
  if (attn) check_vae_latent(H, W, "test_vae_stage");
  if (down) SDB_CHECK(H % 2 == 0 && W % 2 == 0, "test_vae_stage: the downsampler needs even H and W");
  const bool cond_ctx = stage == SDB_VAE_UNET_IN && c.unet_cin != 4;
  SDB_CHECK(cond_ctx == (cond != nullptr), "test_vae_stage: cond [n][cin-4][H][W] is given exactly for SDB_VAE_UNET_IN on a 9- or "
                                           "8-channel context");
  SDB_CHECK(!cond_ctx || c.unet_cin != 9 || n % 2 == 0, "test_vae_stage: a 9-channel conv_in runs on the two CFG halves: n even");
  SDB_CHECK(stage != SDB_VAE_ENC_OUT || tap, "test_vae_stage: SDB_VAE_ENC_OUT needs tap for the quant slice");
  const int HW = H * W;
  Fwd f(c, n);
  f.init_sums(4);
  float* d_x = (cin == 4) ? upload(c, x, (size_t)n * 4 * HW) : nullptr;
  const float* d_cond = cond_ctx ? upload(c, cond, (size_t)n * (c.unet_cin - 4) * HW) : nullptr;
  Act a;
  if (cin != 4) a = stage_activation(f, x, cin, H, W, flags & 1);
  // the UNet's conv_in output carries the fp16 copy the first ResBlock's skip reads
  Act o = stage == SDB_VAE_UNET_IN ? f.act16(H, W, cout) : f.act(down ? H / 2 : H, down ? W / 2 : W, cout);
  Half2Ptr otap;
  float* y = nullptr;   // NCHW outputs of the small-Cout conv and the quant slice
  float* q = nullptr;
  const size_t qcount = (size_t)n * ((flags & 2) ? 5 : 4) * HW;
  ActOp g;
  {
    TraceScope ts(c, trace);
    switch (stage) {
      case SDB_VAE_DEC_IN:
        vae_dec_conv_in(f, d_x, scale, o);
        break;
      case SDB_VAE_DEC_ATTN:
      case SDB_VAE_ENC_ATTN: {
        otap = f.half2((size_t)n * HW * 512, true);
        const bool dec = stage == SDB_VAE_DEC_ATTN;
        run_vae_attention(f, dec ? m.mid_attn : e.mid_attn, a, o, &otap);
        g = f.gn_operand(o, nullptr, dec ? m.mid_block2.norm1 : e.mid_block2.norm1, true, true);  // the next ResnetBlock's norm1
        break;
      }
      case SDB_VAE_DEC_OUT:
      case SDB_VAE_UNET_OUT:
      case SDB_VAE_ENC_OUT:
        y = c.work.get<float>((size_t)n * cout * HW);
        if (stage == SDB_VAE_DEC_OUT) norm_conv_out(f, a, m.vae_norm_out, m.vae_conv_out, 3, y);
        if (stage == SDB_VAE_UNET_OUT) norm_conv_out(f, a, m.norm_out, m.conv_out, 4, y);
        if (stage == SDB_VAE_ENC_OUT) {
          norm_conv_out(f, a, e.norm_out, e.conv_out, 8, y);
          // strided + scaled: as encode_images writes the masked-image latent into channels 1-4 of the inpainting tensor [n,5,H,W]
          q = upload(c, tap, qcount);
          if (flags & 2)
            vae_enc_quant(f, y, HW, q + HW, 5ll * HW, scale);
          else
            vae_enc_quant(f, y, HW, q, 0, 1.f);
        }
        break;
      case SDB_VAE_ENC_IN:
        vae_enc_conv_in(f, d_x, o);
        break;
      case SDB_VAE_UNET_IN: {
        UNetIO io{d_x, nullptr, nullptr, H, W};
        unet_cond_io(c, n, d_x, d_cond, io);
        unet_conv_in(f, m.in_blocks[0], io, o);
        break;
      }
      default:
        vae_enc_down(f, e.blocks[di].down, a, o);
        g = f.gn_operand(o, nullptr, e.blocks[di + 1].res[0].norm1, true, true);  // the next block's first ResnetBlock
        break;
    }
    ts.write();
  }
  if (y) {
    SDB_CUDA(cudaMemcpyAsync(out, y, (size_t)n * cout * HW * 4, cudaMemcpyDeviceToHost, c.stream));
    if (q) SDB_CUDA(cudaMemcpyAsync(tap, q, qcount * 4, cudaMemcpyDeviceToHost, c.stream));
    SDB_CUDA(cudaStreamSynchronize(c.stream));
    return;
  }
  fetch_act(c, o, out);
  if (out16) fetch_half2(c, o.raw16, n, cout, o.H, o.W, out16);
  if (tap && attn) fetch_half2(c, otap, n, 512, H, W, tap);
  if (out_norm && g.p.hi) fetch_half2(c, g.p, n, cout, o.H, o.W, out_norm);
}

// ================================================================================ CLIP block test entry
void model_test_clip_block(Ctx& c, int index, const float* x, int n, int L, int flags, float* out, float* taps, int32_t* trace) {
  Model& m = M(c);
  const int nblk = (int)m.clip.blocks.size();
  SDB_CHECK(index >= 0 && index <= nblk, "test_clip_block: index is a block 0..11, or 12 for the final LayerNorm");
  SDB_CHECK(n >= 1 && L >= 1 && L <= 77 && x && out, "test_clip_block: arguments (1 <= L <= 77)");
  SDB_CHECK((flags & ~1) == 0, "test_clip_block: flags are 1 (pad rows hold large finite junk instead of zeros)");
  const int D = 768;
  Fwd f(c, n);
  const ClipBufs b = clip_bufs(f, n, L);
  const int Lp = b.Lp, Mr = b.Mr;
  // x [n][L][768] staged at the row pitch Lp, as embed_tokens_launch leaves the embedding: pad rows zero, or junk that must never
  // reach a real row
  std::vector<float> hx((size_t)Mr * D, 0.f);
  for (int s = 0; s < n; ++s)
    for (int l = 0; l < Lp; ++l)
      for (int j = 0; j < D; ++j) {
        const size_t r = (size_t)s * Lp + l;
        if (l < L)
          hx[r * D + j] = x[((size_t)s * L + l) * D + j];
        else if (flags & 1)
          hx[r * D + j] = 2.0e4f * (float)((r * 7919 + (size_t)j * 104729) % 2001) / 1000.f - 2.0e4f;
      }
  SDB_CUDA(cudaMemcpyAsync(b.x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice, c.stream));
  ClipTaps tp;
  if (taps && index < nblk) {
    tp.ln1 = f.half2((size_t)Mr * D, true), tp.ln2 = f.half2((size_t)Mr * D, true), tp.o = f.half2((size_t)Mr * D, true);
    tp.h = f.half2((size_t)Mr * 4 * D, true);
    tp.qk = c.work.get<__half>((size_t)Mr * 2 * D);
    tp.vT = c.work.get<__half>((size_t)D * b.Mp);
    tp.x_attn = c.work.get<float>((size_t)Mr * D);
  }
  float* y = index < nblk ? b.x : c.work.get<float>((size_t)Mr * D);
  {
    TraceScope ts(c, trace);
    if (index < nblk)
      run_clip_block(f, m.clip.blocks[index], b, tp.qk ? &tp : nullptr);
    else
      clip_layernorm(c, b, m.clip.ln_final, Half2Ptr{}, y);
    ts.write();
  }
  // real rows only, [n][L][width]
  auto real_rows = [&](const std::vector<float>& src, int width, int col0, int pitch, float* dst) {
    for (int s = 0; s < n; ++s)
      for (int l = 0; l < L; ++l)
        std::copy(&src[((size_t)s * Lp + l) * pitch + col0], &src[((size_t)s * Lp + l) * pitch + col0] + width,
                  dst + ((size_t)s * L + l) * width);
  };
  auto fetch32 = [&](const float* d, size_t count) {
    std::vector<float> h(count);
    SDB_CUDA(cudaMemcpyAsync(h.data(), d, count * 4, cudaMemcpyDeviceToHost, c.stream));
    SDB_CUDA(cudaStreamSynchronize(c.stream));
    return h;
  };
  auto fetch16 = [&](Half2Ptr p, size_t count) {
    std::vector<float> v(count);
    fetch_pair(c, p, count, v.data());
    return v;
  };
  real_rows(fetch32(y, (size_t)Mr * D), D, 0, D, out);
  if (!tp.qk) return;
  const size_t tc = (size_t)n * L * D;  // one [n][L][768] tap
  real_rows(fetch16(tp.ln1, (size_t)Mr * D), D, 0, D, taps);
  const std::vector<float> qk = fetch16({tp.qk, nullptr}, (size_t)Mr * 2 * D);
  real_rows(qk, D, 0, 2 * D, taps + tc);
  real_rows(qk, D, D, 2 * D, taps + 2 * tc);
  const std::vector<float> vT = fetch16({tp.vT, nullptr}, (size_t)D * b.Mp);
  for (int s = 0; s < n; ++s)
    for (int l = 0; l < L; ++l)
      for (int j = 0; j < D; ++j) taps[3 * tc + ((size_t)s * L + l) * D + j] = vT[(size_t)j * b.Mp + (size_t)s * Lp + l];
  real_rows(fetch16(tp.o, (size_t)Mr * D), D, 0, D, taps + 4 * tc);
  real_rows(fetch32(tp.x_attn, (size_t)Mr * D), D, 0, D, taps + 5 * tc);
  real_rows(fetch16(tp.ln2, (size_t)Mr * D), D, 0, D, taps + 6 * tc);
  real_rows(fetch16(tp.h, (size_t)Mr * 4 * D), 4 * D, 0, 4 * D, taps + 7 * tc);
}

}  // namespace sdb
