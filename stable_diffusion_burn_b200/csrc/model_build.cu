// model_build.cu — tensor registry (reference dump-dir names), arenas, synthetic weights, weight packing.
#include <cmath>
#include <cstdlib>

#include "model.cuh"
#include "model_def.cuh"

namespace sdb {


// ------------------------------------------------------------------ registry builder
struct Builder {
  Ctx& c;
  size_t off = 0;
  int add(const std::string& name, std::initializer_list<int64_t> dims, int kind, int fan_in) {
    TensorInfo t;
    t.name = name;
    t.ndim = (int)dims.size();
    int i = 0;
    t.count = 1;
    for (auto d : dims) t.dims[i++] = d, t.count *= d;
    t.kind = kind, t.fan_in = fan_in;
    off = (off + 63) & ~size_t(63);  // 256-byte aligned tensors
    t.offset = off;
    off += t.count;
    c.index[name] = (int)c.tensors.size();
    c.tensors.push_back(t);
    return (int)c.tensors.size() - 1;
  }
  void scalar(const std::string& rel, float v) { c.meta.push_back(MetaCheck{rel, {v}, false}); }
  void pair(const std::string& rel, float a, float b) { c.meta.push_back(MetaCheck{rel, {a, b}, false}); }
  // the files save_conv2d writes beside weight/bias (python/save.py:52-68, read by load_conv2d load.rs:118-160)
  void conv(ConvW& w, const std::string& name, int cin, int cout, int k, int stride = 1) {
    w.cin = cin, w.cout = cout, w.k = k;
    pair(name + "/stride", (float)stride, (float)stride), pair(name + "/padding", (float)(k / 2), (float)(k / 2));
    pair(name + "/dilation", 1.f, 1.f), pair(name + "/kernel_size", (float)k, (float)k);
    scalar(name + "/n_group", 1.f), scalar(name + "/n_channels_in", (float)cin), scalar(name + "/n_channels_out", (float)cout);
    w.wi = add(name + "/weight", {cout, cin, k, k}, K_CONV_W, cin * k * k);
    w.bi = add(name + "/bias", {cout}, K_CONV_B, cin * k * k);
  }
  // PaddedConv2d(0,1,0,1) stride 2 (save_padded_conv2d python/save.py:70-97): the Conv2d lives in <name>/conv and is saved
  // with padding (0,0); channels / kernel_size / stride / padding sit beside it
  void padded_conv_s2(ConvW& w, const std::string& name, int ch) {
    w.cin = ch, w.cout = ch, w.k = 3;
    const std::string cn = name + "/conv";
    pair(cn + "/stride", 2.f, 2.f), pair(cn + "/padding", 0.f, 0.f), pair(cn + "/dilation", 1.f, 1.f);
    pair(cn + "/kernel_size", 3.f, 3.f);
    scalar(cn + "/n_group", 1.f), scalar(cn + "/n_channels_in", (float)ch), scalar(cn + "/n_channels_out", (float)ch);
    pair(name + "/channels", (float)ch, (float)ch);
    scalar(name + "/kernel_size", 3.f), scalar(name + "/stride", 2.f);
    c.meta.push_back(MetaCheck{name + "/padding", {0.f, 1.f, 0.f, 1.f}, false});
    w.wi = add(cn + "/weight", {ch, ch, 3, 3}, K_CONV_W, ch * 9);
    w.bi = add(cn + "/bias", {ch}, K_CONV_B, ch * 9);
  }
  void lin(LinW& w, const std::string& name, int in, int out, bool bias = true) {
    w.in = in, w.out = out;
    w.wi = add(name + "/weight", {in, out}, K_LIN_W, in);
    if (bias) w.bi = add(name + "/bias", {out}, K_LIN_B, in);
    else c.meta.push_back(MetaCheck{name + "/bias", {}, true});
  }
  // group = true: GroupNorm(32) (save_group_norm save.py:30-38); false: LayerNorm (save_layer_norm :24-28)
  void norm(NormW& w, const std::string& name, int ch, bool group = true) {
    w.c = ch;
    if (group) c.group_norms.insert(name), scalar(name + "/n_group", 32.f), scalar(name + "/n_channel", (float)ch);
    w.gi = add(name + "/weight", {ch}, K_NORM_G, ch);
    w.bi = add(name + "/bias", {ch}, K_NORM_B, ch);
  }
  void resblock(ResBlockW& r, const std::string& name, int cin, int cout) {  // unet/mod.rs:662-697
    r.cin = cin, r.cout = cout;
    norm(r.norm_in, name + "/norm_in", cin);
    conv(r.conv_in, name + "/conv_in", cin, cout, 3);
    lin(r.lin_embed, name + "/lin_embed", 1280, cout);
    norm(r.norm_out, name + "/norm_out", cout);
    conv(r.conv_out, name + "/conv_out", cout, cout, 3);
    r.has_skip = cin != cout;
    if (r.has_skip) conv(r.skip, name + "/skip_connection", cin, cout, 1);
  }
  void mha(AttnW& a, const std::string& name, int ch, int cctx) {  // unet/mod.rs:601-630
    scalar(name + "/n_head", 8.f);  // unet/load.rs:46
    lin(a.query, name + "/query", ch, ch, false);
    lin(a.key, name + "/key", cctx, ch, false);
    lin(a.value, name + "/value", cctx, ch, false);
    lin(a.out, name + "/out", ch, ch);
  }
  void st(SpatialTransformerW& s, const std::string& name, int ch) {  // unet/mod.rs:436-451, 490-508
    s.c = ch, s.heads = 8, s.d = ch / 8;
    s.dpad = (s.d % 16 == 0) ? s.d : ((s.d + 15) / 16) * 16;
    norm(s.norm, name + "/norm", ch);
    conv(s.proj_in, name + "/proj_in", ch, ch, 1);
    const std::string t = name + "/transformer";
    norm(s.ln1, t + "/norm1", ch, false);
    mha(s.attn1, t + "/attn1", ch, ch);
    norm(s.ln2, t + "/norm2", ch, false);
    mha(s.attn2, t + "/attn2", ch, 768);
    norm(s.ln3, t + "/norm3", ch, false);
    lin(s.geglu, t + "/mlp/geglu/proj", ch, 8 * ch);
    lin(s.ff, t + "/mlp/lin", 4 * ch, ch);
    conv(s.proj_out, name + "/proj_out", ch, ch, 1);
  }
  void resnet(ResnetW& r, const std::string& name, int cin, int cout) {  // autoencoder/mod.rs:471-503
    r.cin = cin, r.cout = cout;
    norm(r.norm1, name + "/norm1", cin);
    conv(r.conv1, name + "/conv1", cin, cout, 3);
    norm(r.norm2, name + "/norm2", cout);
    conv(r.conv2, name + "/conv2", cout, cout, 3);
    r.has_nin = cin != cout;
    if (r.has_nin) conv(r.nin, name + "/nin_shortcut", cin, cout, 1);
  }
};

struct BlockSpec {
  const char* field;
  int kind, cin, cout;
};
// unet/mod.rs:41-73 in as_array() order (:161-193)
static const BlockSpec kInBlocks[12] = {
    {"conv", BK_CONV, 4, 320},   {"rt1", BK_RT, 320, 320},    {"rt2", BK_RT, 320, 320},   {"d1", BK_DOWN, 320, 320},
    {"rt3", BK_RT, 320, 640},    {"rt4", BK_RT, 640, 640},    {"d2", BK_DOWN, 640, 640},  {"rt5", BK_RT, 640, 1280},
    {"rt6", BK_RT, 1280, 1280},  {"d3", BK_DOWN, 1280, 1280}, {"r1", BK_R, 1280, 1280},   {"r2", BK_R, 1280, 1280}};
static const BlockSpec kOutBlocks[12] = {
    {"r1", BK_R, 2560, 1280},    {"r2", BK_R, 2560, 1280},    {"ru", BK_RU, 2560, 1280},   {"rt1", BK_RT, 2560, 1280},
    {"rt2", BK_RT, 2560, 1280},  {"rtu1", BK_RTU, 1920, 1280}, {"rt3", BK_RT, 1920, 640},  {"rt4", BK_RT, 1280, 640},
    {"rtu2", BK_RTU, 960, 640},  {"rt5", BK_RT, 960, 320},    {"rt6", BK_RT, 640, 320},    {"rt7", BK_RT, 640, 320}};

static void build_block(Builder& b, UNetBlockW& blk, const std::string& name, const BlockSpec& s) {
  blk.kind = s.kind, blk.cin = s.cin, blk.cout = s.cout;
  switch (s.kind) {
    case BK_CONV:
    case BK_DOWN:
      b.conv(blk.conv, name, s.cin, s.cout, 3, s.kind == BK_DOWN ? 2 : 1);
      break;
    case BK_R:
      b.resblock(blk.res, name, s.cin, s.cout);
      break;
    case BK_RT:
      b.resblock(blk.res, name + "/res", s.cin, s.cout);
      b.st(blk.st, name + "/transformer", s.cout);
      break;
    case BK_RU:
      b.resblock(blk.res, name + "/res", s.cin, s.cout);
      b.conv(blk.conv, name + "/upsample/conv", s.cout, s.cout, 3);
      break;
    case BK_RTU:
      b.resblock(blk.res, name + "/res", s.cin, s.cout);
      b.st(blk.st, name + "/transformer", s.cout);
      b.conv(blk.conv, name + "/upsample/conv", s.cout, s.cout, 3);
      break;
  }
}

static size_t env_gb(const char* name, double dflt) {
  const char* v = getenv(name);
  const double gb = v ? atof(v) : dflt;
  return (size_t)(gb * 1024.0 * 1024.0 * 1024.0);
}

void model_create(Ctx& c) {
  auto* m = new Model();
  c.model = m;
  Builder b{c};
  // ---- UNet (unet/mod.rs:35-93)
  b.lin(m->lin1_time, "unet/lin1_time_embed", 320, 1280);
  b.lin(m->lin2_time, "unet/lin2_time_embed", 1280, 1280);
  m->in_blocks.resize(12);
  m->out_blocks.resize(12);
  int level = 0;
  for (int i = 0; i < 12; ++i) {
    BlockSpec s = kInBlocks[i];
    // 9 for an inpainting UNet (sdb_create_inpaint): latent | mask | masked-image latent; 8 for InstructPix2Pix
    // (sdb_create_pix2pix): latent | image latent
    if (i == 0) s.cin = c.unet_cin;
    build_block(b, m->in_blocks[i], std::string("unet/input_blocks/") + s.field, s);
    m->in_blocks[i].level = level;
    if (i == 0) c.tensors[m->in_blocks[0].conv.bi].fan_in = 4 * 9;  // only the weight of a wider conv_in differs
    if (kInBlocks[i].kind == BK_DOWN) level++;  // following blocks run one level lower (the down conv itself reads level-1 input)
  }
  b.resblock(m->mid_res1, "unet/middle_block/res1", 1280, 1280);
  b.st(m->mid_st, "unet/middle_block/transformer", 1280);
  b.resblock(m->mid_res2, "unet/middle_block/res2", 1280, 1280);
  for (int i = 0; i < 12; ++i) {
    build_block(b, m->out_blocks[i], std::string("unet/output_blocks/") + kOutBlocks[i].field, kOutBlocks[i]);
    m->out_blocks[i].level = level;
    if (kOutBlocks[i].kind == BK_RU || kOutBlocks[i].kind == BK_RTU) level--;
  }
  b.norm(m->norm_out, "unet/norm_out", 320);
  b.conv(m->conv_out, "unet/conv_out", 320, 4, 3);
  // ---- VAE decoder (autoencoder/mod.rs:29-45, 153-192)
  b.conv(m->post_quant, "autoencoder/post_quant_conv", 4, 4, 1);
  const std::string d = "autoencoder/decoder";
  b.conv(m->vae_conv_in, d + "/conv_in", 4, 512, 3);
  b.resnet(m->mid_block1, d + "/mid/block_1", 512, 512);
  b.norm(m->mid_attn.norm, d + "/mid/attn/norm", 512);
  b.conv(m->mid_attn.q, d + "/mid/attn/q", 512, 512, 1);
  b.conv(m->mid_attn.k, d + "/mid/attn/k", 512, 512, 1);
  b.conv(m->mid_attn.v, d + "/mid/attn/v", 512, 512, 1);
  b.conv(m->mid_attn.proj_out, d + "/mid/attn/proj_out", 512, 512, 1);
  b.resnet(m->mid_block2, d + "/mid/block_2", 512, 512);
  static const int dec_ch[4][2] = {{512, 512}, {512, 512}, {512, 256}, {256, 128}};
  for (int i = 0; i < 4; ++i) {
    const std::string bn = d + "/blocks/" + std::to_string(i);
    b.resnet(m->dec[i].res[0], bn + "/res1", dec_ch[i][0], dec_ch[i][1]);
    b.resnet(m->dec[i].res[1], bn + "/res2", dec_ch[i][1], dec_ch[i][1]);
    b.resnet(m->dec[i].res[2], bn + "/res3", dec_ch[i][1], dec_ch[i][1]);
    m->dec[i].has_up = i != 3;
    if (m->dec[i].has_up) b.conv(m->dec[i].up, bn + "/upsampler", dec_ch[i][1], dec_ch[i][1], 3);
  }
  b.scalar(d + "/n_block", 4.f);  // autoencoder/load.rs:139
  b.norm(m->vae_norm_out, d + "/norm_out", 128);
  b.conv(m->vae_conv_out, d + "/conv_out", 128, 3, 3);
  // ---- CLIP text encoder (SURVEY §8f row f1; clip/mod.rs:25-44, CLIPConfig::new(49408,768,12,77,12))
  m->clip.tok_i = b.add("clip/token_embedding/weight", {49408, 768}, K_EMB, 768);
  m->clip.pos_i = b.add("clip/position_embedding/weight", {77, 768}, K_EMB, 768);
  m->clip.blocks.resize(12);
  for (int i = 0; i < 12; ++i) {
    ClipBlockW& cb = m->clip.blocks[i];
    const std::string bn = "clip/blocks/" + std::to_string(i);
    b.norm(cb.attn_ln, bn + "/attn_ln", 768, false);
    b.scalar(bn + "/attn/n_head", 12.f);  // clip/load.rs:32
    b.lin(cb.query, bn + "/attn/query", 768, 768);
    b.lin(cb.key, bn + "/attn/key", 768, 768);
    b.lin(cb.value, bn + "/attn/value", 768, 768);
    b.lin(cb.out, bn + "/attn/out", 768, 768);
    b.norm(cb.mlp_ln, bn + "/mlp_ln", 768, false);
    b.lin(cb.fc1, bn + "/mlp/fc1", 768, 3072);
    b.lin(cb.fc2, bn + "/mlp/fc2", 3072, 768);
  }
  b.norm(m->clip.ln_final, "clip/layer_norm", 768, false);
  b.scalar("clip/n_layer", 12.f);  // clip/load.rs:73
  // ---- VAE encoder + quant_conv (SURVEY §8f row f4; autoencoder/mod.rs:31, 122-145, 249-266)
  {
    EncoderW& e = m->enc;
    const std::string en = "autoencoder/encoder";
    b.conv(e.conv_in, en + "/conv_in", 3, 128, 3);
    static const int enc_ch[4][2] = {{128, 128}, {128, 256}, {256, 512}, {512, 512}};
    for (int i = 0; i < 4; ++i) {
      const std::string bn = en + "/blocks/" + std::to_string(i);
      b.resnet(e.blocks[i].res[0], bn + "/res1", enc_ch[i][0], enc_ch[i][1]);
      b.resnet(e.blocks[i].res[1], bn + "/res2", enc_ch[i][1], enc_ch[i][1]);
      e.blocks[i].has_down = i != 3;
      if (e.blocks[i].has_down) b.padded_conv_s2(e.blocks[i].down, bn + "/downsampler", enc_ch[i][1]);
    }
    b.resnet(e.mid_block1, en + "/mid/block_1", 512, 512);
    b.norm(e.mid_attn.norm, en + "/mid/attn/norm", 512);
    b.conv(e.mid_attn.q, en + "/mid/attn/q", 512, 512, 1);
    b.conv(e.mid_attn.k, en + "/mid/attn/k", 512, 512, 1);
    b.conv(e.mid_attn.v, en + "/mid/attn/v", 512, 512, 1);
    b.conv(e.mid_attn.proj_out, en + "/mid/attn/proj_out", 512, 512, 1);
    b.resnet(e.mid_block2, en + "/mid/block_2", 512, 512);
    b.scalar(en + "/n_block", 4.f);  // autoencoder/load.rs:163
    b.norm(e.norm_out, en + "/norm_out", 512);
    b.conv(e.conv_out, en + "/conv_out", 512, 8, 3);
    b.conv(e.quant, "autoencoder/quant_conv", 8, 8, 1);
  }
  // ---- sampler schedule (stablediffusion/mod.rs:44)
  m->alphas_i = b.add("alpha_cumulative_products", {1000}, K_SCHED, 1);

  // execution-order lists
  for (auto& blk : m->in_blocks)
    if (blk.kind >= BK_R) m->resblocks.push_back(&blk.res);
  m->resblocks.push_back(&m->mid_res1);
  m->resblocks.push_back(&m->mid_res2);
  for (auto& blk : m->out_blocks)
    if (blk.kind >= BK_R) m->resblocks.push_back(&blk.res);
  for (auto& blk : m->in_blocks)
    if (blk.kind == BK_RT || blk.kind == BK_RTU) m->sts.push_back(&blk.st);
  m->sts.push_back(&m->mid_st);
  for (auto& blk : m->out_blocks)
    if (blk.kind == BK_RT || blk.kind == BK_RTU) m->sts.push_back(&blk.st);

  c.master.init((b.off + 64) * sizeof(float));
  c.master.off = b.off * sizeof(float);
  c.packed.init(env_gb("SDB_PACKED_GB", 6.5));
  c.work.init(env_gb("SDB_WORK_GB", 24.0));
  SDB_CUDA(cudaMalloc(&c.splitk_tickets, 65536 * sizeof(unsigned int)));
  SDB_CUDA(cudaMemsetAsync(c.splitk_tickets, 0, 65536 * sizeof(unsigned int), c.stream));
  SDB_CUDA(cudaMemsetAsync(c.master.base, 0, c.master.cap, c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

void check_conv_in_shape(const Ctx& c, const std::string& what, int ndim, const int64_t* dims) {
  if (ndim != 4 || dims[1] == c.unet_cin) return;  // other mismatches get the generic shape message
  const char* use = dims[1] == 9   ? "a 9-channel inpainting UNet loads into a context from sdb_create_inpaint"
                    : dims[1] == 8 ? "an 8-channel InstructPix2Pix UNet loads into a context from sdb_create_pix2pix"
                                   : "a 4-channel UNet loads into a context from sdb_create";
  char msg[400];
  snprintf(msg, sizeof(msg),
           "%s: unet/input_blocks/conv/weight is [%lld,%lld,%lld,%lld] but this context's conv_in is [320,%d,3,3]; %s",
           what.c_str(), (long long)dims[0], (long long)dims[1], (long long)dims[2], (long long)dims[3], c.unet_cin, use);
  throw Error(msg);
}

void model_destroy(Ctx& c) {
  auto* m = reinterpret_cast<Model*>(c.model);
  if (!m) return;
  model_invalidate_graphs(c);
  if (c.splitk_tickets) cudaFree(c.splitk_tickets), c.splitk_tickets = nullptr;
  delete m;
  c.model = nullptr;
}

// ------------------------------------------------------------------ synthetic weights (== synth.py)
static uint32_t fnv1a32(const std::string& s) {
  uint32_t h = 0x811C9DC5u;
  for (unsigned char ch : s) {
    h ^= ch;
    h *= 0x01000193u;
  }
  return h;
}
static uint32_t mix32_host(uint32_t x) {
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

void model_init_synthetic(Ctx& c, uint32_t seed) {
  auto* m = reinterpret_cast<Model*>(c.model);
  float* base = reinterpret_cast<float*>(c.master.base);
  std::vector<SynthDesc> table;
  long long nchunks = 0;
  for (const TensorInfo& t : c.tensors) {
    if (t.kind == K_SCHED) continue;
    float bound = 0.f, offset = 0.f;
    switch (t.kind) {
      case K_CONV_W:
      case K_LIN_W:
        bound = (float)(std::sqrt(3.0) / std::sqrt((double)t.fan_in));
        break;
      case K_CONV_B:
      case K_LIN_B:
        bound = (float)(1.0 / std::sqrt((double)t.fan_in));
        break;
      case K_NORM_G:
        bound = 0.1f, offset = 1.0f;
        break;
      case K_NORM_B:
        bound = 0.1f;
        break;
      case K_EMB:
        bound = (float)std::sqrt(3.0);
        break;
    }
    const uint32_t key = mix32_host(fnv1a32(t.name) + seed);
    table.push_back(SynthDesc{(long long)t.offset, (long long)t.count, nchunks, key, bound, offset});
    nchunks += (t.count + 65535) / 65536;
  }
  {  // one launch for the whole registry; the descriptor table is staged through the work arena
    c.work.reset();
    SynthDesc* d_table = c.work.get<SynthDesc>(table.size());
    SDB_CUDA(cudaMemcpyAsync(d_table, table.data(), table.size() * sizeof(SynthDesc), cudaMemcpyHostToDevice, c.stream));
    synth_fill_table_launch(base, d_table, (int)table.size(), nchunks, c.stream);
  }
  // SD-v1 scaled-linear schedule (synth.alpha_cumulative_products)
  std::vector<float> a(1000);
  const double b0 = std::sqrt(0.00085), b1 = std::sqrt(0.012);
  double prod = 1.0;
  for (int i = 0; i < 1000; ++i) {
    // numpy.linspace: start + i*step with step = (stop-start)/(num-1)
    const double s = (i == 999) ? b1 : b0 + (double)i * ((b1 - b0) / 999.0);
    prod *= 1.0 - s * s;
    a[i] = (float)prod;
  }
  SDB_CUDA(cudaMemcpyAsync(base + c.tensors[m->alphas_i].offset, a.data(), 1000 * sizeof(float), cudaMemcpyHostToDevice,
                           c.stream));
  SDB_CUDA(cudaStreamSynchronize(c.stream));
}

}  // namespace sdb
