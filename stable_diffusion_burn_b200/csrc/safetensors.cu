// safetensors.cu — SD-1.x single-file .safetensors checkpoints (the original LDM layout) read straight into the master arena
// (DESIGN §7 f13). Header and key map are validated on the host before any byte of the arena is written; the tensor bytes then
// stream through two pinned host buffers into device staging, and one kernel launch per chunk widens F16 / BF16 to fp32 and
// re-lays each Linear weight from the file's [out][in] to the registry's [in][out].
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstring>
#include <map>

#include "model.cuh"
#include "model_def.cuh"

namespace sdb {

// ------------------------------------------------------------------------------------------------------------ the key map
// The LDM module tree (model.diffusion_model / first_stage_model / cond_stage_model.transformer.text_model) against the
// registry, as the reference's converter applies it: load_state_dict into python/dump.py's StableDiffusion (the LDM names),
// then the savers of python/unet.py, autoencoder.py and clip.py (the registry names; save.py:17-21 writes Linear weights
// transposed). tests/golden/ldm_keymap.json.gz holds the same map derived from the reference itself.
struct MapEntry {
  std::string key;  // LDM key
  std::string reg;  // registry name
  int ndim = 0;
  int64_t dims[4] = {1, 1, 1, 1};  // registry shape (the file holds a transposed Linear weight as [out][in])
  bool transpose = false;
};

namespace {

struct MapBuilder {
  std::vector<MapEntry> e;
  void t(const std::string& k, const std::string& r, std::initializer_list<int64_t> d, bool tr = false) {
    MapEntry m;
    m.key = k, m.reg = r, m.ndim = (int)d.size(), m.transpose = tr;
    int i = 0;
    for (int64_t v : d) m.dims[i++] = v;
    e.push_back(m);
  }
  void conv(const std::string& k, const std::string& r, int64_t cin, int64_t cout, int64_t ks) {
    t(k + ".weight", r + "/weight", {cout, cin, ks, ks}), t(k + ".bias", r + "/bias", {cout});
  }
  void lin(const std::string& k, const std::string& r, int64_t in, int64_t out, bool bias = true) {
    t(k + ".weight", r + "/weight", {in, out}, true);
    if (bias) t(k + ".bias", r + "/bias", {out});
  }
  void norm(const std::string& k, const std::string& r, int64_t ch) {
    t(k + ".weight", r + "/weight", {ch}), t(k + ".bias", r + "/bias", {ch});
  }
  // ResBlock (dump.py: in_layers [GroupNorm, silu, Conv2d], emb_layers [silu, Linear], out_layers [GroupNorm, silu, id, Conv2d])
  void resblock(const std::string& k, const std::string& r, int64_t cin, int64_t cout) {
    norm(k + ".in_layers.0", r + "/norm_in", cin);
    conv(k + ".in_layers.2", r + "/conv_in", cin, cout, 3);
    lin(k + ".emb_layers.1", r + "/lin_embed", 1280, cout);
    norm(k + ".out_layers.0", r + "/norm_out", cout);
    conv(k + ".out_layers.3", r + "/conv_out", cout, cout, 3);
    if (cin != cout) conv(k + ".skip_connection", r + "/skip_connection", cin, cout, 1);
  }
  void attn(const std::string& k, const std::string& r, int64_t ch, int64_t cctx) {
    lin(k + ".to_q", r + "/query", ch, ch, false);
    lin(k + ".to_k", r + "/key", cctx, ch, false);
    lin(k + ".to_v", r + "/value", cctx, ch, false);
    lin(k + ".to_out.0", r + "/out", ch, ch);
  }
  void st(const std::string& k, const std::string& r, int64_t ch) {
    norm(k + ".norm", r + "/norm", ch);
    conv(k + ".proj_in", r + "/proj_in", ch, ch, 1);
    const std::string b = k + ".transformer_blocks.0", rt = r + "/transformer";
    norm(b + ".norm1", rt + "/norm1", ch);
    attn(b + ".attn1", rt + "/attn1", ch, ch);
    norm(b + ".norm2", rt + "/norm2", ch);
    attn(b + ".attn2", rt + "/attn2", ch, 768);
    norm(b + ".norm3", rt + "/norm3", ch);
    lin(b + ".ff.net.0.proj", rt + "/mlp/geglu/proj", ch, 8 * ch);
    lin(b + ".ff.net.2", rt + "/mlp/lin", 4 * ch, ch);
    conv(k + ".proj_out", r + "/proj_out", ch, ch, 1);
  }
  void resnet(const std::string& k, const std::string& r, int64_t cin, int64_t cout) {
    norm(k + ".norm1", r + "/norm1", cin);
    conv(k + ".conv1", r + "/conv1", cin, cout, 3);
    norm(k + ".norm2", r + "/norm2", cout);
    conv(k + ".conv2", r + "/conv2", cout, cout, 3);
    if (cin != cout) conv(k + ".nin_shortcut", r + "/nin_shortcut", cin, cout, 1);
  }
  void mid(const std::string& k, const std::string& r) {
    resnet(k + ".block_1", r + "/block_1", 512, 512);
    norm(k + ".attn_1.norm", r + "/attn/norm", 512);
    for (const char* p : {"q", "k", "v", "proj_out"}) conv(k + ".attn_1." + p, r + "/attn/" + p, 512, 512, 1);
    resnet(k + ".block_2", r + "/block_2", 512, 512);
  }
};

// UNet blocks in LDM order (dump.py UNetModel.input_blocks / output_blocks): registry field, kind, channels
struct UBlock {
  const char* field;
  int kind, cin, cout;
};
const UBlock kIn[12] = {{"conv", BK_CONV, 4, 320},   {"rt1", BK_RT, 320, 320},   {"rt2", BK_RT, 320, 320},
                        {"d1", BK_DOWN, 320, 320},   {"rt3", BK_RT, 320, 640},   {"rt4", BK_RT, 640, 640},
                        {"d2", BK_DOWN, 640, 640},   {"rt5", BK_RT, 640, 1280},  {"rt6", BK_RT, 1280, 1280},
                        {"d3", BK_DOWN, 1280, 1280}, {"r1", BK_R, 1280, 1280},   {"r2", BK_R, 1280, 1280}};
const UBlock kOut[12] = {{"r1", BK_R, 2560, 1280},    {"r2", BK_R, 2560, 1280},   {"ru", BK_RU, 2560, 1280},
                         {"rt1", BK_RT, 2560, 1280},  {"rt2", BK_RT, 2560, 1280}, {"rtu1", BK_RTU, 1920, 1280},
                         {"rt3", BK_RT, 1920, 640},   {"rt4", BK_RT, 1280, 640},  {"rtu2", BK_RTU, 960, 640},
                         {"rt5", BK_RT, 960, 320},    {"rt6", BK_RT, 640, 320},   {"rt7", BK_RT, 640, 320}};

void unet_map(MapBuilder& b, int conv_in_width) {
  const std::string K = "model.diffusion_model.", R = "unet/";
  b.lin(K + "time_embed.0", R + "lin1_time_embed", 320, 1280);
  b.lin(K + "time_embed.2", R + "lin2_time_embed", 1280, 1280);
  for (int i = 0; i < 12; ++i) {
    const UBlock& s = kIn[i];
    const std::string k = K + "input_blocks." + std::to_string(i), r = R + "input_blocks/" + s.field;
    if (s.kind == BK_CONV) b.conv(k + ".0", r, conv_in_width, s.cout, 3);
    if (s.kind == BK_DOWN) b.conv(k + ".0.op", r, s.cin, s.cout, 3);  // Downsample.op
    if (s.kind == BK_R) b.resblock(k + ".0", r, s.cin, s.cout);
    if (s.kind == BK_RT) b.resblock(k + ".0", r + "/res", s.cin, s.cout), b.st(k + ".1", r + "/transformer", s.cout);
  }
  b.resblock(K + "middle_block.0", R + "middle_block/res1", 1280, 1280);
  b.st(K + "middle_block.1", R + "middle_block/transformer", 1280);
  b.resblock(K + "middle_block.2", R + "middle_block/res2", 1280, 1280);
  for (int i = 0; i < 12; ++i) {
    const UBlock& s = kOut[i];
    const std::string k = K + "output_blocks." + std::to_string(i), r = R + "output_blocks/" + s.field;
    if (s.kind == BK_R) {
      b.resblock(k + ".0", r, s.cin, s.cout);
      continue;
    }
    b.resblock(k + ".0", r + "/res", s.cin, s.cout);
    if (s.kind == BK_RT || s.kind == BK_RTU) b.st(k + ".1", r + "/transformer", s.cout);
    // Upsample.conv: the block's second (RU) or third (RTU) module
    if (s.kind == BK_RU) b.conv(k + ".1.conv", r + "/upsample/conv", s.cout, s.cout, 3);
    if (s.kind == BK_RTU) b.conv(k + ".2.conv", r + "/upsample/conv", s.cout, s.cout, 3);
  }
  b.norm(K + "out.0", R + "norm_out", 320);
  b.conv(K + "out.2", R + "conv_out", 320, 4, 3);
}

// prefix: "first_stage_model." in a full checkpoint, "" in a standalone VAE file
void vae_map(MapBuilder& b, const std::string& K) {
  const std::string R = "autoencoder/";
  b.conv(K + "post_quant_conv", R + "post_quant_conv", 4, 4, 1);
  b.conv(K + "quant_conv", R + "quant_conv", 8, 8, 1);
  // decoder: Decoder.up[i] runs in reverse (dump.py: `for l in self.up[::-1]`), so up.3 is the registry's blocks/0
  const std::string d = K + "decoder", rd = R + "decoder";
  b.conv(d + ".conv_in", rd + "/conv_in", 4, 512, 3);
  b.mid(d + ".mid", rd + "/mid");
  static const int64_t dec[4][2] = {{512, 512}, {512, 512}, {512, 256}, {256, 128}};
  for (int i = 0; i < 4; ++i) {
    const std::string k = d + ".up." + std::to_string(3 - i), r = rd + "/blocks/" + std::to_string(i);
    b.resnet(k + ".block.0", r + "/res1", dec[i][0], dec[i][1]);
    b.resnet(k + ".block.1", r + "/res2", dec[i][1], dec[i][1]);
    b.resnet(k + ".block.2", r + "/res3", dec[i][1], dec[i][1]);
    if (i != 3) b.conv(k + ".upsample.conv", r + "/upsampler", dec[i][1], dec[i][1], 3);
  }
  b.norm(d + ".norm_out", rd + "/norm_out", 128);
  b.conv(d + ".conv_out", rd + "/conv_out", 128, 3, 3);
  const std::string e = K + "encoder", re = R + "encoder";
  b.conv(e + ".conv_in", re + "/conv_in", 3, 128, 3);
  static const int64_t enc[4][2] = {{128, 128}, {128, 256}, {256, 512}, {512, 512}};
  for (int i = 0; i < 4; ++i) {
    const std::string k = e + ".down." + std::to_string(i), r = re + "/blocks/" + std::to_string(i);
    b.resnet(k + ".block.0", r + "/res1", enc[i][0], enc[i][1]);
    b.resnet(k + ".block.1", r + "/res2", enc[i][1], enc[i][1]);
    if (i != 3) b.conv(k + ".downsample.conv", r + "/downsampler/conv", enc[i][1], enc[i][1], 3);
  }
  b.mid(e + ".mid", re + "/mid");
  b.norm(e + ".norm_out", re + "/norm_out", 512);
  b.conv(e + ".conv_out", re + "/conv_out", 512, 8, 3);
}

void clip_map(MapBuilder& b) {
  const std::string K = "cond_stage_model.transformer.text_model.", R = "clip/";
  b.t(K + "embeddings.token_embedding.weight", R + "token_embedding/weight", {49408, 768});
  b.t(K + "embeddings.position_embedding.weight", R + "position_embedding/weight", {77, 768});
  for (int i = 0; i < 12; ++i) {
    const std::string k = K + "encoder.layers." + std::to_string(i), r = R + "blocks/" + std::to_string(i);
    b.norm(k + ".layer_norm1", r + "/attn_ln", 768);
    b.lin(k + ".self_attn.q_proj", r + "/attn/query", 768, 768);
    b.lin(k + ".self_attn.k_proj", r + "/attn/key", 768, 768);
    b.lin(k + ".self_attn.v_proj", r + "/attn/value", 768, 768);
    b.lin(k + ".self_attn.out_proj", r + "/attn/out", 768, 768);
    b.norm(k + ".layer_norm2", r + "/mlp_ln", 768);
    b.lin(k + ".mlp.fc1", r + "/mlp/fc1", 768, 3072);
    b.lin(k + ".mlp.fc2", r + "/mlp/fc2", 3072, 768);
  }
  b.norm(K + "final_layer_norm", R + "layer_norm", 768);
}

bool starts(const std::string& s, const char* p) { return s.compare(0, strlen(p), p) == 0; }

std::string shape_str(int ndim, const int64_t* d) {
  std::string s = "[";
  for (int i = 0; i < ndim; ++i) s += (i ? "," : "") + std::to_string(d[i]);
  return s + "]";
}

// ------------------------------------------------------------------------------------------------------- header parser
// The safetensors subset of JSON: one flat object whose members are {"dtype": string, "shape": [uint...], "data_offsets":
// [uint, uint]} in any order, plus an optional "__metadata__" object of string values. Everything else is an error: the
// header comes from outside the program.
enum : int { DT_F32 = 0, DT_F16 = 1, DT_BF16 = 2, DT_OTHER = 3 };

struct HeaderEntry {
  std::string key, dtype;
  int ndim = 0;
  int64_t dims[8] = {0};
  uint64_t begin = 0, end = 0;
  uint64_t count = 1;  // elements
};

struct Parser {
  const std::string& s;
  const std::string& what;
  size_t i = 0;
  [[noreturn]] void fail(const std::string& m) const {
    throw Error(what + ": malformed safetensors header at byte " + std::to_string(i) + ": " + m);
  }
  void ws() {
    while (i < s.size() && (s[i] == ' ' || s[i] == '\t' || s[i] == '\n' || s[i] == '\r')) ++i;
  }
  void expect(char ch) {
    ws();
    if (i >= s.size() || s[i] != ch) fail(std::string("expected '") + ch + "'");
    ++i;
  }
  bool peek(char ch) {
    ws();
    return i < s.size() && s[i] == ch;
  }
  static void utf8(std::string& out, uint32_t cp) {
    if (cp < 0x80) out += (char)cp;
    else if (cp < 0x800) out += (char)(0xC0 | cp >> 6), out += (char)(0x80 | (cp & 0x3F));
    else if (cp < 0x10000) out += (char)(0xE0 | cp >> 12), out += (char)(0x80 | (cp >> 6 & 0x3F)), out += (char)(0x80 | (cp & 0x3F));
    else
      out += (char)(0xF0 | cp >> 18), out += (char)(0x80 | (cp >> 12 & 0x3F)), out += (char)(0x80 | (cp >> 6 & 0x3F)),
          out += (char)(0x80 | (cp & 0x3F));
  }
  uint32_t hex4() {
    if (i + 4 > s.size()) fail("truncated \\u escape");
    uint32_t v = 0;
    for (int k = 0; k < 4; ++k) {
      const char ch = s[i++];
      v <<= 4;
      if (ch >= '0' && ch <= '9') v |= ch - '0';
      else if (ch >= 'a' && ch <= 'f') v |= ch - 'a' + 10;
      else if (ch >= 'A' && ch <= 'F') v |= ch - 'A' + 10;
      else fail("bad \\u escape");
    }
    return v;
  }
  std::string str() {
    expect('"');
    std::string out;
    while (true) {
      if (i >= s.size()) fail("unterminated string");
      const unsigned char ch = s[i++];
      if (ch == '"') return out;
      if (ch < 0x20) fail("control character in a string");
      if (ch != '\\') {
        out += (char)ch;
        continue;
      }
      if (i >= s.size()) fail("unterminated string");
      const char e = s[i++];
      switch (e) {
        case '"': out += '"'; break;
        case '\\': out += '\\'; break;
        case '/': out += '/'; break;
        case 'b': out += '\b'; break;
        case 'f': out += '\f'; break;
        case 'n': out += '\n'; break;
        case 'r': out += '\r'; break;
        case 't': out += '\t'; break;
        case 'u': {
          uint32_t cp = hex4();
          if (cp >= 0xD800 && cp < 0xDC00) {  // a surrogate pair
            if (i + 2 > s.size() || s[i] != '\\' || s[i + 1] != 'u') fail("unpaired surrogate");
            i += 2;
            const uint32_t lo = hex4();
            if (lo < 0xDC00 || lo >= 0xE000) fail("unpaired surrogate");
            cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
          } else if (cp >= 0xDC00 && cp < 0xE000) {
            fail("unpaired surrogate");
          }
          utf8(out, cp);
          break;
        }
        default: fail("bad escape");
      }
    }
  }
  // a JSON integer that must be >= 0 and fit int64: no sign, fraction or exponent
  uint64_t uint(const std::string& key) {
    ws();
    if (i < s.size() && s[i] == '-') fail(key + ": negative value");
    if (i >= s.size() || s[i] < '0' || s[i] > '9') fail(key + ": expected a non-negative integer");
    if (s[i] == '0' && i + 1 < s.size() && s[i + 1] >= '0' && s[i + 1] <= '9') fail(key + ": leading zero");
    uint64_t v = 0;
    while (i < s.size() && s[i] >= '0' && s[i] <= '9') {
      const uint64_t dg = (uint64_t)(s[i++] - '0');
      if (v > ((uint64_t)INT64_MAX - dg) / 10) fail(key + ": integer overflows int64");
      v = v * 10 + dg;
    }
    if (i < s.size() && (s[i] == '.' || s[i] == 'e' || s[i] == 'E')) fail(key + ": expected an integer");
    return v;
  }
  void metadata() {
    expect('{');
    if (peek('}')) {
      ++i;
      return;
    }
    do {
      str();
      expect(':');
      ws();
      if (i >= s.size() || s[i] != '"') fail("__metadata__ values must be strings");
      str();
    } while (peek(',') && ++i);
    expect('}');
  }
  HeaderEntry tensor(const std::string& key) {
    HeaderEntry h;
    h.key = key;
    bool has_dtype = false, has_shape = false, has_off = false;
    expect('{');
    do {
      const std::string f = str();
      expect(':');
      if (f == "dtype" && !has_dtype) {
        ws();
        if (i >= s.size() || s[i] != '"') fail(key + ": dtype must be a string");
        h.dtype = str(), has_dtype = true;
      } else if (f == "shape" && !has_shape) {
        expect('[');
        if (peek(']')) {
          ++i;
        } else {
          do {
            if (h.ndim == 8) fail(key + ": more than 8 dimensions");
            h.dims[h.ndim++] = (int64_t)uint(key + " shape");
          } while (peek(',') && ++i);
          expect(']');
        }
        has_shape = true;
      } else if (f == "data_offsets" && !has_off) {
        expect('[');
        h.begin = uint(key + " data_offsets");
        expect(',');
        h.end = uint(key + " data_offsets");
        expect(']');
        has_off = true;
      } else {
        fail(key + ": unexpected or repeated member \"" + f + "\"");
      }
    } while (peek(',') && ++i);
    expect('}');
    if (!(has_dtype && has_shape && has_off)) fail(key + ": needs dtype, shape and data_offsets");
    return h;
  }
  std::vector<HeaderEntry> parse() {
    std::vector<HeaderEntry> out;
    std::map<std::string, int> seen;
    expect('{');
    if (!peek('}')) {
      bool meta = false;
      do {
        const std::string key = str();
        expect(':');
        if (key == "__metadata__") {
          if (meta) fail("__metadata__ given twice");
          meta = true;
          metadata();
          continue;
        }
        if (!seen.emplace(key, (int)out.size()).second) fail("tensor " + key + " given twice");
        out.push_back(tensor(key));
      } while (peek(',') && ++i);
    }
    expect('}');
    ws();
    if (i != s.size()) fail("trailing content after the header object");
    return out;
  }
};

int dtype_code(const std::string& d) { return d == "F32" ? DT_F32 : d == "F16" ? DT_F16 : d == "BF16" ? DT_BF16 : DT_OTHER; }

// bytes per element of the dtypes the safetensors format defines (0: unknown, its size is not checked)
int dtype_bytes(const std::string& d) {
  if (d == "F64" || d == "I64" || d == "U64") return 8;
  if (d == "F32" || d == "I32" || d == "U32") return 4;
  if (d == "F16" || d == "BF16" || d == "I16" || d == "U16") return 2;
  if (d == "I8" || d == "U8" || d == "BOOL" || d == "F8_E4M3" || d == "F8_E5M2") return 1;
  return 0;
}

struct Fd {
  int fd = -1;
  ~Fd() {
    if (fd >= 0) close(fd);
  }
};

void pread_all(int fd, void* dst, uint64_t bytes, uint64_t off, const std::string& what) {
  char* p = static_cast<char*>(dst);
  while (bytes) {
    const ssize_t r = pread(fd, p, (size_t)std::min<uint64_t>(bytes, 1ull << 30), (off_t)off);
    if (r < 0 && errno == EINTR) continue;
    if (r < 0) throw Error(what + ": read failed: " + strerror(errno));
    if (r == 0) throw Error(what + ": the file ended early (it changed while it was read?)");
    p += r, bytes -= (uint64_t)r, off += (uint64_t)r;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------- the plan
// One mapped tensor: where its bytes lie in the file, what it becomes in the master arena
struct StItem {
  uint64_t begin = 0, end = 0;  // absolute file offsets
  int dtype = DT_F32;
  int64_t rows = 1, cols = 1;  // the file's shape as [rows][cols] (a transposed Linear weight: [out][in])
  size_t dst = 0;              // float offset in the master arena
  bool transpose = false;
};
struct StPlan {
  int kind = SDB_CKPT_FULL;
  int width = 0;  // conv_in input channels (0 for a VAE-only file)
  bool has_sched = false;
  std::vector<StItem> items;  // in file order
};

// Validates the whole file (header, map, shapes, dtypes, byte ranges) against its size; with a context, against that context's
// registry too. Reads the header only.
static StPlan st_plan(int fd, const std::string& path, const Ctx* c) {
  struct stat sb;
  if (fstat(fd, &sb) != 0) throw Error(path + ": fstat failed: " + strerror(errno));
  const uint64_t fsize = (uint64_t)sb.st_size;
  if (fsize < 8) throw Error(path + ": not a safetensors file: " + std::to_string(fsize) + " bytes, shorter than the header length");
  unsigned char lb[8];
  pread_all(fd, lb, 8, 0, path);
  uint64_t hlen = 0;
  for (int k = 7; k >= 0; --k) hlen = hlen << 8 | lb[k];
  constexpr uint64_t kMaxHeader = 100ull << 20;
  if (hlen > kMaxHeader)
    throw Error(path + ": header length " + std::to_string(hlen) + " is over the 100 MB limit of a safetensors header");
  if (8 + hlen > fsize)
    throw Error(path + ": header length " + std::to_string(hlen) + " runs past the end of the file (" + std::to_string(fsize) +
                " bytes)");
  std::string text(hlen, '\0');
  if (hlen) pread_all(fd, &text[0], hlen, 8, path);
  std::vector<HeaderEntry> hdr = Parser{text, path}.parse();
  const uint64_t body = 8 + hlen, body_size = fsize - body;
  // every entry's byte range, mapped or not, lies in the file and fits its dtype and shape
  for (HeaderEntry& h : hdr) {
    const std::string where = path + ": tensor " + h.key;
    if (h.begin > h.end || h.end > body_size)
      throw Error(where + ": data_offsets [" + std::to_string(h.begin) + "," + std::to_string(h.end) + "] lie outside the " +
                  std::to_string(body_size) + " data bytes of the file");
    for (int k = 0; k < h.ndim; ++k) {
      const uint64_t d = (uint64_t)h.dims[k];
      if (d && h.count > (uint64_t)INT64_MAX / 8 / d) throw Error(where + ": shape " + shape_str(h.ndim, h.dims) + " overflows");
      h.count *= d;
    }
    const int nb = dtype_bytes(h.dtype);
    if (nb && h.end - h.begin != h.count * nb)
      throw Error(where + ": data_offsets [" + std::to_string(h.begin) + "," + std::to_string(h.end) + "] hold " +
                  std::to_string(h.end - h.begin) + " bytes, but " + h.dtype + " " + shape_str(h.ndim, h.dims) + " is " +
                  std::to_string(h.count * nb) + " bytes");
  }

  // which checkpoint this is
  bool full = false, vae = false;
  for (const HeaderEntry& h : hdr) {
    if (starts(h.key, "conditioner."))
      throw Error(path + ": key " + h.key + " is an SDXL checkpoint's (conditioner.*); this library runs SD-1.x");
    if (starts(h.key, "cond_stage_model.model."))
      throw Error(path + ": key " + h.key + " is an SD-2.x checkpoint's (OpenCLIP text encoder, cond_stage_model.model.*); this "
                  "library runs SD-1.x");
    if (starts(h.key, "model.diffusion_model.") || starts(h.key, "first_stage_model.") || starts(h.key, "cond_stage_model."))
      full = true;
    if (starts(h.key, "encoder.") || starts(h.key, "decoder.") || starts(h.key, "quant_conv.") || starts(h.key, "post_quant_conv."))
      vae = true;
  }
  if (!full && !vae)
    throw Error(path + ": no SD-1.x checkpoint keys (model.diffusion_model.*, first_stage_model.*, cond_stage_model.*) and no "
                "VAE keys (encoder.*, decoder.*, quant_conv.*, post_quant_conv.*)");
  StPlan plan;
  plan.kind = full ? SDB_CKPT_FULL : SDB_CKPT_VAE;

  MapBuilder mb;
  if (full) {
    const std::string ck = "model.diffusion_model.input_blocks.0.0.weight";
    auto it = std::find_if(hdr.begin(), hdr.end(), [&](const HeaderEntry& h) { return h.key == ck; });
    if (it == hdr.end()) throw Error(path + ": missing " + ck + " (registry unet/input_blocks/conv/weight)");
    if (c) {
      check_conv_in_shape(*c, path, it->ndim, it->dims);
      plan.width = c->unet_cin;
    } else {
      const int64_t w = it->ndim == 4 ? it->dims[1] : -1;
      if (w != 4 && w != 8 && w != 9)
        throw Error(path + ": " + ck + " is " + shape_str(it->ndim, it->dims) + ": a conv_in of 4, 8 or 9 input channels "
                    "([320,C,3,3]) is needed");
      plan.width = (int)w;
    }
    unet_map(mb, plan.width);
    vae_map(mb, "first_stage_model.");
    clip_map(mb);
  } else {
    vae_map(mb, "");
  }
  std::unordered_map<std::string, int> keyix;
  for (size_t k = 0; k < mb.e.size(); ++k) keyix[mb.e[k].key] = (int)k;
  // the map against this context's registry: the same names and shapes, every tensor but the schedule once
  if (c) {
    size_t want = 0;
    for (const TensorInfo& t : c->tensors)
      want += t.kind != K_SCHED && (full || starts(t.name, "autoencoder/"));
    SDB_CHECK(want == mb.e.size(), "the checkpoint key map does not cover the registry");
    for (const MapEntry& m : mb.e) {
      SDB_CHECK(c->has(m.reg), "the checkpoint key map names " + m.reg + ", which is not in the registry");
      const TensorInfo& t = c->tensors[c->index.at(m.reg)];
      SDB_CHECK(t.ndim == m.ndim && std::equal(t.dims, t.dims + t.ndim, m.dims), "the checkpoint key map's shape of " + m.reg);
    }
  }

  std::vector<int> hit(mb.e.size(), -1);
  for (const HeaderEntry& h : hdr) {
    const std::string where = path + ": tensor " + h.key;
    // the key's place in the map: a registry tensor, the schedule, or nothing (ignored)
    std::string key = h.key;
    const char* old_clip = "cond_stage_model.transformer.";
    if (full && starts(key, old_clip) && !starts(key, "cond_stage_model.transformer.text_model.")) {
      const std::string rest = key.substr(strlen(old_clip));
      if (starts(rest, "embeddings.") || starts(rest, "encoder.") || starts(rest, "final_layer_norm."))
        key = "cond_stage_model.transformer.text_model." + rest;  // the older spelling without text_model.
    }
    const bool ignored = full ? (!starts(key, "model.diffusion_model.") && !starts(key, "first_stage_model.") &&
                                 !starts(key, "cond_stage_model.")) ||
                                    starts(key, "first_stage_model.loss.") ||
                                    key == "cond_stage_model.transformer.text_model.embeddings.position_ids"
                              : !(starts(key, "encoder.") || starts(key, "decoder.") || starts(key, "quant_conv.") ||
                                  starts(key, "post_quant_conv."));
    const bool sched = full && key == "alphas_cumprod";
    if (ignored && !sched) continue;
    StItem it;
    it.begin = body + h.begin, it.end = body + h.end;
    it.dtype = dtype_code(h.dtype);
    if (it.dtype == DT_OTHER) throw Error(where + " has dtype " + h.dtype + "; a mapped tensor must be F32, F16 or BF16");
    if (sched) {
      if (h.ndim != 1 || h.dims[0] != 1000) throw Error(where + " is " + shape_str(h.ndim, h.dims) + "; the schedule is [1000]");
      it.cols = 1000;
      it.dst = c ? c->tensors[c->index.at("alpha_cumulative_products")].offset : 0;
      plan.has_sched = true;
      plan.items.push_back(it);
      continue;
    }
    auto f = keyix.find(key);
    if (f == keyix.end()) throw Error(where + " is not a tensor of the SD-1.x model (no registry tensor maps to it)");
    const MapEntry& m = mb.e[f->second];
    if (hit[f->second] >= 0) throw Error(where + ": " + m.reg + " is given twice (also by " + hdr[hit[f->second]].key + ")");
    hit[f->second] = (int)(&h - hdr.data());
    int64_t want[4];
    for (int k = 0; k < m.ndim; ++k) want[k] = m.transpose ? m.dims[m.ndim - 1 - k] : m.dims[k];
    if (h.ndim != m.ndim || !std::equal(want, want + m.ndim, h.dims))
      throw Error(where + " is " + shape_str(h.ndim, h.dims) + "; " + m.reg + " needs " + shape_str(m.ndim, want));
    it.transpose = m.transpose;
    it.rows = m.transpose ? want[0] : 1;
    it.cols = m.transpose ? want[1] : (int64_t)h.count;
    it.dst = c ? c->tensors[c->index.at(m.reg)].offset : 0;
    plan.items.push_back(it);
  }
  for (size_t k = 0; k < mb.e.size(); ++k)
    if (hit[k] < 0) throw Error(path + ": missing " + mb.e[k].key + " (registry " + mb.e[k].reg + ")");
  std::sort(plan.items.begin(), plan.items.end(), [](const StItem& a, const StItem& b) { return a.begin < b.begin; });
  return plan;
}

// --------------------------------------------------------------------------------------------------------- the kernel
// One descriptor per tensor of a chunk: a copy runs in blocks of kCopyBlock elements, a transpose in 32x32 tiles.
struct ConvertDesc {
  long long src;      // byte offset in the device staging buffer (16-byte aligned)
  long long dst;      // float offset in the master arena (the registry aligns tensors to 256 bytes)
  long long rows, cols;  // copy: rows = 1
  long long block0;   // first block of this tensor in the launch
  int dtype, transpose;
};
constexpr int kConvertThreads = 256;
constexpr long long kCopyBlock = kConvertThreads * 8;  // 8 elements per thread

__device__ __forceinline__ float widen16(uint32_t h, int dtype) {
  if (dtype == DT_BF16) return __uint_as_float(h << 16);
  // F16: exact for every finite value; inf / NaN keep their payload (no quieting), as numpy's astype does
  if ((h & 0x7C00u) == 0x7C00u) return __uint_as_float((h & 0x8000u) << 16 | 0x7F800000u | (h & 0x3FFu) << 13);
  return __half2float(__ushort_as_half((unsigned short)h));
}
__device__ __forceinline__ float widen(const unsigned char* p, long long i, int dtype) {
  if (dtype == DT_F32) return reinterpret_cast<const float*>(p)[i];
  return widen16(reinterpret_cast<const uint16_t*>(p)[i], dtype);
}

__global__ void __launch_bounds__(kConvertThreads)
convert_tensors_kernel(const ConvertDesc* __restrict__ desc, int ndesc, const unsigned char* __restrict__ staging,
                       float* __restrict__ master) {
  __shared__ float tile[32][33];
  int lo = 0, hi = ndesc - 1;
  while (lo < hi) {  // last tensor whose first block is <= blockIdx.x
    const int mid = (lo + hi + 1) >> 1;
    if (desc[mid].block0 <= (long long)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const ConvertDesc d = desc[lo];
  const long long b = (long long)blockIdx.x - d.block0;
  const unsigned char* src = staging + d.src;
  float* dst = master + d.dst;
  if (!d.transpose) {
    const long long n = d.rows * d.cols, i0 = b * kCopyBlock + (long long)threadIdx.x * 8;
    if (i0 + 8 <= n) {  // vectorised: 16 or 32 source bytes, two float4 stores
      float v[8];
      if (d.dtype == DT_F32) {
        const float4 a = reinterpret_cast<const float4*>(src)[i0 / 4], c = reinterpret_cast<const float4*>(src)[i0 / 4 + 1];
        v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = c.x, v[5] = c.y, v[6] = c.z, v[7] = c.w;
      } else {
        const uint4 a = reinterpret_cast<const uint4*>(src)[i0 / 8];
        const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) v[2 * k] = widen16(w[k] & 0xFFFFu, d.dtype), v[2 * k + 1] = widen16(w[k] >> 16, d.dtype);
      }
      reinterpret_cast<float4*>(dst + i0)[0] = make_float4(v[0], v[1], v[2], v[3]);
      reinterpret_cast<float4*>(dst + i0)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      for (long long i = i0; i < n && i < i0 + 8; ++i) dst[i] = widen(src, i, d.dtype);
    }
    return;
  }
  // transpose [rows][cols] -> [cols][rows] through a 32x32 tile: reads along a source row, writes along a destination row
  const long long tcols = (d.cols + 31) / 32;
  const long long r0 = (b / tcols) * 32, c0 = (b % tcols) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const long long r = r0 + ty + 8 * k, cc = c0 + tx;
    if (r < d.rows && cc < d.cols) tile[ty + 8 * k][tx] = widen(src, r * d.cols + cc, d.dtype);
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const long long cc = c0 + ty + 8 * k, r = r0 + tx;
    if (r < d.rows && cc < d.cols) dst[cc * d.rows + r] = tile[tx][ty + 8 * k];
  }
}

static long long convert_blocks(const StItem& it) {
  if (it.transpose) return ((it.rows + 31) / 32) * ((it.cols + 31) / 32);
  return (it.rows * it.cols + kCopyBlock - 1) / kCopyBlock;
}

// ------------------------------------------------------------------------------------------------------------- the load
namespace {
struct Pinned {
  void* p = nullptr;
  ~Pinned() {
    if (p) cudaFreeHost(p);
  }
};
struct Events {
  cudaEvent_t e[2] = {nullptr, nullptr};
  ~Events() {
    for (cudaEvent_t x : e)
      if (x) cudaEventDestroy(x);
  }
};
uint64_t align16(uint64_t v) { return (v + 15) & ~uint64_t(15); }
}  // namespace

void safetensors_probe(const char* path_c, int* kind, int* conv_in_width) {
  SDB_CHECK(path_c && *path_c, "null checkpoint path");
  const std::string path = path_c;
  Fd f;
  f.fd = open(path_c, O_RDONLY | O_CLOEXEC);
  if (f.fd < 0) throw Error("cannot open " + path + ": " + strerror(errno));
  const StPlan p = st_plan(f.fd, path, nullptr);
  if (kind) *kind = p.kind;
  if (conv_in_width) *conv_in_width = p.width;
}

void model_load_safetensors(Ctx& c, const char* path_c) {
  SDB_CHECK(path_c && *path_c, "null checkpoint path");
  const std::string path = path_c;
  Fd f;
  f.fd = open(path_c, O_RDONLY | O_CLOEXEC);
  if (f.fd < 0) throw Error("cannot open " + path + ": " + strerror(errno));
  const StPlan plan = st_plan(f.fd, path, &c);

  // chunks in file order: at least 64 MB and at least the largest tensor (16-byte aligned slots in the staging buffer)
  uint64_t cap = 64ull << 20;
  for (const StItem& it : plan.items) cap = std::max(cap, align16(it.end - it.begin));
  struct Chunk {
    size_t first = 0, count = 0;
    uint64_t bytes = 0;
  };
  std::vector<Chunk> chunks;
  std::vector<ConvertDesc> desc(plan.items.size());
  for (size_t k = 0; k < plan.items.size(); ++k) {
    const StItem& it = plan.items[k];
    const uint64_t sz = it.end - it.begin;
    if (chunks.empty() || chunks.back().bytes + sz > cap) chunks.push_back(Chunk{k, 0, 0});
    Chunk& ch = chunks.back();
    const long long block0 = ch.count ? desc[k - 1].block0 + convert_blocks(plan.items[k - 1]) : 0;
    desc[k] = ConvertDesc{(long long)ch.bytes, (long long)it.dst, it.rows, it.cols, block0, it.dtype, it.transpose ? 1 : 0};
    ch.bytes = align16(ch.bytes + sz), ch.count++;
  }

  // from here on the master arena is overwritten: the context is not finalized until the next sdb_finalize_weights
  c.finalized = false;
  model_invalidate_graphs(c);
  if (plan.kind == SDB_CKPT_FULL) {
    c.norm_eps.clear();
  } else {
    for (auto it = c.norm_eps.begin(); it != c.norm_eps.end();)
      it = starts(it->first, "autoencoder/") ? c.norm_eps.erase(it) : std::next(it);
  }
  c.work.reset();
  unsigned char* d_stage = c.work.get<unsigned char>(cap);
  ConvertDesc* d_desc = c.work.get<ConvertDesc>(desc.size() + 1);
  SDB_CUDA(cudaMemcpyAsync(d_desc, desc.data(), desc.size() * sizeof(ConvertDesc), cudaMemcpyHostToDevice, c.stream));
  Pinned host[2];
  Events ev;
  struct Drain {  // a failed read must not free a pinned buffer that a copy still reads
    cudaStream_t s;
    ~Drain() { cudaStreamSynchronize(s); }
  } drain{c.stream};
  for (int k = 0; k < 2; ++k) {
    SDB_CUDA(cudaHostAlloc(&host[k].p, cap, cudaHostAllocDefault));
    SDB_CUDA(cudaEventCreateWithFlags(&ev.e[k], cudaEventDisableTiming));
  }
  float* master = reinterpret_cast<float*>(c.master.base);
  for (size_t n = 0; n < chunks.size(); ++n) {
    const Chunk& ch = chunks[n];
    const int slot = (int)(n & 1);
    unsigned char* hb = static_cast<unsigned char*>(host[slot].p);
    SDB_CUDA(cudaEventSynchronize(ev.e[slot]));  // the copy out of this buffer two chunks ago has finished
    // the chunk's tensors, one read per run of tensors that lie back to back in the file and in the buffer
    for (size_t k = ch.first; k < ch.first + ch.count;) {
      size_t e = k + 1;
      while (e < ch.first + ch.count && plan.items[e].begin == plan.items[e - 1].end &&
             (uint64_t)desc[e].src == (uint64_t)desc[e - 1].src + (plan.items[e - 1].end - plan.items[e - 1].begin))
        ++e;
      pread_all(f.fd, hb + desc[k].src, plan.items[e - 1].end - plan.items[k].begin, plan.items[k].begin, path);
      k = e;
    }
    SDB_CUDA(cudaMemcpyAsync(d_stage, hb, ch.bytes, cudaMemcpyHostToDevice, c.stream));
    SDB_CUDA(cudaEventRecord(ev.e[slot], c.stream));
    const StItem& last = plan.items[ch.first + ch.count - 1];
    const long long blocks = desc[ch.first + ch.count - 1].block0 + convert_blocks(last);
    convert_tensors_kernel<<<(unsigned)blocks, kConvertThreads, 0, c.stream>>>(d_desc + ch.first, (int)ch.count, d_stage, master);
    SDB_CUDA(cudaGetLastError());
  }
  if (plan.kind == SDB_CKPT_FULL && !plan.has_sched) {
    // no alphas_cumprod in the file: the SD-v1 scaled-linear schedule, the values sdb_init_synthetic writes
    std::vector<float> a(1000);
    const double b0 = std::sqrt(0.00085), b1 = std::sqrt(0.012);
    double prod = 1.0;
    for (int i = 0; i < 1000; ++i) {
      const double s = (i == 999) ? b1 : b0 + (double)i * ((b1 - b0) / 999.0);  // numpy.linspace
      prod *= 1.0 - s * s;
      a[i] = (float)prod;
    }
    SDB_CUDA(cudaMemcpyAsync(c.master_ptr("alpha_cumulative_products"), a.data(), 1000 * sizeof(float), cudaMemcpyHostToDevice,
                             c.stream));
  }
  SDB_CUDA(cudaStreamSynchronize(c.stream));
  c.work.reset();
}

}  // namespace sdb
