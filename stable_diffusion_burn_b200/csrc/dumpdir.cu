// dumpdir.cu — reader for the reference's "dump-dir" weight format (SURVEY §8f row f2). Host code only.
//
// Format (writer python/save.py:6-15, reader src/model/load.rs:17-47): every tensor is a 1-D little-endian f32 .npy
// whose first D values are the shape and the rest the row-major data; scalars are [1.0, value]. Directory names are the
// Rust field names, so <root>/<registry name>.npy is the file of every tensor in the registry. Linear weights are stored
// [in,out] (save.py:19), conv weights OIHW. Beside the tensors sit configuration scalars (eps, n_group, stride, n_head, ...)
// which the reference reads into its module configs; here the topology is compiled in, so they are VALIDATED against it
// (a mismatch is an error, never silently ignored) and the norm eps values are honoured per layer.
#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "model.cuh"

namespace sdb {

// ---- .npy (format 1.0 / 2.0 / 3.0), '<f4', C order, 1-D
bool npy_read_f32(const std::string& file, std::vector<float>& out) {
  FILE* f = std::fopen(file.c_str(), "rb");
  if (!f) {
    SDB_CHECK(errno == ENOENT || errno == ENOTDIR, "cannot open " + file + ": " + std::strerror(errno));
    return false;
  }
  struct Closer {
    FILE* f;
    ~Closer() { std::fclose(f); }
  } closer{f};
  unsigned char head[12];
  SDB_CHECK(std::fread(head, 1, 10, f) == 10 && std::memcmp(head, "\x93NUMPY", 6) == 0, file + ": not an .npy file");
  const int major = head[6];
  size_t hlen = head[8] | (head[9] << 8);
  if (major >= 2) {
    SDB_CHECK(std::fread(head + 10, 1, 2, f) == 2, file + ": truncated header");
    hlen |= (size_t)head[10] << 16 | (size_t)head[11] << 24;
  }
  SDB_CHECK(major >= 1 && major <= 3 && hlen < (1u << 20), file + ": unsupported .npy version");
  std::string hdr(hlen, '\0');
  SDB_CHECK(std::fread(&hdr[0], 1, hlen, f) == hlen, file + ": truncated header");
  SDB_CHECK(hdr.find("'<f4'") != std::string::npos, file + ": dtype must be little-endian float32 (NpyData<f32>, load.rs:39)");
  SDB_CHECK(hdr.find("'fortran_order': False") != std::string::npos, file + ": fortran_order must be False");
  const size_t sp = hdr.find("'shape':");
  SDB_CHECK(sp != std::string::npos, file + ": no shape in header");
  const size_t lp = hdr.find('(', sp), rp = hdr.find(')', sp);
  SDB_CHECK(lp != std::string::npos && rp != std::string::npos && rp > lp, file + ": malformed shape");
  long long count = 1;
  int ndim = 0;
  for (size_t i = lp + 1; i < rp;) {
    while (i < rp && (hdr[i] == ' ' || hdr[i] == ',')) ++i;
    if (i >= rp) break;
    char* end = nullptr;
    const long long d = std::strtoll(hdr.c_str() + i, &end, 10);
    SDB_CHECK(end != hdr.c_str() + i && d >= 0, file + ": malformed shape");
    count *= d, ++ndim;
    i = end - hdr.c_str();
  }
  SDB_CHECK(ndim == 1, file + ": dump-dir tensors are 1-D [dims..., values...] arrays (save.py:10-15)");
  out.resize((size_t)count);
  SDB_CHECK(std::fread(out.data(), sizeof(float), (size_t)count, f) == (size_t)count, file + ": truncated data");
  return true;
}

// load_tensor::<B, D> (src/model/load.rs:30-47): splits [dims..., values...]; checks the element count
long long dump_tensor_read(const std::string& file, int ndim, int64_t* dims, std::vector<float>& payload) {
  SDB_CHECK(npy_read_f32(file, payload), "missing file " + file);
  SDB_CHECK((long long)payload.size() >= ndim, file + ": shorter than its rank");
  long long count = 1;
  for (int i = 0; i < ndim; ++i) {
    const float d = payload[i];
    SDB_CHECK(d >= 0 && d == std::floor(d) && d < 1e9f, file + ": leading values are not a shape");
    dims[i] = (int64_t)d, count *= dims[i];
  }
  SDB_CHECK((long long)payload.size() == ndim + count, file + ": element count does not match its leading shape values");
  return count;
}

static bool read_scalar(const std::string& file, float& v) {  // save_scalar: [1.0, value]
  std::vector<float> p;
  if (!npy_read_f32(file, p)) return false;
  SDB_CHECK(p.size() == 2 && p[0] == 1.0f, file + ": not a dump-dir scalar ([1.0, value])");
  v = p[1];
  return true;
}

static std::string dir_of(const std::string& name) { return name.substr(0, name.rfind('/')); }

void model_load_dump_dir(Ctx& c, const char* root_c) {
  SDB_CHECK(root_c && *root_c, "null dump-dir path");
  const std::string root = root_c;
  std::vector<float> buf;
  int64_t dims[4];
  float v = 0.f;
  // load_stable_diffusion (src/model/stablediffusion/load.rs:20-21)
  SDB_CHECK(read_scalar(root + "/n_steps.npy", v), "missing file " + root + "/n_steps.npy");
  SDB_CHECK(v == 1000.f, "n_steps must be 1000 (the sampler's schedule length)");
  // a 4- / 9-channel conv_in that does not fit this context gets a message naming the create entry to use, before the
  // configuration scalar unet/input_blocks/conv/n_channels_in reports it as a plain topology difference
  if (npy_read_f32(root + "/unet/input_blocks/conv/weight.npy", buf) && buf.size() >= 4) {
    const int64_t d[4] = {(int64_t)buf[0], (int64_t)buf[1], (int64_t)buf[2], (int64_t)buf[3]};
    check_conv_in_shape(c, root, 4, d);
  }
  // configuration scalars recorded while the registry was built
  for (const MetaCheck& m : c.meta) {
    const std::string file = root + "/" + m.relpath + ".npy";
    if (m.must_be_absent) {
      std::vector<float> tmp;
      SDB_CHECK(!npy_read_f32(file, tmp), file + " exists, but this layer has no such tensor in the compiled topology");
      continue;
    }
    std::vector<float> p;
    SDB_CHECK(npy_read_f32(file, p), "missing file " + file);
    std::vector<float> want;
    want.push_back((float)m.values.size());
    want.insert(want.end(), m.values.begin(), m.values.end());
    SDB_CHECK(p == want, file + ": value differs from the compiled SD-v1.4 topology");
  }
  // from here on the master arena is overwritten tensor by tensor: a failure midway must not leave the context "finalized"
  // on stale packed weights (ADVICE r1)
  c.finalized = false;
  model_invalidate_graphs(c);
  c.norm_eps.clear();
  std::vector<float> fill;
  for (const TensorInfo& t : c.tensors) {
    const bool sched = t.name == "alpha_cumulative_products";
    const std::string file = root + "/" + (sched ? std::string("alphas_cumprod") : t.name) + ".npy";
    float* dst = reinterpret_cast<float*>(c.master.base) + t.offset;
    std::vector<float> probe;
    const bool is_norm = t.kind == K_NORM_G || t.kind == K_NORM_B;
    const bool is_bias = t.kind == K_CONV_B || t.kind == K_LIN_B;
    if (is_norm && t.kind == K_NORM_G) {
      // load_group_norm / load_layer_norm both require eps (groupnorm/load.rs:19, load.rs:95)
      const std::string d = dir_of(t.name);
      SDB_CHECK(read_scalar(root + "/" + d + "/eps.npy", v), "missing file " + root + "/" + d + "/eps.npy");
      SDB_CHECK(v > 0.f && v < 1e-2f, root + "/" + d + "/eps.npy: implausible eps");
      c.norm_eps[d] = v;
    }
    if (!npy_read_f32(file, buf)) {
      // optional tensors are detected by file absence: Linear/Conv bias -> None (load.rs:70,123), GroupNorm
      // weight/bias -> ones/zeros (groupnorm/load.rs:21-30). LayerNorm requires both (load.rs:93-94).
      const bool group_norm = is_norm && c.group_norms.count(dir_of(t.name));
      SDB_CHECK(is_bias || group_norm, "missing file " + file);
      fill.assign((size_t)t.count, t.kind == K_NORM_G ? 1.f : 0.f);
      SDB_CUDA(cudaMemcpy(dst, fill.data(), t.count * sizeof(float), cudaMemcpyHostToDevice));
      continue;
    }
    SDB_CHECK((long long)buf.size() >= t.ndim, file + ": shorter than its rank");
    for (int i = 0; i < t.ndim; ++i)
      SDB_CHECK(buf[i] == (float)t.dims[i], file + ": shape differs from the registry entry " + t.name);
    SDB_CHECK((long long)buf.size() == t.ndim + t.count, file + ": element count does not match its shape");
    SDB_CUDA(cudaMemcpy(dst, buf.data() + t.ndim, t.count * sizeof(float), cudaMemcpyHostToDevice));
  }
  (void)dims;
  c.finalized = false;
}

}  // namespace sdb
