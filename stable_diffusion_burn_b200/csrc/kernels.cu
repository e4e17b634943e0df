// kernels.cu — HBM-bound kernels around the tensor-core GEMMs: GroupNorm statistics, operand staging
// (GroupNorm-apply + SiLU + fp16 hi/lo split, stride-2 phase layout), LayerNorm, the
// small CUDA-core convolutions (Cin = 4, Cout <= 4), sampler elementwise ops, weight packing.
// All activations are NHWC; loads/stores are 8- or 16-byte vectors, coalesced along channels.
#include "kernels.cuh"

#include <algorithm>

namespace sdb {

static inline int ceil_div(long long a, long long b) { return int((a + b - 1) / b); }

__device__ __forceinline__ void split_store8(const float (&f)[8], __half* hi, __half* lo) {
  __half2 h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const HalfPair2 s = split_f16x2(f[2 * j], f[2 * j + 1]);
    h[j] = s.hi, l[j] = s.lo;
  }
  *reinterpret_cast<uint4*>(hi) = *reinterpret_cast<uint4*>(h);
  if (lo) *reinterpret_cast<uint4*>(lo) = *reinterpret_cast<uint4*>(l);
}

__device__ __forceinline__ void split_store1(float f, __half* hi, __half* lo, size_t o) {
  const HalfPair2 s = split_f16x2(f, 0.f);
  hi[o] = __low2half(s.hi);
  if (lo) lo[o] = __low2half(s.lo);
}

// ============================================================ GroupNorm statistics
// Deterministic two-level reduction (no floating-point atomics): every CTA reduces its pixel chunk per group in a
// fixed order and writes a partial; the last CTA of an image (ticket counter) folds the partials in chunk order.
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, int C, int HW, int pix_per_cta,
                                                       double* __restrict__ sums, float* __restrict__ partials,
                                                       unsigned int* __restrict__ tickets) {
  pdl_enter();
  __shared__ float s_pair[2][1280];  // per channel-pair (sum, sumsq), C <= 2560
  __shared__ bool s_last;
  const int n = blockIdx.y;
  const int gs = C / 32;
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  // thread -> (channel pair, pixel lane): narrow tensors (C/2 < 256) spread the spare threads over pixels
  const int npair = C / 2;
  const int pg = npair >= 256 ? 1 : 256 / npair;          // pixel lanes per channel pair
  const int nslot = npair >= 256 ? npair : npair * pg;    // (pixel lane, pair) partials, <= 1280
  for (int slot = threadIdx.x; slot < nslot; slot += blockDim.x) {
    const int cp = slot % npair, pl = slot / npair;
    const float* ptr = x + (size_t)n * HW * C + cp * 2;
    float s = 0.f, q = 0.f;
    int p = p0 + pl;
    for (; p + 3 * pg < p1; p += 4 * pg) {
      float2 v0 = *reinterpret_cast<const float2*>(ptr + (size_t)p * C);
      float2 v1 = *reinterpret_cast<const float2*>(ptr + (size_t)(p + pg) * C);
      float2 v2 = *reinterpret_cast<const float2*>(ptr + (size_t)(p + 2 * pg) * C);
      float2 v3 = *reinterpret_cast<const float2*>(ptr + (size_t)(p + 3 * pg) * C);
      s += (v0.x + v0.y) + (v1.x + v1.y) + (v2.x + v2.y) + (v3.x + v3.y);
      q += (v0.x * v0.x + v0.y * v0.y) + (v1.x * v1.x + v1.y * v1.y) + (v2.x * v2.x + v2.y * v2.y) +
           (v3.x * v3.x + v3.y * v3.y);
    }
    for (; p < p1; p += pg) {
      float2 v = *reinterpret_cast<const float2*>(ptr + (size_t)p * C);
      s += v.x + v.y;
      q += v.x * v.x + v.y * v.y;
    }
    s_pair[0][slot] = s;
    s_pair[1][slot] = q;
  }
  __syncthreads();
  const int chunks = gridDim.x;
  if (threadIdx.x < 64) {  // thread = (group, stat): fold the group's channel pairs in index order
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
    const int pairs = gs / 2;
    float acc = 0.f;
    for (int l = 0; l < (npair >= 256 ? 1 : pg); ++l)
      for (int i = 0; i < pairs; ++i) acc += s_pair[which][l * npair + g * pairs + i];
    partials[((size_t)n * chunks + blockIdx.x) * 64 + threadIdx.x] = acc;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&tickets[n], 1u) == (unsigned)(chunks - 1);
  __syncthreads();
  if (s_last && threadIdx.x < 64) {
    __threadfence();
    double acc = 0.0;
    for (int ch = 0; ch < chunks; ++ch) acc += (double)partials[((size_t)n * chunks + ch) * 64 + threadIdx.x];
    sums[(size_t)n * 64 + threadIdx.x] = acc;  // [n][32][2]
  }
}

size_t gn_stats_partial_floats(int n, int HW) {
  int pix = (int)((((long long)HW * n) + 591) / 592);
  if (pix < 16) pix = 16;
  return (size_t)n * ceil_div(HW, pix) * 64;
}

void gn_stats_launch(const float* x, int C, int n, int HW, double* sums, float* partials, unsigned int* tickets,
                     cudaStream_t st) {
  SDB_CHECK(C % 64 == 0 && C <= 2560, "GroupNorm channels");
  int pix = (int)((((long long)HW * n) + 591) / 592);
  if (pix < 16) pix = 16;
  dim3 grid(ceil_div(HW, pix), n);
  launch_k(gn_stats_kernel, grid, dim3(256), 0, st, x, C, HW, pix, sums, partials, tickets);
  SDB_CUDA(cudaGetLastError());
}

// per-(image, channel) affine from the group sums: y = x*scale + shift
__device__ __forceinline__ void gn_affine(const double* sums, int n, int c, int gs, double inv_cnt, float eps,
                                          const float* gamma, const float* beta, float& scale, float& shift) {
  const int g = c / gs;
  const double s = sums[((size_t)n * 32 + g) * 2 + 0], q = sums[((size_t)n * 32 + g) * 2 + 1];
  const double mean = s * inv_cnt;
  double var = q * inv_cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  scale = rstd * gamma[c];
  shift = beta[c] - (float)mean * scale;
}

// ============================================================ operand staging
__global__ void __launch_bounds__(256)
prep_operand_kernel(const float* __restrict__ x0, int C0, const float* __restrict__ x1, int C1, int H, int W,
                    int pix_per_cta, int phase2, __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  pdl_enter();
  const int n = blockIdx.y;
  const int C = C0 + C1, HW = H * W;
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  const int c8n = C / 8;
  const int items = (p1 - p0) * c8n;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int p = p0 + i / c8n;
    const int c = (i % c8n) * 8;
    const float* src = (c < C0) ? x0 + ((size_t)n * HW + p) * C0 + c : x1 + ((size_t)n * HW + p) * C1 + (c - C0);
    float4 a = *reinterpret_cast<const float4*>(src);
    float4 b = *reinterpret_cast<const float4*>(src + 4);
    float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    const int h = p / W, w = p % W;
    if (phase2) {
      const int ph = (h & 1) * 2 + (w & 1);
      const size_t o = ((((size_t)n * 4 + ph) * (H / 2) + (h >> 1)) * (W / 2) + (w >> 1)) * C + c;
      split_store8(f, out_hi + o, out_lo ? out_lo + o : nullptr);
    } else {
      const size_t o = ((size_t)n * HW + p) * C + c;
      split_store8(f, out_hi + o, out_lo ? out_lo + o : nullptr);
    }
  }
}

void prep_operand_launch(const float* x0, int C0, const float* x1, int C1, int n, int H, int W, bool phase2, Half2Ptr out,
                         cudaStream_t st) {
  const int C = C0 + C1, HW = H * W;
  SDB_CHECK(C % 8 == 0 && C0 % 8 == 0, "operand channels must be multiples of 8");
  int pix = (int)((((long long)HW * n) + 1183) / 1184);
  if (pix < 8) pix = 8;
  dim3 grid(ceil_div(HW, pix), n);
  launch_k(prep_operand_kernel, grid, dim3(256), 0, st, x0, C0, x1, C1, H, W, pix, phase2 ? 1 : 0, out.hi, out.lo);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ fused GroupNorm: statistics + apply in ONE launch
// Phase 1: per-CTA group partials of the CTA's pixel chunk (fixed-order, deterministic), published to global memory.
// After an in-kernel rendezvous of the image's CTAs every CTA folds all partials (same order everywhere). Phase 2:
// normalise + SiLU + fp16 hi/lo split of the same chunk (second read hits L2). The grid never exceeds 4 CTAs per SM,
// so every CTA is resident and the wait cannot deadlock.
__global__ void __launch_bounds__(256)
gn_fused_kernel(const float* __restrict__ x0, int C0, const float* __restrict__ x1, int C1, int H, int W, int pix_per_cta,
                int silu, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                __half* __restrict__ out_hi, __half* __restrict__ out_lo, float* __restrict__ partials,
                unsigned int* __restrict__ tickets) {
  pdl_enter();
  extern __shared__ float s_dyn[];  // scale[C], shift[C]
  __shared__ float s_pair[2][1280];
  const int n = blockIdx.y;
  const int C = C0 + C1, gs = C / 32, HW = H * W;
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  // ---- phase 1
  // thread -> (channel pair, pixel lane): narrow tensors (C/2 < 256) spread the spare threads over pixels
  const int npair = C / 2;
  const int pg = npair >= 256 ? 1 : 256 / npair;          // pixel lanes per channel pair
  const int nslot = npair >= 256 ? npair : npair * pg;    // (pixel lane, pair) partials, <= 1280
  for (int slot = threadIdx.x; slot < nslot; slot += blockDim.x) {
    const int cp = slot % npair, pl = slot / npair;
    const int c = cp * 2;
    const float* ptr;
    int stride;
    if (c < C0) {
      ptr = x0 + (size_t)n * HW * C0 + c;
      stride = C0;
    } else {
      ptr = x1 + (size_t)n * HW * C1 + (c - C0);
      stride = C1;
    }
    float s = 0.f, q = 0.f;
    int p = p0 + pl;
    for (; p + 3 * pg < p1; p += 4 * pg) {
      float2 v0 = *reinterpret_cast<const float2*>(ptr + (size_t)p * stride);
      float2 v1 = *reinterpret_cast<const float2*>(ptr + (size_t)(p + pg) * stride);
      float2 v2 = *reinterpret_cast<const float2*>(ptr + (size_t)(p + 2 * pg) * stride);
      float2 v3 = *reinterpret_cast<const float2*>(ptr + (size_t)(p + 3 * pg) * stride);
      s += (v0.x + v0.y) + (v1.x + v1.y) + (v2.x + v2.y) + (v3.x + v3.y);
      q += (v0.x * v0.x + v0.y * v0.y) + (v1.x * v1.x + v1.y * v1.y) + (v2.x * v2.x + v2.y * v2.y) +
           (v3.x * v3.x + v3.y * v3.y);
    }
    for (; p < p1; p += pg) {
      float2 v = *reinterpret_cast<const float2*>(ptr + (size_t)p * stride);
      s += v.x + v.y;
      q += v.x * v.x + v.y * v.y;
    }
    s_pair[0][slot] = s;
    s_pair[1][slot] = q;
  }
  __syncthreads();
  const int chunks = gridDim.x;
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
    const int pairs = gs / 2;
    float acc = 0.f;
    for (int l = 0; l < (npair >= 256 ? 1 : pg); ++l)
      for (int i = 0; i < pairs; ++i) acc += s_pair[which][l * npair + g * pairs + i];
    partials[((size_t)n * chunks + blockIdx.x) * 64 + threadIdx.x] = acc;
  }
  __threadfence();
  __syncthreads();
  // ---- rendezvous of the image's CTAs (all co-resident), then EVERY CTA folds the partials itself in the same fixed
  // order: no single-CTA serial tail and no second flag round trip; the result is identical in every CTA.
  if (threadIdx.x == 0) {
    atomicAdd(&tickets[n], 1u);
    const long long t0 = clock64();
    while (atomicAdd(&tickets[n], 0u) < (unsigned)chunks) {
      __nanosleep(64);
      if (clock64() - t0 > 4000000000ll) __trap();  // ~2 s: a lost CTA becomes a launch failure, not a hung GPU
    }
    __threadfence();
  }
  __syncthreads();
  __shared__ double s_fold[4][64];
  __shared__ double s_sum[64];
  {
    const int stat = threadIdx.x & 63, part = threadIdx.x >> 6;
    const int per = (chunks + 3) / 4;
    const int c0 = part * per, c1 = min(chunks, c0 + per);
    const float* src = partials + (size_t)n * chunks * 64 + stat;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    int ch = c0;
    for (; ch + 3 < c1; ch += 4) {
      const float v0 = __ldcg(src + (size_t)ch * 64), v1 = __ldcg(src + (size_t)(ch + 1) * 64);
      const float v2 = __ldcg(src + (size_t)(ch + 2) * 64), v3 = __ldcg(src + (size_t)(ch + 3) * 64);
      a0 += (double)v0, a1 += (double)v1, a2 += (double)v2, a3 += (double)v3;
    }
    for (; ch < c1; ++ch) a0 += (double)__ldcg(src + (size_t)ch * 64);
    s_fold[part][stat] = (a0 + a1) + (a2 + a3);
  }
  __syncthreads();
  if (threadIdx.x < 64)
    s_sum[threadIdx.x] = ((s_fold[0][threadIdx.x] + s_fold[1][threadIdx.x]) + s_fold[2][threadIdx.x]) + s_fold[3][threadIdx.x];
  __syncthreads();
  // ---- phase 2
  float* s_scale = s_dyn;
  float* s_shift = s_dyn + C;
  {
    const double inv_cnt = 1.0 / ((double)gs * HW);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const int g = c / gs;
      const double sm = s_sum[g * 2 + 0], sq = s_sum[g * 2 + 1];
      const double mean = sm * inv_cnt;
      double var = sq * inv_cnt - mean * mean;
      if (var < 0.0) var = 0.0;
      const float rstd = (float)(1.0 / sqrt(var + (double)eps));
      const float sc = rstd * gamma[c];
      s_scale[c] = sc;
      s_shift[c] = beta[c] - (float)mean * sc;
    }
  }
  __syncthreads();
  const int c8n = C / 8;
  const int items = (p1 - p0) * c8n;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int p = p0 + i / c8n;
    const int c = (i % c8n) * 8;
    const float* src = (c < C0) ? x0 + ((size_t)n * HW + p) * C0 + c : x1 + ((size_t)n * HW + p) * C1 + (c - C0);
    float4 a = *reinterpret_cast<const float4*>(src);
    float4 b = *reinterpret_cast<const float4*>(src + 4);
    float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = f[j] * s_scale[c + j] + s_shift[c + j];
    if (silu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = silu_f(f[j]);
    }
    const size_t o = ((size_t)n * HW + p) * C + c;
    split_store8(f, out_hi + o, out_lo ? out_lo + o : nullptr);
  }
}

// ============================================================ GroupNorm apply from producer-side statistics
// The GEMM that wrote the tensor also left per-(image, slot, channel-bucket) partial sums (gemm_tc.cuh: gn_part). Every CTA folds
// the partials of its image in a fixed order (fp64), derives the per-channel affine and makes ONE pass over its pixel chunk:
// x read once, no statistics pass, no grid rendezvous. Reads the two sources of cat([x0, x1]) directly.
__global__ void __launch_bounds__(256)
gn_apply_kernel(const GnSrc s0, const GnSrc s1, int bucket, int H, int W, int pix_per_cta, int silu,
                const float* __restrict__ gamma, const float* __restrict__ beta, float eps, __half* __restrict__ out_hi,
                __half* __restrict__ out_lo) {
  pdl_enter();
  extern __shared__ float s_dyn[];  // scale[C], shift[C]
  __shared__ double s_bsum[2 * 256];  // (sum, sumsq) per channel bucket of the concat, C / bucket <= 256
  __shared__ double s_gsum[64];
  const int n = blockIdx.y;
  const int C0 = s0.C, C1 = s1.C, C = C0 + C1, gs = C / 32, HW = H * W;
  const int nb0 = C0 / bucket, nbt = C / bucket;
  // fold of the producer's partial slots. A serial walk would be a chain of L2 round trips: the slots of one
  // (bucket, stat) item are spread over `lanes` threads, four loads in flight each, and the lanes are combined in index order
  // (fixed order everywhere -> every CTA of the image derives bit-identical statistics)
  __shared__ double s_lane[512];
  {
    const int items = 2 * nbt;
    const int lanes = items >= 256 ? 1 : 256 / items;
    for (int idx = threadIdx.x; idx < items * lanes; idx += blockDim.x) {
      const int t = idx % items, lane = idx / items;
      const int b = t >> 1, which = t & 1;
      const GnSrc& s = b < nb0 ? s0 : s1;
      const int nbk = s.C / bucket, bb = b < nb0 ? b : b - nb0;
      const float* p = s.part + ((size_t)n * s.cap * nbk + bb) * 2 + which;
      const size_t st = (size_t)nbk * 2;
      double a = 0.0;
      int sl = lane;
      for (; sl + 3 * lanes < s.slots; sl += 4 * lanes) {
        const float v0 = __ldcg(p + sl * st), v1 = __ldcg(p + (sl + lanes) * st);
        const float v2 = __ldcg(p + (sl + 2 * lanes) * st), v3 = __ldcg(p + (sl + 3 * lanes) * st);
        a += (double)v0, a += (double)v1, a += (double)v2, a += (double)v3;
      }
      for (; sl < s.slots; sl += lanes) a += (double)__ldcg(p + sl * st);
      s_lane[lane * items + t] = a;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < items; t += blockDim.x) {
      double a = 0.0;
      for (int l = 0; l < lanes; ++l) a += s_lane[l * items + t];
      s_bsum[t] = a;
    }
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1, bpg = gs / bucket;
    double a = 0.0;
    for (int i = 0; i < bpg; ++i) a += s_bsum[(g * bpg + i) * 2 + which];
    s_gsum[threadIdx.x] = a;
  }
  __syncthreads();
  float* s_scale = s_dyn;
  float* s_shift = s_dyn + C;
  {
    const double inv_cnt = 1.0 / ((double)gs * HW);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const int g = c / gs;
      const double mean = s_gsum[g * 2] * inv_cnt;
      double var = s_gsum[g * 2 + 1] * inv_cnt - mean * mean;
      if (var < 0.0) var = 0.0;
      const float sc = (float)(1.0 / sqrt(var + (double)eps)) * gamma[c];
      s_scale[c] = sc;
      s_shift[c] = beta[c] - (float)mean * sc;
    }
  }
  __syncthreads();
  const int p0 = blockIdx.x * pix_per_cta, p1 = min(HW, p0 + pix_per_cta);
  const int c8n = C / 8;
  const int items = (p1 - p0) * c8n;
  const float* x0 = s0.x;
  const float* x1 = s1.x;
  auto src_of = [&](int i, int& p, int& c) {
    p = p0 + i / c8n;
    c = (i - (i / c8n) * c8n) * 8;
    return (c < C0) ? x0 + ((size_t)n * HW + p) * C0 + c : x1 + ((size_t)n * HW + p) * C1 + (c - C0);
  };
  auto finish = [&](float4 a, float4 b, int p, int c) {
    float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = fmaf(f[j], s_scale[c + j], s_shift[c + j]);
    if (silu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = silu_f(f[j]);
    }
    const size_t o = ((size_t)n * HW + p) * C + c;
    split_store8(f, out_hi + o, out_lo ? out_lo + o : nullptr);
  };
  // two items per thread and iteration: 4 independent 16-byte loads in flight before the first use
  int i = threadIdx.x;
  for (; i + (int)blockDim.x < items; i += 2 * blockDim.x) {
    int pa, ca, pb, cb;
    const float* sa = src_of(i, pa, ca);
    const float* sb = src_of(i + blockDim.x, pb, cb);
    const float4 a0 = __ldcs(reinterpret_cast<const float4*>(sa)), a1 = __ldcs(reinterpret_cast<const float4*>(sa + 4));
    const float4 b0 = __ldcs(reinterpret_cast<const float4*>(sb)), b1 = __ldcs(reinterpret_cast<const float4*>(sb + 4));
    finish(a0, a1, pa, ca);
    finish(b0, b1, pb, cb);
  }
  if (i < items) {
    int pa, ca;
    const float* sa = src_of(i, pa, ca);
    finish(*reinterpret_cast<const float4*>(sa), *reinterpret_cast<const float4*>(sa + 4), pa, ca);
  }
}

// Large images leave thousands of partial slots (one per 128-pixel tile): a first pass folds groups of 64 slots (fp64 inside,
// fixed order) so that the apply kernel's per-CTA fold stays short. in [n][cap][nbk][2] -> out [n][ceil(slots/64)][nbk][2].
__global__ void __launch_bounds__(256)
gn_fold_kernel(const float* __restrict__ part, int cap, int slots, int nbk2, float* __restrict__ out) {
  pdl_enter();
  const int n = blockIdx.y, chunk = blockIdx.x, nchunks = gridDim.x;
  const int s0 = chunk * 64, s1 = min(slots, s0 + 64);
  for (int t = threadIdx.x; t < nbk2; t += blockDim.x) {
    const float* p = part + ((size_t)n * cap + s0) * nbk2 + t;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    int sl = 0;
    const int cnt = s1 - s0;
    for (; sl + 3 < cnt; sl += 4) {
      a0 += (double)__ldcg(p + (size_t)sl * nbk2), a1 += (double)__ldcg(p + (size_t)(sl + 1) * nbk2);
      a2 += (double)__ldcg(p + (size_t)(sl + 2) * nbk2), a3 += (double)__ldcg(p + (size_t)(sl + 3) * nbk2);
    }
    for (; sl < cnt; ++sl) a0 += (double)__ldcg(p + (size_t)sl * nbk2);
    out[((size_t)n * nchunks + chunk) * nbk2 + t] = (float)((a0 + a1) + (a2 + a3));
  }
}
int gn_fold_slots(int slots) { return (slots + 63) / 64; }
void gn_fold_launch(const float* part, int cap, int slots, int nbk, int n, float* out, cudaStream_t st) {
  dim3 grid(gn_fold_slots(slots), n);
  launch_k(gn_fold_kernel, grid, dim3(256), 0, st, part, cap, slots, nbk * 2, out);
  SDB_CUDA(cudaGetLastError());
}

// group sums [n][32][2] (double) of ONE tensor from the producer's (possibly pre-folded) partial slots: what gn_stats_kernel
// computes by reading the tensor, here from a few KB of partials
__global__ void __launch_bounds__(256)
gn_sums_from_partials_kernel(const float* __restrict__ part, int cap, int slots, int nbk, int bpg, double* __restrict__ sums) {
  pdl_enter();
  __shared__ double s_b[512];
  const int n = blockIdx.x;
  for (int t = threadIdx.x; t < 2 * nbk; t += blockDim.x) {
    const float* p = part + (size_t)n * cap * nbk * 2 + t;
    double a = 0.0;
    for (int sl = 0; sl < slots; ++sl) a += (double)__ldcg(p + (size_t)sl * nbk * 2);
    s_b[t] = a;
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
    double a = 0.0;
    for (int i = 0; i < bpg; ++i) a += s_b[(g * bpg + i) * 2 + which];
    sums[(size_t)n * 64 + threadIdx.x] = a;
  }
}
void gn_sums_from_partials_launch(const float* part, int cap, int slots, int nbk, int C, int bucket, int n, double* sums,
                                  cudaStream_t st) {
  SDB_CHECK(nbk <= 256 && (C / 32) % bucket == 0, "group sums from partials: geometry");
  launch_k(gn_sums_from_partials_kernel, dim3(n), dim3(256), 0, st, part, cap, slots, nbk, (C / 32) / bucket, sums);
  SDB_CUDA(cudaGetLastError());
}

void gn_apply_launch(const GnSrc& s0, const GnSrc& s1, int bucket, int n, int H, int W, int silu, const float* gamma,
                     const float* beta, float eps, Half2Ptr out, cudaStream_t st) {
  const int C = s0.C + s1.C, HW = H * W;
  SDB_CHECK(C % 64 == 0 && s0.C % 8 == 0 && C <= 2560 && bucket > 0 && s0.C % bucket == 0 && s1.C % bucket == 0 &&
                (C / 32) % bucket == 0 && C / bucket <= 256,
            "GroupNorm apply: channel / bucket geometry");
  // every CTA repeats the fold of its image's partials (8-24 KB from L2), so the grid is kept small, at least one pixel per CTA
  constexpr int kGnApplyCtasPerSm = 4;
  const int ctas = kGnApplyCtasPerSm * g_num_sms;
  int pix = (int)((((long long)HW * n) + ctas - 1) / ctas);
  if (pix < 1) pix = 1;
  dim3 grid(ceil_div(HW, pix), n);
  launch_k(gn_apply_kernel, grid, dim3(256), (size_t)2 * C * sizeof(float), st, s0, s1, bucket, H, W, pix, silu, gamma, beta, eps,
           out.hi, out.lo);
  SDB_CUDA(cudaGetLastError());
}

static int gn_fused_pix(int n, int HW) {
  constexpr int kGnFusedMinPix = 1;  // pixels per CTA floor: small feature maps are latency-bound, so they get many small CTAs
  int pix = (int)((((long long)HW * n) + 295) / 296);  // <= 296 CTAs (2 per SM): short fold, always co-resident
  return pix < kGnFusedMinPix ? kGnFusedMinPix : pix;
}
size_t gn_fused_partial_floats(int n, int HW) { return (size_t)n * ceil_div(HW, gn_fused_pix(n, HW)) * 64; }

void gn_fused_launch(const float* x0, int C0, const float* x1, int C1, int n, int H, int W, int silu, const float* gamma,
                     const float* beta, float eps, Half2Ptr out, float* partials, unsigned int* tickets, cudaStream_t st) {
  const int C = C0 + C1, HW = H * W;
  SDB_CHECK(C % 64 == 0 && C0 % 8 == 0 && C <= 2560, "GroupNorm channels");
  const int pix = gn_fused_pix(n, HW);
  dim3 grid(ceil_div(HW, pix), n);
  SDB_CHECK((long long)grid.x * grid.y <= 592, "fused GroupNorm grid must stay co-resident");
  launch_k(gn_fused_kernel, grid, dim3(256), (size_t)2 * C * sizeof(float), st, x0, C0, x1, C1, H, W, pix, silu, gamma, beta, eps, out.hi,
           out.lo, partials, tickets);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ LayerNorm: one warp per row
template <int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, int rows, int C, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                 float* __restrict__ out_f32) {
  pdl_enter();
  const int row = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int c8n = C / 8;
  const float* xr = x + (size_t)row * C;
  float v[MAXV][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int c8 = lane + k * 32;
    if (c8 < c8n) {
      float4 a = *reinterpret_cast<const float4*>(xr + c8 * 8);
      float4 b = *reinterpret_cast<const float4*>(xr + c8 * 8 + 4);
      v[k][0] = a.x, v[k][1] = a.y, v[k][2] = a.z, v[k][3] = a.w, v[k][4] = b.x, v[k][5] = b.y, v[k][6] = b.z, v[k][7] = b.w;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[k][j];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int c8 = lane + k * 32;
    if (c8 < c8n) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[k][j] - mean;
        q += d * d;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int c8 = lane + k * 32;
    if (c8 < c8n) {
      float f[8];
      const int c = c8 * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = (v[k][j] - mean) * rstd * gamma[c + j] + beta[c + j];
      if (out_hi) split_store8(f, out_hi + (size_t)row * C + c, out_lo ? out_lo + (size_t)row * C + c : nullptr);
      if (out_f32) {
        *reinterpret_cast<float4*>(out_f32 + (size_t)row * C + c) = make_float4(f[0], f[1], f[2], f[3]);
        *reinterpret_cast<float4*>(out_f32 + (size_t)row * C + c + 4) = make_float4(f[4], f[5], f[6], f[7]);
      }
    }
  }
}
void layernorm_launch(const float* x, int rows, int C, const float* gamma, const float* beta, float eps,
                      Half2Ptr out, float* out_f32, cudaStream_t st) {
  SDB_CHECK(C % 8 == 0 && C <= 1280, "LayerNorm width");
  const int grid = ceil_div(rows, 8);
  if (C <= 512)
    launch_k(layernorm_kernel<2>, dim3(grid), dim3(256), 0, st, x, rows, C, gamma, beta, eps, out.hi, out.lo, out_f32);
  else
    launch_k(layernorm_kernel<5>, dim3(grid), dim3(256), 0, st, x, rows, C, gamma, beta, eps, out.hi, out.lo, out_f32);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ conversions
__global__ void convert_f16_kernel(const float* __restrict__ x, long long count8, __half* __restrict__ hi,
                                   __half* __restrict__ lo) {
  pdl_enter();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count8; i += (long long)gridDim.x * blockDim.x) {
    float4 a = *reinterpret_cast<const float4*>(x + i * 8);
    float4 b = *reinterpret_cast<const float4*>(x + i * 8 + 4);
    float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    split_store8(f, hi + i * 8, lo ? lo + i * 8 : nullptr);
  }
}
void convert_f16_launch(const float* x, long long count, Half2Ptr out, cudaStream_t st) {
  SDB_CHECK(count % 8 == 0, "convert count");
  const long long c8 = count / 8;
  int grid = (int)((c8 + 255) / 256);
  if (grid > g_num_sms * 8) grid = g_num_sms * 8;
  convert_f16_kernel<<<grid, 256, 0, st>>>(x, c8, out.hi, out.lo);
  SDB_CUDA(cudaGetLastError());
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int C, int HW, float* __restrict__ y, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % C);
    const long long r = i / C;
    const int p = int(r % HW);
    const long long n = r / HW;
    y[i] = x[(n * C + c) * HW + p];
  }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, int C, int HW, float* __restrict__ y, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int p = int(i % HW);
    const long long r = i / HW;
    const int c = int(r % C);
    const long long n = r / C;
    y[i] = x[(n * HW + p) * C + c];
  }
}
void nchw_to_nhwc_launch(const float* x, int n, int C, int H, int W, float* y, cudaStream_t st) {
  const long long total = (long long)n * C * H * W;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  nchw_to_nhwc_kernel<<<grid, 256, 0, st>>>(x, C, H * W, y, total);
  SDB_CUDA(cudaGetLastError());
}
void nhwc_to_nchw_launch(const float* x, int n, int C, int H, int W, float* y, cudaStream_t st) {
  const long long total = (long long)n * C * H * W;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  nhwc_to_nchw_kernel<<<grid, 256, 0, st>>>(x, C, H * W, y, total);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ conv 3x3, Cin = 4 (fp32, CUDA cores)
// block = 64 pixels x (Cout/..) ; thread (pix, co-lane): weights staged in smem as [36][Cout]
__global__ void __launch_bounds__(256)
conv3x3_cin4_kernel(const float* __restrict__ x, int H, int W, const float* __restrict__ w, const float* __restrict__ b,
                    int Cout, const float* __restrict__ pre_w, const float* __restrict__ pre_b, float pre_scale,
                    float* __restrict__ y, __half* __restrict__ y_hi, __half* __restrict__ y_lo) {
  pdl_enter();
  extern __shared__ float sm[];
  float* s_w = sm;                  // [36][Cout]
  float* s_in = sm + 36 * Cout;     // [PIX][36]
  constexpr int PIX = 32;
  const int n = blockIdx.y;
  const int HW = H * W;
  const int p0 = blockIdx.x * PIX;
  for (int i = threadIdx.x; i < 36 * Cout; i += blockDim.x) {
    const int k = i / Cout, co = i % Cout;  // k = ci*9 + tap (OIHW inner order)
    s_w[i] = w[(size_t)co * 36 + k];
  }
  for (int i = threadIdx.x; i < PIX * 36; i += blockDim.x) {
    const int pl = i / 36, k = i % 36;
    const int ci = k / 9, tap = k % 9;
    const int p = p0 + pl;
    float v = 0.f;
    if (p < HW) {
      const int h = p / W + tap / 3 - 1, ww = p % W + tap % 3 - 1;
      if (h >= 0 && h < H && ww >= 0 && ww < W) {
        const float* xp = x + (size_t)n * 4 * HW + (size_t)h * W + ww;
        if (pre_w) {
          float acc = pre_b[ci];
#pragma unroll
          for (int cj = 0; cj < 4; ++cj) acc += pre_w[ci * 4 + cj] * (xp[(size_t)cj * HW] * pre_scale);
          v = acc;
        } else {
          v = xp[(size_t)ci * HW];
        }
      }
    }
    s_in[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < PIX * Cout; i += blockDim.x) {
    const int pl = i / Cout, co = i % Cout;
    const int p = p0 + pl;
    if (p >= HW) continue;
    float acc = b ? b[co] : 0.f;
#pragma unroll
    for (int k = 0; k < 36; ++k) acc += s_in[pl * 36 + k] * s_w[k * Cout + co];
    const size_t o = ((size_t)n * HW + p) * Cout + co;
    y[o] = acc;
    if (y_hi) split_store1(acc, y_hi, y_lo, o);  // fp16 hi/lo copy for a consumer that takes this tensor as a raw GEMM operand
  }
}
void conv3x3_cin4_launch(const float* x_nchw, int n, int H, int W, const float* w, const float* b, int Cout,
                         const float* pre_w, const float* pre_b, float pre_scale, float* y, Half2Ptr y16, cudaStream_t st) {
  const size_t smem = (size_t)(36 * Cout + 32 * 36) * sizeof(float);
  static DeviceOnce once;
  if (once.first())
    SDB_CUDA(cudaFuncSetAttribute(conv3x3_cin4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
  dim3 grid(ceil_div(H * W, 32), n);
  launch_k(conv3x3_cin4_kernel, grid, dim3(256), smem, st, x_nchw, H, W, w, b, Cout, pre_w, pre_b, pre_scale, y, y16.hi,
           y16.lo);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ conv 3x3, Cin = 8 or 9: a conditioned UNet's conv_in
// The conv3x3_cin4 scheme over CIN*9 taps: the inpainting UNet (CIN 9, DESIGN §7 f9) and the InstructPix2Pix UNet (CIN 8, f10).
// Channels 0-3 come from x (sample stride xs), channels 4..CIN-1 from cond (sample stride cs, sample index modulo cmod: the two
// CFG halves of an inpainting step read one copy; the three guidance groups of an edit step each have their own). The taps
// accumulate in OIHW order from the bias, as conv3x3_cin4_kernel does, so zero weights on channels 4..CIN-1 give its result bit
// for bit. Weights [CIN*9][Cout] fill 101 KB (CIN 9) / 90 KB (CIN 8) of shared memory and every CTA stages all of them: PIX
// output pixels per CTA amortise that staging.
template <int CIN, int PIX>
__global__ void __launch_bounds__(256)
conv3x3_cin_cond_kernel(const float* __restrict__ x, long long xs, const float* __restrict__ cond, long long cs, int cmod, int H,
                        int W, const float* __restrict__ w, const float* __restrict__ b, int Cout, float* __restrict__ y,
                        __half* __restrict__ y_hi, __half* __restrict__ y_lo) {
  constexpr int K = CIN * 9;
  pdl_enter();
  extern __shared__ float sm[];
  float* s_w = sm;                  // [K][Cout]
  float* s_in = sm + K * Cout;      // [PIX][K]
  const int n = blockIdx.y;
  const int HW = H * W;
  const int p0 = blockIdx.x * PIX;
  for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) {
    const int k = i / Cout, co = i % Cout;  // k = ci*9 + tap (OIHW inner order)
    s_w[i] = w[(size_t)co * K + k];
  }
  const float* xn = x + (size_t)n * xs;
  const float* cn = cond + (size_t)(n % cmod) * cs - (size_t)4 * HW;  // channel ci >= 4 at cn + ci*HW
  for (int i = threadIdx.x; i < PIX * K; i += blockDim.x) {
    const int pl = i / K, k = i % K;
    const int ci = k / 9, tap = k % 9;
    const int p = p0 + pl;
    float v = 0.f;
    if (p < HW) {
      const int h = p / W + tap / 3 - 1, ww = p % W + tap % 3 - 1;
      if (h >= 0 && h < H && ww >= 0 && ww < W) v = (ci < 4 ? xn : cn)[(size_t)ci * HW + (size_t)h * W + ww];
    }
    s_in[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < PIX * Cout; i += blockDim.x) {
    const int pl = i / Cout, co = i % Cout;
    const int p = p0 + pl;
    if (p >= HW) continue;
    float acc = b ? b[co] : 0.f;
#pragma unroll 9
    for (int k = 0; k < K; ++k) acc += s_in[pl * K + k] * s_w[k * Cout + co];
    const size_t o = ((size_t)n * HW + p) * Cout + co;
    y[o] = acc;
    if (y_hi) split_store1(acc, y_hi, y_lo, o);
  }
}
template <int CIN>
static void conv3x3_cin_cond_go(const float* x, long long x_stride, const float* cond, long long cond_stride, int cond_mod, int n,
                                int H, int W, const float* w, const float* b, int Cout, float* y, Half2Ptr y16, cudaStream_t st) {
  constexpr int PIX = kConvCinCondPix;
  const size_t smem = (size_t)(CIN * 9 * Cout + PIX * CIN * 9) * sizeof(float);
  static DeviceOnce once;
  if (once.first())
    SDB_CUDA(cudaFuncSetAttribute(conv3x3_cin_cond_kernel<CIN, PIX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(ceil_div(H * W, PIX), n);
  launch_k(conv3x3_cin_cond_kernel<CIN, PIX>, grid, dim3(256), smem, st, x, x_stride, cond, cond_stride, cond_mod, H, W, w, b,
           Cout, y, y16.hi, y16.lo);
  SDB_CUDA(cudaGetLastError());
}
void conv3x3_cin_cond_launch(int cin, const float* x, long long x_stride, const float* cond, long long cond_stride, int cond_mod,
                             int n, int H, int W, const float* w, const float* b, int Cout, float* y, Half2Ptr y16, cudaStream_t st) {
  SDB_CHECK(cin == 8 || cin == 9, "conv3x3_cin_cond_launch: cin must be 8 or 9");
  (cin == 8 ? conv3x3_cin_cond_go<8> : conv3x3_cin_cond_go<9>)(x, x_stride, cond, cond_stride, cond_mod, n, H, W, w, b, Cout, y,
                                                              y16, st);
}

// ============================================================ conv 3x3, Cout <= 8, fused GroupNorm + SiLU (fp32, CUDA cores)
// The last conv of the UNet (320 -> 4), of the VAE decoder (128 -> 3 at 512x512: 134 MB of input) and of the encoder (512 -> 8).
// HBM-bound by construction (Cout is tiny), so the kernel is organised around reading x ONCE with wide coalesced loads:
//   CTA = 8 x 32 output pixels, 256 threads, one pixel each; channels in chunks of 16. Per chunk the (8+2) x (32+2) halo tile is
//   loaded (float4, 64 B contiguous per pixel), GroupNorm + SiLU applied on the way in, and stored channel-quad-major
//   [4][pixel][4] so that the warp's float4 reads are conflict-free; the chunk's weights sit beside it (broadcast reads).
// Each x element crosses HBM/L2 1.33 times (halo), against 9 times for a tap-by-tap warp-per-pixel kernel.
// TH = rows of the CTA tile (threads = 32 * TH): 8 for large images; 2 for small ones, where an 8-row tile would leave most SMs
// idle (UNet conv_out at 64x64, batch 2: 32 CTAs with TH = 8). With so few warps per SM nothing hides the latency of a
// chunk's loads, so the small variant takes 64 channels per round (5 rounds for 320 channels instead of 20).
// KS = channel-split groups inside the CTA (threads = 32 * TH * KS): group ks takes the channel chunks ks, ks + KS, ... with its own
// halo tile and weight slice, and the groups' partial sums are added in group order at the end (deterministic). The small-image
// variant uses it to put 10 warps on an SM instead of 2: at 64x64, batch 2 the 128 two-warp CTAs left every SM with two warps
// and the kernel latency-bound.
template <int COUT, int TH, int CK, int KS = 1>
__global__ void __launch_bounds__(32 * TH * KS)
conv3x3_small_cout_kernel(const float* __restrict__ x, int H, int W, int C, const double* __restrict__ sums,
                          const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                          const float* __restrict__ wp, const float* __restrict__ b, float* __restrict__ y) {
  pdl_enter();
  constexpr int TW = 32, HP = TH + 2, WP = TW + 2, NPIX = HP * WP, GT = 32 * TH;  // GT = threads of one group
  constexpr int GROUP_F4 = (CK / 4) * NPIX + 9 * COUT * (CK / 4);                  // float4s of one group's tile + weights
  extern __shared__ float sm[];
  float* s_scale = sm;                           // [C]
  float* s_shift = sm + C;                       // [C]
  const int ks = threadIdx.x / GT, gtid = threadIdx.x - ks * GT;
  float4* s_act = reinterpret_cast<float4*>(sm + 2 * C) + (size_t)ks * GROUP_F4;   // [CK/4][NPIX] float4 (this group's)
  float4* s_w = s_act + (CK / 4) * NPIX;         // [9][COUT][CK/4] float4
  const int n = blockIdx.z;
  const int HW = H * W;
  const int h0 = blockIdx.y * TH, w0 = blockIdx.x * TW;
  {
    const int gs = C / 32;
    const double inv_cnt = 1.0 / ((double)gs * HW);
    for (int c = threadIdx.x; c < C; c += blockDim.x) gn_affine(sums, n, c, gs, inv_cnt, eps, gamma, beta, s_scale[c], s_shift[c]);
  }
  const int tx = gtid & 31, ty = gtid >> 5;
  float acc[COUT];
#pragma unroll
  for (int o = 0; o < COUT; ++o) acc[o] = 0.f;
  for (int c0 = ks * CK; c0 < C; c0 += CK * KS) {  // the launcher guarantees (C / CK) % KS == 0: every group runs the same rounds
    __syncthreads();  // the previous chunk's reads are done (and, first time round, the affine table is written)
    // halo tile: NPIX pixels x 4 channel quads
    for (int i = gtid; i < NPIX * (CK / 4); i += GT) {
      const int pix = i / (CK / 4), q = i % (CK / 4);
      const int hh = h0 - 1 + pix / WP, ww = w0 - 1 + pix % WP;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
        const int c = c0 + q * 4;
        v = __ldcs(reinterpret_cast<const float4*>(x + ((size_t)n * HW + (size_t)hh * W + ww) * C + c));
        v.x = silu_f(fmaf(v.x, s_scale[c], s_shift[c])), v.y = silu_f(fmaf(v.y, s_scale[c + 1], s_shift[c + 1]));
        v.z = silu_f(fmaf(v.z, s_scale[c + 2], s_shift[c + 2])), v.w = silu_f(fmaf(v.w, s_scale[c + 3], s_shift[c + 3]));
      }
      s_act[q * NPIX + pix] = v;  // zero outside the image == the conv's zero padding of the NORMALISED tensor
    }
    for (int i = gtid; i < 9 * COUT * (CK / 4); i += GT) {
      const int q = i % (CK / 4), o = (i / (CK / 4)) % COUT, tap = i / ((CK / 4) * COUT);
      s_w[i] = *reinterpret_cast<const float4*>(wp + ((size_t)o * 9 + tap) * C + c0 + q * 4);
    }
    __syncthreads();
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int pix = (ty + tap / 3) * WP + tx + tap % 3;
#pragma unroll
      for (int q = 0; q < CK / 4; ++q) {
        const float4 a = s_act[q * NPIX + pix];
#pragma unroll
        for (int o = 0; o < COUT; ++o) {
          const float4 wv = s_w[(tap * COUT + o) * (CK / 4) + q];
          acc[o] = fmaf(a.x, wv.x, fmaf(a.y, wv.y, fmaf(a.z, wv.z, fmaf(a.w, wv.w, acc[o]))));
        }
      }
    }
  }
  if (KS > 1) {
    // partial sums of the groups -> shared memory (over the tiles, which are dead now), added in group order by group 0
    __syncthreads();
    float* s_red = sm + 2 * C;  // [KS][COUT][GT]
#pragma unroll
    for (int o = 0; o < COUT; ++o) s_red[(ks * COUT + o) * GT + gtid] = acc[o];
    __syncthreads();
    if (ks == 0) {
#pragma unroll
      for (int o = 0; o < COUT; ++o) {
        float a = s_red[o * GT + gtid];
        for (int k = 1; k < KS; ++k) a += s_red[(k * COUT + o) * GT + gtid];
        acc[o] = a;
      }
    }
  }
  const int h = h0 + ty, w = w0 + tx;
  if (ks == 0 && h < H && w < W) {
#pragma unroll
    for (int o = 0; o < COUT; ++o) y[((size_t)n * COUT + o) * HW + (size_t)h * W + w] = acc[o] + b[o];
  }
}
SmallCoutVariant conv3x3_small_cout_launch(const float* x, int n, int H, int W, int C, const double* sums, const float* gamma,
                                           const float* beta, float eps, const float* w_packed, const float* b, int Cout,
                                           float* y_nchw, cudaStream_t st) {
  SDB_CHECK(C % 16 == 0, "conv3x3_small_cout: channels must be a multiple of 16");
  // too few 8-row tiles to fill the machine -> 2-row tiles, 32 channels per round and group, the channel chunks split over
  // KS = 5 or 4 groups of two warps (10 / 8 warps per CTA; 320 = 10 x 32 and 512 = 16 x 32 channels)
  const bool small = (long long)ceil_div(W, 32) * ceil_div(H, 8) * n < 2 * g_num_sms && C % 32 == 0;
  const int ksplit = !small ? 1 : ((C / 32) % 5 == 0 ? 5 : ((C / 32) % 4 == 0 ? 4 : 1));
  const int th = small ? 2 : 8, ck = small ? 32 : 16;
  dim3 grid(ceil_div(W, 32), ceil_div(H, th), n), block(32 * th * ksplit);
  auto smem = [&](int cout) {
    return (size_t)(2 * C + std::max(ksplit * (ck * (th + 2) * 34 + 9 * cout * ck), ksplit * cout * 32 * th)) * sizeof(float);
  };
#define SDB_SMALL_KS(CO, KSV)                                                                                                       \
  {                                                                                                                                 \
    static DeviceOnce once;                                                                                                         \
    if (once.first())                                                                                                               \
      SDB_CUDA(cudaFuncSetAttribute(conv3x3_small_cout_kernel<CO, 2, 32, KSV>, cudaFuncAttributeMaxDynamicSharedMemorySize,         \
                                    160 * 1024));                                                                                   \
    SDB_CHECK(smem(CO) <= 160 * 1024, "conv3x3_small_cout: shared memory");                                                         \
    launch_k(conv3x3_small_cout_kernel<CO, 2, 32, KSV>, grid, block, smem(CO), st, x, H, W, C, sums, gamma, beta, eps, w_packed, b, \
             y_nchw);                                                                                                               \
  }
#define SDB_SMALL_CONV(CO)                                                                                                          \
  if (small) {                                                                                                                      \
    if (ksplit == 5) SDB_SMALL_KS(CO, 5) else if (ksplit == 4) SDB_SMALL_KS(CO, 4) else SDB_SMALL_KS(CO, 1)                          \
  } else                                                                                                                            \
    launch_k(conv3x3_small_cout_kernel<CO, 8, 16>, grid, block, smem(CO), st, x, H, W, C, sums, gamma, beta, eps, w_packed, b, y_nchw)
  if (Cout == 4) {
    SDB_SMALL_CONV(4);
  } else if (Cout == 3) {
    SDB_SMALL_CONV(3);
  } else if (Cout == 8) {
    SDB_SMALL_CONV(8);
  } else {
    throw Error("conv3x3_small_cout: Cout must be 3, 4 or 8");
  }
#undef SDB_SMALL_CONV
#undef SDB_SMALL_KS
  SDB_CUDA(cudaGetLastError());
  return {th, ck, ksplit};
}

// quant_conv (1x1, 8 -> 8) followed by the slice [0..4) of Autoencoder::encode_image (autoencoder/mod.rs:60-66): NCHW in/out
__global__ void quant_conv_slice_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                        int HW, float* __restrict__ y) {
  const int n = blockIdx.y;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = x[((size_t)n * 8 + j) * HW + p];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float acc = b[c];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += w[c * 8 + j] * v[j];
      y[((size_t)n * 4 + c) * HW + p] = acc;
    }
  }
}
void quant_conv_slice_launch(const float* x, const float* w, const float* b, int n, int HW, float* y, cudaStream_t st) {
  dim3 grid(std::min(ceil_div(HW, 256), 1024), n);
  quant_conv_slice_kernel<<<grid, 256, 0, st>>>(x, w, b, HW, y);
  SDB_CUDA(cudaGetLastError());
}

// quant_conv_slice_kernel writing fl(y * scale) at a per-sample stride: the inpainting path's masked-image latent lands scaled
// in channels 1-4 of the conditioning tensor [n,5,HW] (ys = 5 HW) in the encoder's own launch
__global__ void quant_conv_slice_scaled_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                               int HW, long long ys, float scale, float* __restrict__ y) {
  const int n = blockIdx.y;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = x[((size_t)n * 8 + j) * HW + p];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float acc = b[c];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += w[c * 8 + j] * v[j];
      y[(size_t)n * ys + (size_t)c * HW + p] = __fmul_rn(acc, scale);
    }
  }
}
void quant_conv_slice_scaled_launch(const float* x, const float* w, const float* b, int n, int HW, long long y_stride, float scale,
                                    float* y, cudaStream_t st) {
  dim3 grid(std::min(ceil_div(HW, 256), 1024), n);
  quant_conv_slice_scaled_kernel<<<grid, 256, 0, st>>>(x, w, b, HW, y_stride, scale, y);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ time embedding + GEMV
// y[N] = act(x[K] W[K][N] + b); a block owns 32 outputs, 8 k-slices reduced through smem.
// t_dev != null: x is the sinusoidal timestep embedding (reference unet/mod.rs:24-29), K must be 320. T: the timestep's type, int
// (the schedule's timesteps) or float (a real t, DESIGN §7 f15); at an integer t both give the same (float)t and the same rows.
template <class T>
__global__ void __launch_bounds__(256)
gemv_kernel(const float* __restrict__ x, const T* __restrict__ t_dev, const float* __restrict__ W,
            const float* __restrict__ b, int K, int N, int silu, float* __restrict__ y) {
  pdl_enter();
  __shared__ float s_part[8][32];
  __shared__ float s_x[1280];
  if (t_dev) {
    const T t = *t_dev;
    for (int i = threadIdx.x; i < 160; i += blockDim.x) {
      // freqs = exp(arange(half) * (-ln(10000)/half)); args = t*freqs; [cos | sin]
      const float f = expf((float)i * (float)(-9.210340371976184 / 160.0));
      const float a = (float)t * f;
      s_x[i] = cosf(a);
      s_x[160 + i] = sinf(a);
    }
  } else {
    for (int i = threadIdx.x; i < K; i += blockDim.x) s_x[i] = x[i];
  }
  __syncthreads();
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ks = threadIdx.x >> 5;  // 0..7
  float acc = 0.f;
  if (col < N)
    for (int k = ks; k < K; k += 8) acc += s_x[k] * W[(size_t)k * N + col];
  s_part[ks][threadIdx.x & 31] = acc;
  __syncthreads();
  if (ks == 0 && col < N) {
    float s = b ? b[col] : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += s_part[j][threadIdx.x & 31];
    y[col] = silu ? silu_f(s) : s;
  }
}
void gemv_launch(const float* x, const float* W, const float* b, int K, int N, float* y, cudaStream_t st) {
  SDB_CHECK(K <= 1280, "gemv K");
  launch_k(gemv_kernel<int>, dim3(ceil_div(N, 32)), dim3(256), 0, st, x, (const int*)nullptr, W, b, K, N, 0, y);
  SDB_CUDA(cudaGetLastError());
}
// emb_silu = silu(lin2(silu(lin1(timestep_embedding(t)))))  — two multi-CTA GEMVs
template <class T>
static void time_embed_go(const T* t, const float* w1, const float* b1, const float* w2, const float* b2, float* hidden,
                          float* emb_silu, cudaStream_t st) {
  launch_k(gemv_kernel<T>, dim3(40), dim3(256), 0, st, (const float*)nullptr, t, w1, b1, 320, 1280, 1, hidden);
  launch_k(gemv_kernel<int>, dim3(40), dim3(256), 0, st, (const float*)hidden, (const int*)nullptr, w2, b2, 1280, 1280, 1,
           emb_silu);
  SDB_CUDA(cudaGetLastError());
}
void time_embed_launch(const int* t, const float* w1, const float* b1, const float* w2, const float* b2, float* hidden,
                       float* emb_silu, cudaStream_t st) {
  time_embed_go(t, w1, b1, w2, b2, hidden, emb_silu, st);
}
void time_embed_launch(const float* t, const float* w1, const float* b1, const float* w2, const float* b2, float* hidden,
                       float* emb_silu, cudaStream_t st) {
  time_embed_go(t, w1, b1, w2, b2, hidden, emb_silu, st);
}

// Time embedding for ALL timesteps of a sampling schedule in one pass (the rows depend on t alone: sample_latent computes them once
// per call instead of once per step; the weights of the 22 lin_embed layers, 103 MB of fp32, stream once per R rows instead of
// once per step). Same arithmetic, in the same order, as gemv_kernel: the rows are bit-identical to the per-step path.
//   y[row][N] = act(x[row][K] W[K][N] + b),  row = blockIdx.y * R + r
// t_embed != null: x is the sinusoidal embedding of t_embed[row] (K = 320; T as gemv_kernel's). t_rowmap != null: output row
// index = t_rowmap[row].
template <int R, class T>
__global__ void __launch_bounds__(256)
gemv_rows_kernel(const float* __restrict__ x, const T* __restrict__ t_embed, const int* __restrict__ t_rowmap, int rows,
                 const float* __restrict__ W, const float* __restrict__ b, int K, int N, int silu, float* __restrict__ y,
                 long long y_stride) {
  pdl_enter();
  __shared__ float s_part[R][8][32];
  __shared__ float s_x[R][1280];
  const int r0 = blockIdx.y * R, nr = min(R, rows - r0);
  for (int r = 0; r < nr; ++r) {
    if (t_embed) {
      const T t = t_embed[r0 + r];
      for (int i = threadIdx.x; i < 160; i += blockDim.x) {
        const float f = expf((float)i * (float)(-9.210340371976184 / 160.0));
        const float a = (float)t * f;
        s_x[r][i] = cosf(a);
        s_x[r][160 + i] = sinf(a);
      }
    } else {
      for (int i = threadIdx.x; i < K; i += blockDim.x) s_x[r][i] = x[(size_t)(r0 + r) * K + i];
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int col = blockIdx.x * 32 + lane;
  const int ks = threadIdx.x >> 5;  // 0..7
  float acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = 0.f;
  if (col < N)
    for (int k = ks; k < K; k += 8) {
      const float w = W[(size_t)k * N + col];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] += s_x[r][k] * w;  // rows >= nr read stale shared memory and are never stored
    }
#pragma unroll
  for (int r = 0; r < R; ++r) s_part[r][ks][lane] = acc[r];
  __syncthreads();
  if (ks == 0 && col < N) {
    for (int r = 0; r < nr; ++r) {
      float s = b ? b[col] : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += s_part[r][j][lane];
      const long long orow = t_rowmap ? t_rowmap[r0 + r] : (r0 + r);
      y[orow * y_stride + col] = silu ? silu_f(s) : s;
    }
  }
}
// Row j of the call's timesteps t_embed[j] goes to emb_all row row_of[j] (emb_all[row_of[j]][N]): the in-graph selection needs no
// step counter. The DDIM grid's rows are its timestep values (t_embed = row_of); the Karras grid's real t of step j goes to row j.
template <class T>
static void time_embed_rows_go(const T* t_embed, const int* row_of, int rows, const float* w1, const float* b1, const float* w2,
                               const float* b2, const float* w_all, const float* b_all, int n_all, float* hidden, float* emb_silu,
                               float* emb_all, cudaStream_t st) {
  constexpr int R = 5;
  const dim3 gy(40, ceil_div(rows, R));
  launch_k(gemv_rows_kernel<R, T>, gy, dim3(256), 0, st, (const float*)nullptr, t_embed, (const int*)nullptr, rows, w1, b1, 320,
           1280, 1, hidden, (long long)1280);
  launch_k(gemv_rows_kernel<R, int>, gy, dim3(256), 0, st, (const float*)hidden, (const int*)nullptr, (const int*)nullptr, rows, w2,
           b2, 1280, 1280, 1, emb_silu, (long long)1280);
  launch_k(gemv_rows_kernel<R, int>, dim3(ceil_div(n_all, 32), ceil_div(rows, R)), dim3(256), 0, st, (const float*)emb_silu,
           (const int*)nullptr, row_of, rows, w_all, b_all, 1280, n_all, 0, emb_all, (long long)n_all);
  SDB_CUDA(cudaGetLastError());
}
void time_embed_rows_launch(const int* t_dev, int rows, const float* w1, const float* b1, const float* w2, const float* b2,
                            const float* w_all, const float* b_all, int n_all, float* hidden, float* emb_silu, float* emb_all,
                            cudaStream_t st) {
  time_embed_rows_go(t_dev, t_dev, rows, w1, b1, w2, b2, w_all, b_all, n_all, hidden, emb_silu, emb_all, st);
}
void time_embed_rows_launch(const float* t_dev, const int* row_of, int rows, const float* w1, const float* b1, const float* w2,
                            const float* b2, const float* w_all, const float* b_all, int n_all, float* hidden, float* emb_silu,
                            float* emb_all, cudaStream_t st) {
  time_embed_rows_go(t_dev, row_of, rows, w1, b1, w2, b2, w_all, b_all, n_all, hidden, emb_silu, emb_all, st);
}
// out[N] = emb_all[*t_dev][N]: the one launch of the UNet step graph that replaces the three GEMVs
__global__ void __launch_bounds__(256)
emb_select_kernel(const float* __restrict__ emb_all, const int* __restrict__ t_dev, int N, float* __restrict__ out) {
  pdl_enter();
  const float4* src = reinterpret_cast<const float4*>(emb_all + (size_t)(*t_dev) * N);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N / 4; i += gridDim.x * blockDim.x)
    reinterpret_cast<float4*>(out)[i] = src[i];
}
void emb_select_launch(const float* emb_all, const int* t_dev, int N, float* out, cudaStream_t st) {
  SDB_CHECK(N % 4 == 0, "emb_select: N must be a multiple of 4");
  launch_k(emb_select_kernel, dim3(ceil_div(N / 4, 256)), dim3(256), 0, st, emb_all, t_dev, N, out);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ CLIP token + position embedding
// x[s][l][:] = E[tok[s][l]] + Pos[l] for l < L, zero rows up to Lp (reference clip/mod.rs:62-68)
__global__ void embed_tokens_kernel(const int* __restrict__ tok, const float* __restrict__ E, const float* __restrict__ Pos,
                                    int L, int Lp, int D, int vocab, float* __restrict__ x) {
  pdl_enter();
  const int row = blockIdx.x;  // s*Lp + l
  const int s = row / Lp, l = row % Lp;
  float4* dst = reinterpret_cast<float4*>(x + (size_t)row * D);
  if (l >= L) {
    for (int i = threadIdx.x; i < D / 4; i += blockDim.x) dst[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  int id = tok[s * L + l];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  const float4* e = reinterpret_cast<const float4*>(E + (size_t)id * D);
  const float4* pp = reinterpret_cast<const float4*>(Pos + (size_t)l * D);
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) {
    const float4 a = e[i], b = pp[i];
    dst[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}
void embed_tokens_launch(const int* tok, const float* E, const float* Pos, int n, int L, int Lp, int D, int vocab, float* x,
                         cudaStream_t st) {
  launch_k(embed_tokens_kernel, dim3(n * Lp), dim3(192), 0, st, tok, E, Pos, L, Lp, D, vocab, x);
}

// y = a + b (merged conv biases at finalize)
__global__ void add_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, float* __restrict__ y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = a[i] + b[i];
}
void add_vec_launch(const float* a, const float* b, int n, float* y, cudaStream_t st) {
  add_vec_kernel<<<ceil_div(n, 256), 256, 0, st>>>(a, b, n, y);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ sampler elementwise
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}
// Counter-hash Box-Muller N(0,1): element i of the stream keyed by (k0, k1). The init latent (randn_launch) and the per-step
// noise of stochastic DDIM (step_noise_keys) are both this function, evaluated in registers where they are consumed.
__device__ __forceinline__ float randn_at(long long i, uint32_t k0, uint32_t k1) {
  const uint32_t a = mix32((uint32_t)i ^ k0), b = mix32(((uint32_t)i * 0x9E3779B9u) ^ k1);
  const float u1 = ((a >> 8) + 1) * (1.0f / 16777216.0f);  // (0,1]
  const float u2 = (b >> 8) * (1.0f / 16777216.0f);
  return sqrtf(-2.0f * logf(u1)) * cosf(6.283185307179586f * u2);
}

// The init-latent keys of a seed (randn_launch)
__host__ __device__ __forceinline__ void init_noise_keys(uint64_t seed, uint32_t* k0, uint32_t* k1) {
  *k0 = (uint32_t)seed * 2654435761u + 1u;
  *k1 = (uint32_t)(seed >> 32) ^ 0x5bd1e995u;
}
// The init-latent keys of the seed, mixed with the timestep. k1 also takes k0: seeds that differ in their low word only would
// otherwise share k1, hence the angle of every Box-Muller pair, and their streams would correlate (at pi/4).
__host__ __device__ void step_noise_keys(uint64_t seed, int t, uint32_t* k0, uint32_t* k1) {
  *k0 = ((uint32_t)seed * 2654435761u + 1u) ^ mix32(0x3C6EF372u + (uint32_t)t);
  *k1 = ((uint32_t)(seed >> 32) ^ 0x5bd1e995u) ^ mix32(*k0 ^ 0xA54FF53Au);
}

// One fused guidance + update step of the sampler (DESIGN §7 f5, f6), per latent element i < count:
//   pred = u + (c - u) scale, x0 = (x - sqrt(1 - a_t) pred) / sqrt(a_t)                        (every kind)
//   STEP_DDIM        x' = sqrt(a_prev) x0 + dir_coef pred                        (eta = 0: sample_latent's own step)
//   STEP_DDIM_ETA    x' = sqrt(a_prev) x0 + dir_coef pred + s z,  z = randn_at(i, k0, k1)
//   STEP_DPMPP_2M    D = x0 (first order) or c1 x0 - c2 x0_prev (second order); x0_prev <- x0; x' = cx x + cd D
// BLEND (masked img2img): the step's result nl is blended with the known latent noised to the step's target level,
// x = w nl + (1 - w) (sqrt(a_prev) z0 + sqrt(1 - a_prev) eps), w = mask[sample][pixel % plane]. nl is the same expression in
// both instantiations, so an all-ones mask reproduces the unmasked step bit for bit. The blend and the new samplers' updates
// are written with _rn intrinsics (no FMA contraction) so that a test can restate them exactly in float32. STEP_DDIM is the
// expression sample_latent has always used; its instantiations keep the instructions they had.
// PER_SAMPLE (a batch of different requests, DESIGN §7 f7): the scale and the eta noise key of sample i / (4 plane) come from
// s.scales / s.noise_seeds, and z is drawn at the index within the sample. The arithmetic is the same expression.
// GROUPS = 3 (InstructPix2Pix, DESIGN §7 f10): eu = e_U, ec = e_I and ec + count = e_T, and the guidance is
// pred = e_U + s_T (e_T - e_I) + s_I (e_I - e_U) with scale = s_T, scale_i = s_I, left to right with _rn intrinsics; the UNet input
// batch holds the latent three times.
template <int KIND, bool BLEND, bool PER_SAMPLE = false, int GROUPS = 2>
__device__ __forceinline__ void cfg_step(const float* __restrict__ eu, const float* __restrict__ ec, float* __restrict__ lat,
                                         long long count, float scale, float sqrt_1m_at, float sqrt_at, float sqrt_aprev,
                                         float dir_coef, const float* __restrict__ z0, const float* __restrict__ e0,
                                         const float* __restrict__ w, int plane, const SamplerStep& s, float scale_i = 0.f) {
  pdl_enter();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    const float u = eu[i], c = ec[i];
    float sc = scale;
    long long zi = i;  // index of z in its stream
    uint32_t k0 = s.k0, k1 = s.k1;
    if constexpr (PER_SAMPLE) {
      const long long smp = i / (4ll * plane);
      sc = s.scales[smp];
      if constexpr (KIND == STEP_DDIM_ETA) {
        zi = i - smp * 4ll * plane;
        step_noise_keys(s.noise_seeds[smp], s.t, &k0, &k1);
      }
    }
    float pred;
    if constexpr (GROUPS == 3)
      pred = __fadd_rn(__fadd_rn(u, __fmul_rn(sc, __fsub_rn(ec[i + count], c))), __fmul_rn(scale_i, __fsub_rn(c, u)));
    else
      pred = u + (c - u) * sc;                            // stablediffusion/mod.rs:190-191
    const float x = lat[i];
    const float x0 = (x - pred * sqrt_1m_at) / sqrt_at;   // :152
    float nl;
    if constexpr (KIND == STEP_DDIM) {
      nl = x0 * sqrt_aprev + pred * dir_coef;             // :153-155 (sigma = 0)
    } else if constexpr (KIND == STEP_DDIM_ETA) {         // :153-155 with sigma = s
      nl = __fadd_rn(__fadd_rn(__fmul_rn(sqrt_aprev, x0), __fmul_rn(dir_coef, pred)), __fmul_rn(s.s, randn_at(zi, k0, k1)));
    } else {
      const float d = s.second ? __fsub_rn(__fmul_rn(s.c1, x0), __fmul_rn(s.c2, s.hist[i])) : x0;
      s.hist[i] = x0;
      nl = __fadd_rn(__fmul_rn(s.cx, x), __fmul_rn(s.cd, d));
    }
    if constexpr (BLEND) {
      const float ka = KIND == STEP_DDIM ? sqrt_aprev : s.ka, kb = KIND == STEP_DDIM ? dir_coef : s.kb;
      const int p = (int)(i % plane);
      const float wi = w[(i / (4ll * plane)) * plane + p];
      const float known = __fadd_rn(__fmul_rn(ka, z0[i]), __fmul_rn(kb, e0[i]));
      nl = __fadd_rn(__fmul_rn(wi, nl), __fmul_rn(__fsub_rn(1.0f, wi), known));
    }
    lat[i] = nl;
    lat[i + count] = nl;  // the UNet input batch holds the latent twice (uncond half | cond half)
    if constexpr (GROUPS == 3) lat[i + 2 * count] = nl;
  }
}
// GROUPS = 3 reads e_I and e_T from one eps [3][count] at eu; the two-group kinds take ec from the launcher
template <int KIND, bool BLEND, bool PER_SAMPLE, int GROUPS>
__global__ void cfg_step_kernel(const float* __restrict__ eu, const float* __restrict__ ec, float* __restrict__ lat,
                                long long count, float scale, float sqrt_1m_at, float sqrt_at, float sqrt_aprev, float dir_coef,
                                float scale_i, const float* __restrict__ z0, const float* __restrict__ e0,
                                const float* __restrict__ w, int plane, const SamplerStep s) {
  cfg_step<KIND, BLEND, PER_SAMPLE, GROUPS>(eu, GROUPS == 3 ? eu + count : ec, lat, count, scale, sqrt_1m_at, sqrt_at, sqrt_aprev,
                                            dir_coef, z0, e0, w, plane, s, scale_i);
}
// the five instantiations of one kind: three groups (no blend, uniform), or two groups with or without blend and per-sample inputs
template <int KIND>
static void cfg_step_go(const CfgStepArgs& a, dim3 grid, cudaStream_t st) {
  const bool blend = a.w != nullptr, per_sample = a.s.scales != nullptr;
  auto go = [&](auto kernel) {
    launch_k(kernel, grid, dim3(256), 0, st, a.eu, a.ec, a.lat, a.count, a.scale, a.sqrt_1m_at, a.sqrt_at, a.sqrt_aprev, a.dir_coef,
             a.scale_i, a.z0, a.e0, a.w, a.plane, a.s);
  };
  if (a.groups == 3)
    go(cfg_step_kernel<KIND, false, false, 3>);
  else if (per_sample)
    blend ? go(cfg_step_kernel<KIND, true, true, 2>) : go(cfg_step_kernel<KIND, false, true, 2>);
  else
    blend ? go(cfg_step_kernel<KIND, true, false, 2>) : go(cfg_step_kernel<KIND, false, false, 2>);
}
void cfg_step_launch(const CfgStepArgs& a, cudaStream_t st) {
  const bool blend = a.w != nullptr, per_sample = a.s.scales != nullptr;
  SDB_CHECK(a.groups == 2 || (a.groups == 3 && !blend && !per_sample), "cfg_step_launch: groups");
  SDB_CHECK(!per_sample || (a.plane > 0 && (a.kind != STEP_DDIM_ETA || a.s.noise_seeds)), "cfg_step_launch: per-sample inputs");
  int grid = (int)((a.count + 255) / 256);
  if (grid > g_num_sms * 8) grid = g_num_sms * 8;
  if (a.kind == STEP_DDIM)
    cfg_step_go<STEP_DDIM>(a, dim3(grid), st);
  else if (a.kind == STEP_DDIM_ETA)
    cfg_step_go<STEP_DDIM_ETA>(a, dim3(grid), st);
  else if (a.kind == STEP_DPMPP_2M)
    cfg_step_go<STEP_DPMPP_2M>(a, dim3(grid), st);
  else
    SDB_CHECK(false, "cfg_step_launch: kind");
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ img2img staging
// u8 HWC RGB [nb][Hp][Wp][3] -> the encoder's input [nb][4][Hp][Wp], x = v / 127.5 - 1 (the inverse of latent_to_image's
// (x + 1) / 2 * 255), fourth plane zero
__global__ void u8_to_enc_input_kernel(const uint8_t* __restrict__ rgb, long long plane, long long total, float* __restrict__ out) {
  pdl_enter();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % plane, r = i / plane;
    const int ch = (int)(r % 4);
    const long long s = r / 4;
    out[i] = ch == 3 ? 0.f : __fsub_rn(__fdiv_rn((float)rgb[(s * plane + p) * 3 + ch], 127.5f), 1.0f);
  }
}
void u8_to_enc_input_launch(const uint8_t* rgb, int nb, int Hp, int Wp, float* out, cudaStream_t st) {
  const long long plane = (long long)Hp * Wp, total = (long long)nb * 4 * plane;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  launch_k(u8_to_enc_input_kernel, dim3(grid), dim3(256), 0, st, rgb, plane, total, out);
  SDB_CUDA(cudaGetLastError());
}

// Once per img2img call. Latent elements i < count: z0 *= 0.18215 in place, start latent sa z0 + sb eps into both halves of the
// UNet input batch. Then, with a mask, one thread per latent cell j < n*H*W: w = (sum of the 8x8 mask block) / (64 * 255).
__global__ void img2img_prep_kernel(float* __restrict__ z0, const float* __restrict__ eps, float* __restrict__ xb, long long count,
                                    float sa, float sb, const uint8_t* __restrict__ mask, float* __restrict__ w, int H, int W) {
  pdl_enter();
  const long long cells = mask ? count / 4 : 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count + cells; i += (long long)gridDim.x * blockDim.x) {
    if (i < count) {
      const float z = __fmul_rn(z0[i], 0.18215f);
      const float x = __fadd_rn(__fmul_rn(sa, z), __fmul_rn(sb, eps[i]));
      z0[i] = z;
      xb[i] = x;
      xb[i + count] = x;
    } else {
      const long long j = i - count;
      const int x = (int)(j % W), y = (int)((j / W) % H);
      const long long s = j / ((long long)H * W);
      const uint8_t* m = mask + (s * 8 * H + 8 * y) * 8 * W + 8 * x;
      int sum = 0;
      for (int r = 0; r < 8; ++r)
        for (int q = 0; q < 8; ++q) sum += m[(long long)r * 8 * W + q];
      w[j] = __fdiv_rn((float)sum, 16320.0f);
    }
  }
}
void img2img_prep_launch(float* z0, const float* eps, float* xb, long long count, float sa, float sb, const uint8_t* mask, float* w,
                         int H, int W, cudaStream_t st) {
  const long long total = count + (mask ? count / 4 : 0);
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 8) grid = g_num_sms * 8;
  launch_k(img2img_prep_kernel, dim3(grid), dim3(256), 0, st, z0, eps, xb, count, sa, sb, mask, w, H, W);
  SDB_CUDA(cudaGetLastError());
}

// 9-channel inpainting (DESIGN §7 f9), once per call. Elements i < nb*4*plane: the encoder input of the masked image,
// x_m = (mask >= 128) ? 0 : fl(fl(v / 127.5) - 1), fourth plane zero (u8_to_enc_input's layout). Then one thread per latent cell
// j < nb*H*W: the latent mask m[8h][8w] >= 128 (nearest pick), 1 or 0, into channel 0 of cond [nb,5,H,W].
__global__ void inpaint_prep_kernel(const uint8_t* __restrict__ rgb, const uint8_t* __restrict__ mask, int Hp, int Wp, long long count,
                                    float* __restrict__ out, float* __restrict__ cond) {
  pdl_enter();
  const long long plane = (long long)Hp * Wp;
  const int H = Hp / 8, W = Wp / 8;
  const long long cells = count / (4 * 64);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count + cells; i += (long long)gridDim.x * blockDim.x) {
    if (i < count) {
      const long long p = i % plane, r = i / plane;
      const int ch = (int)(r % 4);
      const long long s = r / 4;
      const bool hole = mask[s * plane + p] >= 128;
      out[i] = (ch == 3 || hole) ? 0.f : __fsub_rn(__fdiv_rn((float)rgb[(s * plane + p) * 3 + ch], 127.5f), 1.0f);
    } else {
      const long long j = i - count;
      const int xx = (int)(j % W), yy = (int)((j / W) % H);
      const long long s = j / ((long long)H * W);
      cond[s * 5 * H * W + (long long)yy * W + xx] = mask[s * plane + (long long)(8 * yy) * Wp + 8 * xx] >= 128 ? 1.f : 0.f;
    }
  }
}
void inpaint_prep_launch(const uint8_t* rgb, const uint8_t* mask, int nb, int Hp, int Wp, float* enc_in, float* cond,
                         cudaStream_t st) {
  const long long count = (long long)nb * 4 * Hp * Wp, total = count + count / 256;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  launch_k(inpaint_prep_kernel, dim3(grid), dim3(256), 0, st, rgb, mask, Hp, Wp, count, enc_in, cond);
  SDB_CUDA(cudaGetLastError());
}

__global__ void cfg_combine_kernel(const float* __restrict__ eu, const float* __restrict__ ec, long long count, float scale,
                                   float* __restrict__ pred) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
    pred[i] = eu[i] + (ec[i] - eu[i]) * scale;  // stablediffusion/mod.rs:190-191
}
void cfg_combine_launch(const float* eps_u, const float* eps_c, long long count, float scale, float* pred, cudaStream_t st) {
  int grid = (int)((count + 255) / 256);
  if (grid > g_num_sms * 8) grid = g_num_sms * 8;
  cfg_combine_kernel<<<grid, 256, 0, st>>>(eps_u, eps_c, count, scale, pred);
  SDB_CUDA(cudaGetLastError());
}

__global__ void to_rgb8_kernel(const float* __restrict__ img, int HW, long long total, uint8_t* __restrict__ rgb) {
  pdl_enter();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % 3);
    const long long r = i / 3;
    const int p = int(r % HW);
    const long long n = r / HW;
    float v = img[(n * 3 + c) * HW + p];
    v = (v + 1.0f) / 2.0f * 255.0f;             // stablediffusion/mod.rs:79-84
    // :96  v.to_f64().min(255.0).max(0.0) as u8  (NaN -> min gives 255)
    float m = (v != v) ? 255.0f : fminf(v, 255.0f);
    m = fmaxf(m, 0.0f);
    rgb[i] = (uint8_t)m;                        // truncation toward zero
  }
}
void to_rgb8_launch(const float* img_nchw, int n, int H, int W, uint8_t* rgb, cudaStream_t st) {
  const long long total = (long long)n * 3 * H * W;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  to_rgb8_kernel<<<grid, 256, 0, st>>>(img_nchw, H * W, total, rgb);
  SDB_CUDA(cudaGetLastError());
}


__global__ void randn_kernel(float* __restrict__ x, long long count, uint32_t k0, uint32_t k1) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
    x[i] = randn_at(i, k0, k1);
}
static void randn_keys_launch(float* x, long long count, uint32_t k0, uint32_t k1, cudaStream_t st) {
  int grid = (int)((count + 255) / 256);
  if (grid > g_num_sms * 8) grid = g_num_sms * 8;
  randn_kernel<<<grid, 256, 0, st>>>(x, count, k0, k1);
  SDB_CUDA(cudaGetLastError());
}
void randn_launch(float* x, long long count, uint64_t seed, cudaStream_t st) {
  uint32_t k0, k1;
  init_noise_keys(seed, &k0, &k1);
  randn_keys_launch(x, count, k0, k1, st);
}
__global__ void randn_seeds_kernel(float* __restrict__ x, long long per, long long count, const uint64_t* __restrict__ seeds) {
  pdl_enter();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    const long long s = i / per;
    uint32_t k0, k1;
    init_noise_keys(seeds[s], &k0, &k1);
    x[i] = randn_at(i - s * per, k0, k1);
  }
}
void randn_seeds_launch(float* x, int n, long long per, const uint64_t* seeds, cudaStream_t st) {
  const long long count = (long long)n * per;
  int grid = (int)((count + 255) / 256);
  if (grid > g_num_sms * 8) grid = g_num_sms * 8;
  launch_k(randn_seeds_kernel, dim3(grid), dim3(256), 0, st, x, per, count, seeds);
  SDB_CUDA(cudaGetLastError());
}

__global__ void stage_cfg_context_kernel(const float* __restrict__ cond, int L, const float* __restrict__ uncond, long long ustride,
                                         const int* __restrict__ lens, int n, int Lpad, long long total, float* __restrict__ out) {
  pdl_enter();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % 768);
    const long long rr = i / 768;
    const int r = (int)(rr % Lpad), b = (int)(rr / Lpad);
    float v = 0.f;
    if (r < lens[b])
      v = b < n ? uncond[b * ustride + (long long)r * 768 + col] : cond[((long long)(b - n) * L + r) * 768 + col];
    out[i] = v;
  }
}
void stage_cfg_context_launch(const float* cond, int L, const float* uncond, long long ustride, const int* lens, int n, int Lpad,
                              float* out, cudaStream_t st, int groups) {
  // groups - 1 unconditional groups (rows b < (groups - 1) n) read uncond[b * ustride], then one prompt group
  const long long total = (long long)groups * n * Lpad * 768;
  n *= groups - 1;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  launch_k(stage_cfg_context_kernel, dim3(grid), dim3(256), 0, st, cond, L, uncond, ustride, lens, n, Lpad, total, out);
  SDB_CUDA(cudaGetLastError());
}
void step_noise_launch(float* x, long long count, uint64_t seed, int t, cudaStream_t st) {
  uint32_t k0, k1;
  step_noise_keys(seed, t, &k0, &k1);
  randn_keys_launch(x, count, k0, k1, st);
}

// ============================================================ weight packing
__global__ void pack_conv_kernel(const float* __restrict__ w, int Cout, int Cin, int kk, __half* hi, __half* lo) {
  const long long total = (long long)Cout * kk * Cin;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % Cin);
    const long long r = i / Cin;
    const int tap = int(r % kk);
    const long long co = r / kk;
    split_store1(w[(co * Cin + c) * kk + tap], hi, lo, (size_t)i);
  }
}
void pack_conv_launch(const float* w, int Cout, int Cin, int ksize, Half2Ptr out, cudaStream_t st) {
  const long long total = (long long)Cout * ksize * ksize * Cin;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  pack_conv_kernel<<<grid, 256, 0, st>>>(w, Cout, Cin, ksize * ksize, out.hi, out.lo);
  SDB_CUDA(cudaGetLastError());
}

// nearest-2x upsample folded into the following 3x3 conv: output phase (a,b) in {0,1}^2 sees a 2x2 window of
// the low-res source; window tap (i,j) accumulates the 3x3 taps that land on the same source pixel:
//   a=0: rows {0} -> i=0, {1,2} -> i=1 ;  a=1: rows {0,1} -> i=0, {2} -> i=1   (same for columns)
__global__ void pack_conv_up2_kernel(const float* __restrict__ w, int Cout, int Cin, __half* hi, __half* lo) {
  const long long total = (long long)4 * Cout * 4 * Cin;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % Cin);
    long long r = i / Cin;
    const int wt = int(r % 4);
    r /= 4;
    const int co = int(r % Cout);
    const int phase = int(r / Cout);
    const int a = phase >> 1, b = phase & 1, ti = wt >> 1, tj = wt & 1;
    float acc = 0.f;
    for (int kh = 0; kh < 3; ++kh) {
      const int ii = (a == 0) ? (kh == 0 ? 0 : 1) : (kh == 2 ? 1 : 0);
      if (ii != ti) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int jj = (b == 0) ? (kw == 0 ? 0 : 1) : (kw == 2 ? 1 : 0);
        if (jj != tj) continue;
        acc += w[(((size_t)co * Cin + c) * 3 + kh) * 3 + kw];
      }
    }
    split_store1(acc, hi, lo, (size_t)i);
  }
}
void pack_conv_up2_launch(const float* w, int Cout, int Cin, Half2Ptr out, cudaStream_t st) {
  const long long total = (long long)16 * Cout * Cin;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  pack_conv_up2_kernel<<<grid, 256, 0, st>>>(w, Cout, Cin, out.hi, out.lo);
  SDB_CUDA(cudaGetLastError());
}

__global__ void pack_linear_kernel(const float* __restrict__ w, int in, int out, int ldw, int col0, __half* hi, __half* lo,
                                   int row_offset, const float* __restrict__ in_scale) {
  // tiled transpose [in][out] -> [out][in]; in_scale (optional) multiplies input feature i: a LayerNorm's gamma folded into
  // the weights of the GEMM that consumes the normalised tensor
  __shared__ float tile[32][33];
  const int o0 = blockIdx.x * 32, i0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int i = i0 + r, o = o0 + threadIdx.x;
    tile[r][threadIdx.x] = (i < in && o < out) ? w[(size_t)i * ldw + col0 + o] * (in_scale ? in_scale[i] : 1.0f) : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int o = o0 + r, i = i0 + threadIdx.x;
    if (o < out && i < in) split_store1(tile[threadIdx.x][r], hi, lo, (size_t)(row_offset + o) * in + i);
  }
}
void pack_linear_launch(const float* w, int in, int out, Half2Ptr dst, int row_offset, cudaStream_t st, int ldw,
                        int col0, const float* in_scale) {
  dim3 grid(ceil_div(out, 32), ceil_div(in, 32)), block(32, 8);
  pack_linear_kernel<<<grid, block, 0, st>>>(w, in, out, ldw ? ldw : out, col0, dst.hi, dst.lo, row_offset, in_scale);
  SDB_CUDA(cudaGetLastError());
}

// row sums of a packed fp16 matrix [rows][K]: s_hi[r] = sum_k hi[r][k], s_full[r] = sum_k (hi + lo)[r][k] (fp32 accumulation
// in a fixed order: one warp per row, lanes stride K, xor-tree) — the "u" vector of a LayerNorm folded into a GEMM: it must be
// the sum of exactly the values the tensor cores multiply, or the mean would not cancel
__global__ void __launch_bounds__(256) rowsum_f16_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, int rows,
                                                         int K, float* __restrict__ s_hi, float* __restrict__ s_full) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float a = 0.f, b = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float h = __half2float(hi[(size_t)row * K + k]);
    a += h;
    b += h + (lo ? __half2float(lo[(size_t)row * K + k]) : 0.f);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o), b += __shfl_xor_sync(0xffffffffu, b, o);
  if (lane == 0) {
    if (s_hi) s_hi[row] = a;
    if (s_full) s_full[row] = b;
  }
}
void rowsum_f16_launch(Half2Ptr m, int rows, int K, float* s_hi, float* s_full, cudaStream_t st) {
  rowsum_f16_kernel<<<ceil_div(rows, 8), 256, 0, st>>>(m.hi, m.lo, rows, K, s_hi, s_full);
  SDB_CUDA(cudaGetLastError());
}

__global__ void pack_geglu_kernel(const float* __restrict__ w, const float* __restrict__ b, int in, int h4, int half_tile,
                                  __half* hi, __half* lo, float* bias_packed, const float* __restrict__ in_scale) {
  // packed row pr in [0, 2*h4): tile j = pr / (2*half_tile); within tile q = pr % (2*half_tile);
  // q < half_tile -> x column j*half_tile + q ; else gate column h4 + j*half_tile + (q - half_tile)
  const long long total = (long long)2 * h4 * in;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int i = int(idx % in);
    const int pr = int(idx / in);
    const int j = pr / (2 * half_tile), q = pr % (2 * half_tile);
    const int col = (q < half_tile) ? j * half_tile + q : h4 + j * half_tile + (q - half_tile);
    split_store1(w[(size_t)i * (2 * h4) + col] * (in_scale ? in_scale[i] : 1.0f), hi, lo, (size_t)idx);
    if (i == 0 && bias_packed) bias_packed[pr] = b[col];
  }
}
void pack_geglu_launch(const float* w, const float* b, int in, int h4, int half_tile, Half2Ptr dst, float* bias_packed,
                       cudaStream_t st, const float* in_scale) {
  const long long total = (long long)2 * h4 * in;
  int grid = (int)((total + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  pack_geglu_kernel<<<grid, 256, 0, st>>>(w, b, in, h4, half_tile, dst.hi, dst.lo, bias_packed, in_scale);
  SDB_CUDA(cudaGetLastError());
}

__global__ void pack_small_cout_kernel(const float* __restrict__ w, int Cout, int Cin, float* __restrict__ out) {
  const int total = Cout * 9 * Cin;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % Cin, tap = (i / Cin) % 9, co = i / (9 * Cin);
    out[i] = w[((size_t)co * Cin + c) * 9 + tap];
  }
}
void pack_small_cout_launch(const float* w, int Cout, int Cin, float* out, cudaStream_t st) {
  pack_small_cout_kernel<<<ceil_div(Cout * 9 * Cin, 256), 256, 0, st>>>(w, Cout, Cin, out);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ row softmax (VAE attention, 1 head, d = 512)
// P[r][:] = softmax(S[r][:] * scale) -> fp16 hi(/lo); one CTA per row, row kept in registers
template <int PER>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ S, int cols, float scale_log2, __half* __restrict__ hi,
                    __half* __restrict__ lo) {
  __shared__ float red[8];
  const size_t row = blockIdx.x;
  const float* sr = S + row * cols;
  float v[PER];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int i = threadIdx.x + k * 256;
    v[k] = i < cols ? sr[i] * scale_log2 : -INFINITY;
    mx = fmaxf(mx, v[k]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) mx = fmaxf(mx, red[k]);
  __syncthreads();
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    v[k] = exp2f(v[k] - mx);
    sum += v[k];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) sum += red[k];
  const float inv = 1.0f / sum;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int i = threadIdx.x + k * 256;
    if (i < cols) split_store1(v[k] * inv, hi, lo, row * cols + i);
  }
}
int softmax_rows_launch(const float* S, long long rows, int cols, float scale, Half2Ptr out, cudaStream_t st) {
  const float sl2 = scale * 1.4426950408889634f;
  int per;
  if (cols <= 4096)
    softmax_rows_kernel<16><<<(unsigned)rows, 256, 0, st>>>(S, cols, sl2, out.hi, out.lo), per = 16;
  else if (cols <= kSoftmaxRowsMax)
    softmax_rows_kernel<36><<<(unsigned)rows, 256, 0, st>>>(S, cols, sl2, out.hi, out.lo), per = 36;
  else
    throw Error("softmax_rows: row too long");
  SDB_CUDA(cudaGetLastError());
  return per;
}

// ============================================================ synthetic weights
__global__ void synth_fill_kernel(float* __restrict__ dst, long long count, uint32_t key, float bound, float offset) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t h = mix32((uint32_t)i ^ key);
    const float u = (float)(h >> 8) * (1.0f / 16777216.0f);
    // (u*2 - 1) is exact; one rounding for *bound, one for +offset — same as the numpy generator
    dst[i] = __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(u, 2.0f), 1.0f), bound), offset);
  }
}
void synth_fill_launch(float* dst, long long count, uint32_t key, float bound, float offset, cudaStream_t st) {
  int grid = (int)((count + 255) / 256);
  if (grid > g_num_sms * 16) grid = g_num_sms * 16;
  synth_fill_kernel<<<grid, 256, 0, st>>>(dst, count, key, bound, offset);
  SDB_CUDA(cudaGetLastError());
}

// every tensor of the registry in ONE launch: a block walks 64K-element chunks; chunk -> tensor by binary search over the
// chunk prefix sums (one launch per tensor — 1131 of them — used to drown every other kernel in a profiler's launch list)
__global__ void __launch_bounds__(256)
synth_fill_table_kernel(float* __restrict__ base, const SynthDesc* __restrict__ desc, int ntensors, long long nchunks) {
  constexpr long long CH = 65536;
  for (long long ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    int lo = 0, hi = ntensors - 1;
    while (lo < hi) {  // last tensor whose first chunk is <= ch
      const int mid = (lo + hi + 1) >> 1;
      if (desc[mid].chunk0 <= ch) lo = mid; else hi = mid - 1;
    }
    const SynthDesc d = desc[lo];
    const long long i0 = (ch - d.chunk0) * CH, i1 = min(d.count, i0 + CH);
    float* dst = base + d.offset;
    for (long long i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
      const uint32_t h = mix32((uint32_t)i ^ d.key);
      const float u = (float)(h >> 8) * (1.0f / 16777216.0f);
      dst[i] = __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(u, 2.0f), 1.0f), d.bound), d.shift);
    }
  }
}
void synth_fill_table_launch(float* base, const SynthDesc* d_desc, int ntensors, long long nchunks, cudaStream_t st) {
  const int grid = (int)std::min<long long>(nchunks, g_num_sms * 16);
  synth_fill_table_kernel<<<grid, 256, 0, st>>>(base, d_desc, ntensors, nchunks);
  SDB_CUDA(cudaGetLastError());
}

// ============================================================ LoRA merge (DESIGN §7 f8)
// One CTA = one 64 x 64 tile of one tensor's W_eff (tile -> tensor by binary search over the tile prefix sums). For each term the
// up / down chunks of 32 ranks are staged in shared memory as [k][64 rows] and [k][64 cols]; a thread owns rows ty + 16 i and
// cols tx + 16 j (i, j < 4), so for a fixed (i, j) a half-warp reads and writes 16 consecutive elements of the row-major tensor.
// The term's dot product d runs k-ascending in fp32 FMAs and folds into tot with one more FMA: the order is fixed, so the
// result is reproducible, and with dyadic factors exact.
constexpr int kLoraTile = 64, kLoraKc = 32;
__global__ void __launch_bounds__(256)
lora_merge_kernel(const LoraTensorDesc* __restrict__ tens, int ntensors, const LoraTermDesc* __restrict__ terms) {
  __shared__ float sa[kLoraKc][kLoraTile + 1];  // [k][row of the tile]
  __shared__ float sb[kLoraKc][kLoraTile + 1];  // [k][col of the tile]
  const long long tile = blockIdx.x;
  int lo = 0, hi = ntensors - 1;
  while (lo < hi) {  // last tensor whose first tile is <= tile
    const int mid = (lo + hi + 1) >> 1;
    if (tens[mid].tile0 <= tile) lo = mid; else hi = mid - 1;
  }
  const LoraTensorDesc t = tens[lo];
  const int tl = (int)(tile - t.tile0);
  const int row0 = (tl / t.tiles_c) * kLoraTile, col0 = (tl % t.tiles_c) * kLoraTile;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  // conv: rows index out (up), cols index fan-in (down); Linear [in][out]: rows index fan-in (down), cols index out (up)
  const int fan_in = t.transposed ? t.rows : t.cols;
  float tot[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) tot[i][j] = 0.f;
  for (int q = 0; q < t.nterms; ++q) {
    const LoraTermDesc tm = terms[t.term0 + q];
    float (*su)[kLoraTile + 1] = t.transposed ? sb : sa;  // where the up chunk goes
    float (*sd)[kLoraTile + 1] = t.transposed ? sa : sb;  // where the down chunk goes
    const int u0 = t.transposed ? col0 : row0, d0 = t.transposed ? row0 : col0;
    const int u_lim = t.transposed ? t.cols : t.rows, d_lim = t.transposed ? t.rows : t.cols;
    float d[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) d[i][j] = 0.f;
    for (int k0 = 0; k0 < tm.r; k0 += kLoraKc) {
      const int kc = min(kLoraKc, tm.r - k0);
      __syncthreads();  // the previous chunk has been consumed
      for (int e = threadIdx.x; e < kLoraKc * kLoraTile; e += 256) {
        const int kk = e % kLoraKc, i = e / kLoraKc;  // up [out][r]: consecutive threads walk k
        su[kk][i] = (kk < kc && u0 + i < u_lim) ? tm.up[(long long)(u0 + i) * tm.r + k0 + kk] : 0.f;
        const int kd = e / kLoraTile, id = e % kLoraTile;  // down [r][fan-in]: consecutive threads walk fan-in
        sd[kd][id] = (kd < kc && d0 + id < d_lim) ? tm.down[(long long)(k0 + kd) * fan_in + d0 + id] : 0.f;
      }
      __syncthreads();
      for (int kk = 0; kk < kc; ++kk) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = sa[kk][ty + 16 * i], b[i] = sb[kk][tx + 16 * i];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) d[i][j] = __fmaf_rn(a[i], b[j], d[i][j]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) tot[i][j] = __fmaf_rn(tm.s, d[i][j], tot[i][j]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = row0 + ty + 16 * i;
    if (r >= t.rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int cc = col0 + tx + 16 * j;
      if (cc < t.cols) {
        const long long idx = (long long)r * t.cols + cc;
        t.out[idx] = __fadd_rn(t.base[idx], tot[i][j]);
      }
    }
  }
}
void lora_merge_launch(const LoraTensorDesc* d_tensors, int ntensors, const LoraTermDesc* d_terms, long long ntiles, cudaStream_t st) {
  SDB_CHECK(ntiles > 0 && ntiles < (1LL << 31), "lora merge: tile count");
  lora_merge_kernel<<<(unsigned)ntiles, 256, 0, st>>>(d_tensors, ntensors, d_terms);
  SDB_CUDA(cudaGetLastError());
}

}  // namespace sdb
