// gemm_tc.cu — wgmma implicit-GEMM for conv3x3 / conv1x1 / Linear on sm_90a.
//
// Replaces burn nn::conv::Conv2d / nn::Linear on the reference hot path
// (call sites: src/model/unet/mod.rs:716,726,729 ResBlock convs; :468,479 proj_in/out;
//  :645-651 q/k/v/out; :580,553 GEGLU/ff; src/model/autoencoder/mod.rs:513-528, 567-606).
//
// gemm_tc_kernel: one CTA = one 128 x BN output tile (x one K split). Warp roles:
//   warpgroup 0    : TMA producer (warp 0: cp.async.bulk.tensor 5-D activation boxes + 2-D weight boxes; warps 1-3 idle)
//   warpgroups 1-2 : consumers. Each issues wgmma m64nBNk16 (fp16 x fp16 -> fp32 in registers) for 64 of the 128 rows, then
//                    both write the accumulator to shared memory as a row-major fp32 image and run the epilogue from it
//                    (bias / residual / statistics -> global)
// gemm_tc_persistent_kernel (LayerNorm-consuming and GEGLU epilogues): the same roles, at most one CTA per SM running a
// sequence of tiles, the epilogue straight from the accumulator registers while the producer loads the next tile.
// Multi-pass products (PASSES = 2, 3) add the low-order fp16 halves of the operands
// (A_lo*B_hi, A_hi*B_lo) into the same accumulator for fp32-class accuracy.
#include "gemm_tc.cuh"

#include <algorithm>
#include <cstring>

namespace sdb {

static constexpr int BM = 128;
static constexpr int BK = 64;  // fp16 elements per k chunk = 128 bytes = one swizzle row
static constexpr int A_TILE_BYTES = BM * BK * 2;

template <int BN, int PASSES>
struct StageLayout {
  static constexpr int B_TILE_BYTES = BN * BK * 2;
  static constexpr int A_TILES = PASSES >= 2 ? 2 : 1;
  static constexpr int B_TILES = PASSES >= 3 ? 2 : 1;
  static constexpr int BYTES = A_TILES * A_TILE_BYTES + B_TILES * B_TILE_BYTES;
};
// The epilogue's view of the accumulator: [128 rows][BN] fp32 in shared memory (over the idle pipeline stages), rows padded by
// 16 B so that the 128-bit reads of 4 rows x 32 columns per warp instruction are bank-conflict free; after it, 32 KB of scratch
// for the GroupNorm column sums.
template <int BN>
struct AccLayout {
  static constexpr int PITCH = (BN + 4) * 4;
  static constexpr int BYTES = BM * PITCH;
  static constexpr int GN_BYTES = 32 * 1024;
};
static constexpr int EW = 8;  // consumer / epilogue warps (two warpgroups)

// QuickGELU x*sigmoid(1.702x), the CLIP MLP activation (act = 1)
__device__ __forceinline__ float quick_gelu(float x) { return __fdividef(x, 1.0f + __expf(-1.702f * x)); }
// Activation + fp32 / fp16(hi,lo) stores of 4 consecutive columns of one output row. Deliberately NOT inlined: the epilogue
// runs once per CTA, so its cost is dominated by cold instruction fetch (ncu: stall_no_inst); one shared copy of this
// body instead of one per unrolled row keeps the epilogue's code footprint small.
__device__ __noinline__ void epilogue_store(float4 f, unsigned int o32, unsigned int o16, float* out_f32, __half* out_f16,
                                            __half* out_f16_lo, int act) {
  if (act == 1) f.x = quick_gelu(f.x), f.y = quick_gelu(f.y), f.z = quick_gelu(f.z), f.w = quick_gelu(f.w);
  if (out_f32) *reinterpret_cast<float4*>(out_f32 + o32) = f;
  if (out_f16) {
    const HalfPair2 s0 = split_f16x2(f.x, f.y), s1 = split_f16x2(f.z, f.w);
    __half2 h[2] = {s0.hi, s1.hi};
    *reinterpret_cast<uint2*>(out_f16 + o16) = *reinterpret_cast<uint2*>(h);
    if (out_f16_lo) {
      __half2 l[2] = {s0.lo, s1.lo};
      *reinterpret_cast<uint2*>(out_f16_lo + o16) = *reinterpret_cast<uint2*>(l);
    }
  }
}

// 4 x 4 transpose of 32-bit values inside each quad of lanes (q = lane % 4): lane q ends with {x[q] of lane 0, ..., x[q] of
// lane 3}. Two butterfly stages: lanes q and q ^ 1 swap the elements whose bit 0 differs from theirs (the 2 x 2 blocks
// transpose), then lanes q and q ^ 2 swap on bit 1 (the blocks change places). The register epilogue uses it to turn 4 column
// pairs per lane into 8 consecutive columns per lane.
__device__ __forceinline__ uint4 quad_transpose(uint32_t (&x)[4], int q) {
  const bool e = q & 1, f = q & 2;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const uint32_t v = __shfl_xor_sync(0xffffffffu, e ? x[2 * j] : x[2 * j + 1], 1);
    if (e) x[2 * j] = v; else x[2 * j + 1] = v;
  }
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const uint32_t v = __shfl_xor_sync(0xffffffffu, f ? x[c] : x[2 + c], 2);
    if (f) x[c] = v; else x[2 + c] = v;
  }
  return make_uint4(x[0], x[1], x[2], x[3]);
}

// 4 consecutive columns of a residual kept as an fp16 hi + lo pair, as fp32 hi + lo
__device__ __forceinline__ float4 res_pair4(const __half* hi, const __half* lo) {
  const uint2 h = *reinterpret_cast<const uint2*>(hi);
  const uint2 l = *reinterpret_cast<const uint2*>(lo);
  const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(&h.x)), h1 = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
  const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(&l.x)), l1 = __half22float2(*reinterpret_cast<const __half2*>(&l.y));
  return make_float4(h0.x + l0.x, h0.y + l0.y, h1.x + l1.x, h1.y + l1.y);
}

// Bucket reduction of the per-quarter column sums an epilogue left in shared memory (cs[q][col] = (sum, sumsq) of the 32 rows of
// lane quarter q), written as this tile's GroupNorm partials. `nq` quarters per image slice (4 = the whole tile is one image).
// which images the 128 rows of this tile belong to: g_tn images per tile (1, 2 or 4), the first one, the tile's index inside it
struct GnTile {
  int tn, img0, tile, nimg;
};
__device__ __forceinline__ GnTile gn_tile_of(const GemmParams& p, int n0, int th, int tw) {
  GnTile g;
  if (p.gn_rpi) {  // flattened rows: blockIdx.x is the row tile
    g.nimg = p.gn_nimg;
    if (p.gn_rpi >= BM)
      g.tn = 1, g.img0 = (tw * BM) / p.gn_rpi, g.tile = ((tw * BM) % p.gn_rpi) / BM;
    else
      g.tn = BM / p.gn_rpi, g.img0 = tw * g.tn, g.tile = 0;
  } else {
    g.tn = p.TN, g.img0 = n0, g.tile = th * p.tiles_w + tw, g.nimg = p.nimg;
  }
  return g;
}
__device__ __forceinline__ void gn_write_partials(const GemmParams& p, const float2* cs, int BN, int te, int nthreads, const GnTile g,
                                                  int col0, int z) {
  const int nbk_tile = BN / p.gn_bucket, nbk_total = p.N / p.gn_bucket;
  const int qpi = 4 / g.tn;  // lane quarters per image (1, 2 or 4 images per tile: checked by run_gemm)
  const int slot = p.gn_slot0 + g.tile * p.split_k + z;
  // thread = (bucket, quarter): 4 adjacent lanes hold the quarters of one bucket and combine them with shuffles in a fixed
  // order (nbk_tile * 4 <= 256 threads: BN <= 256, bucket >= 4); whole warps take part so that the shuffles are convergent
  (void)nthreads;
  if (te < ((nbk_tile * 4 + 31) & ~31)) {
    const int b = te >> 2, q = te & 3;
    float sm = 0.f, sq = 0.f;
    if (b < nbk_tile) {
      const float2* src = cs + q * BN + b * p.gn_bucket;
      for (int c = 0; c < p.gn_bucket; ++c) sm += src[c].x, sq += src[c].y;
    }
    if (qpi >= 2) sm += __shfl_xor_sync(0xffffffffu, sm, 1), sq += __shfl_xor_sync(0xffffffffu, sq, 1);
    if (qpi == 4) sm += __shfl_xor_sync(0xffffffffu, sm, 2), sq += __shfl_xor_sync(0xffffffffu, sq, 2);
    const int k = q / qpi, img = g.img0 + k, c0 = b * p.gn_bucket;
    if (b < nbk_tile && (q % qpi) == 0 && img < g.nimg && col0 + c0 < p.N) {
      float2* dst = reinterpret_cast<float2*>(p.gn_part) + ((size_t)img * p.gn_cap + slot) * nbk_total + (col0 + c0) / p.gn_bucket;
      *dst = make_float2(sm, sq);
    }
  }
}

// EPI selects what the epilogue does beside bias / residual / stores. It is a compile-time choice because the once-per-CTA
// epilogue is instruction-issue bound: statistics code that is merely skipped at run time still costs issue slots.
//   EPI_PLAIN  nothing more          EPI_GN   GroupNorm statistics of the output tensor (column sums per channel bucket)
//   EPI_LNS    LayerNorm row statistics of the output rows (partial sum / sum of squares per N-tile share)
//   EPI_LNC    the A operand is the RAW input of a LayerNorm whose gamma is folded into the weights: the normalisation is applied
//              here as a rank-1 correction, out = rstd_r * (acc - mean_r * u_c) + v_c  (u = column sums of the folded weights,
//              v = beta^T W + bias arrives as `bias`), from the row statistics the producer of A left (EPI_LNS)
//   EPI_GEGLU / EPI_GEGLU_LNC   x * gelu_erf(gate) on column-interleaved (x | gate) tiles (unet/mod.rs:578-592), without / with
//              the LayerNorm-consuming correction
enum : int { EPI_PLAIN = 0, EPI_GN = 1, EPI_LNS = 2, EPI_LNC = 3, EPI_GEGLU = 4, EPI_GEGLU_LNC = 5 };

template <int BN, int PASSES, int STAGES>
__host__ __device__ constexpr int region_bytes() {
  return STAGES * StageLayout<BN, PASSES>::BYTES > AccLayout<BN>::BYTES + AccLayout<BN>::GN_BYTES
             ? STAGES * StageLayout<BN, PASSES>::BYTES
             : AccLayout<BN>::BYTES + AccLayout<BN>::GN_BYTES;
}

template <int BN, int PASSES, int STAGES, int EPI>
__global__ void __launch_bounds__(128 + 32 * EW, 1)
gemm_tc_kernel(const __grid_constant__ GemmMaps maps, const GemmParams p) {
  static_assert(EPI == EPI_PLAIN || EPI == EPI_GN || EPI == EPI_LNS, "the register epilogues run in gemm_tc_persistent_kernel");
  constexpr bool kGN = EPI == EPI_GN, kLNS = EPI == EPI_LNS;
  using L = StageLayout<BN, PASSES>;
  constexpr int EG = EW / 4;                                    // warps sharing one 32-row quarter of the tile
  constexpr int CSTEP = 32 * EG;                                // column stride between the chunks of one warp
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle atoms
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + region_bytes<BN, PASSES, STAGES>());
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  long long* const dbg = (p.dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) ? p.dbg : nullptr;
  if (dbg && threadIdx.x == 0) dbg[0] = clock64();

  // ---- tile coordinates
  int mt = blockIdx.x;
  const int tw = mt % p.tiles_w;
  mt /= p.tiles_w;
  const int th = mt % p.tiles_h;
  const int tn = mt / p.tiles_h;
  const int w0 = tw * p.TW, h0 = th * p.TH, n0 = tn * p.TN;
  const int col0 = blockIdx.y * BN;

  const int main_iters = p.num_taps * p.kc;
  const int total_iters = main_iters + p.xkc;
  const int per_split = (total_iters + p.split_k - 1) / p.split_k;
  // grid.z is the K split — or, for the folded nearest-2x upsample conv (p.up2, never split), the output phase (a, b): the four
  // 2x2-tap phase convolutions of one layer run as ONE launch; phase shifts the taps, the weight rows and the output pixel
  const int up_a = p.up2 ? (int)(blockIdx.z >> 1) : 0, up_b = p.up2 ? (int)(blockIdx.z & 1) : 0;
  const int kz = p.up2 ? 0 : (int)blockIdx.z;
  const int b_row0 = col0 + (p.up2 ? (int)blockIdx.z * p.N : 0);  // first weight row of this tile (phase-major packing)
  const int it_begin = kz * per_split;
  const int it_end = min(total_iters, it_begin + per_split);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], EW);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&maps.a[0][0]);
    tma_prefetch_desc(&maps.b[0]);
    if (p.kc0 < p.kc) tma_prefetch_desc(&maps.a[1][0]);
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) dbg[1] = clock64();
  // Programmatic dependent launch: everything above overlapped the previous kernel's tail. From here on each role waits for the
  // previous kernel (griddepcontrol.wait) only where it first touches data that kernel may have written:
  //   producer : WEIGHTS are immutable, so the weight tiles of the first STAGES k-chunks are issued BEFORE the wait; activation
  //              tiles after it
  //   consumers: wait before the epilogue's first read of residual rows; all of this kernel's stores follow it
  if (warp == 0) {
    // ===================================================== TMA producer (one elected lane: see elect_one in common.cuh)
    if (elect_one()) {
      // iteration -> (activation source, channel chunk, tap shift) and the weight map / K coordinate that go with it
      auto load_b = [&](int it, int s) {
        const CUtensorMap* bm = it < main_iters ? maps.b : maps.bx;
        const int bk = (it < main_iters ? it : it - main_iters) * BK;
        uint8_t* sb = smem + s * L::BYTES + L::A_TILES * A_TILE_BYTES;
        tma_load_2d(sb, &bm[0], &full_bar[s], bk, b_row0);
        if (PASSES >= 3) tma_load_2d(sb + L::B_TILE_BYTES, &bm[1], &full_bar[s], bk, b_row0);
      };
      auto load_a = [&](int it, int s) {
        int src, c0, cw, ch, cp;
        if (it < main_iters) {
          const int tap = it / p.kc;
          const int cc = it - tap * p.kc;
          src = cc >= p.kc0 ? 1 : 0;
          c0 = (cc - (src ? p.kc0 : 0)) * BK;
          cw = w0 + p.tap_dw[tap] + up_b, ch = h0 + p.tap_dh[tap] + up_a, cp = p.tap_ph[tap];
        } else {
          const int e = it - main_iters;
          src = e >= p.xkc0 ? 3 : 2;
          c0 = (e - (src == 3 ? p.xkc0 : 0)) * BK;
          cw = w0, ch = h0, cp = 0;
        }
        uint8_t* st = smem + s * L::BYTES;
        tma_load_5d(st, &maps.a[src][0], &full_bar[s], c0, cw, ch, cp, n0);
        if (PASSES >= 2) tma_load_5d(st + A_TILE_BYTES, &maps.a[src][1], &full_bar[s], c0, cw, ch, cp, n0);
      };
      // ---- before the wait: weights only (the pipeline slots are all free: fresh barriers)
      const int npre = min(STAGES, it_end - it_begin);
      for (int i = 0; i < npre; ++i) {
        mbar_expect_tx(&full_bar[i], L::BYTES);
        load_b(it_begin + i, i);
      }
      pdl_wait();
      for (int i = 0; i < npre; ++i) load_a(it_begin + i, i);
      if (dbg) dbg[2] = clock64();
      // ---- steady state
      int s = npre == STAGES ? 0 : npre;
      uint32_t ph = npre == STAGES ? 1 : 0;
      for (int it = it_begin + npre; it < it_end; ++it) {
        mbar_wait(&empty_bar[s], ph ^ 1);
        mbar_expect_tx(&full_bar[s], L::BYTES);
        load_a(it, s);
        load_b(it, s);
        if (++s == STAGES) {
          s = 0;
          ph ^= 1;
        }
      }
    }
  } else if (warp >= 4) {
    // ===================================================== consumers: wgmma mainloop, then the epilogue
    pdl_wait();  // residual rows below may come from the previous kernel; every store of this kernel follows
    const int wg = (warp - 4) >> 2;  // rows [64 wg, 64 wg + 64) of the tile
    {
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int s = 0, prev = -1;
      uint32_t ph = 0;
      for (int it = it_begin; it < it_end; ++it) {
        mbar_wait(&full_bar[s], ph);
        if (dbg && threadIdx.x == 128 && it == it_begin) dbg[3] = clock64();
        const uint32_t a_hi = smem_u32(smem + s * L::BYTES) + wg * (64 * 128);
        const uint32_t a_lo = a_hi + A_TILE_BYTES;
        const uint32_t b_hi = smem_u32(smem + s * L::BYTES) + L::A_TILES * A_TILE_BYTES;
        const uint32_t b_lo = b_hi + L::B_TILE_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint32_t koff = k * 32;  // 16 fp16 = 32 bytes inside the 128B swizzle row
          const uint64_t da = make_sdesc_sw128(a_hi + koff);
          const uint64_t db = make_sdesc_sw128(b_hi + koff);
          Wgmma<BN>::template ss<0>(acc, da, db, 1);
          if (PASSES >= 2) Wgmma<BN>::template ss<0>(acc, make_sdesc_sw128(a_lo + koff), db, 1);
          if (PASSES >= 3) Wgmma<BN>::template ss<0>(acc, da, make_sdesc_sw128(b_lo + koff), 1);
        }
        wgmma_commit();
        // one group stays in flight: the products of the previous stage are complete, so its slot goes back to the producer
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == STAGES) {
          s = 0;
          ph ^= 1;
        }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (dbg && threadIdx.x == 128) dbg[4] = clock64();
      // every consumer's products are complete before the accumulator image overwrites the stages
      asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");
      float* img = reinterpret_cast<float*>(smem);
      const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BN / 2; j += 2) {
        const int row = r0 + 8 * ((j >> 1) & 1), col = 8 * (j >> 2) + 2 * (lane & 3);
        *reinterpret_cast<float2*>(img + row * (AccLayout<BN>::PITCH / 4) + col) = make_float2(acc[j], acc[j + 1]);
      }
      asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");
    }
    // The epilogue reads the accumulator image row-wise: warp w serves the 32-row quarter q = w % 4 and its share `half` of
    // the 32-column chunks. A row-per-thread store pattern would touch 32 cache lines per instruction, so rows are read and
    // written as 4 rows x 128 contiguous bytes per warp instruction.
    const int q = warp & 3;             // 32-row quarter of the tile this warp serves
    const int half = (warp - 4) >> 2;   // which share of the column chunks this warp owns (0..EG-1)
    const int r = q * 32 + lane;        // accumulator row
    const int pw = w0 + r % p.TW;
    const int phh = h0 + (r / p.TW) % p.TH;
    const int pn = n0 + r / (p.TW * p.TH);
    const int row_ok = ((pw < p.W) && (phh < p.H) && (pn < p.nimg)) ? 1 : 0;
    // output row index (< 2^31 rows); -1 marks a row outside the tensor
    const int m = row_ok ? ((pn * p.OH + phh * p.os + p.oa + up_a) * p.OW + pw * p.os + p.ob + up_b) : -1;

    // ---- work that needs no accumulator, done while the main loop runs: the element offsets of the 8 rows this lane
    // serves in every column chunk (rr = 4 i + sub), the bias of each chunk, and the first chunk's residual addends. The
    // epilogue is a chain of L2 round trips: everything issued here is off that chain.
    const int sub = lane >> 3;          // row within a group of 4
    const int cq = (lane & 7) * 4;      // 4-column group inside the 32-column chunk
    constexpr int NCHUNK = (BN + CSTEP - 1) / CSTEP;
    int mr8[8], ao[8];
    float4 bvs[NCHUNK], ad[8];
    const bool res_pair = p.res_hi != nullptr;  // the residual lives as an fp16 hi + lo pair (row stride ldc16)
    const bool plain = p.split_k == 1;
    {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + sub;
        const int mr = __shfl_sync(0xffffffffu, m, rr);
        mr8[i] = mr;
        ao[i] = res_pair ? mr * p.ldc16 : mr * p.ldc;
        ad[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < NCHUNK; ++j) {
        const int col = col0 + half * 32 + j * CSTEP + cq;
        bvs[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (plain && p.bias && half * 32 + j * CSTEP < BN && col < p.N) bvs[j] = *reinterpret_cast<const float4*>(p.bias + col);
      }
    }
    auto issue_addends = [&](int col) {
      if (col >= p.N) return;
      if (res_pair) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (mr8[i] >= 0) ad[i] = res_pair4(p.res_hi + (unsigned)(ao[i] + col), p.res_lo + (unsigned)(ao[i] + col));
        return;
      }
      if (p.residual == nullptr) return;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (mr8[i] >= 0) ad[i] = *reinterpret_cast<const float4*>(p.residual + (unsigned)(ao[i] + col));
    };
    // the residual may be produced by the previous kernel (always complete: stream order) or be this launch's own
    // output buffer written by an EARLIER launch (in-place accumulate): both are safe to read before the MMAs finish
    const bool pre_issued = plain;
    if (pre_issued) issue_addends(col0 + half * 32 + cq);

    pdl_trigger();  // the epilogue starts: the next kernel of the stream may begin its own prologue
    if (dbg && threadIdx.x == 128) dbg[5] = clock64();
    constexpr uint32_t TROW = AccLayout<BN>::PITCH;
    const uint32_t arow = smem_u32(smem) + q * 32 * TROW;  // row 32 q of the accumulator image
    auto unstage = [&](uint32_t t, int rr) {
      float4 f;
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(f.x), "=f"(f.y), "=f"(f.z), "=f"(f.w)
                   : "r"(t + rr * TROW + cq * 4)
                   : "memory");
      return f;
    };
    // element offsets fit 32 bits (run_gemm checks rows * ld < 2^31): one IMAD per row instead of 64-bit address chains
    // GroupNorm statistics of the output (p.gn_part): per-quarter column sums, in the scratch after the accumulator image
    float2* const gn_cs = reinterpret_cast<float2*>(smem + AccLayout<BN>::BYTES);
    const GnTile gnt = gn_tile_of(p, n0, th, tw);
    auto store_out = [&](float4 f, int mr, int col) {
      epilogue_store(f, (unsigned)(mr * p.ldc + col), (unsigned)(mr * p.ldc16 + col), p.out_f32, p.out_f16, p.out_f16_lo, p.act);
    };

    if (p.split_k > 1) {
      // raw partial sums -> workspace [split][M][N]
      const size_t Mtot = (size_t)p.nimg * p.OH * p.OW;
      float* wsbase = p.ws + (size_t)kz * Mtot * p.N;
#pragma unroll 1
      for (int c = half * 32; c < BN; c += CSTEP) {
        const int col = col0 + c + cq;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int rr = i * 4 + sub;
          const int mr = __shfl_sync(0xffffffffu, m, rr);
          if (mr >= 0 && col < p.N) __stcg(reinterpret_cast<float4*>(wsbase + (size_t)mr * p.N + col), unstage(arow + c * 4, rr));
        }
      }
      __threadfence();
      asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");  // all epilogue warps have published their part of the tile
      // Tile-level rendezvous of the split_k CTAs (all co-resident: run_gemm keeps ctas*split within one wave), then
      // every CTA folds its own slice of the tile rows in z order (deterministic) and runs the epilogue on it.
      unsigned int* tk = p.tickets + 2 * ((size_t)blockIdx.y * gridDim.x + blockIdx.x);
      if (warp == 4 && lane == 0) {
        atomicAdd(tk, 1u);
        const long long t0 = clock64();
        while (atomicAdd(tk, 0u) < (unsigned)p.split_k) {
          __nanosleep(32);
          if (clock64() - t0 > 4000000000ll) __trap();
        }
        __threadfence();
      }
      asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");
      {
        const int rows_per = (BM + p.split_k - 1) / p.split_k;
        const int r0 = kz * rows_per, r1 = min(BM, r0 + rows_per);
        constexpr int C4 = BN / 4;
        // thread -> (row lane, fixed 4-column group): a thread's GroupNorm column sums stay in registers across its rows
        constexpr int RL = (EW * 32) / C4;  // row lanes
        const int te = threadIdx.x - 128;
        const int rlane = te / C4, cg4 = te - rlane * C4;
        const int rpi = BM / gnt.tn;  // rows per image inside the tile
        float4* const gn_red = reinterpret_cast<float4*>(smem + AccLayout<BN>::BYTES);  // [RL][TN][C4][2] float4, <= 32 KB
#pragma unroll 1
        for (int k = 0; k < gnt.tn; ++k) {
        float4 gsum = make_float4(0.f, 0.f, 0.f, 0.f), gsq = gsum;
        const int row_a = max(r0, k * rpi), row_b = min(r1, (k + 1) * rpi);
#pragma unroll 1
        for (int rl = row_a + rlane; rlane < RL && rl < row_b; rl += RL) {
          const int col = col0 + cg4 * 4;
          const int qw = w0 + rl % p.TW, qh = h0 + (rl / p.TW) % p.TH, qn = n0 + rl / (p.TW * p.TH);
          if (qw < p.W && qh < p.H && qn < p.nimg && col < p.N) {
            const int mr = (qn * p.OH + qh * p.os + p.oa) * p.OW + qw * p.os + p.ob;
            // the addends first, then the partials four at a time: independent loads in flight together, summed in z order
            float4 bv = make_float4(0.f, 0.f, 0.f, 0.f), rs = bv;
            if (p.bias) bv = *reinterpret_cast<const float4*>(p.bias + col);
            if (p.residual) rs = *reinterpret_cast<const float4*>(p.residual + (size_t)mr * p.ldc + col);
            if (p.res_hi) rs = res_pair4(p.res_hi + (size_t)mr * p.ldc16 + col, p.res_lo + (size_t)mr * p.ldc16 + col);
            const float* wp = p.ws + (size_t)mr * p.N + col;
            const size_t zs = Mtot * p.N;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            int z = 0;
#pragma unroll 1
            for (; z + 4 <= p.split_k; z += 4) {
              const float4 v0 = __ldcg(reinterpret_cast<const float4*>(wp + (size_t)z * zs));
              const float4 v1 = __ldcg(reinterpret_cast<const float4*>(wp + (size_t)(z + 1) * zs));
              const float4 v2 = __ldcg(reinterpret_cast<const float4*>(wp + (size_t)(z + 2) * zs));
              const float4 v3 = __ldcg(reinterpret_cast<const float4*>(wp + (size_t)(z + 3) * zs));
              acc.x += v0.x, acc.y += v0.y, acc.z += v0.z, acc.w += v0.w;
              acc.x += v1.x, acc.y += v1.y, acc.z += v1.z, acc.w += v1.w;
              acc.x += v2.x, acc.y += v2.y, acc.z += v2.z, acc.w += v2.w;
              acc.x += v3.x, acc.y += v3.y, acc.z += v3.z, acc.w += v3.w;
            }
#pragma unroll 1
            for (; z < p.split_k; ++z) {
              const float4 v = __ldcg(reinterpret_cast<const float4*>(wp + (size_t)z * zs));
              acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
            }
            acc.x += bv.x + rs.x, acc.y += bv.y + rs.y;
            acc.z += bv.z + rs.z, acc.w += bv.w + rs.w;
            if constexpr (kGN) {
              gsum.x += acc.x, gsum.y += acc.y, gsum.z += acc.z, gsum.w += acc.w;
              gsq.x = fmaf(acc.x, acc.x, gsq.x), gsq.y = fmaf(acc.y, acc.y, gsq.y), gsq.z = fmaf(acc.z, acc.z, gsq.z), gsq.w = fmaf(acc.w, acc.w, gsq.w);
            }
            store_out(acc, mr, col);
          }
        }
        if (kGN && rlane < RL) {
          gn_red[((rlane * gnt.tn + k) * C4 + cg4) * 2] = gsum;
          gn_red[((rlane * gnt.tn + k) * C4 + cg4) * 2 + 1] = gsq;
        }
        }
        if constexpr (kGN) {
          // fold the row lanes in a fixed order, then the channel buckets: this CTA's partial for its slice of the tile rows
          asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");
          const int nbk_tile = BN / p.gn_bucket, nbk_total = p.N / p.gn_bucket;
          const int slot = p.gn_slot0 + gnt.tile * p.split_k + kz;
          const float* red = reinterpret_cast<const float*>(gn_red);
          for (int it = te; it < gnt.tn * nbk_tile; it += EW * 32) {
            const int k = it / nbk_tile, b = it - k * nbk_tile;
            const int img = gnt.img0 + k, c0 = b * p.gn_bucket;
            if (img >= gnt.nimg || col0 + c0 >= p.N) continue;
            float sm = 0.f, sq = 0.f;
            for (int l = 0; l < RL; ++l)
              for (int cc = c0; cc < c0 + p.gn_bucket; ++cc) {
                const int base = (((l * gnt.tn + k) * C4 + (cc >> 2)) * 2) * 4 + (cc & 3);
                sm += red[base], sq += red[base + 4];
              }
            float2* dst = reinterpret_cast<float2*>(p.gn_part) + ((size_t)img * p.gn_cap + slot) * nbk_total + (col0 + c0) / p.gn_bucket;
            *dst = make_float2(sm, sq);
          }
        }
      }
      asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");
      if (warp == 4 && lane == 0) {
        // last CTA to finish resets both counters: the buffer is all zero again for the next launch
        if (atomicAdd(tk + 1, 1u) == (unsigned)(p.split_k - 1)) {
          tk[0] = 0u;
          tk[1] = 0u;
        }
      }
    } else {
      constexpr int NCH = NCHUNK;  // column chunks per warp (the warps of a lane quarter interleave them)
      if (!pre_issued) issue_addends(col0 + half * 32 + cq);
      float lrs[8], lrq[8];  // EPI_LNS: this lane's share of the row sums of its 8 rows
#pragma unroll
      for (int k = 0; k < 8; ++k) lrs[k] = 0.f, lrq[k] = 0.f;
      (void)lrs, (void)lrq;
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        const int c = half * 32 + j * CSTEP;
        if (c < BN) {
          const int col = col0 + c + cq;
          float4 gsum = make_float4(0.f, 0.f, 0.f, 0.f), gsq = gsum;
          (void)gsum, (void)gsq;
          if (col < p.N) {
            const uint32_t tl = arow + c * 4 + sub * TROW + cq * 4;
#pragma unroll
            for (int b4 = 0; b4 < 2; ++b4) {
              float4 t[4];
#pragma unroll
              for (int i = 0; i < 4; ++i)
                asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                             : "=f"(t[i].x), "=f"(t[i].y), "=f"(t[i].z), "=f"(t[i].w)
                             : "r"(tl + (b4 * 4 + i) * 4 * TROW)
                             : "memory");
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int k = b4 * 4 + i;
                if (mr8[k] < 0) continue;
                float4 f = t[i];
                f.x += bvs[j].x + ad[k].x, f.y += bvs[j].y + ad[k].y, f.z += bvs[j].z + ad[k].z, f.w += bvs[j].w + ad[k].w;
                if constexpr (kLNS) {
                  lrs[k] += (f.x + f.y) + (f.z + f.w);
                  lrq[k] = fmaf(f.x, f.x, fmaf(f.y, f.y, fmaf(f.z, f.z, fmaf(f.w, f.w, lrq[k]))));
                }
                if constexpr (kGN) {
                  gsum.x += f.x, gsum.y += f.y, gsum.z += f.z, gsum.w += f.w;
                  gsq.x = fmaf(f.x, f.x, gsq.x), gsq.y = fmaf(f.y, f.y, gsq.y), gsq.z = fmaf(f.z, f.z, gsq.z), gsq.w = fmaf(f.w, f.w, gsq.w);
                }
                epilogue_store(f, (unsigned)(mr8[k] * p.ldc + col), (unsigned)(mr8[k] * p.ldc16 + col), p.out_f32, p.out_f16,
                               p.out_f16_lo, p.act);
              }
            }
          }
          if constexpr (kGN) {
            // the 4 lanes that hold the same columns (sub = 0..3) fold in a fixed order; sub 0 publishes the quarter's 32-row sums
#pragma unroll
            for (int o = 8; o <= 16; o <<= 1) {
              gsum.x += __shfl_xor_sync(0xffffffffu, gsum.x, o), gsum.y += __shfl_xor_sync(0xffffffffu, gsum.y, o);
              gsum.z += __shfl_xor_sync(0xffffffffu, gsum.z, o), gsum.w += __shfl_xor_sync(0xffffffffu, gsum.w, o);
              gsq.x += __shfl_xor_sync(0xffffffffu, gsq.x, o), gsq.y += __shfl_xor_sync(0xffffffffu, gsq.y, o);
              gsq.z += __shfl_xor_sync(0xffffffffu, gsq.z, o), gsq.w += __shfl_xor_sync(0xffffffffu, gsq.w, o);
            }
            if (sub == 0) {
              float2* d = gn_cs + q * BN + c + cq;
              d[0] = make_float2(gsum.x, gsq.x), d[1] = make_float2(gsum.y, gsq.y);
              d[2] = make_float2(gsum.z, gsq.z), d[3] = make_float2(gsum.w, gsq.w);
            }
          }
          // the next chunk's addends travel while its accumulator columns are read and staged
          if (j + 1 < NCH && c + CSTEP < BN) issue_addends(col0 + c + CSTEP + cq);
        }
      }
      if constexpr (kLNS) {
        // the 8 lanes that share a row (same sub) fold their column groups in a fixed order; one of them publishes this warp's
        // partial for the row: slot = (N tile, share of the chunks). The consumer adds the slots in index order.
#pragma unroll
        for (int k = 0; k < 8; ++k) {
#pragma unroll
          for (int o = 1; o <= 4; o <<= 1) {
            lrs[k] += __shfl_xor_sync(0xffffffffu, lrs[k], o);
            lrq[k] += __shfl_xor_sync(0xffffffffu, lrq[k], o);
          }
        }
        if ((lane & 7) == 0) {
          // two slots per N tile whatever the warp count (the consumer's slot count is a function of N alone)
          const int slot = blockIdx.y * 2 + half;
#pragma unroll
          for (int k = 0; k < 8; ++k)
            if (mr8[k] >= 0) {
              float2* d = reinterpret_cast<float2*>(p.ln_out) + (size_t)mr8[k] * p.ln_slots + slot;
              d[0] = make_float2(lrs[k], lrq[k]);
              if (EG == 1) d[1] = make_float2(0.f, 0.f);
            }
        }
      }
      if constexpr (kGN) {
        asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");  // every quarter's column sums are in shared memory
        gn_write_partials(p, gn_cs, BN, threadIdx.x - 128, EW * 32, gnt, col0, p.up2 ? (int)blockIdx.z * p.gn_phase_slots : 0);
      }
    }
    if (dbg && threadIdx.x == 128) dbg[6] = clock64();
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) dbg[7] = clock64();
}

// The output tile a CTA works on: linear tile index t -> (m tile, n tile, z), m tile fastest, then n tile, then z (the K split,
// or the output phase of the folded upsample conv). It is the order in which the hardware dispatched the 3-D grid of one CTA
// per tile, so a persistent CTA taking tiles c, c + G, c + 2G, ... keeps the L2 reuse of the weight tiles that order gives.
struct GemmTile {
  int mt, nt, z;
  int tw, th, w0, h0, n0, col0;
  int up_a, up_b, kz, b_row0;
  int it_begin, it_end;
};
template <int BN>
__device__ __forceinline__ GemmTile gemm_tile_of(const GemmParams& p, int t, int m_tiles, int n_tiles) {
  GemmTile T;
  T.mt = t % m_tiles;
  T.nt = (t / m_tiles) % n_tiles;
  T.z = t / (m_tiles * n_tiles);
  T.tw = T.mt % p.tiles_w;
  T.th = (T.mt / p.tiles_w) % p.tiles_h;
  T.w0 = T.tw * p.TW, T.h0 = T.th * p.TH, T.n0 = (T.mt / (p.tiles_w * p.tiles_h)) * p.TN;
  T.col0 = T.nt * BN;
  // z is the K split — or, for the folded nearest-2x upsample conv (p.up2, never split), the output phase (a, b): the four
  // 2x2-tap phase convolutions of one layer run as ONE launch; phase shifts the taps, the weight rows and the output pixel
  T.up_a = p.up2 ? (T.z >> 1) : 0, T.up_b = p.up2 ? (T.z & 1) : 0;
  T.kz = p.up2 ? 0 : T.z;
  T.b_row0 = T.col0 + (p.up2 ? T.z * p.N : 0);  // first weight row of this tile (phase-major packing)
  const int total_iters = p.num_taps * p.kc + p.xkc;
  const int per_split = (total_iters + p.split_k - 1) / p.split_k;
  T.it_begin = T.kz * per_split;
  T.it_end = min(total_iters, T.it_begin + per_split);
  return T;
}
// output row index of accumulator row r of a tile (< 2^31 rows); -1 marks a row outside the tensor
__device__ __forceinline__ int gemm_row_of(const GemmParams& p, const GemmTile& T, int r) {
  const int pw = T.w0 + r % p.TW;
  const int phh = T.h0 + (r / p.TW) % p.TH;
  const int pn = T.n0 + r / (p.TW * p.TH);
  return (pw < p.W && phh < p.H && pn < p.nimg) ? ((pn * p.OH + phh * p.os + p.oa + T.up_a) * p.OW + pw * p.os + p.ob + T.up_b) : -1;
}

// The instances whose epilogue runs from the accumulator registers — the LayerNorm-consuming and GEGLU projections, the
// short-K multi-wave launches of the transformer blocks: they never write the accumulator image over the operand ring, so one
// CTA runs a sequence of tiles (persistent grid) and the producer loads the next tile's operands while the consumers run the
// epilogue of the current one. Their per-column addends (bias, LayerNorm column sums) are staged in shared memory once per
// tile. The GroupNorm / LayerNorm-statistics epilogues and the split-K fold reduce across the rows or columns of the tile and
// keep the shared-memory image (one tile per CTA). So do the plain instances: their per-row residual cannot be staged, and read
// from global memory between the stores of a register epilogue it puts one L2 round trip per column pair on the critical path.
template <int EPI>
__host__ __device__ constexpr bool epi_from_registers() {
  return EPI == EPI_LNC || EPI == EPI_GEGLU || EPI == EPI_GEGLU_LNC;
}
// bias and LayerNorm column sums of one tile for the register epilogue, after the ring's barriers
template <int BN, int EPI>
__host__ __device__ constexpr int epi_stage_bytes() {
  return epi_from_registers<EPI>() ? 2 * BN * 4 : 0;
}

// The LayerNorm-consuming and GEGLU instances (epi_from_registers): the same producer / consumer roles and mainloop as
// gemm_tc_kernel, run over a sequence of tiles per CTA, and the epilogue from the accumulator registers. gemm_tc_kernel keeps
// its one-tile form: built from this tile loop, its instances measured 2 % slower in the mainloop (DESIGN.md §4).
template <int BN, int PASSES, int STAGES, int EPI>
__global__ void __launch_bounds__(128 + 32 * EW, 1)
gemm_tc_persistent_kernel(const __grid_constant__ GemmMaps maps, const GemmParams p) {
  static_assert(epi_from_registers<EPI>(), "the shared-memory epilogues run in gemm_tc_kernel");
  constexpr bool kLNC = EPI == EPI_LNC || EPI == EPI_GEGLU_LNC;
  constexpr bool kGEGLU = EPI == EPI_GEGLU || EPI == EPI_GEGLU_LNC;
  using L = StageLayout<BN, PASSES>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle atoms
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + region_bytes<BN, PASSES, STAGES>());
  uint64_t* empty_bar = full_bar + STAGES;
  float* const stage_bias = reinterpret_cast<float*>(empty_bar + STAGES);  // this tile's [BN] bias, then [BN] column sums
  float* const stage_u = stage_bias + BN;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // ---- the tiles of this CTA: a 1-D grid of at most one CTA per SM, CTA c runs tiles c, c + G, c + 2G, ... (never split in K:
  // run_gemm does not split a LayerNorm-consuming or GEGLU GEMM)
  const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
  const int n_tiles = (p.N + BN - 1) / BN;
  const int ntiles = m_tiles * n_tiles * (p.up2 ? 4 : 1);
  const int t0 = blockIdx.x, tstep = gridDim.x;
  long long* const dbg = (p.dbg && t0 == 0) ? p.dbg : nullptr;
  if (dbg && threadIdx.x == 0) dbg[0] = clock64();
  const int main_iters = p.num_taps * p.kc;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], EW);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&maps.a[0][0]);
    tma_prefetch_desc(&maps.b[0]);
    if (p.kc0 < p.kc) tma_prefetch_desc(&maps.a[1][0]);
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) dbg[1] = clock64();
  // Programmatic dependent launch: everything above overlapped the previous kernel's tail. From here on each role waits for the
  // previous kernel (griddepcontrol.wait) only where it first touches data that kernel may have written:
  //   producer : WEIGHTS are immutable, so the weight tiles of the first STAGES k-chunks of the first tile are issued BEFORE the
  //              wait; activation tiles after it
  //   consumers: wait before the first read of the LayerNorm row statistics; all of this kernel's stores follow it
  if (warp == 0) {
    // ===================================================== TMA producer (one elected lane: see elect_one in common.cuh)
    if (elect_one()) {
      // ring slot and phase run on across the tiles of this CTA
      int s = 0;
      uint32_t ph = 0;
#pragma unroll 1
      for (int t = t0; t < ntiles; t += tstep) {
        const GemmTile T = gemm_tile_of<BN>(p, t, m_tiles, n_tiles);
        // iteration -> (activation source, channel chunk, tap shift) and the weight map / K coordinate that go with it
        auto load_b = [&](int it, int s) {
          const CUtensorMap* bm = it < main_iters ? maps.b : maps.bx;
          const int bk = (it < main_iters ? it : it - main_iters) * BK;
          uint8_t* sb = smem + s * L::BYTES + L::A_TILES * A_TILE_BYTES;
          tma_load_2d(sb, &bm[0], &full_bar[s], bk, T.b_row0);
          if (PASSES >= 3) tma_load_2d(sb + L::B_TILE_BYTES, &bm[1], &full_bar[s], bk, T.b_row0);
        };
        auto load_a = [&](int it, int s) {
          int src, c0, cw, ch, cp;
          if (it < main_iters) {
            const int tap = it / p.kc;
            const int cc = it - tap * p.kc;
            src = cc >= p.kc0 ? 1 : 0;
            c0 = (cc - (src ? p.kc0 : 0)) * BK;
            cw = T.w0 + p.tap_dw[tap] + T.up_b, ch = T.h0 + p.tap_dh[tap] + T.up_a, cp = p.tap_ph[tap];
          } else {
            const int e = it - main_iters;
            src = e >= p.xkc0 ? 3 : 2;
            c0 = (e - (src == 3 ? p.xkc0 : 0)) * BK;
            cw = T.w0, ch = T.h0, cp = 0;
          }
          uint8_t* st = smem + s * L::BYTES;
          tma_load_5d(st, &maps.a[src][0], &full_bar[s], c0, cw, ch, cp, T.n0);
          if (PASSES >= 2) tma_load_5d(st + A_TILE_BYTES, &maps.a[src][1], &full_bar[s], c0, cw, ch, cp, T.n0);
        };
        int it = T.it_begin;
        if (t == t0) {
          // ---- first tile, before the wait: weights only (the pipeline slots are all free: fresh barriers)
          const int npre = min(STAGES, T.it_end - T.it_begin);
          for (int i = 0; i < npre; ++i) {
            mbar_expect_tx(&full_bar[i], L::BYTES);
            load_b(it + i, i);
          }
          pdl_wait();
          for (int i = 0; i < npre; ++i) load_a(it + i, i);
          if (dbg) dbg[2] = clock64();
          it += npre;
          s = npre == STAGES ? 0 : npre;
          ph = npre == STAGES ? 1 : 0;
        }
        // ---- steady state: a slot is refilled as soon as the consumers release it, also while they run an epilogue
        for (; it < T.it_end; ++it) {
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], L::BYTES);
          load_a(it, s);
          load_b(it, s);
          if (++s == STAGES) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================================================== consumers: wgmma mainloop, then the epilogue
    pdl_wait();  // the row statistics below come from the previous kernel; every store of this kernel follows
    const int wg = (warp - 4) >> 2;  // rows [64 wg, 64 wg + 64) of the tile
    int s = 0;
    uint32_t ph = 0;
#pragma unroll 1
    for (int t = t0; t < ntiles; t += tstep) {
      const GemmTile T = gemm_tile_of<BN>(p, t, m_tiles, n_tiles);
      const bool first = t == t0;
      const int col0 = T.col0;
      // This thread's accumulator rows are ra = 64 wg + 16 (warp % 4) + lane / 4 and ra + 8. Their output rows, and for a
      // LayerNorm-consuming GEMM their partial row statistics, are requested before the mainloop so that those loads travel while
      // the products run.
      const int ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);
      int mrow[2] = {-1, -1};
      constexpr int LNPRE = 8;  // row-statistics slots loaded ahead of the mainloop (the rest after it)
      float2 lnv[2][LNPRE];
      // this tile's bias and LayerNorm column sums: one column per consumer thread, staged after the mainloop
      const int te = threadIdx.x - 128;
      float sbias = 0.f, su = 0.f;
      if (te < BN && col0 + te < p.N) {
        if (p.bias) sbias = p.bias[col0 + te];
        if constexpr (kLNC) su = p.ln_u[col0 + te];
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mrow[h] = gemm_row_of(p, T, ra + 8 * h);
        if constexpr (kLNC) {
          const float2* sp = reinterpret_cast<const float2*>(p.ln_in) + (size_t)mrow[h] * p.ln_in_slots;
#pragma unroll
          for (int i = 0; i < LNPRE; ++i) lnv[h][i] = (mrow[h] >= 0 && i < p.ln_in_slots) ? sp[i] : make_float2(0.f, 0.f);
        }
      }
      float acc[BN / 2];
      {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int it = T.it_begin; it < T.it_end; ++it) {
          mbar_wait(&full_bar[s], ph);
          if (dbg && threadIdx.x == 128 && first && it == T.it_begin) dbg[3] = clock64();
          const uint32_t a_hi = smem_u32(smem + s * L::BYTES) + wg * (64 * 128);
          const uint32_t a_lo = a_hi + A_TILE_BYTES;
          const uint32_t b_hi = smem_u32(smem + s * L::BYTES) + L::A_TILES * A_TILE_BYTES;
          const uint32_t b_lo = b_hi + L::B_TILE_BYTES;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            const uint32_t koff = k * 32;  // 16 fp16 = 32 bytes inside the 128B swizzle row
            const uint64_t da = make_sdesc_sw128(a_hi + koff);
            const uint64_t db = make_sdesc_sw128(b_hi + koff);
            Wgmma<BN>::template ss<0>(acc, da, db, 1);
            if (PASSES >= 2) Wgmma<BN>::template ss<0>(acc, make_sdesc_sw128(a_lo + koff), db, 1);
            if (PASSES >= 3) Wgmma<BN>::template ss<0>(acc, da, make_sdesc_sw128(b_lo + koff), 1);
          }
          wgmma_commit();
          // one group stays in flight: the products of the previous stage are complete, so its slot goes back to the producer
          wgmma_wait<1>();
          if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
          prev = s;
          if (++s == STAGES) {
            s = 0;
            ph ^= 1;
          }
        }
        wgmma_wait<0>();
        reg_fence(acc);
        if (dbg && threadIdx.x == 128 && first) dbg[4] = clock64();
        // the last stage goes back too: the producer fills the ring with the next tile's operands during this epilogue
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
        asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");  // the previous tile's epilogue has read the staging
        if (te < BN) stage_bias[te] = sbias, stage_u[te] = su;
        asm volatile("bar.sync 1, %0;" ::"n"(EW * 32) : "memory");
      }
      {
        // ---- epilogue from the accumulator registers. acc[4 jj + 2 h + e] is row ra + 8 h, tile column 8 jj + 2 (lane % 4) + e.
        // Every element is the expression of the shared-memory epilogue it replaces, in the same order.
        if (t + tstep >= ntiles) pdl_trigger();  // the last tile's epilogue starts: the next kernel may begin its prologue
        if (dbg && threadIdx.x == 128 && first) dbg[5] = clock64();
        const int cp = 2 * (lane & 3);
        float ln_mu[2] = {0.f, 0.f}, ln_rs[2] = {0.f, 0.f};
        if constexpr (kLNC) {
          // EPI_LNC: mean / rstd of each row, from the partial row sums the producer of A left, added in slot order
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (mrow[h] >= 0) {
              float sm = 0.f, sq = 0.f;
#pragma unroll
              for (int i = 0; i < LNPRE; ++i)
                if (i < p.ln_in_slots) sm += lnv[h][i].x, sq += lnv[h][i].y;
              const float2* sp = reinterpret_cast<const float2*>(p.ln_in) + (size_t)mrow[h] * p.ln_in_slots;
              for (int i = LNPRE; i < p.ln_in_slots; ++i) {
                const float2 v = sp[i];
                sm += v.x, sq += v.y;
              }
              const float inv = 1.0f / (float)p.ln_C;
              ln_mu[h] = sm * inv;
              ln_rs[h] = rsqrtf(fmaxf(sq * inv - ln_mu[h] * ln_mu[h], 0.f) + p.ln_eps);
            }
          }
        }
        // Stores go out 32 columns at a time: the 4 lanes of a row exchange their column pairs (quad_transpose) so that each
        // lane writes 8 consecutive fp16 columns with one 16-byte store, 64 contiguous bytes per row and warp instruction.
        // Rows outside the tensor take part in the exchange and skip the store (the 4 lanes of a quad share their rows). A
        // group's values are computed for both rows before any branch: run-time choices (activation, fp32 output) are taken
        // once per group, so that the arithmetic of 8 column pairs interleaves.
        const int q4 = lane & 3;
        auto store_f16 = [&](uint32_t (&hi)[2][4], uint32_t (&lo)[2][4], int ocol) {
          if (!p.out_f16) return;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const unsigned o16 = (unsigned)(mrow[h] * p.ldc16 + ocol + 8 * q4);
            const uint4 vh = quad_transpose(hi[h], q4);
            if (mrow[h] >= 0) *reinterpret_cast<uint4*>(p.out_f16 + o16) = vh;
            if (p.out_f16_lo) {
              const uint4 vl = quad_transpose(lo[h], q4);
              if (mrow[h] >= 0) *reinterpret_cast<uint4*>(p.out_f16_lo + o16) = vl;
            }
          }
        };
        if constexpr (kGEGLU) {
          // tile columns [0,BN/2) = x, [BN/2,BN) = gate: both halves of an output column are in this thread (jj and jj + BN/16)
          constexpr int HB = BN / 2;
          const int ocol0 = T.nt * HB;
#pragma unroll
          for (int g = 0; g < HB / 32; ++g) {
            uint32_t hi[2][4], lo[2][4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int jj = 4 * g + k, c = 8 * jj + cp;
              const float2 bx = *reinterpret_cast<const float2*>(stage_bias + c);
              const float2 bg = *reinterpret_cast<const float2*>(stage_bias + HB + c);
              float2 ux = make_float2(0.f, 0.f), ug = ux;
              if constexpr (kLNC) {
                ux = *reinterpret_cast<const float2*>(stage_u + c);
                ug = *reinterpret_cast<const float2*>(stage_u + HB + c);
              }
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float2 tx = make_float2(acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1]);
                float2 tg = make_float2(acc[4 * (jj + HB / 8) + 2 * h], acc[4 * (jj + HB / 8) + 2 * h + 1]);
                if constexpr (kLNC) {
                  const float rmu = ln_mu[h], rrs = ln_rs[h];
                  tx.x = rrs * (tx.x - rmu * ux.x), tx.y = rrs * (tx.y - rmu * ux.y);
                  tg.x = rrs * (tg.x - rmu * ug.x), tg.y = rrs * (tg.y - rmu * ug.y);
                }
                float2 y;
                y.x = (tx.x + bx.x) * gelu_erf_fast(tg.x + bg.x);
                y.y = (tx.y + bx.y) * gelu_erf_fast(tg.y + bg.y);
                const HalfPair2 s2 = split_f16x2(y.x, y.y);
                hi[h][k] = *reinterpret_cast<const uint32_t*>(&s2.hi), lo[h][k] = *reinterpret_cast<const uint32_t*>(&s2.lo);
              }
            }
            store_f16(hi, lo, ocol0 + 32 * g);
          }
        } else {
          // LayerNorm folded in: rstd * (acc - mean * u) ; beta^T W + bias comes in through the bias (no residual: run_gemm
          // checks)
#pragma unroll
          for (int g = 0; g < BN / 32; ++g) {
            if (col0 + 32 * g >= p.N) continue;  // N is a multiple of 32: a group is all in or all out
            float2 f[2][4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int c = 32 * g + 8 * k + cp;
              const float2 bv = *reinterpret_cast<const float2*>(stage_bias + c);
              const float2 us = *reinterpret_cast<const float2*>(stage_u + c);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float2 v = make_float2(acc[4 * (4 * g + k) + 2 * h], acc[4 * (4 * g + k) + 2 * h + 1]);
                v.x = ln_rs[h] * (v.x - ln_mu[h] * us.x), v.y = ln_rs[h] * (v.y - ln_mu[h] * us.y);
                v.x += bv.x, v.y += bv.y;
                f[h][k] = v;
              }
            }
            if (p.act == 1) {
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int k = 0; k < 4; ++k) f[h][k].x = quick_gelu(f[h][k].x), f[h][k].y = quick_gelu(f[h][k].y);
            }
            if (p.out_f32) {
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int k = 0; k < 4; ++k)
                  if (mrow[h] >= 0) *reinterpret_cast<float2*>(p.out_f32 + (unsigned)(mrow[h] * p.ldc + col0 + 32 * g + 8 * k + cp)) = f[h][k];
            }
            uint32_t hi[2][4], lo[2][4];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const HalfPair2 s2 = split_f16x2(f[h][k].x, f[h][k].y);
                hi[h][k] = *reinterpret_cast<const uint32_t*>(&s2.hi), lo[h][k] = *reinterpret_cast<const uint32_t*>(&s2.lo);
              }
            store_f16(hi, lo, col0 + 32 * g);
          }
        }
        if (dbg && threadIdx.x == 128 && first) dbg[6] = clock64();
      }
    }
  }
  __syncthreads();
  if (dbg && threadIdx.x == 0) dbg[7] = clock64();
}

// ------------------------------------------------------------------ launcher
// Opt-in maximum of dynamic shared memory per block on sm_90 (227 KB); the kernel adds 1 KB of alignment pad and two 8-byte
// barriers per stage to the ring.
static constexpr int SMEM_OPTIN_MAX = 227 * 1024;
template <int BN, int PASSES>
constexpr int pick_stages() {
  // as many stages as fit in the opt-in maximum, capped at 8. The 3-pass BN = 160 tile (72 KB stages, the bulk of the
  // UNet's tensor work) needs 3: with one wgmma group in flight a freed slot then has two stages of products, not one, to be
  // refilled in, and its mainloop keeps the tensor pipe busy (DESIGN.md §4, "Measured").
  constexpr int per = StageLayout<BN, PASSES>::BYTES;
  constexpr int n = (SMEM_OPTIN_MAX - 1024) / (per + 2 * 8);
  return n > 8 ? 8 : n;
}

template <int BN, int PASSES, int STAGES, int EPI>
static void launch_epi(const GemmMaps& maps, const GemmParams& p, cudaStream_t stream) {
  constexpr int smem = region_bytes<BN, PASSES, STAGES>() + 2 * STAGES * 8 + epi_stage_bytes<BN, EPI>() + 1024;
  static_assert(smem <= SMEM_OPTIN_MAX, "shared memory per block");
  static_assert(4 * BN * 8 <= AccLayout<BN>::GN_BYTES && 2 * (EW * 32) * 4 * 16 <= AccLayout<BN>::GN_BYTES,
                "GroupNorm column sums must fit in the scratch after the accumulator image");
  static DeviceOnce once;
  const bool first = once.first();
  auto go = [&](void (*kernel)(const GemmMaps, const GemmParams), dim3 grid) {
    if (first) SDB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    launch_k(kernel, grid, dim3(128 + 32 * EW), (size_t)smem, stream, maps, p);
  };
  const int m_tiles = p.tiles_n * p.tiles_h * p.tiles_w, n_tiles = (p.N + BN - 1) / BN;
  if constexpr (epi_from_registers<EPI>()) {
    // at most one CTA per SM, each running every gridDim.x-th tile
    SDB_CHECK(p.split_k == 1 && p.ldc16 % 8 == 0 && reinterpret_cast<uintptr_t>(p.out_f16) % 16 == 0 &&
                  reinterpret_cast<uintptr_t>(p.out_f16_lo) % 16 == 0,
              "register epilogue: no K split, fp16 outputs written 8 columns (16 bytes) at a time");
    go(gemm_tc_persistent_kernel<BN, PASSES, STAGES, EPI>, dim3(std::min(m_tiles * n_tiles * (p.up2 ? 4 : 1), g_num_sms)));
  } else {
    go(gemm_tc_kernel<BN, PASSES, STAGES, EPI>, dim3(m_tiles, n_tiles, p.up2 ? 4 : p.split_k));
  }
}
// the statistics-producing epilogues exist for the tile widths their tensors use (run_gemm picks those widths for them)
template <int BN, int PASSES, int STAGES>
static void launch_inst(const GemmMaps& maps, const GemmParams& p, cudaStream_t stream) {
  SDB_CHECK((p.gn_part != nullptr) + (p.ln_out != nullptr) + (p.ln_in != nullptr) <= 1, "one statistics role per launch");
  if constexpr (BN == 128) {
    if (p.geglu) {
      SDB_CHECK(!p.gn_part && !p.ln_out && p.split_k == 1, "GEGLU epilogue: no statistics output, no split-K");
      return p.ln_in ? launch_epi<BN, PASSES, STAGES, EPI_GEGLU_LNC>(maps, p, stream)
                     : launch_epi<BN, PASSES, STAGES, EPI_GEGLU>(maps, p, stream);
    }
  }
  SDB_CHECK(!p.geglu, "the GEGLU epilogue is built for 128-wide tiles");
  if constexpr (BN >= 128) {
    if (p.gn_part) return launch_epi<BN, PASSES, STAGES, EPI_GN>(maps, p, stream);
  }
  if constexpr (BN == 160) {
    if (p.ln_out) return launch_epi<BN, PASSES, STAGES, EPI_LNS>(maps, p, stream);
  }
  if constexpr (BN == 128 || BN == 160) {
    if (p.ln_in) return launch_epi<BN, PASSES, STAGES, EPI_LNC>(maps, p, stream);
  }
  SDB_CHECK(!p.gn_part && !p.ln_out && !p.ln_in, "this statistics epilogue is not built for this tile width");
  launch_epi<BN, PASSES, STAGES, EPI_PLAIN>(maps, p, stream);
}

template <int BN, int PASSES>
static void launch_bn(const GemmMaps& maps, const GemmParams& p, cudaStream_t stream) {
  launch_inst<BN, PASSES, pick_stages<BN, PASSES>()>(maps, p, stream);
}

int gemm_tc_stages(int BN, int passes) {
  SDB_CHECK(passes >= 1 && passes <= 3, "passes");
  constexpr int t[4][3] = {{pick_stages<64, 1>(), pick_stages<64, 2>(), pick_stages<64, 3>()},
                           {pick_stages<128, 1>(), pick_stages<128, 2>(), pick_stages<128, 3>()},
                           {pick_stages<160, 1>(), pick_stages<160, 2>(), pick_stages<160, 3>()},
                           {pick_stages<256, 1>(), pick_stages<256, 2>(), pick_stages<256, 3>()}};
  switch (BN) {
    case 64: return t[0][passes - 1];
    case 128: return t[1][passes - 1];
    case 160: return t[2][passes - 1];
    case 256: return t[3][passes - 1];
    default: throw Error("unsupported BN");
  }
}

void gemm_tc_launch(const GemmMaps& maps, const GemmParams& p, int BN, int passes, cudaStream_t stream) {
  SDB_CHECK(p.TN * p.TH * p.TW == BM, "M tile must cover 128 rows");
  SDB_CHECK(p.N % 32 == 0, "N must be a multiple of 32");
#define SDB_DISPATCH(bn)                                             \
  case bn:                                                           \
    if (passes == 1) launch_bn<bn, 1>(maps, p, stream);              \
    else if (passes == 2) launch_bn<bn, 2>(maps, p, stream);         \
    else launch_bn<bn, 3>(maps, p, stream);                          \
    break;
  switch (BN) {
    SDB_DISPATCH(64)
    SDB_DISPATCH(128)
    SDB_DISPATCH(160)
    SDB_DISPATCH(256)
    default:
      throw Error("unsupported BN");
  }
#undef SDB_DISPATCH
}

}  // namespace sdb
