// attention.cu — fused QK^T . softmax . PV on wgmma (flash-style streaming softmax, no N^2 tensor in HBM).
//
// Replaces qkv_attention (reference src/model/attention.rs:5-45 == src/backend.rs:88-128, mask = None):
//   softmax((q d^-1/4)(k d^-1/4)^T) v  ==  softmax(q k^T d^-1/2) v.
//
// One CTA = 128 query rows of one (sample, head). Warp roles:
//   warpgroup 0    : TMA producers — warp 0 the Q tile once, then K tiles [128 keys][d]; warp 1 the V tiles (ST-stage rings)
//   warpgroups 1-2 : 64 query rows each. S = Q K^T with wgmma (Q and K from shared memory, S in registers: m64n128), running
//                    max / sum in fp32 (exp2 with the d^-1/2 scale folded in), P converted in registers to the A fragment of
//                    O += P V (wgmma with A from registers, O in registers), lazy O rescale, O / l written as fp16 hi(/lo).
//                    Software-pipelined: the softmax of one key tile runs while the tensor cores compute the P V product of the
//                    previous one, and the two warpgroups take turns issuing their wgmmas (ping-pong on named barriers).
#include "attention.cuh"

#include <type_traits>

namespace sdb {

// VMN = false: V arrives transposed, V^T [d][keys] (K-major B operand of P.V: two boxes of [DPAD rows][64 keys]).
// VMN = true : V arrives as the projection wrote it, V [keys][d] (MN-major B operand: DC boxes of [128 keys][64 channels]) —
//              no transposing GEMM in front of the kernel.
// QK3 = true : q and k arrive as fp16 hi + lo pairs and S = q_hi k_hi^T + q_lo k_hi^T + q_hi k_lo^T (the 3-term split product of
//              the GEMMs): the logits are fp32-class. With single fp16 operands a logit of magnitude ~30 (peaked softmax of a
//              trained checkpoint) carries an absolute error ~1e-2, i.e. ~1 % on the dominant probabilities — the largest
//              single error source of a UNet step on realistic-statistics weights (tests/test_realstats_gpu.py).
template <int DPAD, bool VMN = false, bool QK3 = false>
struct AttnCfg {
  static constexpr int DC = (DPAD + 63) / 64;                          // 64-wide chunks of the head dim
  static constexpr int QK_PARTS = QK3 ? 2 : 1;                          // hi (+ lo) copies of the Q and K tiles
  static constexpr int Q_HALF = DC * 128 * 128;                         // [128 rows][64] x DC, 128 B rows
  static constexpr int Q_TILE = QK_PARTS * Q_HALF;
  static constexpr int K_HALF = DC * 128 * 128;
  static constexpr int K_BYTES = QK_PARTS * K_HALF;
  static constexpr int V_CHUNK = VMN ? 128 * 128 : ((DPAD * 128 + 1023) / 1024) * 1024;   // VMN: [128 keys][64 ch]; else [DPAD rows][64 keys]
  static constexpr int V_BYTES = (VMN ? DC : 2) * V_CHUNK;
  static constexpr int V_TX = VMN ? DC * 128 * 128 : 2 * DPAD * 128;    // bytes one V stage receives
  static constexpr int FIXED = Q_TILE + 512 + 1024;
  // K/V pipeline stages: two when they fit in the 227 KB of shared memory a block may use
  static constexpr int ST = (FIXED + 2 * (K_BYTES + V_BYTES) <= 226 * 1024) ? 2 : 1;
  static constexpr int SMEM = FIXED + ST * (K_BYTES + V_BYTES);
  static_assert(SMEM <= 226 * 1024, "smem budget");
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int DPAD, bool VMN, bool QK3>
__global__ void __launch_bounds__(384, 1)
attention_kernel(const __grid_constant__ CUtensorMap mq, const __grid_constant__ CUtensorMap mk,
                 const __grid_constant__ CUtensorMap mv, const __grid_constant__ CUtensorMap mq_lo,
                 const __grid_constant__ CUtensorMap mk_lo, const AttnParams p) {
  using Cfg = AttnCfg<DPAD, VMN, QK3>;
  constexpr int DC = Cfg::DC, ST = Cfg::ST;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::Q_TILE;                  // ST stages
  uint8_t* sV = sK + ST * Cfg::K_BYTES;            // ST stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ST * Cfg::V_BYTES);
  uint64_t* q_full = bars;             // 1
  uint64_t* k_full = q_full + 1;       // ST
  uint64_t* k_empty = k_full + ST;     // ST (one arrival per softmax warp)
  uint64_t* v_full = k_empty + ST;     // ST
  uint64_t* v_empty = v_full + ST;     // ST (one arrival per softmax warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // stamps go through p.dbg (a kernel parameter) rather than a pointer copy that would hold two registers through the loop
  const bool dbg = p.dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0;
  constexpr int DJ0 = 8;  // stamped key tiles: DJ0 .. DJ0+3
  if (dbg && threadIdx.x == 0) p.dbg[255] = clock64();
  pdl_trigger();
  const int q0 = blockIdx.x * 128;
  const int h = blockIdx.y;
  const int s = blockIdx.z;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < ST; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    fence_mbar_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&mq);
    tma_prefetch_desc(&mk);
    tma_prefetch_desc(&mv);
  }
  __syncthreads();
  pdl_wait();
  // a device-side length of 0 (or beyond Nk) would leave T = 0 and the epilogue waiting forever: clamp to [1, Nk]
  const int kvlen = p.kvlen ? max(1, min(p.kvlen[s], p.Nk)) : p.Nk;
  const int T = (kvlen + 127) / 128;

  if (warp < 4) {
    // ======================================================================= TMA producers
    // warp 0 loads Q and the K tiles, warp 1 the V tiles: the consumers free a K stage a whole softmax before the V stage of the
    // same tile, so the next K load must not queue behind the wait for that V stage
    if (warp == 0 && elect_one()) {
      mbar_expect_tx(q_full, Cfg::Q_TILE);
#pragma unroll
      for (int c = 0; c < DC; ++c) {
        tma_load_2d(sQ + c * 16384, &mq, q_full, p.q_col0 + h * DPAD + c * 64, s * p.q_rows_per_sample + q0);
        if (QK3) tma_load_2d(sQ + Cfg::Q_HALF + c * 16384, &mq_lo, q_full, p.q_col0 + h * DPAD + c * 64, s * p.q_rows_per_sample + q0);
      }
      for (int j = 0; j < T; ++j) {
        const int st = j % ST;
        const uint32_t ph = (j / ST) & 1;
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_expect_tx(&k_full[st], Cfg::K_BYTES);
#pragma unroll
        for (int c = 0; c < DC; ++c) {
          tma_load_2d(sK + st * Cfg::K_BYTES + c * 16384, &mk, &k_full[st], p.k_col0 + h * DPAD + c * 64,
                      s * p.k_rows_per_sample + j * 128);
          if (QK3)
            tma_load_2d(sK + st * Cfg::K_BYTES + Cfg::K_HALF + c * 16384, &mk_lo, &k_full[st], p.k_col0 + h * DPAD + c * 64,
                        s * p.k_rows_per_sample + j * 128);
        }
      }
    } else if (warp == 1 && elect_one()) {
      for (int j = 0; j < T; ++j) {
        const int st = j % ST;
        const uint32_t ph = (j / ST) & 1;
        mbar_wait(&v_empty[st], ph ^ 1);
        mbar_expect_tx(&v_full[st], Cfg::V_TX);
        if (VMN) {
#pragma unroll
          for (int c = 0; c < DC; ++c)  // [128 keys][64 channels] boxes; channels past the head (or the matrix) are never multiplied
            tma_load_2d(sV + st * Cfg::V_BYTES + c * Cfg::V_CHUNK, &mv, &v_full[st], p.v_col0 + h * DPAD + c * 64,
                        s * p.k_rows_per_sample + j * 128);
        } else {
#pragma unroll
          for (int c = 0; c < 2; ++c)
            tma_load_2d(sV + st * Cfg::V_BYTES + c * Cfg::V_CHUNK, &mv, &v_full[st],
                        s * p.k_rows_per_sample + j * 128 + c * 64, h * p.d);
        }
      }
    }
  } else {
    // ======================================================================= softmax warpgroups + epilogue
    // accumulator layout of m64nN (see Wgmma in common.cuh): this thread holds rows rw + 8 hh (hh = 0, 1) of the warpgroup's
    // 64, columns 8 (i / 4) + 2 (lane % 4) + i % 2 of element i, with hh = (i / 2) % 2
    const int wg = (warp - 4) >> 2;
    const int rw = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // row inside the CTA's 128
    const int cl = 2 * (lane & 3);
    const float sl2 = p.scale * 1.4426950408889634f;  // d^-1/2 * log2(e)
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float o[DPAD / 2];
#pragma unroll
    for (int i = 0; i < DPAD / 2; ++i) o[i] = 0.f;
    const uint32_t qa = smem_u32(sQ) + wg * (64 * 128);
    // keys per S sub-tile: the 128-key tile in one m64n128 product, or for d = 160 in two m64n64 halves (S, P and O of a 128-key
    // product do not fit the registers beside an 80-register O: the wgmma would be serialised and the thread would spill)
    constexpr int KW = DPAD > 128 ? 64 : 128, NSUB = 128 / KW;
    // Software pipeline over the key sub-tiles u = 0 .. U-1 (keys [KW (u % NSUB), + KW) of tile u / NSUB). Iteration u issues
    // S_u = Q K_u^T, then O += P_{u-1} V_{u-1}, waits for S_u alone and exponentiates it on the CUDA cores while the tensor cores
    // run the P V product; then it waits for that product, rescales O and packs P_u for the next iteration. Each output element
    // sees the operations of the serial schedule in the same order (O <- alpha_u O, then O += P_u V_u), with the same row
    // maxima, exponent arguments and partial-sum folds: the result is bit-identical to computing the sub-tiles one at a time.
    const int U = T * NSUB;
    float sv[KW / 2];     // S_u, exponentiated in place (P_u in fp32)
    uint32_t pa[KW / 4];  // P_{u-1} as fp16 pairs: the A fragments of the KW / 16 k-steps of P V, read by wgmmas in flight
    float alpha[2];       // O rescale factor of the sub-tile just exponentiated (per row half)
    // SDB_ATTN_DBG timeline of key tiles DJ0 .. DJ0+3 (their first sub-tile): 0 S issued, 1 S ready, 2 softmax done,
    // 3 PV issued, 4 PV done
    auto sstamp = [&](int u, int k) {
      const int j = u / NSUB;
      if (dbg && threadIdx.x == 128 && u % NSUB == 0 && j >= DJ0 && j < DJ0 + 4) p.dbg[(j - DJ0) * 8 + k] = clock64();
    };
    auto issue_s = [&](int u) {
      const int j = u / NSUB, sub = u % NSUB, st = j % ST;
      if (sub == 0) mbar_wait(&k_full[st], (j / ST) & 1);
#pragma unroll
      for (int i = 0; i < KW / 2; ++i) sv[i] = 0.f;
      const uint32_t ka = smem_u32(sK + st * Cfg::K_BYTES) + sub * KW * 128;  // key rows [sub KW, sub KW + KW) of the tile
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DPAD / 16; ++kk) {
        const uint32_t off = (kk / 4) * 16384 + (kk % 4) * 32;
        Wgmma<KW>::template ss<0>(sv, make_sdesc_sw128(qa + off), make_sdesc_sw128(ka + off), 1);
        if (QK3) {  // + q_lo k_hi^T + q_hi k_lo^T
          Wgmma<KW>::template ss<0>(sv, make_sdesc_sw128(qa + Cfg::Q_HALF + off), make_sdesc_sw128(ka + off), 1);
          Wgmma<KW>::template ss<0>(sv, make_sdesc_sw128(qa + off), make_sdesc_sw128(ka + Cfg::K_HALF + off), 1);
        }
      }
      wgmma_commit();
      sstamp(u, 0);
    };
    auto s_ready = [&](int u) {  // after the wait for S_u: the K stage is free once its last sub-tile is multiplied
      reg_fence(sv);
      const int j = u / NSUB;
      if (u % NSUB == NSUB - 1 && lane == 0) mbar_arrive(&k_empty[j % ST]);
      sstamp(u, 1);
    };
    auto issue_pv = [&](int u) {
      const int j = u / NSUB, sub = u % NSUB, st = j % ST;
      if (sub == 0) mbar_wait(&v_full[st], (j / ST) & 1);
      const uint32_t va = smem_u32(sV + st * Cfg::V_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KW / 16; ++kk) {
        const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
        const int kg = sub * (KW / 16) + kk;  // 16-key step inside the 128-key tile
        // K-major V^T: 16 keys = 32 bytes inside a 128-byte row; MN-major V: 16 keys = 16 rows of 128 bytes
        if (VMN)
          Wgmma<DPAD>::template rs<1>(o, a, make_sdesc_sw128_mn(va + kg * 2048, Cfg::V_CHUNK), 1);
        else
          Wgmma<DPAD>::template rs<0>(o, a, make_sdesc_sw128(va + (kg / 4) * Cfg::V_CHUNK + (kg % 4) * 32), 1);
      }
      wgmma_commit();
      sstamp(u, 3);
    };
    auto pv_done = [&](int u) {  // after the wait for P_u V_u: the V stage is free once its last sub-tile is multiplied
      reg_fence(o);
      const int j = u / NSUB;
      if (u % NSUB == NSUB - 1 && lane == 0) mbar_arrive(&v_empty[j % ST]);
      sstamp(u, 4);
    };
    // S_u -> P_u (fp32, in sv), alpha; running maximum and sum. Sub-tiles with every key valid for both rows (all but the last
    // of a short sequence) take a copy of the code without the key mask: the same values, without a compare per element.
    auto softmax = [&](int u) {
      const int j = u / NSUB, sub = u % NSUB;
      // valid keys of this sub-tile per row (<= 0: none), less this thread's column offset cl: column 8 (i / 4) + cl + i % 2 of
      // element i is a valid key when 8 (i / 4) + i % 2 < vcl (compile-time left sides, no column registers)
      int vcl[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        int vt = min(128, kvlen - j * 128);
        if (p.causal) vt = max(1, min(vt, q0 + rw + 8 * hh - j * 128 + 1));  // additive -inf mask above the diagonal
        vcl[hh] = vt - sub * KW - cl;
      }
      auto run = [&](auto full_c) {
        constexpr bool full = decltype(full_c)::value;
        // 4 independent max chains per row, then the 4 lanes that share a row
        float mxa[2][4];
#pragma unroll
        for (int a = 0; a < 4; ++a) mxa[0][a] = mxa[1][a] = -INFINITY;
#pragma unroll
        for (int i = 0; i < KW / 2; ++i) {
          const int hh = (i >> 1) & 1;
          if (full || 8 * (i >> 2) + (i & 1) < vcl[hh]) mxa[hh][(i >> 2) & 3] = fmaxf(mxa[hh][(i >> 2) & 3], sv[i]);
        }
        float m_new[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float mx = fmaxf(fmaxf(mxa[hh][0], mxa[hh][1]), fmaxf(mxa[hh][2], mxa[hh][3]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          // Lazy rescale with a threshold: the running maximum is only a reference point (softmax is shift invariant), so it is
          // moved — and O / l rescaled — only when the row's maximum grew by more than 2^8; otherwise the tile is exponentiated
          // against the stale reference and P may reach 256 (exact in fp16, fp32 sums).
          const float m_cand = fmaxf(m_run[hh], mx * sl2);
          const bool resc = m_cand > m_run[hh] + 8.0f;  // first tile: m_run = -inf -> true
          m_new[hh] = resc ? m_cand : m_run[hh];
          alpha[hh] = resc ? ex2(m_run[hh] - m_new[hh]) : 1.0f;  // 0 on the first tile
        }
        float sum[2][2] = {{0.f, 0.f}, {0.f, 0.f}};  // independent partial row sums (ILP), folded in fixed order below
#pragma unroll
        for (int i = 0; i < KW / 2; i += 2) {
          const int hh = (i >> 1) & 1, c8 = 8 * (i >> 2);
          float p0 = ex2(fmaf(sv[i], sl2, -m_new[hh]));
          float p1 = ex2(fmaf(sv[i + 1], sl2, -m_new[hh]));
          if (!full) {
            p0 = (c8 < vcl[hh]) ? p0 : 0.f;
            p1 = (c8 + 1 < vcl[hh]) ? p1 : 0.f;
          }
          sum[hh][(i >> 2) & 1] += p0 + p1;  // fp32 terms; the fp16 rounding of P is unbiased and averages out over the row
          sv[i] = p0;
          sv[i + 1] = p1;
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float t = sum[hh][0] + sum[hh][1];
          t += __shfl_xor_sync(0xffffffffu, t, 1);
          t += __shfl_xor_sync(0xffffffffu, t, 2);
          l_run[hh] = l_run[hh] * alpha[hh] + t;
          m_run[hh] = m_new[hh];
        }
      };
      if (vcl[0] >= KW - cl && vcl[1] >= KW - cl)
        run(std::true_type());
      else
        run(std::false_type());
      sstamp(u, 2);
    };
    // once P_{u-1} V_{u-1} is done: O <- alpha_u O, and P_u to fp16 A fragments (pa is read by the P V wgmmas until then)
    auto rescale_pack = [&]() {
      if (alpha[0] != 1.0f || alpha[1] != 1.0f) {
#pragma unroll
        for (int i = 0; i < DPAD / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
      }
#pragma unroll
      for (int i = 0; i < KW / 2; i += 2) pa[i >> 1] = pack_h2(sv[i], sv[i + 1]);
    };

    // Ping-pong of the two warpgroups (named barriers 2 and 3): a warpgroup issues the wgmmas of a round only after the other
    // one has issued those of its previous round, so the tensor cores take the two in turn while the other exponentiates.
    // Warpgroup 1 lets warpgroup 0 go first and skips its last hand-over, so no arrival is left pending at exit.
    auto turn_begin = [&]() {
      if (wg == 0)
        asm volatile("bar.sync 2, 256;" ::: "memory");
      else
        asm volatile("bar.sync 3, 256;" ::: "memory");
    };
    auto turn_end = [&](bool last) {
      if (wg == 0)
        asm volatile("bar.arrive 3, 256;" ::: "memory");
      else if (!last)
        asm volatile("bar.arrive 2, 256;" ::: "memory");
    };
    if (wg == 1) turn_end(false);

    mbar_wait(q_full, 0);
    turn_begin();
    issue_s(0);
    turn_end(false);
    wgmma_wait<0>();
    s_ready(0);
    softmax(0);
    rescale_pack();
    for (int u = 1; u < U; ++u) {
      turn_begin();
      issue_s(u);
      issue_pv(u - 1);
      turn_end(false);
      wgmma_wait<1>();  // S_u; P_{u-1} V_{u-1} may still run
      s_ready(u);
      softmax(u);
      wgmma_wait<0>();
      pv_done(u - 1);
      rescale_pack();
    }
    turn_begin();
    issue_pv(U - 1);
    turn_end(true);
    wgmma_wait<0>();
    pv_done(U - 1);
    // ---- epilogue: O / l -> fp16 hi(/lo)
    const float inv_l[2] = {1.0f / l_run[0], 1.0f / l_run[1]};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int qrow = q0 + rw + 8 * hh;
      if (qrow >= p.Nq) continue;
      const size_t orow = (size_t)(s * p.q_rows_per_sample + qrow) * p.ldo + h * p.d;
#pragma unroll
      for (int i = 2 * hh; i < DPAD / 2; i += 4) {
        const int col = 8 * (i >> 2) + cl;
        if (col < p.d) {
          const float f0 = o[i] * inv_l[hh], f1 = o[i + 1] * inv_l[hh];
          const HalfPair2 sp = split_f16x2(f0, f1);
          *reinterpret_cast<__half2*>(p.out_hi + orow + col) = sp.hi;
          if (p.out_lo) *reinterpret_cast<__half2*>(p.out_lo + orow + col) = sp.lo;
        }
      }
    }
  }
  __syncthreads();
}

template <int DPAD, bool VMN, bool QK3>
static void launch_attn2(const AttnMaps& m, const AttnParams& p, cudaStream_t st) {
  constexpr int smem = AttnCfg<DPAD, VMN, QK3>::SMEM;
  static DeviceOnce once;
  if (once.first())
    SDB_CUDA(cudaFuncSetAttribute(attention_kernel<DPAD, VMN, QK3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  dim3 grid((p.Nq + 127) / 128, p.heads, p.nb);
  launch_k(attention_kernel<DPAD, VMN, QK3>, grid, dim3(384), (size_t)smem, st, m.q, m.k, m.v, m.q_lo, m.k_lo, p);
}
template <int DPAD>
static void launch_attn(const AttnMaps& m, const AttnParams& p, cudaStream_t st) {
  if (p.v_mn)
    launch_attn2<DPAD, true, false>(m, p, st);
  else
    launch_attn2<DPAD, false, false>(m, p, st);
}

bool attention_supports_qk3(int dpad) { return dpad == 48 || dpad == 80; }

void attention_launch(const AttnMaps& m, const AttnParams& p, cudaStream_t st) {
  if (p.qk3) {
    // split q / k operands (levels 0-1 of the UNet: V always MN-major there)
    SDB_CHECK(p.v_mn && attention_supports_qk3(p.dpad), "split q/k attention: head dim / V layout");
    if (p.dpad == 48)
      launch_attn2<48, true, true>(m, p, st);
    else
      launch_attn2<80, true, true>(m, p, st);
    return;
  }
  switch (p.dpad) {
    case 48:
      launch_attn<48>(m, p, st);
      break;
    case 64:
      launch_attn<64>(m, p, st);
      break;
    case 80:
      launch_attn<80>(m, p, st);
      break;
    case 160:
      launch_attn<160>(m, p, st);
      break;
    default:
      throw Error("attention: unsupported head dim " + std::to_string(p.dpad));
  }
}

}  // namespace sdb
