// attention.cuh — launch descriptor of the fused attention kernel.
#pragma once
#include "common.cuh"

namespace sdb {

struct AttnParams {
  int nb, heads, d, dpad;
  int Nq, Nk;                 // query rows per sample / maximum key rows per sample
  int q_rows_per_sample;      // row stride between samples in the Q matrix (and in the output)
  int k_rows_per_sample;      // row stride between samples in K (= column stride in V^T)
  int q_col0, k_col0;         // first column of head 0 inside the Q / K matrices
  int qk3;                    // 1: q and k are fp16 hi + lo pairs, S is the 3-term split product (fp32-class logits)
  int v_mn, v_col0;           // v_mn = 1: V is a [keys][ldv] matrix (head h at columns v_col0 + h*dpad) consumed MN-major;
                              // v_mn = 0: V^T [heads*d][ldv] (sample s at columns s*k_rows)
  const int* kvlen;           // [nb] valid keys per sample, or null (= Nk)
  int causal;                 // 1: query row i attends to keys 0..i only
  float scale;                // d^-1/2
  __half* out_hi;             // [nb*Nq][ldo], head h at columns h*d
  __half* out_lo;             // optional residual half
  int ldo;
  long long* dbg;             // bring-up aid (SDB_ATTN_DBG): clock64 stamps of CTA (0,0,0), key tiles 8..11, or null
};

struct AttnMaps {
  CUtensorMap q, k, v, q_lo, k_lo;  // q_lo / k_lo: the lo halves (same geometry) when p.qk3, else copies of q / k
};
void attention_launch(const AttnMaps& m, const AttnParams& p, cudaStream_t st);
bool attention_supports_qk3(int dpad);

}  // namespace sdb
