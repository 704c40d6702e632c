#pragma once
#include "common.cuh"

namespace ssb {

struct AttnArgs {
  const int4* utt_q = nullptr;  // query layout table
  const int4* utt_k = nullptr;  // key/value layout table
  int B = 0;
  int max_q = 0;                // max query length (grid sizing)
  int heads = 2;                // head dim is fixed at 128
  const float* Q = nullptr; int ldq = 0;
  const float* K = nullptr; int ldk = 0;
  const float* V = nullptr; int ldv = 0;
  const float* keymask = nullptr;  // per key row (guarded), 1 = attend, 0 = -inf; may be null
  float scale = 1.0f;              // applied to q (hd^-0.5)
  float* out = nullptr; int ldo = 0;
};

int attention(Ctx& ctx, const AttnArgs& a);

// wgmma / TMA attention for long batches (attention_tc.cu).  Operands are fp16 hi/lo planes:
//   Q  [rows_q, ldq], head h at columns qcol0 + 128 h;   K [rows_k, ldk], head h at columns kcol0 + 128 h;
//   V^T [heads * 128, ldvt]: row = head * 128 + d, column = key row of the K/V layout (transpose_planes below).
// Output: fp32 [rows_q, ldo] and / or fp16 hi/lo planes [rows_q, ldh] (head h at columns 128 h).
struct AttnTCArgs {
  const int4* utt_q = nullptr;
  const int4* utt_k = nullptr;
  int B = 0, max_q = 0, heads = 2;
  const __half* Qh = nullptr; const __half* Ql = nullptr; int64_t rows_q = 0; int ldq = 0; int qcol0 = 0;
  const __half* Kh = nullptr; const __half* Kl = nullptr; int64_t rows_k = 0; int ldk = 0; int kcol0 = 0;
  const __half* Vth = nullptr; const __half* Vtl = nullptr; int64_t ldvt = 0;
  const float* keymask = nullptr;
  float scale = 1.0f;
  float* out = nullptr; int ldo = 0;
  __half* oh = nullptr; __half* ol = nullptr; int ldh = 0;
};
int attention_tc(Ctx& ctx, const AttnTCArgs& a);
bool attention_tc_enabled();           // process-wide switch for the long-batch paths (ssb_set_attention_tensor_cores; default on)
int set_attention_tc_enabled(int on);
// planes [rows, ld] (columns col0 .. col0 + C) -> transposed planes [C, ldt]; columns rows .. ldt are zero-filled
int transpose_planes(Ctx& ctx, const __half* xh, const __half* xl, int ld, int col0, int64_t rows, int C, __half* th, __half* tl,
                     int64_t ldt);

}  // namespace ssb
