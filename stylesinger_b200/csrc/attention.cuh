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

// attention() refuses (before any launch) heads outside {1, 2}, B > 65535 (gridDim.z), no output, an ld that is not a
// multiple of 4 or a pointer that is not 16-byte aligned (the float4 loads and stores), and an ld narrower than heads x 128
// columns.  attention_check() is that check alone, for callers that must refuse before launching anything else.
int attention_check(const AttnArgs& a);
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
// attention_tc() refuses (before any launch) heads outside {1, 2}, B > 65535, no output (out, or both planes), an ld or
// column offset that is not a multiple of 8 (TMA strides and inner coordinates are 16-byte multiples), a pointer that is
// not 16-byte aligned, a column window past its ld (qcol0 + heads x 128 > ldq, kcol0 + heads x 128 > ldk: TMA would
// read zero fill), an output narrower than heads x 128 columns, and V^T narrower than the key rows (ldvt < rows_k).
int attention_tc_check(const AttnTCArgs& a);
int attention_tc(Ctx& ctx, const AttnTCArgs& a);
// launches so far of attention_kernel [0] and attention_tc_kernel [1] (ssb_attention_launch_count)
extern std::atomic<long long> g_attn_launches[2];
bool attention_tc_enabled();          // process-wide switch for the long-batch paths (ssb_set_attention_tensor_cores; default on)
int set_attention_tc_enabled(int on);
// planes [rows, ld] (columns col0 .. col0 + C) -> transposed planes [C, ldt]; columns rows .. ldt are zero-filled.
// Refuses C not a multiple of 32, ldt < rows and a column window col0 + C past ld.
int transpose_planes(Ctx& ctx, const __half* xh, const __half* xl, int ld, int col0, int64_t rows, int C, __half* th, __half* tl,
                     int64_t ldt);

}  // namespace ssb
