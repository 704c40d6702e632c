// Persistent wgmma sampler kernel: phase table + launch (see sampler_tc.cu).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace ssb {

enum SPhaseMode { SP_GATE = 0, SP_RES_SKIP = 1, SP_INPROJ = 2, SP_SKIPPROJ = 3, SP_MEL_SAMPLE = 4, SP_F0_SAMPLE = 5 };

// One GEMM phase of the persistent sampler: D[128 x 64 tiles] = A1 (*) W1, then a fused epilogue.
struct SPhase {
  int a1;              // tensor-map index of the A operand's hi plane (lo = +1)
  int w1;              // tensor-map index of the weights' hi plane (lo = +1), box [64 x 64]
  int taps, kchunks, dil, center, N, NT;
  int mode;
  const float* bias;   // [N]
  float wscale;        // ConvTC::wscale of the weights w1: the epilogue takes acc * wscale + bias
  float* out;          // fp32 output (x, or the sampler state x_t [rows,80])
  int ldo;
  __half* oh;          // fp16 hi/lo planes output
  __half* ol;
  int ldh;
  const float* res;    // RES_SKIP: residual stream in
  int ld_res;
  float beta;
  const float* vec2;   // step bias added before the planes are written
  const float* add;    // GATE: hoisted conditioner projection of this layer [rows, ld_add] (packed gate column order)
  int ld_add;
  float* skip;         // RES_SKIP: skip accumulator
  int ld_skip, C, skip_init;
  __half* sh;          // RES_SKIP (last layer): planes of the finished skip sum
  __half* sl;
  const float* tab;    // MEL_SAMPLE: 8 schedule scalars of this step
  const float* noise;  // MEL_SAMPLE: tight [total, 80] noise of this step, or null (Philox)
  unsigned long long stream_id;        // Philox stream of the Gaussian draws, keyed per utterance (SeqDev::rng)
  unsigned long long stream2;          // F0_SAMPLE: Philox stream of the uniform draws
  int n_valid;         // MEL_SAMPLE / SKIPPROJ: valid output columns
  int sync_after;      // 1: grid barrier after this entry; 0: the next entry is independent (e.g. the other F0 net)
  int goff;            // tile-group rotation: group g is processed by cluster (g + goff) % nclusters
  int no_clip;         // MEL_SAMPLE: 1 = use x0 as predicted, no clamp to [-1, 1] (ProDiff p_sample, prodiff.py:143-148)
  // F0_SAMPLE (GaussianMultinomialDiffusion step, gaussian_multinomial_diffusion.py:325-333,398-413) + next DDiffNet input
  int tstep, has_next;
  float log_eps;
  int32_t* uv;         // class state [rows]
  const float* clip_lo;
  const float* clip_hi;
  const float* tab2;   // multinomial schedule scalars of this step
  const float* noise2; // tight [total, 2] uniform noise of this step, or null
  const float* in_w;   // DDiffNet input_projection weight / bias [C/2], uv embedding [2][C/2]
  const float* in_b;
  const float* uv_emb;
  float* x_next;       // residual stream of the next step [rows, C]
};

int sampler_tc_max_ctas();
int sampler_tc_max_clusters(int cs);  // co-resident clusters of size cs (cooperative launch limit)
// runs the phases over the row tiles of `s`; the sampling phases draw with s.rng.  single_pass: one hi*hi wgmma per K step
// (the lo planes are not read) instead of the 3-pass hi/lo split.
int launch_sampler_tc(Ctx& ctx, const CUtensorMap* maps_dev, const SPhase* phases_dev, int nphases, const SeqDev& s,
                      int max_nt, unsigned* barrier_ctr, int cs, bool single_pass);
int x80_planes(Ctx& ctx, const float* x, int64_t rows, __half* hi, __half* lo);

}  // namespace ssb
