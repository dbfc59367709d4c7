// Epilogue activations shared by the GEMM kernels (gemm.cu, linear_w8.cu).
#pragma once
#include "../../include/b200mix.h"

namespace b200 {

// Epilogue activations. All are of the form x * sigmoid(q(x)) and cost one ex2 + one rcp on the MUFU pipe, so a
// GEGLU / SiLU epilogue stays well inside the tensor-core time of its tile.
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float x_sigmoid_neg_log2(float x, float neg_q_log2e) {  // x / (1 + 2^neg_q_log2e)
  return __fdividef(x, 1.0f + ex2_approx(neg_q_log2e));
}
__device__ __forceinline__ float act_silu(float x) { return x_sigmoid_neg_log2(x, -1.4426950408889634f * x); }
// Exact-erf GELU  x * Phi(x)  with  Phi(x) = sigmoid(2 x (c0 + c1 x^2 + c2 x^4)),  coefficients fitted (minimax over
// [-7,7]) so that |gelu_fast - gelu_erf| <= 3.1e-5 absolute: 250x below the bf16 rounding of the output. The quartic
// coefficient is negative, so the polynomial is only evaluated for x^2 <= 49 (ACT_X2_MAX): beyond |x| = 7 the exponent
// continues linearly (slope 2 * 1.788), where both Phi and the sigmoid differ from 0 / 1 by < 1e-12, and it
// saturates to exactly x (x -> +inf) and exactly 0 (x -> -inf: 2^(+big) = inf, x / inf = 0) like erf-GELU does
// (the reference asserts gelu(-100) == 0 and gelu(20) == 20, ppdiffusers/tests/models/test_activations.py:55-63).
constexpr float ACT_X2_MAX = 49.0f;
__device__ __forceinline__ float act_gelu_erf(float x) {
  const float k = -2.0f * 1.4426950408889634f;
  const float c0 = 7.97627599e-01f * k, c1 = 3.69255429e-02f * k, c2 = -3.41174308e-04f * k;
  const float x2 = fminf(x * x, ACT_X2_MAX);
  return x_sigmoid_neg_log2(x, x * fmaf(fmaf(c2, x2, c1), x2, c0));
}
// tanh-GELU: 0.5 x (1 + tanh(u)) == x * sigmoid(2u), u = sqrt(2/pi) (x + 0.044715 x^3)   (identity, not an approximation)
__device__ __forceinline__ float act_gelu_tanh(float x) {
  const float k = -2.0f * 1.4426950408889634f * 0.7978845608028654f;
  return x_sigmoid_neg_log2(x, x * fmaf(k * 0.044715f, x * x, k));
}
__device__ __forceinline__ float act_quick_gelu(float x) { return x_sigmoid_neg_log2(x, -1.702f * 1.4426950408889634f * x); }

// All four share the form x / (1 + 2^(x (c0 + c1 x^2 + c2 x^4))); the coefficients are picked ONCE per kernel so the
// unrolled per-element code is branch-free (a switch per element serialises the 32 MUFU chains of a chunk: measured
// 16 us instead of 5 us per 128x256 tile). With c1 = c2 = 0 the polynomial is exactly c0, so every activation keeps the
// bits of its dedicated function above.
struct ActCoef {
  float c0, c1, c2;
};
__device__ __forceinline__ ActCoef act_coef(int act, int glu) {
  const float l2e = 1.4426950408889634f;
  if (glu == B200MIX_GLU_GEGLU) act = B200MIX_ACT_GELU_ERF;
  else if (glu) act = B200MIX_ACT_SILU;
  ActCoef a = {0.0f, 0.0f, 0.0f};
  switch (act) {
    case B200MIX_ACT_SILU: a.c0 = -l2e; break;
    case B200MIX_ACT_GELU_ERF: {
      const float k = -2.0f * l2e;
      a.c0 = 7.97627599e-01f * k, a.c1 = 3.69255429e-02f * k, a.c2 = -3.41174308e-04f * k;
      break;
    }
    case B200MIX_ACT_GELU_TANH: {
      const float k = -2.0f * l2e * 0.7978845608028654f;
      a.c0 = k, a.c1 = k * 0.044715f;
      break;
    }
    case B200MIX_ACT_QUICK_GELU: a.c0 = -1.702f * l2e; break;
    default: break;
  }
  return a;
}
__device__ __forceinline__ float act_eval(float x, const ActCoef& a) {
  // x^2 is clamped to the range the erf-GELU polynomial was fitted on (see act_gelu_erf); SiLU / quick-GELU have
  // c1 = c2 = 0 and tanh-GELU is saturated to 1 ulp long before |x| = 7, so the clamp changes none of them
  const float x2 = fminf(x * x, ACT_X2_MAX);
  return x_sigmoid_neg_log2(x, x * fmaf(fmaf(a.c2, x2, a.c1), x2, a.c0));
}

}  // namespace b200
