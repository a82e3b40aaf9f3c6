// kgx_testhooks.cuh -- device side of the kgx_test_field hook (include/kgx.h): one primitive per thread, applied to operands
// copied in from the host, so that the tests can feed the branch-free field / distance / jump-rule primitives of
// kgx_field.cuh, kgx_curve.cuh and kgx_kernel.cuh the boundary values that random walks never produce.
#pragma once
#include "../../include/kgx.h"   // KGX_TF_* op codes
#include "kgx_kernel.cuh"
#include "kgx_curve.cuh"

namespace kgx {

// Operands a, b and the result: 8 words per element.  Ops whose result is narrower than a field element zero the rest.
__global__ void test_field_kernel(int op, int n, const u32* a, const u32* b, u32* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u32 x[8], y[8], r[8];
#pragma unroll
  for (int w = 0; w < 8; w++) { x[w] = a[i * 8 + w]; y[w] = b[i * 8 + w]; r[w] = 0; }
  switch (op) {
    case KGX_TF_MUL: fe_mul(r, x, y); break;
    case KGX_TF_SQR: fe_sqr(r, x); break;
    case KGX_TF_SUB: fe_sub(r, x, y); break;
    case KGX_TF_INV: fe_inv(r, x); break;
    case KGX_TF_MUL_INPLACE: fe_mul(x, x, y); fe_copy(r, x); break;          // the aliased forms of the jump pass
    case KGX_TF_SQR_INPLACE: fe_sqr(x, x); fe_copy(r, x); break;
    case KGX_TF_SUB_INPLACE: fe_sub(x, x, y); fe_copy(r, x); break;
    case KGX_TF_GT_HALF: r[0] = fe_gt_half_mask(x); break;
    case KGX_TF_CNEG: fe_cneg(x, y[0]); fe_copy(r, x); break;
    case KGX_TF_D128_ADD: d128_add(x, y[0], y[1], y[2], y[3]); for (int w = 0; w < 4; w++) r[w] = x[w]; break;
    case KGX_TF_D128_CNEG: d128_cneg(x, y[0]); for (int w = 0; w < 4; w++) r[w] = x[w]; break;
    case KGX_TF_IS_ZERO: r[0] = fe_is_zero_modp(x) ? 1u : 0u; break;
    case KGX_TF_NEG: fe_neg(r, x); break;
    case KGX_TF_DBL: fe_dbl(r, x); break;
    case KGX_TF_JUMP_INDEX:
      r[0] = jump_index<true>(x[0], y[0], (int)y[1]);
      r[1] = jump_index<false>(x[0], y[0], (int)y[1]);
      break;
    case KGX_TF_SYM_NEXT_AUX: r[0] = sym_next_aux(y[0], x[0], x[1], (int)y[1]); break;
  }
#pragma unroll
  for (int w = 0; w < 8; w++) out[i * 8 + w] = r[w];
}

}  // namespace kgx
