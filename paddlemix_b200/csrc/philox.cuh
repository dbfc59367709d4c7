// Counter-based random numbers shared by the samplers: Philox4x32-10 (Salmon et al., SC'11; Random123's
// philox4x32-10), and the standard-normal transform of b200mix_iddpm_step. oracle/generation.py restates both on the CPU.
#pragma once
#include <cstdint>

namespace b200 {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k.x += 0x9E3779B9u;
      k.y += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// Four standard normals for element group g (elements 4g .. 4g+3) at `step`:
//   (r0, r1, r2, r3) = philox4x32_10(counter = (step, g mod 2^32, g div 2^32, 0), key = (seed mod 2^32, seed div 2^32))
//   u_k = (r_k + 0.5) * 2^-32                                   (in (0, 1), exact in fp64)
//   z0 = fp32(sqrt(-2 ln u0) cos(2 pi u1)),  z1 = fp32(sqrt(-2 ln u0) sin(2 pi u1))
//   z2 = fp32(sqrt(-2 ln u2) cos(2 pi u3)),  z3 = fp32(sqrt(-2 ln u2) sin(2 pi u3))
// Box-Muller in fp64, each result rounded once to fp32; 2 pi is the fp64 constant 6.283185307179586.
__device__ __forceinline__ void philox_normal4(unsigned long long seed, uint32_t step, unsigned long long g, float z[4]) {
  const uint4 r = philox4x32_10(make_uint4(step, (uint32_t)g, (uint32_t)(g >> 32), 0u),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const double u0 = ((double)w[2 * p] + 0.5) * 2.3283064365386963e-10;  // 2^-32
    const double u1 = ((double)w[2 * p + 1] + 0.5) * 2.3283064365386963e-10;
    const double rad = sqrt(__dmul_rn(-2.0, log(u0)));
    double s, c;
    sincos(__dmul_rn(6.283185307179586, u1), &s, &c);
    z[2 * p] = (float)__dmul_rn(rad, c);
    z[2 * p + 1] = (float)__dmul_rn(rad, s);
  }
}

}  // namespace b200
