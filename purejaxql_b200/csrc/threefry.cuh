// jax.random (threefry2x32) semantics, as consumed by the PQN hot path.
//
// Replaces, on device, the PRNG arithmetic the reference reaches through
// jax.random.split / uniform / randint / choice / normal at
//   purejaxql/pqn_minatar.py:107-112 (per-env key split), :116-125 (eps-greedy),
//   :183 (3-way split of the scan carry), and inside gymnax Environment.step.
// Both counter layouts are supported (`part` = jax_threefry_partitionable):
//   part=0  "original" layout, default for the reference's pinned jax<=0.4.38
//   part=1  "partitionable" layout, default from jax 0.5
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PQN_HD __host__ __device__ __forceinline__
#else
#define PQN_HD inline
#ifndef __restrict__
#define __restrict__ __restrict
#endif
#endif

namespace pqn {

struct Key {
  uint32_t k0, k1;
};

PQN_HD uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

// Threefry-2x32, 20 rounds (Random123).
PQN_HD void threefry2x32(uint32_t k0, uint32_t k1, uint32_t& x0, uint32_t& x1) {
  const uint32_t k2 = k0 ^ k1 ^ 0x1BD11BDAu;
  x0 += k0;
  x1 += k1;
#define PQN_TF_R(r) \
  x0 += x1;         \
  x1 = rotl32(x1, r) ^ x0;
  PQN_TF_R(13) PQN_TF_R(15) PQN_TF_R(26) PQN_TF_R(6)
  x0 += k1; x1 += k2 + 1u;
  PQN_TF_R(17) PQN_TF_R(29) PQN_TF_R(16) PQN_TF_R(24)
  x0 += k2; x1 += k0 + 2u;
  PQN_TF_R(13) PQN_TF_R(15) PQN_TF_R(26) PQN_TF_R(6)
  x0 += k0; x1 += k1 + 3u;
  PQN_TF_R(17) PQN_TF_R(29) PQN_TF_R(16) PQN_TF_R(24)
  x0 += k1; x1 += k2 + 4u;
  PQN_TF_R(13) PQN_TF_R(15) PQN_TF_R(26) PQN_TF_R(6)
  x0 += k2; x1 += k0 + 5u;
#undef PQN_TF_R
}

// Word j (0 <= j < 2*num) of the flat output of the original-layout
// threefry_2x32(key, iota(2*num)): blocks are (c, c+num), outputs concat(y0, y1).
PQN_HD uint32_t split_word_original(Key k, uint32_t num, uint32_t j) {
  uint32_t c = (j < num) ? j : j - num;
  uint32_t x0 = c, x1 = c + num;
  threefry2x32(k.k0, k.k1, x0, x1);
  return (j < num) ? x0 : x1;
}

// jax.random.split(key, num)[i]
PQN_HD Key split_at(Key k, uint32_t num, uint32_t i, int part) {
  Key out;
  if (part) {
    uint32_t x0 = 0u, x1 = i;
    threefry2x32(k.k0, k.k1, x0, x1);
    out.k0 = x0;
    out.k1 = x1;
  } else {
    out.k0 = split_word_original(k, num, 2u * i);
    out.k1 = split_word_original(k, num, 2u * i + 1u);
  }
  return out;
}

// jax.random.split(key) -> both children (num = 2); 2 blocks in the original
// layout ((0,2) -> a0,b0 ; (1,3) -> a1,b1 ; child0 = (a0,a1), child1 = (b0,b1)).
PQN_HD void split2(Key k, int part, Key& c0, Key& c1) {
  if (part) {
    uint32_t a0 = 0u, a1 = 0u, b0 = 0u, b1 = 1u;
    threefry2x32(k.k0, k.k1, a0, a1);
    threefry2x32(k.k0, k.k1, b0, b1);
    c0.k0 = a0; c0.k1 = a1; c1.k0 = b0; c1.k1 = b1;
  } else {
    uint32_t a0 = 0u, b0 = 2u, a1 = 1u, b1 = 3u;
    threefry2x32(k.k0, k.k1, a0, b0);
    threefry2x32(k.k0, k.k1, a1, b1);
    c0.k0 = a0; c0.k1 = a1; c1.k0 = b0; c1.k1 = b1;
  }
}

// jax.random.split(key, 3): original layout blocks (0,3),(1,4),(2,5) ->
// out = [a0,a1,a2,b0,b1,b2] -> children (a0,a1),(a2,b0),(b1,b2).
PQN_HD void split3(Key k, int part, Key& c0, Key& c1, Key& c2) {
  if (part) {
    c0 = split_at(k, 3, 0, 1); c1 = split_at(k, 3, 1, 1); c2 = split_at(k, 3, 2, 1);
  } else {
    uint32_t a0 = 0u, b0 = 3u, a1 = 1u, b1 = 4u, a2 = 2u, b2 = 5u;
    threefry2x32(k.k0, k.k1, a0, b0);
    threefry2x32(k.k0, k.k1, a1, b1);
    threefry2x32(k.k0, k.k1, a2, b2);
    c0.k0 = a0; c0.k1 = a1; c1.k0 = a2; c1.k1 = b0; c2.k0 = b1; c2.k1 = b2;
  }
}

// random_bits(key, 32, shape)[i] for a shape with n elements.
PQN_HD uint32_t bits_at(Key k, uint32_t n, uint32_t i, int part) {
  if (part) {
    uint32_t x0 = 0u, x1 = i;
    threefry2x32(k.k0, k.k1, x0, x1);
    return x0 ^ x1;
  }
  const uint32_t half = (n + 1u) >> 1;
  const bool lo = i < half;
  const uint32_t c = lo ? i : i - half;
  uint32_t x0 = c, x1 = c + half;
  if ((n & 1u) && c == half - 1u) x1 = 0u;  // the odd-size pad counter is a literal 0
  threefry2x32(k.k0, k.k1, x0, x1);
  return lo ? x0 : x1;
}

// random_bits(key, 32, ()) : scalar draw.
PQN_HD uint32_t bits_scalar(Key k, int part) { return bits_at(k, 1u, 0u, part); }

PQN_HD float bits_to_unit_float(uint32_t bits) {
  const uint32_t fb = (bits >> 9) | 0x3F800000u;
#if defined(__CUDA_ARCH__)
  return __uint_as_float(fb) - 1.0f;
#else
  union { uint32_t u; float f; } cv;
  cv.u = fb;
  return cv.f - 1.0f;
#endif
}

// jax.random.uniform(key, (), f32, minval, maxval)
PQN_HD float uniform_from_bits(uint32_t bits, float minval, float maxval) {
  float f = bits_to_unit_float(bits) * (maxval - minval) + minval;
  return f < minval ? minval : f;
}
PQN_HD float uniform_scalar(Key k, int part) { return uniform_from_bits(bits_scalar(k, part), 0.0f, 1.0f); }

// ---------------------------------------------------------------------------
// jax.random.normal(key, shape, f32): jax 0.4.x `_normal_real`,
//   u = uniform(key, shape, lo = nextafter(-1, 0), hi = 1);  sqrt(2) * lax.erf_inv(u)
// with lax.erf_inv lowered (chlo.erf_inv) to XLA's fp32 form of M. Giles' approximation ("Approximating the erfinv
// function", GPU Computing Gems Jade Edition, 2011):
//   w = -log1p(-x * x)
//   w < 5:  t = w - 2.5,      p = Horner over the 9 "central" coefficients in t
//   else:   t = sqrt(w) - 3,  p = Horner over the 9 "tail" coefficients in t
//   erf_inv(x) = x * inf where |x| == 1, else p * x
// The uniform here is 2 f - (1 - 2^-24) for f = (bits >> 9) * 2^-23: exact in fp32, never 0 and never +-1, so the
// normal takes exactly 2^23 values, one per value of bits >> 9, and the |x| == 1 case cannot occur.  Both branches
// occur (w >= 5 for |u| > 0.9966).
//
// Two points of XLA:GPU's code generation are recollection, not checked against a live jax, and fix the bits:
//  (1) log1p is libdevice's log1pf, applied to the rounded product x * x.  This code calls log1pf (libdevice's on the
//      device, the C library's on the host) on __fmul_rn(x, x), which no -fmad setting fuses into log1pf's first add.
//  (2) LLVM's NVPTX backend contracts each Horner step p * t + c into one fma (its default fma level fuses an fmul
//      feeding an fadd).  The steps are written as fmaf, so the bits do not depend on the -fmad of the unit that
//      includes this header.  jax on the CPU does not contract and gives a different last bit in some values.
// tests/golden/make_gaussian_bandit_golden_from_ref.py records jax's values on the CPU and on a CUDA device.
PQN_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
PQN_HD float sqrt_rn(float a) {
#if defined(__CUDA_ARCH__)
  return __fsqrt_rn(a);
#else
  return sqrtf(a);
#endif
}

// w = -log1p(-x * x), the argument of erf_inv's polynomial
PQN_HD float erf_inv_w(float x) { return -log1pf(-mul_rn(x, x)); }

// erf_inv(x) given w = erf_inv_w(x): the polynomial part, which is exact fp32 arithmetic with no library call
PQN_HD float erf_inv_from_w(float x, float w) {
  float p;
  if (w < 5.0f) {
    const float t = w - 2.5f;
    p = 2.81022636e-08f;
    p = fmaf(p, t, 3.43273939e-07f);
    p = fmaf(p, t, -3.5233877e-06f);
    p = fmaf(p, t, -4.39150654e-06f);
    p = fmaf(p, t, 0.00021858087f);
    p = fmaf(p, t, -0.00125372503f);
    p = fmaf(p, t, -0.00417768164f);
    p = fmaf(p, t, 0.246640727f);
    p = fmaf(p, t, 1.50140941f);
  } else {
    const float t = sqrt_rn(w) - 3.0f;
    p = -0.000200214257f;
    p = fmaf(p, t, 0.000100950558f);
    p = fmaf(p, t, 0.00134934322f);
    p = fmaf(p, t, -0.00367342844f);
    p = fmaf(p, t, 0.00573950773f);
    p = fmaf(p, t, -0.0076224613f);
    p = fmaf(p, t, 0.00943887047f);
    p = fmaf(p, t, 1.00167406f);
    p = fmaf(p, t, 2.83297682f);
  }
  return (x == 1.0f || x == -1.0f) ? x * INFINITY : p * x;
}

PQN_HD float erf_inv(float x) { return erf_inv_from_w(x, erf_inv_w(x)); }

// jax.random.normal's value for the 32 random bits of one element
PQN_HD float normal_from_bits(uint32_t bits) {
  const float u = uniform_from_bits(bits, -0.99999994f /* nextafter(-1, 0) = -(1 - 2^-24) */, 1.0f);
  return mul_rn(1.41421356237309504880f /* sqrt(2), rounded to fp32 */, erf_inv(u));
}
// jax.random.normal(key, ())
PQN_HD float normal_scalar(Key k, int part) { return normal_from_bits(bits_scalar(k, part)); }

// jax.random.randint(key, (), 0, span) with 1 <= span < 2^16 (small action sets):
//   k1,k2 = split(key); off = ((hi % span) * mult + lo % span) % span,
//   mult = ((2^16 % span)^2) % span, all in uint32.
PQN_HD int32_t randint_scalar(Key k, uint32_t span, int part) {
  Key k1, k2;
  split2(k, part, k1, k2);
  const uint32_t hi = bits_scalar(k1, part);
  const uint32_t lo = bits_scalar(k2, part);
  uint32_t mult = 65536u % span;
  mult = (mult * mult) % span;
  const uint32_t off = ((hi % span) * mult + (lo % span)) % span;
  return (int32_t)off;
}

// randint(key, (n,), lo, hi)[i] — vector draw element (used by Freeway etc.)
PQN_HD int32_t randint_at(Key k, uint32_t n, uint32_t i, int32_t minval, int32_t maxval, int part) {
  Key k1, k2;
  split2(k, part, k1, k2);
  const uint32_t hi = bits_at(k1, n, i, part);
  const uint32_t lo = bits_at(k2, n, i, part);
  uint32_t span = (uint32_t)(maxval - minval);
  if (maxval <= minval) span = 1u;
  uint32_t mult = 65536u % span;
  mult = (mult * mult) % span;
  const uint32_t off = ((hi % span) * mult + (lo % span)) % span;
  return minval + (int32_t)off;
}

}  // namespace pqn
