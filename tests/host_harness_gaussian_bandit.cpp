// CPU logic harness of jax.random.normal and GaussianBandit-misc — TEST INFRASTRUCTURE ONLY (built by
// tests/test_gaussian_bandit_host.py).  Compiles the same __host__ __device__ functions the CUDA kernels use
// (threefry.cuh's normal_from_bits and erf_inv, env_misc.cuh's GaussianBanditEnv) with g++, driving the env in the
// order the kernels of pqn_env.cu call it (the loops of host_harness_misc.cpp, included here), so that both can be
// checked against the NumPy oracles without a GPU.  The product never calls this.
//
// On the host, log1pf is the C library's; on the device it is libdevice's.  h_log1pf and h_erf_inv_from_w let the
// tests take that one library call apart from the rest, which is exact fp32 arithmetic on both.
#include "host_harness_misc.cpp"

extern "C" {
PQN_HARNESS(gaussian_bandit, GaussianBanditEnv)

void h_normal_from_bits(const uint32_t* bits, float* out, int64_t n) {
  for (int64_t i = 0; i < n; ++i) out[i] = normal_from_bits(bits[i]);
}
void h_normal_scalar(const uint32_t* keys, float* out, int64_t n, int part) {
  for (int64_t i = 0; i < n; ++i) out[i] = normal_scalar(Key{keys[2 * i], keys[2 * i + 1]}, part);
}
void h_log1pf(const float* x, float* out, int64_t n) {
  for (int64_t i = 0; i < n; ++i) out[i] = log1pf(x[i]);
}
void h_erf_inv_from_w(const float* x, const float* w, float* out, int64_t n) {
  for (int64_t i = 0; i < n; ++i) out[i] = erf_inv_from_w(x[i], w[i]);
}
}
