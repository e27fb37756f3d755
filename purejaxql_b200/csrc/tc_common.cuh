// PTX wrappers and constants of the wgmma / mma.sync / TMA / mbarrier GEMM path (sm_90a).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace pqn {
namespace tc {

constexpr int TC_CONSUMERS = 256;        // two consumer warpgroups: rows 0-63 and 64-127 of the 128 x 128 tile
constexpr int TC_THREADS = TC_CONSUMERS + 32;   // + one TMA producer warp (warp 8)
constexpr int TC_BK16 = 64;              // fp16 elements per k-block = one 128-byte swizzle row
constexpr int TC_BK = 32;                // fp32 (TF32 path) elements per k-block = one 128-byte swizzle row
constexpr int TC_STAGES = 2;             // 2 x 64 KB operand stages + the 66 KB fp32 tile fit in 227 KB
constexpr int TC_PROMOTE = 4;            // k-blocks per register main chain (16 k-steps) before promotion to the fp32 tile
constexpr int TC_TILE_BYTES = 128 * TC_BK16 * 2;  // 16 KB: 128 rows x 128 bytes
// fp16 split: x = hi + lo' * 2^-11 with hi = fp16(x), lo' = fp16((x - hi) * 2^11): 22 significant bits, the scaled lo'
// stays a normal fp16 number down to |x| ~ 1e-7.  The two cross products accumulate in their own `corr` register
// accumulator in units of 2^-11.
constexpr float TC_LO_SCALE = 2048.0f, TC_LO_INV = 1.0f / 2048.0f;
constexpr int TC_A_HI = 0, TC_A_LO = TC_TILE_BYTES, TC_B_HI = 2 * TC_TILE_BYTES, TC_B_LO = 3 * TC_TILE_BYTES;
constexpr int TC_STAGE_BYTES = 4 * TC_TILE_BYTES;  // 64 KB
constexpr int TC_ACC_LD = 132;           // floats per row of the fp32 result tile (conflict-free 16-byte row reads)
constexpr int TC_SP_FLOATS = 384 + 8 * 128 + 8;   // per-seed epilogue parameters (LN scale/bias, Q-head)
constexpr int TC_SMEM_BYTES = TC_STAGES * TC_STAGE_BYTES + 128 * TC_ACC_LD * 4 + TC_SP_FLOATS * 4 + 256 /*barriers*/ +
                              1024 /*align slack*/;
// TMA-store epilogues: warpgroup wg stages its 64 x 128 fp32 result as four SWIZZLE_128B boxes of [64 rows][32 floats]
// at byte wg * TC_OUT_STAGE_WG of the fp32 tile region, which lies inside the tile rows that warpgroup owns
constexpr int TC_OUT_BOX_BYTES = 64 * 32 * 4;     // 8 KB
constexpr int TC_OUT_STAGE_WG = 34 * 1024;
static_assert(TC_OUT_STAGE_WG >= 64 * TC_ACC_LD * 4 && TC_OUT_STAGE_WG + 4 * TC_OUT_BOX_BYTES <= 128 * TC_ACC_LD * 4,
              "each warpgroup's output staging lies within its own 64 rows of the fp32 tile, 1024-byte aligned");
#define PQN_TC_MAX_A 8

enum Epilogue : int { EPI_STORE = 0, EPI_LN_TRAIN = 1, EPI_LN_HEAD = 2, EPI_RELU_MASK = 3, EPI_RELU_BITS = 4 };

struct GemmShape {
  int S;         // batch (seeds)
  int M;         // rows of D that exist (rows >= M are not stored)
  int m_tiles, n_tiles, k_blocks;
  int split3;    // TF32 kernel only: 0 single pass, 1 3xTF32 with A_lo from memory, 2 3xTF32 with A_lo derived in the
                 // kernel (the fp16 kernel always takes both planes of both operands)
  int k_split;   // >1: the k-blocks of every output tile are divided over k_split CTAs; partial ks goes to
                 // out + ks * EpiParams::split_stride (EPI_STORE only) and a reduce kernel adds them in order
};

struct EpiParams {
  int64_t split_stride;  // elements between the partial outputs of a split-K launch
  float out_scale;  // result = (main + corr * 2^-11) * out_scale (undoes the operand pre-scaling); 0 => 1
  // EPI_STORE / EPI_RELU_MASK
  float* out;
  const float* mask;
  const uint32_t* relu_bits;  // EPI_RELU_BITS: [S][rows][ld_out / 32] words, bit c of a row = (activation c > 0)
  int64_t ld_out, out_seed_stride;
  // EPI_LN_*
  const float* params;
  int64_t P, off_b, off_scale, off_bias, off_hw, off_hb;
  int A, rows;
  float *H, *XHAT, *RSTD, *Q;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ float tf32_lo(float x) {
  const float hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);  // what a TF32 tensor-core read keeps of x
  return x - hi;                                                       // exact in fp32
}

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!ok);
}

// ---- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// shared -> global tensor store; completion is tracked per issuing thread by bulk async-groups
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory sources of all committed bulk stores have been read (the staging area may be rewritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// all committed bulk stores are complete
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// makes this thread's generic-proxy shared-memory writes visible to a following TMA (async-proxy) read
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads/writes across the asynchronous MMAs
__device__ __forceinline__ void fence_operands(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] . B[16 x 128], fp16 operands from shared memory, fp32 accumulate in registers.
// TA / TB = 1: the operand is MN-major in shared memory (transposed read).  scale_d = 0 overwrites D.
// D fragment of thread t of the warpgroup: rows 16 * (t / 32) + (t % 32) / 4 (+ 8), columns 8 j + 2 (t % 4) (+ 1):
// d[4j], d[4j+1] on the first row, d[4j+2], d[4j+3] on the second.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_m64n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
      "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

// The same product with A[64 x 16] from registers: each warp of the warpgroup holds rows 16 (warp % 4) .. + 15 in the
// mma.sync m16n8k16 A layout, a[0] = (row g, k 2t, 2t+1), a[1] = (g + 8, 2t ..), a[2] = (g, 2t + 8 ..),
// a[3] = (g + 8, 2t + 8 ..) with g = lane / 4, t = lane % 4, low half = lower k.  B from shared memory, TB as above.
// The registers of a[] are read asynchronously: they must not be rewritten before the wgmma has retired.
template <int TB>
__device__ __forceinline__ void wgmma_f16_m64n128_ra(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b,
                                                     uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
      "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, %70;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d), "n"(TB));
}

// Shared-memory matrix descriptor (sm_90 GMMA: start >> 4 at bits 0-13, LBO >> 4 at 16-29, SBO >> 4 at 32-45,
// layout type at 62-63, 1 = SWIZZLE_128B) for a fp16 operand tile as TMA writes it; k-step `ks` = 16 k values:
//   K-major : 128-byte rows (64 k), 8-row swizzle atoms every 1024 B (SBO); the k-step advances 32 B in the row.
//   MN-major: TMA boxes of [64 k rows][64 mn = 128 B] at 8192 B (LBO: next 64 MN elements), 8-row k atoms of
//             1024 B (SBO); one k-step (16 k rows) = 2048 B.
// Tile bases are 1024-byte aligned, so the swizzle phase (base offset) is 0.
template <int MN>
__device__ __forceinline__ uint64_t make_gdesc16(uint32_t tile_addr, int ks) {
  const uint32_t addr = MN ? tile_addr + ks * 2048 : tile_addr + ks * 32;
  const uint64_t lbo = MN ? (8192u >> 4) : 1u;
  const uint64_t sbo = 1024u >> 4;
  return (uint64_t)((addr >> 4) & 0x3FFFu) | (lbo << 16) | (sbo << 32) | (1ull << 62);
}

// fp16 split of an fp32 value (see TC_LO_SCALE); saturates instead of overflowing to inf
__device__ __forceinline__ void split16(float x, __half& hi, __half& lo) {
  x = fminf(fmaxf(x, -65000.0f), 65000.0f);
  hi = __float2half_rn(x);
  lo = __float2half_rn((x - __half2float(hi)) * TC_LO_SCALE);
}
// SAT = false: the caller guarantees |x| < 65504 (e.g. LayerNorm outputs: |xhat| <= sqrt(n - 1))
template <bool SAT = true>
__device__ __forceinline__ void split16x2(float x0, float x1, __half2& hi, __half2& lo) {
  if (SAT) {
    x0 = fminf(fmaxf(x0, -65000.0f), 65000.0f);
    x1 = fminf(fmaxf(x1, -65000.0f), 65000.0f);
  }
  hi = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(hi);
  lo = __floats2half2_rn((x0 - hf.x) * TC_LO_SCALE, (x1 - hf.y) * TC_LO_SCALE);
}

// host-side pieces used by other translation units (pqn_net.cu)
// fp32 tensor [seeds][mid][inner] with a {32, box_mid, 1} box, SWIZZLE_128B for both majors
int make_tmap(CUtensorMap* tm, const float* base, uint64_t inner, uint64_t mid, uint64_t seeds, uint64_t mid_stride_elems,
              uint64_t seed_stride_elems, uint32_t box_mid);
// the TF32 kernel: t = {A, A_lo, B, B_lo} fp32 maps, gs.k_blocks counts 32-element k-blocks
int launch_gemm(int a_mn, int b_mn, int epi, const CUtensorMap* t, const GemmShape& gs, const EpiParams& ep, cudaStream_t st,
                int kernel_id = -1);
// fp16 tensor [seeds][mid][inner] with a {64, box_mid, 1} box (128 bytes x box_mid), SWIZZLE_128B for both majors
int make_tmap16(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t mid, uint64_t seeds, uint64_t mid_stride_elems,
                uint64_t seed_stride_elems, uint32_t box_mid);
// the fp16-split kernel: t = {A_hi, A_lo', B_hi, B_lo'} fp16 maps, gs.k_blocks counts 64-element k-blocks
int launch_gemm16(int a_mn, int b_mn, int epi, const CUtensorMap* t, const GemmShape& gs, const EpiParams& ep,
                  cudaStream_t st, int kernel_id = -1);

}  // namespace tc
}  // namespace pqn
