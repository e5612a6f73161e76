// Grouped, persistent 3xTF32 GEMM on the Hopper tensor cores (wgmma.mma_async, kind tf32) for the actor / critic /
// discriminator MLPs.
//
// Same contract as phc_gemm (gemm.cu): C[M,N] (+)= epi(alpha * sum_k A(m,k) B(n,k)), both operand major-nesses, fp32 in and
// out, fp32-equivalent numerics.  The reference trains in fp32 and the parity bar is 1e-5, so every fp32 product is made of
// three tensor-core products: x = hi + lo with hi = trunc_tf32(x) and lo = rna_tf32(x - hi) (hi + lo = x to 2^-22 |x|), and
// per k-step D += A_lo*B_hi, D += A_hi*B_lo, D += A_hi*B_hi.  The dropped A_lo*B_lo term is <= 2^-20 |ab|.
//
// wgmma reads tf32 operands from shared memory in K-major order only, so the CTA's threads stage every k-block themselves:
// global -> registers (16-byte loads for both operand orders) -> hi / lo split -> shared memory in the canonical no-swizzle
// K-major layout (8-row x 16-byte core matrices; LBO = 128 B between the core matrices along K, SBO = BK * 32 B between 8-row
// groups).  The k-loop is a software pipeline over a ring of three shared-memory stages: while the wgmmas of k-block i run,
// k-block i + 1 is split and stored into the next stage, and then the global loads of k-block i + 2 are issued and stay in
// flight across the k-block boundary.  wgmma.wait_group 1 keeps one batch queued behind the running one, so the tensor pipe
// is not drained at k-block boundaries; the barrier after it only frees the stage of k-block i - 1 for reuse.
//
// CTA = 256 threads = 2 warpgroups; a tile is 128 x BN (each warpgroup owns 64 rows: one m64nBNk8 wgmma per product and k-step).
//   BN = 128, BK = 32 (default): 3 x 64 KB of shared memory;   BN = 256, BK = 16 (phc_gemm_tc5s_set_tile(256)): 3 x 48 KB.
// One launch takes up to PHC_GEMM_GROUP_MAX independent problems (the same layer of actor, critic and discriminator; dW and dX
// of one layer): their tiles form one list walked by one persistent CTA per SM, in static striding or drawn from a global
// counter (dynamic, the default: a CTA that got long tiles draws fewer of them).
// Split-K slices of one output tile add into C in slice order (a per-tile turnstile in global memory), never by float atomics; so do
// problems of one launch that accumulate into the same C (their slices are numbered one after the other, in problem order): the
// result does not depend on which CTA finishes first, so a run is reproducible bit for bit.  A launch with ordered problems always
// draws its tiles dynamically; a slice then only waits for a lower-numbered tile that a running CTA has already drawn.
// phc_gemm_tc5 is the same kernel with operands pre-split in global memory (hi / lo arrays loaded instead of split).
// A 3xTF32 problem with 128 x 128 tiles that comes with a weight image of B (PhcGemmDesc.B_img) skips the staging: B arrives
// pre-split by bulk copy and A goes from global memory straight into the wgmma register fragment (the image loop below).  One
// that also comes with an image of A (PhcGemmDesc.A_img: the weight gradient, whose operands are both mn-major activations,
// imaged once per launch instead of once per tile) takes both operands by bulk copy into the staged loop's stages (the pair loop).
// A problem with PhcGemmDesc.C_img (128 x 128 tiles, 3xTF32, not accumulating) also writes its output's image from the epilogue:
// a 128 x 128 output tile is exactly four 128 x 32 image blocks, so the next layer's forward or input-gradient GEMM gets its A
// image without a separate pass and runs on the pair loop, which keeps three k-blocks of both operands in flight and does no
// per-thread global loads (the image loop issues 16 scalar A loads per thread and k-block, one k-block ahead).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <type_traits>

#include "../../include/phc_b200.h"
#include "phc_common.cuh"

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

namespace phc {
namespace wg {

constexpr int BM = 128, NUM_THREADS = 256, MAX_PROBLEMS = PHC_GEMM_GROUP_MAX;

template <int BN>
struct Cfg {
  static constexpr int BK = BN == 128 ? 32 : 16;
  static constexpr int A_TILE = BM * BK * 4;
  static constexpr int B_TILE = BN * BK * 4;
  static constexpr int STAGE = 2 * (A_TILE + B_TILE);           // [A hi | A lo | B hi | B lo]
  static constexpr int STAGES = 3;
  static constexpr int SMEM = STAGES * STAGE;
  static constexpr int SBO = BK * 32;                           // bytes between 8-row groups
  static constexpr int A_PER = BM * BK / NUM_THREADS;           // staged elements per thread
  static constexpr int B_PER = BN * BK / NUM_THREADS;
};

// Weight images (PhcGemmDesc.B_img, made by phc_gemm_make_images): B pre-split and pre-laid-out for the 128 x 128 x 32 tile.
// One block of IMG_BLOCK floats per (128-row n-tile, 32-wide k-block), block (nt, kb) at nt * ceil(K / 32) + kb; each block is
// [hi | lo], every half a 128 x 32 tile in the no-swizzle K-major layout the staged loop writes, zero outside N x K.  A stage of B
// is then one bulk copy, and A goes to wgmma from registers (see the image loop in gemm_wgmma_kernel).
constexpr int IMG_ROWS = 128, IMG_BK = 32, IMG_HALF = IMG_ROWS * IMG_BK, IMG_BLOCK = 2 * IMG_HALF;
constexpr int IMG_STAGES = 4;             // B ring of the image loop: 4 x 32 KB, inside the staged loop's 3 x 64 KB

struct Prob {
  const float* A; const float* B; const float* A_lo; const float* B_lo;      // A_lo / B_lo: pre-split operands (phc_gemm_tc5)
  const float* B_img;                                                          // weight image of B (128 x 128 tiles only), or NULL
  const float* A_img;                                                          // image of A (only with B_img), or NULL
  float* C; float* C_hi; float* C_lo;                                          // C_hi / C_lo: split copies of the result (phc_gemm_tc5)
  float* C_img;                                                                // image of the result (rows = M, K = N), or NULL
  const float* bias;
  float* aux;
  long long lda, ldb, ldc, ldaux;
  int M, N, K;
  float alpha;
  int act, accumulate, a_k, b_k, k_splits;
  int tiles_m, tiles_n, kb_total, kb_per, tile_begin, tile_count;
  unsigned int* turn;   // ordered accumulation: per output tile, the index of the slice whose turn it is to add into C (zero between launches)
  int turn_first, turn_total;   // this problem's first slice number and the slice count of all problems sharing the turnstile
};

struct Params {
  Prob p[MAX_PROBLEMS];
  int count, total_tiles;
  unsigned int* sched;  // dynamic tile scheduler: {next tile, CTAs done} in global memory (both zero between launches); NULL = static striding
};

__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_tf32_n256(float (&d)[128], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db));
}

// the same product with A from registers: a[0..3] is the warp's 16 x 8 tf32 fragment, (row lane / 4 + 8 (i & 1), col lane % 4 + 4 (i >> 1))
__device__ __forceinline__ void wgmma_tf32_n128_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

// mbarrier + bulk copy (the B stages of the image loop; the CTA is its own cluster of one)
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra WAIT;\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// pins register operands of the wgmma A fragment in place: computed before the wgmma.fence that precedes the batch, and kept
// live up to the wait_group that retires it (the compiler would otherwise move the splits past the fence or reuse the registers)
template <int N>
__device__ __forceinline__ void reg_fence(uint32_t (&r)[N][4]) {
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(r[i][j])::"memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory matrix descriptor (sm_90 GMMA): start address, LBO, SBO in 16-byte units, layout type 0 (no swizzle)
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}

template <int BN, typename Acc>
__device__ __forceinline__ void wgmma_tf32(Acc& d, uint64_t da, uint64_t db) {
  if constexpr (BN == 128) wgmma_tf32_n128(d, da, db); else wgmma_tf32_n256(d, da, db);
}

__device__ __forceinline__ float trunc_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
// lo = rna_tf32(x - trunc_tf32(x)): x - trunc is exact in fp32 (13 significant bits), round-to-nearest (ties away) to the 11
// bits a tf32 operand keeps, done with integer arithmetic on the bit pattern
__device__ __forceinline__ float split_lo(float x) {
  const float d = x - trunc_hi(x);
  return __uint_as_float((__float_as_uint(d) + 0x1000u) & 0xFFFFE000u);
}
__device__ __forceinline__ void sts128(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, float a) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(a) : "memory"); }

// Where the 16-byte chunks of an R x BK operand tile come from and go to.  Thread tid stages chunks c = tid + i * 256.
//   k-contiguous: chunk c holds (r, 4 kc .. 4 kc + 3) and lands at byte c * 16 of the tile (lanes of a warp write 512 contiguous
//                 bytes);
//   mn-contiguous: chunk c holds (r .. r + 3, k) with kl = c & 3, rl = (c >> 2) & 7, r = 4 (8 rh + rl), k = 4 kh + kl: a warp reads
//                 128 contiguous bytes of each of 4 k-rows.  Element e of the chunk goes to byte off + 16 e = off ^ (e << 4) of the
//                 tile, off = (r / 8) SBO + kh 128 + (rl & 1) 64 + kl 4 (bits 4-5 of off are zero), by a 4-byte store each.
//                 SBO and 128 are multiples of the 32 banks' 128 bytes, so the bank of element e is 16 (rl & 1) + 4 e + kl; the
//                 j-th store of a thread writes element e = j ^ (rl >> 1), so in each store the 32 lanes (kl, rl) write 32 distinct
//                 banks.
template <int R, int BK>
struct Map {
  static constexpr int KC = BK / 4;
  __device__ static void kmaj(int c, int& r, int& kc) { r = (c & 7) + 8 * (c / (8 * KC)); kc = (c >> 3) % KC; }
  __device__ static void mnmaj(int c, int& r, int& k, uint32_t& off) {
    const int kl = c & 3, rl = (c >> 2) & 7, c2 = c >> 5, rh = c2 % (R / 32), kh = c2 / (R / 32);
    r = 4 * (8 * rh + rl); k = 4 * kh + kl;
    off = (uint32_t)((4 * rh + (rl >> 1)) * BK * 32 + kh * 128 + (rl & 1) * 64 + kl * 4);
  }
};

// global -> registers: PER elements (PER / 4 chunks) of the R x BK tile at (r0, k0), zero outside [0, rows) x [0, K)
template <int R, int BK, int PER>
__device__ __forceinline__ void load_op(float (&v)[PER], const float* __restrict__ g, long long ld, bool kmaj, int r0, int rows, int k0,
                                        int K, int tid) {
  using Mp = Map<R, BK>;
#pragma unroll
  for (int i = 0; i < PER / 4; ++i) {
    int r, k;                                                // the chunk's first element; its 4 elements are contiguous in g
    const float* src;
    if (kmaj) {
      int kc;
      Mp::kmaj(tid + i * NUM_THREADS, r, kc);
      r += r0; k = k0 + 4 * kc;
      src = g + (long long)r * ld + k;
    } else {
      uint32_t off;
      Mp::mnmaj(tid + i * NUM_THREADS, r, k, off);
      r += r0; k += k0;
      src = g + (long long)k * ld + r;
    }
    if (kmaj ? (r < rows && k + 3 < K) : (r + 3 < rows && k < K)) {
      const float4 t = *reinterpret_cast<const float4*>(src);
      v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) v[4 * i + e] = (kmaj ? (r < rows && k + e < K) : (r + e < rows && k < K)) ? src[e] : 0.f;
    }
  }
}

// registers -> shared memory.  MODE 0: hi = trunc_tf32(v), lo = split_lo(v); 1: hi only (single pass); 2: v is hi, w is lo (pre-split)
template <int R, int BK, int PER, int MODE>
__device__ __forceinline__ void store_op(const float (&v)[PER], const float (&w)[PER], uint32_t s_hi, uint32_t s_lo, bool kmaj, int tid) {
  using Mp = Map<R, BK>;
  auto hi = [](float x) { return MODE == 2 ? x : trunc_hi(x); };
  if (kmaj) {
#pragma unroll
    for (int i = 0; i < PER / 4; ++i) {
      const uint32_t off = (uint32_t)(tid + i * NUM_THREADS) * 16u;
      sts128(s_hi + off, hi(v[4 * i]), hi(v[4 * i + 1]), hi(v[4 * i + 2]), hi(v[4 * i + 3]));
      if (MODE == 0) sts128(s_lo + off, split_lo(v[4 * i]), split_lo(v[4 * i + 1]), split_lo(v[4 * i + 2]), split_lo(v[4 * i + 3]));
      if (MODE == 2) sts128(s_lo + off, w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
    }
  } else {
    const int p = (tid >> 3) & 3;                            // rl >> 1 of every chunk of this thread
    // u[j] = x[j ^ p]: the element the j-th store writes
    auto perm = [p](const float* x, float (&u)[4]) {
      u[0] = x[0]; u[1] = x[1]; u[2] = x[2]; u[3] = x[3];
      if (p & 1) { const float t0 = u[0], t2 = u[2]; u[0] = u[1]; u[1] = t0; u[2] = u[3]; u[3] = t2; }
      if (p & 2) { const float t0 = u[0], t1 = u[1]; u[0] = u[2]; u[1] = u[3]; u[2] = t0; u[3] = t1; }
    };
#pragma unroll
    for (int i = 0; i < PER / 4; ++i) {
      int r, k;
      uint32_t off;
      Mp::mnmaj(tid + i * NUM_THREADS, r, k, off);
      off ^= (uint32_t)p << 4;
      float u[4], ul[4];
      perm(&v[4 * i], u);
      if (MODE == 2) perm(&w[4 * i], ul);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t o = off ^ ((uint32_t)j << 4);
        sts32(s_hi + o, hi(u[j]));
        if (MODE == 0) sts32(s_lo + o, split_lo(u[j]));
        if (MODE == 2) sts32(s_lo + o, ul[j]);
      }
    }
  }
}

__device__ __forceinline__ void split_rna(float x, float& h, float& l) {
  uint32_t a, b;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(a) : "f"(x));
  const float res = x - __uint_as_float(a);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(b) : "f"(res));
  h = __uint_as_float(a); l = __uint_as_float(b);
}

// SINGLE: one tensor-core product per fp32 product (plain TF32, ~1e-3 relative): no lo terms.  OUT_IMG: the epilogue writes
// PhcGemmDesc.C_img where a problem has one.  It is a separate instantiation because the extra epilogue code changes how ptxas
// schedules the whole kernel: in the one instantiation, the launches without output images ran 3-11 % slower on the bench
// minibatch (H100 SXM, 700 W).
template <int BN, bool PRESPLIT, bool SINGLE, bool OUT_IMG = false>
__global__ void __launch_bounds__(NUM_THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ Params P) {
  static_assert(!(PRESPLIT && SINGLE), "the pre-split operands are for the 3xTF32 products");
  using C = Cfg<BN>;
  constexpr int BK = C::BK;
  constexpr int MODE = SINGLE ? 1 : PRESPLIT ? 2 : 0;
  // single pass stays on the staged loop: ptxas serialises the wgmmas of its image loop (C7513)
  constexpr bool HAS_IMG = BN == IMG_ROWS && BK == IMG_BK && !PRESPLIT && !SINGLE;
  static_assert(!HAS_IMG || (C::A_TILE == IMG_HALF * 4 && C::B_TILE == IMG_HALF * 4), "an image block pair is one stage");
  static_assert(!OUT_IMG || HAS_IMG, "output images are written by the 3xTF32 kernel with 128 x 128 tiles");
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ int s_tile;
  __shared__ __align__(8) uint64_t s_bar[IMG_STAGES];      // one mbarrier per B stage of the image loop
  __shared__ __align__(8) uint64_t s_pbar[C::STAGES];      // one mbarrier per stage of the pair loop
  const int tid = threadIdx.x, lane = tid & 31, wgi = tid >> 7, wq = (tid >> 5) & 3;
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
  const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(s_bar);
  const uint32_t pbar0 = (uint32_t)__cvta_generic_to_shared(s_pbar);
  const bool dyn = P.sched != nullptr;
  int ring = 0;                                             // k-blocks the image loop has taken through its B ring so far
  uint32_t pphase = 0;                                      // bit s: the parity the pair loop waits for next on stage s
  if constexpr (HAS_IMG) {
    if (tid == 0) {
#pragma unroll
      for (int s = 0; s < IMG_STAGES; ++s) mbar_init(bar0 + 8 * s, 1);
#pragma unroll
      for (int s = 0; s < C::STAGES; ++s) mbar_init(pbar0 + 8 * s, 1);
      mbar_init_fence();
    }
    __syncthreads();
  }

  for (int it = 0;; ++it) {
    int t;
    if (dyn) {
      if (tid == 0) s_tile = (int)atomicAdd(P.sched, 1u);
      __syncthreads();
      t = s_tile;
      __syncthreads();
    } else {
      t = blockIdx.x + it * gridDim.x;
    }
    if (t >= P.total_tiles) break;
    int gi = 0;
#pragma unroll 1
    while (gi + 1 < P.count && t >= P.p[gi].tile_begin + P.p[gi].tile_count) ++gi;
    const Prob& q = P.p[gi];
    const int tl = t - q.tile_begin;
    const int ni = tl % q.tiles_n, rr = tl / q.tiles_n, mi = rr % q.tiles_m, z = rr / q.tiles_m;
    const int m0 = mi * BM, n0 = ni * BN;
    const int kb_begin = z * q.kb_per;
    const int nkb = max(0, min(q.kb_total, kb_begin + q.kb_per) - kb_begin);
    if (nkb == 0) continue;                                 // (uniform) an empty split-K slice adds nothing
    const bool ak = q.a_k != 0, bk = q.b_k != 0;

    float acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    // k-block j of the staged and the pair loop sits in shared-memory stage j % 3 as [A hi | A lo | B hi | B lo]
    auto stage = [&](int j) { return sbase + (uint32_t)((j % C::STAGES) * C::STAGE); };
    auto mma = [&](int j) {                                  // one wgmma batch: every product of k-block j
      const uint32_t s = stage(j);
      const uint32_t a_hi = s + (uint32_t)(wgi * 8 * C::SBO), a_lo = a_hi + C::A_TILE;
      const uint32_t b_hi = s + 2 * C::A_TILE, b_lo = b_hi + C::B_TILE;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 8; ++kk) {
        const uint32_t o = (uint32_t)kk * 256u;
        const uint64_t dAh = smem_desc(a_hi + o, 128, C::SBO), dBh = smem_desc(b_hi + o, 128, C::SBO);
        if constexpr (!SINGLE) {
          wgmma_tf32<BN>(acc, smem_desc(a_lo + o, 128, C::SBO), dBh);
          wgmma_tf32<BN>(acc, dAh, smem_desc(b_lo + o, 128, C::SBO));
        }
        wgmma_tf32<BN>(acc, dAh, dBh);
      }
      wgmma_commit();
    };
    bool staged = true;
    if constexpr (HAS_IMG) {
      if (q.A_img != nullptr) {                              // (uniform) A and B both from their images: the pair loop
        staged = false;
        // The A block and the B block of a k-block are [hi | lo] 32 KB each, in the layout the staged loop writes, so together
        // they fill one stage exactly and the staged loop's mma(j) consumes it: the products, their order and the k order are
        // the staged loop's, and the results are the same bit for bit.  Thread 0 fills stage j % 3 with two bulk copies under
        // that stage's mbarrier, 3 k-blocks ahead; the barrier after wait_group 1 of step j frees the stage of j - 1.  No
        // generic-proxy write touches the stages, so there is no proxy fence.  The stages' mbarriers are not the image loop's:
        // their phases are counted per stage in pphase, whatever ring position the image loop is at.
        const float* aimg = q.A_img + (long long)mi * q.kb_total * IMG_BLOCK;
        const float* bimg = q.B_img + (long long)ni * q.kb_total * IMG_BLOCK;
        auto issue = [&](int j) {
          const uint32_t s = stage(j), bar = pbar0 + 8 * (j % C::STAGES);
          mbar_expect_tx(bar, C::STAGE);
          bulk_g2s(s, aimg + (long long)(kb_begin + j) * IMG_BLOCK, IMG_BLOCK * 4, bar);
          bulk_g2s(s + 2 * C::A_TILE, bimg + (long long)(kb_begin + j) * IMG_BLOCK, IMG_BLOCK * 4, bar);
        };
        if (tid == 0)
          for (int j = 0; j < min(nkb, C::STAGES); ++j) issue(j);
#pragma unroll 1
        for (int j = 0; j < nkb; ++j) {
          const int s = j % C::STAGES;
          mbar_wait(pbar0 + 8 * s, (pphase >> s) & 1u);
          pphase ^= 1u << s;
          mma(j);
          wgmma_wait<1>();
          __syncthreads();
          if (tid == 0 && j >= 1 && j + 2 < nkb) issue(j + 2);
        }
        wgmma_wait<0>();
      } else if (q.B_img != nullptr) {                       // (uniform) B from its weight image, A from registers
        staged = false;
        // B: k-block j arrives in ring slot (ring + j) % IMG_STAGES by one bulk copy that thread 0 issues, IMG_STAGES k-blocks
        // ahead; the barrier after wait_group 1 of step j says that the slot of j - 1 is free again.  No generic-proxy write
        // touches B, so there is no proxy fence.
        // A: every thread loads its own part of the wgmma A fragment straight from global memory and splits it in registers:
        // ar[4 kk + i] = A(r + 8 (i & 1), k0 + 8 kk + c + 4 (i >> 1)), r = the warp's row lane / 4, c = lane % 4.  The loads
        // of k-block j + 1 are in flight during the wgmmas of j.  A batch behind wait_group 1 still reads its A registers,
        // so there are two split sets, used alternately, and the loop is unrolled by two to keep their indices static.
        // The products, their order per k8 and the k order are those of the staged loop: the results are the same bit for bit.
        const int r = m0 + wgi * 64 + wq * 16 + (lane >> 2), c = lane & 3;
        const bool ok0 = r < q.M, ok1 = r + 8 < q.M;
        const float* arow0 = q.A + (long long)(ok0 ? r : 0) * q.lda + c;
        const float* arow1 = q.A + (long long)(ok1 ? r + 8 : 0) * q.lda + c;
        float ar[16];
        auto load_a = [&](int j) {
          const int k0 = (kb_begin + j) * BK;
          const bool full = k0 + BK <= q.K;
#pragma unroll
          for (int e = 0; e < 16; ++e) {
            const int k = k0 + 8 * (e >> 2) + 4 * ((e >> 1) & 1);
            const bool ok = ((e & 1) ? ok1 : ok0) && (full || k + c < q.K);
            ar[e] = ok ? ((e & 1) ? arow1 : arow0)[k] : 0.f;
          }
        };
        uint32_t ah[2][BK / 8][4], al[2][SINGLE ? 1 : BK / 8][4];
        constexpr uint32_t B_BYTES = (SINGLE ? 1 : 2) * IMG_HALF * 4, SLOT = 2 * IMG_HALF * 4;
        const float* img = q.B_img + (long long)ni * q.kb_total * IMG_BLOCK;
        auto issue = [&](int j) {
          const int s = (ring + j) % IMG_STAGES;
          mbar_expect_tx(bar0 + 8 * s, B_BYTES);
          bulk_g2s(sbase + s * SLOT, img + (long long)(kb_begin + j) * IMG_BLOCK, B_BYTES, bar0 + 8 * s);
        };
        if (tid == 0)
          for (int j = 0; j < min(nkb, IMG_STAGES); ++j) issue(j);
        load_a(0);
        auto step = [&](int j, auto set) {
          constexpr int S = decltype(set)::value;
#pragma unroll
          for (int e = 0; e < 16; ++e) {
            ah[S][e >> 2][e & 3] = __float_as_uint(trunc_hi(ar[e]));
            if constexpr (!SINGLE) al[S][e >> 2][e & 3] = __float_as_uint(split_lo(ar[e]));
          }
          if (j + 1 < nkb) load_a(j + 1);
          const int s = (ring + j) % IMG_STAGES;
          mbar_wait(bar0 + 8 * s, (uint32_t)((ring + j) / IMG_STAGES) & 1u);
          uint64_t dB[BK / 8][2];                            // B descriptors (hi, lo) per k8, also made before the fence
#pragma unroll
          for (int kk = 0; kk < BK / 8; ++kk)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              dB[kk][h] = smem_desc(sbase + s * SLOT + h * IMG_HALF * 4 + kk * 256, 128, C::SBO);
              asm volatile("" : "+l"(dB[kk][h])::"memory");
            }
          reg_fence(ah[S]);
          if constexpr (!SINGLE) reg_fence(al[S]);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < BK / 8; ++kk) {
            if constexpr (!SINGLE) {
              wgmma_tf32_n128_rs(acc, al[S][kk], dB[kk][0]);
              wgmma_tf32_n128_rs(acc, ah[S][kk], dB[kk][1]);
            }
            wgmma_tf32_n128_rs(acc, ah[S][kk], dB[kk][0]);
          }
          wgmma_commit();
          wgmma_wait<1>();
          reg_fence(ah[S ^ 1]);                                // the batch of j - 1 is done with its set
          if constexpr (!SINGLE) reg_fence(al[S ^ 1]);
          __syncthreads();
          if (tid == 0 && j >= 1 && j - 1 + IMG_STAGES < nkb) issue(j - 1 + IMG_STAGES);
        };
#pragma unroll 1
        for (int j = 0; j < nkb; j += 2) {
          step(j, std::integral_constant<int, 0>());
          if (j + 1 < nkb) step(j + 1, std::integral_constant<int, 1>());
        }
        wgmma_wait<0>();
        ring += nkb;
      }
    }
    if (staged) {
      // k-block j is staged through the registers v and shared-memory stage j % 3
      struct Regs { float a[C::A_PER], b[C::B_PER], a_lo[PRESPLIT ? C::A_PER : 1], b_lo[PRESPLIT ? C::B_PER : 1]; };
      Regs v;
      auto load = [&](int j) {
        const int k0 = (kb_begin + j) * BK;
        load_op<BM, BK>(v.a, q.A, q.lda, ak, m0, q.M, k0, q.K, tid);
        load_op<BN, BK>(v.b, q.B, q.ldb, bk, n0, q.N, k0, q.K, tid);
        if constexpr (PRESPLIT) {
          load_op<BM, BK>(v.a_lo, q.A_lo, q.lda, ak, m0, q.M, k0, q.K, tid);
          load_op<BN, BK>(v.b_lo, q.B_lo, q.ldb, bk, n0, q.N, k0, q.K, tid);
        }
      };
      auto store = [&](int j) {
        const uint32_t s = stage(j);
        if constexpr (PRESPLIT) {
          store_op<BM, BK, C::A_PER, MODE>(v.a, v.a_lo, s, s + C::A_TILE, ak, tid);
          store_op<BN, BK, C::B_PER, MODE>(v.b, v.b_lo, s + 2 * C::A_TILE, s + 2 * C::A_TILE + C::B_TILE, bk, tid);
        } else {
          store_op<BM, BK, C::A_PER, MODE>(v.a, v.a, s, s + C::A_TILE, ak, tid);
          store_op<BN, BK, C::B_PER, MODE>(v.b, v.b, s + 2 * C::A_TILE, s + 2 * C::A_TILE + C::B_TILE, bk, tid);
        }
        fence_async_smem();                                   // generic-proxy writes -> visible to the tensor core's reads
      };
      // Step j: k-block j's wgmmas go out; k-block j + 1, loaded during step j - 1, is split and stored into the stage of
      // j - 2, whose wgmmas the barrier of step j - 1 saw finish; then the loads of j + 2 are issued.  They come after the store
      // on purpose: fence.proxy.async is a MEMBAR.CTA that waits for every memory access the thread has in flight, global loads
      // included, so loads issued before it would be waited for right there -- which is also why a second register set would
      // not let them start earlier.  Issued after it, they stay in flight through wait_group 1 (which leaves j's batch running
      // behind j - 1's) and the barrier, up to the store of step j + 1.  The barrier makes j + 1's stage visible to both
      // warpgroups and tells them j - 1's stage is free.
      load(0);
      store(0);
      if (nkb > 1) load(1);
      __syncthreads();
  #pragma unroll 1
      for (int j = 0; j < nkb; ++j) {
        mma(j);
        if (j + 1 < nkb) store(j + 1);
        if (j + 2 < nkb) load(j + 2);
        wgmma_wait<1>();
        __syncthreads();
      }
      wgmma_wait<0>();
    }
    __syncthreads();                                         // both warpgroups' last batch is done before its stage is refilled

    const bool ordered = q.turn != nullptr;                 // split-K slice: wait until the slices before it have added into C
    volatile unsigned int* turn = ordered ? q.turn + mi * q.tiles_n + ni : nullptr;
    if (ordered) {
      if (tid == 0) {
        while (*turn != (unsigned)(q.turn_first + z)) __nanosleep(64);
        __threadfence();
      }
      __syncthreads();
    }
    // ---- epilogue straight from the accumulator fragment: acc[4 j + 2 h + c] is (row w*16 + lane/4 + 8 h, col 8 j + 2 (lane%4) + c)
    const int act = q.act;
    const float* bias = (q.bias && z == 0) ? q.bias : nullptr;
    // C_img: the stored value, split like phc_gemm_make_images, at the image position of (row m - m0 of m-tile mi, k = n); the
    // tile's 128 rows and every 32-column k-block it starts below N are written, zeros outside M x N, so the image is the
    // one phc_gemm_make_images would make from C.  A quad's float2 pairs of one k-block half fill 128 contiguous bytes.
    float* cimg = nullptr;
    if constexpr (OUT_IMG) cimg = q.C_img ? q.C_img + (long long)mi * ((q.N + IMG_BK - 1) / IMG_BK) * IMG_BLOCK : nullptr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int rt = wgi * 64 + wq * 16 + (lane >> 2) + 8 * h;   // row within the tile
      const int m = m0 + rt;
      const bool row_ok = m < q.M;
      float* crow = q.C + (long long)m * q.ldc;
      float* arow = (q.aux && act < PHC_ACT_RELU_BITS && row_ok) ? q.aux + (long long)m * q.ldaux : nullptr;
      uint32_t* brow = (q.aux && act >= PHC_ACT_RELU_BITS && row_ok) ? reinterpret_cast<uint32_t*>(q.aux) + (long long)m * q.ldaux : nullptr;
#pragma unroll
      for (int qc = 0; qc < BN / 32; ++qc) {
        const int nb = n0 + 32 * qc;
        if (nb >= q.N) break;                                // warp-uniform
        const uint32_t mbits = (act == PHC_ACT_MASK_BITS && brow) ? brow[nb >> 5] : 0u;
        uint32_t bits = 0;
        // ordered: this tile is C's only writer right now.  The chunk's old C values are read past L1 all at once, before any
        // store, so that their L2 round trips overlap: the turnstile chains the epilogues of an output tile's slices one after
        // the other, so the latency of each epilogue adds up over the slices.
        float old[8];
        if (ordered && row_ok) {
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int n = nb + 8 * (e >> 1) + 2 * (lane & 3) + (e & 1);
            old[e] = n < q.N ? __ldcg(crow + n) : 0.f;
          }
        }
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = 4 * qc + jj;
          const int nl = 8 * jj + 2 * (lane & 3);            // column within the 32-column chunk
          float v[2];
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int n = nb + nl + c;
            float x = q.alpha * acc[4 * j + 2 * h + c];
            if (bias && n < q.N) x += bias[n];
            if (act == PHC_ACT_RELU || act == PHC_ACT_RELU_BITS) x = fmaxf(x, 0.f);
            if (act == PHC_ACT_RELU_BITS) bits |= (x > 0.f ? 1u : 0u) << (nl + c);
            else if (act == PHC_ACT_MASK_BITS) x = ((mbits >> (nl + c)) & 1u) ? x : 0.f;
            else if (arow && n < q.N) {
              if (act == PHC_ACT_SILU) { arow[n] = x; x = silu_f(x); }
              else if (act == PHC_ACT_SILU_BWD) x *= silu_grad_f(arow[n]);
              else x = arow[n] > 0.f ? x : 0.f;              // ReLU backward from the saved activation
            } else if (act == PHC_ACT_SILU) {
              x = silu_f(x);
            }
            v[c] = x;
          }
          if (OUT_IMG && cimg) {
            const float w0 = row_ok && nb + nl < q.N ? v[0] : 0.f, w1 = row_ok && nb + nl + 1 < q.N ? v[1] : 0.f;
            float* o = cimg + (long long)(nb >> 5) * IMG_BLOCK + 256 * (rt >> 3) + 32 * (nl >> 2) + 4 * (rt & 7) + (nl & 3);
            *reinterpret_cast<float2*>(o) = make_float2(trunc_hi(w0), trunc_hi(w1));
            *reinterpret_cast<float2*>(o + IMG_HALF) = make_float2(split_lo(w0), split_lo(w1));
          }
          if (!row_ok) continue;
          const int n = nb + nl;
          if (ordered) {
            if (n < q.N) crow[n] = old[2 * jj] + v[0];
            if (n + 1 < q.N) crow[n + 1] = old[2 * jj + 1] + v[1];
          } else if (q.accumulate) {                         // one writer per element: same result whatever the order
            if (n < q.N) atomicAdd(crow + n, v[0]);
            if (n + 1 < q.N) atomicAdd(crow + n + 1, v[1]);
          } else if (n + 1 < q.N) {
            *reinterpret_cast<float2*>(crow + n) = make_float2(v[0], v[1]);
          } else if (n < q.N) {
            crow[n] = v[0];
          }
          if (PRESPLIT && q.C_hi) {
            float h0, l0, h1, l1;
            split_rna(v[0], h0, l0); split_rna(v[1], h1, l1);
            if (n < q.N) { q.C_hi[(long long)m * q.ldc + n] = h0; q.C_lo[(long long)m * q.ldc + n] = l0; }
            if (n + 1 < q.N) { q.C_hi[(long long)m * q.ldc + n + 1] = h1; q.C_lo[(long long)m * q.ldc + n + 1] = l1; }
          }
        }
        if (act == PHC_ACT_RELU_BITS) {                      // the row's 32 bits are spread over the 4 lanes of a quad
          bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
          bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
          if (brow && (lane & 3) == 0) brow[nb >> 5] = bits;
        }
      }
    }
    if (ordered) {                                          // hand the tile to the next slice (the last one resets the turnstile)
      __threadfence();
      __syncthreads();
      if (tid == 0) *turn = (q.turn_first + z + 1 == q.turn_total) ? 0u : (unsigned)(q.turn_first + z + 1);
    }
  }
  // the last CTA to get here puts both counters back to zero for the next launch (every CTA has drawn its terminating tile by now)
  if (dyn && tid == 0 && atomicInc(P.sched + 1, gridDim.x - 1) == gridDim.x - 1) { __threadfence(); P.sched[0] = 0u; }
}

__global__ void split_lo_kernel(const float* __restrict__ x, float* __restrict__ lo, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) lo[i] = split_lo(x[i]);
}

// x -> hi = rna_tf32(x), lo = rna_tf32(x - hi) over a strided [rows, cols] block
__global__ void split_tf32_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int cols, float* __restrict__ hi,
                                  float* __restrict__ lo, int64_t ldo) {
  const int64_t total = rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols;
    const int c = (int)(i - r * cols);
    split_rna(x[r * ldx + c], hi[r * ldo + c], lo[r * ldo + c]);
  }
}

// Weight images: CTA b writes image block b of the launch, [hi | lo] of one 128 x 32 tile of B in the K-major layout of the
// staged loop (16-byte chunk c = tid + 256 i holds (r, 4 kc .. 4 kc + 3), Map::kmaj), split by the kernel's own trunc_hi / split_lo
constexpr int IMG_JOBS = 64;
struct ImgJob { const float* B; long long ldb; float* img; long long block_begin; int b_k, N, K, kbs; };
struct ImgParams { ImgJob j[IMG_JOBS]; int count; long long total_blocks; };

__global__ void __launch_bounds__(NUM_THREADS) weight_image_kernel(const __grid_constant__ ImgParams P) {
  using Mp = Map<IMG_ROWS, IMG_BK>;
  for (long long b = blockIdx.x; b < P.total_blocks; b += gridDim.x) {
    int i = 0;
    while (i + 1 < P.count && b >= P.j[i + 1].block_begin) ++i;
    const ImgJob& J = P.j[i];
    const long long lb = b - J.block_begin;
    const int n0 = (int)(lb / J.kbs) * IMG_ROWS, k0 = (int)(lb % J.kbs) * IMG_BK;
    float4* hi = reinterpret_cast<float4*>(J.img + lb * IMG_BLOCK);
    float4* lo = hi + IMG_HALF / 4;
#pragma unroll
    for (int it = 0; it < IMG_HALF / 4 / NUM_THREADS; ++it) {
      const int c = threadIdx.x + it * NUM_THREADS;
      int r, kc;
      Mp::kmaj(c, r, kc);
      const int n = n0 + r, k = k0 + 4 * kc;
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e)
        v[e] = (n < J.N && k + e < J.K) ? (J.b_k ? J.B[(long long)n * J.ldb + k + e] : J.B[(long long)(k + e) * J.ldb + n]) : 0.f;
      hi[c] = make_float4(trunc_hi(v[0]), trunc_hi(v[1]), trunc_hi(v[2]), trunc_hi(v[3]));
      lo[c] = make_float4(split_lo(v[0]), split_lo(v[1]), split_lo(v[2]), split_lo(v[3]));
    }
  }
}

static long long image_blocks(int N, int K) { return (long long)((N + IMG_ROWS - 1) / IMG_ROWS) * ((K + IMG_BK - 1) / IMG_BK); }

static int g_single_pass = 0;
static int g_tile = 0;        // 0: default (128), else the tile width 128 | 256
static int g_sched = -1;      // -1: not decided yet (env PHC_TC5S_SCHED = static | dynamic; default dynamic), 0 static, 1 dynamic
// {next tile, CTAs done} pairs of the dynamic scheduler, zero at load time and put back to zero by every launch's last CTA; launches
// rotate through them so that two launches in flight on different streams do not share a pair
constexpr int SCHED_SLOTS = 64;
__device__ unsigned int g_sched_counters[SCHED_SLOTS][2];
// split-K turnstiles, one per output tile of the split-K problems of a launch; launches rotate through the slots like the scheduler pairs
constexpr int TURN_SLOTS = 16, TURN_TILES = 8192;
__device__ unsigned int g_turns[TURN_SLOTS][TURN_TILES];

static int num_sms() {
  static int n = 0;
  if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); if (n <= 0) n = 132; }
  return n;
}

// fills P.p[n] for one problem; returns the number of tiles it adds
static int add_problem(Params& P, int n, int tiles, int bn, const float* A, const float* A_lo, const float* A_img, long long lda, int a_k,
                       const float* B, const float* B_lo, const float* B_img, long long ldb, int b_k, float* Cm, float* C_hi, float* C_lo, float* C_img,
                       long long ldc, int M, int N, int K, float alpha, const float* bias, int act, float* aux, long long ldaux, int accumulate,
                       int k_splits) {
  const int bk = bn == 128 ? Cfg<128>::BK : Cfg<256>::BK;
  Prob& q = P.p[n];
  q.A = A; q.A_lo = A_lo; q.B = B; q.B_lo = B_lo; q.B_img = bn == IMG_ROWS ? B_img : nullptr;
  q.A_img = q.B_img ? A_img : nullptr; q.C = Cm; q.C_hi = C_hi; q.C_lo = C_lo; q.C_img = C_img; q.bias = bias; q.aux = aux;
  q.lda = lda; q.ldb = ldb; q.ldc = ldc; q.ldaux = ldaux; q.M = M; q.N = N; q.K = K; q.alpha = alpha; q.act = act;
  q.accumulate = accumulate ? 1 : 0; q.a_k = a_k ? 1 : 0; q.b_k = b_k ? 1 : 0;
  int ks = k_splits < 1 ? 1 : k_splits;
  q.tiles_m = (M + BM - 1) / BM;
  q.tiles_n = (N + bn - 1) / bn;
  q.kb_total = (K + bk - 1) / bk;
  if (ks > q.kb_total) ks = q.kb_total;
  q.kb_per = (q.kb_total + ks - 1) / ks;
  ks = (q.kb_total + q.kb_per - 1) / q.kb_per;            // no empty slice: every slice takes its turn
  q.k_splits = ks;
  q.turn = nullptr;
  q.tile_begin = tiles;
  q.tile_count = q.tiles_m * q.tiles_n * ks;
  return q.tile_count;
}

template <int BN, bool PRESPLIT, bool SINGLE, bool OUT_IMG = false>
static int launch_kernel(const Params& P, cudaStream_t stream) {
  static bool smem_set = false;
  if (!smem_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<BN, PRESPLIT, SINGLE, OUT_IMG>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM);
    if (e != cudaSuccess) return phc_check_cuda(e, "cudaFuncSetAttribute(gemm_wgmma)");
    smem_set = true;
  }
  const int sms = num_sms();
  const unsigned grid = (unsigned)(P.total_tiles < sms ? P.total_tiles : sms);
  gemm_wgmma_kernel<BN, PRESPLIT, SINGLE, OUT_IMG><<<grid, NUM_THREADS, Cfg<BN>::SMEM, stream>>>(P);
  phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "gemm_wgmma_kernel launch");
}

template <int BN, bool PRESPLIT>
static int launch(Params& P, bool dynamic_sched, bool single, cudaStream_t stream, bool out_img = false) {
  // ordered problems: split-K, or accumulating into the same C as another problem of the launch (which then shares its turnstile)
  int owner[MAX_PROBLEMS];
  bool ordered = false;
  int turn_tiles = 0;
  for (int i = 0; i < P.count; ++i) {
    Prob& q = P.p[i];
    owner[i] = -1;
    for (int j = 0; j < i && q.accumulate; ++j) {
      const Prob& o = P.p[j];
      if (!o.accumulate || o.C != q.C) continue;
      if (o.M != q.M || o.N != q.N || o.ldc != q.ldc) { phc_set_error("phc_gemm_group: problems accumulating into the same C must have the same shape"); return PHC_ERR_INVALID_ARG; }
      owner[i] = owner[j] >= 0 ? owner[j] : j;
      break;
    }
  }
  bool has_members[MAX_PROBLEMS] = {};
  for (int i = 0; i < P.count; ++i)
    if (owner[i] >= 0) has_members[owner[i]] = true;
  for (int i = 0; i < P.count; ++i) {
    Prob& q = P.p[i];
    q.turn_first = 0; q.turn_total = q.k_splits;
    if (q.k_splits > 1 || owner[i] >= 0 || has_members[i]) { ordered = true; if (owner[i] < 0) turn_tiles += q.tiles_m * q.tiles_n; }
  }
  if (turn_tiles > TURN_TILES) { phc_set_error("gemm: more than 8192 ordered output tiles in one launch"); return PHC_ERR_UNSUPPORTED; }
  if (ordered) {
    static unsigned int* tbase = nullptr;
    static unsigned int turn_no = 0;
    if (!tbase) {
      void* p = nullptr;
      cudaError_t es = cudaGetSymbolAddress(&p, g_turns);
      if (es != cudaSuccess) return phc_check_cuda(es, "cudaGetSymbolAddress(g_turns)");
      tbase = static_cast<unsigned int*>(p);
    }
    unsigned int* t = tbase + (size_t)(turn_no++ % TURN_SLOTS) * TURN_TILES;
    for (int i = 0; i < P.count; ++i) {
      Prob& q = P.p[i];
      if (owner[i] >= 0) {                                   // continue the owner's slice numbering on the owner's turnstile
        Prob& o = P.p[owner[i]];
        q.turn = o.turn;
        q.turn_first = o.turn_total;
        o.turn_total += q.k_splits;
      } else if (q.k_splits > 1 || has_members[i]) {
        q.turn = t; t += q.tiles_m * q.tiles_n;
      }
    }
    for (int i = 0; i < P.count; ++i)                        // every member of a turnstile group learns the group's slice count
      if (owner[i] >= 0) P.p[i].turn_total = P.p[owner[i]].turn_total;
    dynamic_sched = true;
  }
  P.sched = nullptr;
  if (dynamic_sched) {
    static unsigned int* base = nullptr;
    static unsigned int launch_no = 0;
    if (!base) {
      void* p = nullptr;
      cudaError_t es = cudaGetSymbolAddress(&p, g_sched_counters);
      if (es != cudaSuccess) return phc_check_cuda(es, "cudaGetSymbolAddress(g_sched_counters)");
      base = static_cast<unsigned int*>(p);
    }
    P.sched = base + 2 * (launch_no++ % SCHED_SLOTS);
  }
  if constexpr (PRESPLIT) return launch_kernel<BN, true, false>(P, stream);
  if constexpr (BN == 128)
    if (out_img) return launch_kernel<BN, false, false, true>(P, stream);   // (validate_group: not with single pass)
  return single ? launch_kernel<BN, false, true>(P, stream) : launch_kernel<BN, false, false>(P, stream);
}

}  // namespace wg
}  // namespace phc

static int validate_group(const PhcGemmDesc* d, int32_t count) {
  using namespace phc::wg;
  if (!d || count < 1 || count > MAX_PROBLEMS) { phc_set_error("phc_gemm_group: 1 <= count <= PHC_GEMM_GROUP_MAX problems"); return PHC_ERR_INVALID_ARG; }
  for (int i = 0; i < count; ++i) {
    const PhcGemmDesc& g = d[i];
    if (!g.A || !g.B || !g.C || g.M < 0 || g.N < 0 || g.K < 1) { phc_set_error("phc_gemm_group: bad problem (NULL operand or negative size)"); return PHC_ERR_INVALID_ARG; }
    if (g.M == 0 || g.N == 0) continue;
    if ((g.lda & 3) || (g.ldb & 3) || (g.ldc & 3)) { phc_set_error("phc_gemm_group: leading dimensions must be multiples of 4 floats (16-byte operand loads)"); return PHC_ERR_INVALID_ARG; }
    for (const void* p : {(const void*)g.A, (const void*)g.B, (const void*)g.C})
      if (reinterpret_cast<uintptr_t>(p) & 15) { phc_set_error("phc_gemm_group: A, B, C must be 16-byte aligned"); return PHC_ERR_INVALID_ARG; }
    const int ks = g.k_splits < 1 ? 1 : g.k_splits;
    if (g.act < 0 || g.act > PHC_ACT_MASK_BITS || ((g.act == PHC_ACT_SILU_BWD || g.act == PHC_ACT_MASK_BITS) && !g.aux)) { phc_set_error("phc_gemm_group: bad activation code"); return PHC_ERR_INVALID_ARG; }
    if (g.act >= PHC_ACT_RELU_BITS && g.aux && ((reinterpret_cast<uintptr_t>(g.aux) & 3) || g.ldaux < (g.N + 31) / 32)) { phc_set_error("phc_gemm_group: bit-mask aux needs ldaux >= ceil(N / 32) words"); return PHC_ERR_INVALID_ARG; }
    if (ks > 1 && (!g.accumulate || g.act || g.aux)) { phc_set_error("phc_gemm_group: split-K needs accumulate=1 and a linear epilogue"); return PHC_ERR_INVALID_ARG; }
    if (g.B_lo && (reinterpret_cast<uintptr_t>(g.B_lo) & 15)) { phc_set_error("phc_gemm_group: B_lo must be 16-byte aligned"); return PHC_ERR_INVALID_ARG; }
    if (g.A_img && ((reinterpret_cast<uintptr_t>(g.A_img) & 15) || !g.B_img)) { phc_set_error("phc_gemm_group: A_img must be 16-byte aligned and comes with B_img only"); return PHC_ERR_INVALID_ARG; }
    if (g.B_img && ((reinterpret_cast<uintptr_t>(g.B_img) & 15) || (!g.a_kmajor && !g.A_img))) { phc_set_error("phc_gemm_group: B_img must be 16-byte aligned and comes with a_kmajor or A_img only"); return PHC_ERR_INVALID_ARG; }
    if (g.C_img && ((reinterpret_cast<uintptr_t>(g.C_img) & 15) || g.accumulate || ks > 1)) { phc_set_error("phc_gemm_group: C_img must be 16-byte aligned and comes without accumulate or split-K"); return PHC_ERR_INVALID_ARG; }
    if (g.C_img && (g_tile == 256 || g_single_pass)) { phc_set_error("phc_gemm_group: C_img is written by the 3xTF32 kernel with 128 x 128 tiles only"); return PHC_ERR_UNSUPPORTED; }
  }
  // write hazards: the C spans [C, C + (M - 1) ldc + N) of two problems may only overlap when both accumulate into the same C with
  // the same shape -- they then share a turnstile and add in problem order; any other overlap would race (plain stores, or
  // unordered atomics of accumulating problems with different C)
  auto span = [](const PhcGemmDesc& g, uintptr_t& lo, uintptr_t& hi) {
    lo = reinterpret_cast<uintptr_t>(g.C);
    hi = lo + (uintptr_t)(((int64_t)g.M - 1) * g.ldc + g.N) * sizeof(float);
  };
  for (int i = 0; i < count; ++i) {
    const PhcGemmDesc& a = d[i];
    if (a.M == 0 || a.N == 0) continue;
    uintptr_t a0, a1;
    span(a, a0, a1);
    for (int j = 0; j < i; ++j) {
      const PhcGemmDesc& b = d[j];
      if (b.M == 0 || b.N == 0) continue;
      uintptr_t b0, b1;
      span(b, b0, b1);
      if (a0 >= b1 || b0 >= a1) continue;
      if (a.accumulate && b.accumulate && a.C == b.C && a.M == b.M && a.N == b.N && a.ldc == b.ldc) continue;
      phc_set_error("phc_gemm_group: two problems write overlapping C ranges (only accumulating problems on the same C with the same M, N, ldc may)");
      return PHC_ERR_INVALID_ARG;
    }
  }
  return PHC_OK;
}

// PhcGemmDesc.B_lo (a pre-split low term of the weights) is validated and not read: the kernel makes the identical lo term itself
// from the fp32 operand it stages anyway.
extern "C" int phc_gemm_group(const PhcGemmDesc* d, int32_t count, void* stream) {
  using namespace phc::wg;
  const int vrc = validate_group(d, count);
  if (vrc != PHC_OK) return vrc;
  if (g_sched < 0) { const char* v = getenv("PHC_TC5S_SCHED"); g_sched = (v && v[0] == 's') ? 0 : 1; }
  const int bn = g_tile == 256 ? 256 : 128;
  static Params P;      // host staging (launches are serialised by the caller's stream order; the struct is copied at launch)
  memset(&P, 0, sizeof(P));
  int tiles = 0, n = 0;
  bool out_img = false;
  for (int i = 0; i < count; ++i) {
    const PhcGemmDesc& g = d[i];
    if (g.M == 0 || g.N == 0) continue;
    out_img |= g.C_img != nullptr;
    tiles += add_problem(P, n, tiles, bn, g.A, nullptr, g.A_img, g.lda, g.a_kmajor, g.B, nullptr, g.B_img, g.ldb, g.b_kmajor, g.C, nullptr, nullptr, g.C_img, g.ldc,
                         g.M, g.N, g.K, g.alpha, g.bias, g.act, g.aux, g.ldaux, g.accumulate, g.k_splits);
    ++n;
  }
  if (n == 0) return PHC_OK;
  P.count = n; P.total_tiles = tiles;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool single = g_single_pass != 0;
  return bn == 256 ? launch<256, false>(P, g_sched == 1, single, st) : launch<128, false>(P, g_sched == 1, single, st, out_img);
}

extern "C" int phc_gemm_tc5s(const float* A, int64_t lda, int32_t a_kmajor, const float* B, int64_t ldb, int32_t b_kmajor, float* C,
                             int64_t ldc, int32_t M, int32_t N, int32_t K, float alpha, const float* bias, int32_t act, float* aux,
                             int64_t ldaux, int32_t accumulate, int32_t k_splits, void* stream) {
  PhcGemmDesc d;
  d.A = A; d.lda = lda; d.a_kmajor = a_kmajor; d.B = B; d.ldb = ldb; d.b_kmajor = b_kmajor; d.C = C; d.ldc = ldc;
  d.M = M; d.N = N; d.K = K; d.alpha = alpha; d.bias = bias; d.act = act; d.aux = aux; d.ldaux = ldaux;
  d.accumulate = accumulate; d.k_splits = k_splits; d.B_lo = nullptr; d.B_img = nullptr; d.A_img = nullptr; d.C_img = nullptr;
  return phc_gemm_group(&d, 1, stream);
}

extern "C" int phc_gemm_tc5(const float* A_hi, const float* A_lo, int64_t lda, int32_t a_kmajor, const float* B_hi,
                            const float* B_lo, int64_t ldb, int32_t b_kmajor, float* C, float* C_hi, float* C_lo, int64_t ldc,
                            int32_t M, int32_t N, int32_t K, float alpha, const float* bias, int32_t relu, float* mask,
                            int64_t ldmask, int32_t accumulate, int32_t k_splits, void* stream) {
  using namespace phc::wg;
  if (!A_hi || !A_lo || !B_hi || !B_lo || !C || M < 0 || N < 0 || K < 1) { phc_set_error("phc_gemm_tc5: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (M == 0 || N == 0) return PHC_OK;
  if ((lda & 3) || (ldb & 3) || (ldc & 1)) { phc_set_error("phc_gemm_tc5: lda, ldb must be multiples of 4 floats, ldc of 2"); return PHC_ERR_INVALID_ARG; }
  for (const void* p : {(const void*)A_hi, (const void*)A_lo, (const void*)B_hi, (const void*)B_lo})
    if (reinterpret_cast<uintptr_t>(p) & 15) { phc_set_error("phc_gemm_tc5: operands must be 16-byte aligned"); return PHC_ERR_INVALID_ARG; }
  if (reinterpret_cast<uintptr_t>(C) & 7) { phc_set_error("phc_gemm_tc5: C must be 8-byte aligned"); return PHC_ERR_INVALID_ARG; }
  if (k_splits < 1) k_splits = 1;
  if (relu < 0 || relu > PHC_ACT_SILU_BWD || (relu == PHC_ACT_SILU_BWD && !mask)) { phc_set_error("phc_gemm_tc5: bad activation code"); return PHC_ERR_INVALID_ARG; }
  if (k_splits > 1 && (!accumulate || relu || mask)) { phc_set_error("phc_gemm_tc5: split-K needs accumulate=1 and a linear epilogue"); return PHC_ERR_INVALID_ARG; }
  if ((C_hi == nullptr) != (C_lo == nullptr) || (C_hi && accumulate)) { phc_set_error("phc_gemm_tc5: C_hi/C_lo come as a pair and not with accumulate"); return PHC_ERR_INVALID_ARG; }
  static Params P;
  memset(&P, 0, sizeof(P));
  P.total_tiles = add_problem(P, 0, 0, 128, A_hi, A_lo, nullptr, lda, a_kmajor, B_hi, B_lo, nullptr, ldb, b_kmajor, C, C_hi, C_lo, nullptr, ldc, M, N, K, alpha, bias,
                              relu, mask, ldmask, accumulate, k_splits);
  P.count = 1;
  return launch<128, true>(P, false, false, static_cast<cudaStream_t>(stream));
}

extern "C" int phc_split_tf32(const float* x, int64_t ldx, int64_t rows, int32_t cols, float* hi, float* lo, int64_t ldo,
                              void* stream) {
  if (!x || !hi || !lo || rows < 0 || cols < 1 || ldx < cols || ldo < cols) { phc_set_error("phc_split_tf32: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (rows == 0) return PHC_OK;
  int64_t g = (rows * cols + 255) / 256; if (g > 132 * 8) g = 132 * 8;
  phc::wg::split_tf32_kernel<<<(unsigned)g, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, ldx, rows, cols, hi, lo, ldo);
  phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "split_tf32_kernel");
}

extern "C" int64_t phc_gemm_image_floats(int32_t N, int32_t K) {
  return N < 1 || K < 1 ? 0 : phc::wg::image_blocks(N, K) * phc::wg::IMG_BLOCK;
}

extern "C" int phc_gemm_make_images(const PhcGemmImageDesc* d, int32_t count, void* stream) {
  using namespace phc::wg;
  if (count < 0 || (count > 0 && !d)) { phc_set_error("phc_gemm_make_images: bad arguments"); return PHC_ERR_INVALID_ARG; }
  for (int i = 0; i < count; ++i) {
    const PhcGemmImageDesc& g = d[i];
    if (!g.B || !g.img || g.N < 1 || g.K < 1 || g.ldb < (g.b_kmajor ? g.K : g.N)) { phc_set_error("phc_gemm_make_images: bad image (NULL pointer, empty or ldb too small)"); return PHC_ERR_INVALID_ARG; }
    if (reinterpret_cast<uintptr_t>(g.img) & 15) { phc_set_error("phc_gemm_make_images: img must be 16-byte aligned"); return PHC_ERR_INVALID_ARG; }
  }
  static ImgParams P;
  for (int i0 = 0; i0 < count; i0 += IMG_JOBS) {
    memset(&P, 0, sizeof(P));
    P.count = count - i0 < IMG_JOBS ? count - i0 : IMG_JOBS;
    long long blocks = 0;
    for (int i = 0; i < P.count; ++i) {
      const PhcGemmImageDesc& g = d[i0 + i];
      P.j[i] = ImgJob{g.B, (long long)g.ldb, g.img, blocks, g.b_kmajor ? 1 : 0, g.N, g.K, (g.K + IMG_BK - 1) / IMG_BK};
      blocks += image_blocks(g.N, g.K);
    }
    P.total_blocks = blocks;
    const long long grid = blocks < 132 * 8 ? blocks : 132 * 8;
    weight_image_kernel<<<(unsigned)grid, NUM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(P);
    phc_count_launches(1);
    const int rc = phc_check_cuda(cudaGetLastError(), "weight_image_kernel launch");
    if (rc != PHC_OK) return rc;
  }
  return PHC_OK;
}

extern "C" int phc_split_lo(const float* x, float* lo, int64_t n, void* stream) {
  if (n < 0 || (n > 0 && (!x || !lo))) { phc_set_error("phc_split_lo: NULL buffer"); return PHC_ERR_INVALID_ARG; }
  if (n == 0) return PHC_OK;
  const int threads = 256;
  int64_t blocks = (n + threads - 1) / threads;
  if (blocks > 132 * 8) blocks = 132 * 8;
  phc::wg::split_lo_kernel<<<(unsigned)blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(x, lo, n);
  phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "split_lo_kernel launch");
}

extern "C" int phc_gemm_set_precision(int32_t mode) {      // PHC_GEMM_FP32_3XTF32 (default) | PHC_GEMM_TF32_SINGLE_PASS
  if (mode != PHC_GEMM_FP32_3XTF32 && mode != PHC_GEMM_TF32_SINGLE_PASS) { phc_set_error("phc_gemm_set_precision: unknown mode"); return PHC_ERR_INVALID_ARG; }
  phc::wg::g_single_pass = mode == PHC_GEMM_TF32_SINGLE_PASS;
  return PHC_OK;
}

extern "C" int phc_gemm_tc5s_set_tile(int32_t width) {     // 128: 128 x 128 x 32 tiles (default); 256: 128 x 256 x 16; 0 = default
  if (width != 0 && width != 128 && width != 256) { phc_set_error("phc_gemm_tc5s_set_tile: 0, 128 or 256"); return PHC_ERR_INVALID_ARG; }
  phc::wg::g_tile = width;
  return PHC_OK;
}

extern "C" int phc_gemm_tc5s_set_sched(int32_t mode) {     // tile order: 0 static striding, 1 dynamic (global counter), -1 default
  if (mode < -1 || mode > 1) { phc_set_error("phc_gemm_tc5s_set_sched: -1, 0 or 1"); return PHC_ERR_INVALID_ARG; }
  phc::wg::g_sched = mode;
  return PHC_OK;
}

extern "C" int phc_gemm_tc5s_set_ctas(int32_t ctas) {      // CTAs per tile: 0 (default) or 1; 2 is accepted and runs the one-CTA tiles
  if (ctas < 0 || ctas > 2) { phc_set_error("phc_gemm_tc5s_set_ctas: 0, 1 or 2"); return PHC_ERR_INVALID_ARG; }
  return PHC_OK;
}
