// Tensor-core GEMM for the actor / critic / discriminator MLPs (forward, input-gradient and weight-gradient forms).
// Reference: the MLPs are plain nn.Linear stacks in fp32 (phc/learning/network_builder.py:105-124,
// amp_network_builder.py:58-249; mixed_precision: False in phc/data/cfg/learning/im.yaml:51) -> cuBLAS SGEMM.
//
//   C[M,N] (+)= epilogue( alpha * sum_k A(m,k) * B(n,k) )
//
// A(m,k) and B(n,k) are addressed through (row, col) strides so that the three layer forms need no transposes:
//   forward      Y = X W^T      : A = X  [M=batch, K=in]   k-contiguous ; B = W  [N=out, K=in]   k-contiguous
//   input grad   dX = dY W      : A = dY [M=batch, K=out]  k-contiguous ; B = W  [K=out, N=in]   n-contiguous
//   weight grad  dW = dY^T X    : A = dY [K=batch, M=out]  m-contiguous ; B = X  [K=batch, N=in] n-contiguous
//
// Precision: fp32-equivalent on the TF32 tensor cores by the 3xTF32 split (a = a_hi + a_lo in registers,
// acc += a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, fp32 accumulate), because the reference trains in fp32 and the parity
// bar is 1e-5; a single TF32/BF16 pass (1e-3) would not meet it.  v1 of this kernel issues warp-level mma.sync
// (m16n8k8) from a cp.async multi-stage pipeline; gemm_wgmma.cu is the wgmma version the learner uses by default.
//
// Epilogue (all optional, applied in this order): alpha scale, + bias[n], ReLU, * (mask[m,n] > 0) (ReLU backward),
// then either store or atomically accumulate into C (split-K weight gradients accumulate into a zeroed bucket).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/phc_b200.h"
#include "phc_common.cuh"

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

namespace phc {

constexpr int BM = 128, BN = 128, BK = 16, STAGES = 4, GEMM_THREADS = 256;
constexpr int WM = 64, WN = 32;                 // warp tile: 2 x 4 warps
constexpr int KPAD = 4;                         // k-contiguous tiles: [rows][BK + 4]   (stride 20 words: conflict free)
constexpr int MPAD = 8;                         // mn-contiguous tiles: [BK][rows + 8]  (stride 136 words: conflict free)
constexpr int TILE_FLOATS = (BM * (BK + KPAD) > BK * (BM + MPAD)) ? BM * (BK + KPAD) : BK * (BM + MPAD);   // 2560

struct GemmArgs {
  const float* A; const float* B; float* C;
  const float* bias;      // [N] or null
  float* mask;            // `aux` of the C ABI: [M, ldmask] or null (read by the backward modes, written by SiLU forward)
  int M, N, K;
  int64_t lda, ldb, ldc, ldmask;
  float alpha;
  int relu;               // PHC_ACT_* activation code
  int accumulate;         // atomicAdd into C instead of store
  int k_splits;           // gridDim.z
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool pred) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  const int sz = pred ? 16 : 0;                                  // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float r = x - __uint_as_float(hi);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// Load one operand tile (ROWS x BK, logical element (r, k)) of a strided matrix into shared memory.
//   KMAJ:  global (r, k) at base[r*ld + k]  -> smem [r][BK+KPAD]
//   !KMAJ: global (r, k) at base[k*ld + r]  -> smem [k][ROWS+MPAD]
// rows / k beyond the matrix are zero filled.  ld % 4 == 0 and 16-byte aligned base are checked on the host; the
// buffers are allocated with their extents rounded up to 4 elements (zero padded), so a 16-byte chunk never crosses
// the end of a row's allocation.
template <bool KMAJ, int ROWS>
__device__ __forceinline__ void load_tile(float* s, const float* __restrict__ g, int64_t ld, int r0, int k0, int R, int Kend,
                                          int tid) {
  if (KMAJ) {
    constexpr int CH = BK / 4;                                   // 16-byte chunks per row
#pragma unroll
    for (int i = tid; i < ROWS * CH; i += GEMM_THREADS) {
      const int r = i / CH, c = i % CH;
      const bool ok = (r0 + r < R) && (k0 + 4 * c < Kend);
      const float* src = ok ? g + (int64_t)(r0 + r) * ld + k0 + 4 * c : g;
      cp_async16(s + r * (BK + KPAD) + 4 * c, src, ok);
    }
  } else {
    constexpr int CH = ROWS / 4;
#pragma unroll
    for (int i = tid; i < BK * CH; i += GEMM_THREADS) {
      const int k = i / CH, c = i % CH;
      const bool ok = (k0 + k < Kend) && (r0 + 4 * c < R);
      const float* src = ok ? g + (int64_t)(k0 + k) * ld + r0 + 4 * c : g;
      cp_async16(s + k * (ROWS + MPAD) + 4 * c, src, ok);
    }
  }
}

template <bool KMAJ, int ROWS>
__device__ __forceinline__ float lds_elem(const float* s, int r, int k) {
  return KMAJ ? s[r * (BK + KPAD) + k] : s[k * (ROWS + MPAD) + r];
}

template <bool A_KMAJ, bool B_KMAJ>
__global__ void __launch_bounds__(GEMM_THREADS, 2) gemm_3xtf32_kernel(const __grid_constant__ GemmArgs g) {
  extern __shared__ __align__(16) float gsm[];
  float* sA = gsm;                                  // [STAGES][TILE_FLOATS]
  float* sB = gsm + STAGES * TILE_FLOATS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = (warp >> 2) * WM, wn = (warp & 3) * WN;       // 2 x 4 warp grid
  const int grp = lane >> 2, tig = lane & 3;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  // K range of this split (multiples of BK)
  const int k_tiles_total = (g.K + BK - 1) / BK;
  const int tiles_per_split = (k_tiles_total + g.k_splits - 1) / g.k_splits;
  const int kt_begin = blockIdx.z * tiles_per_split;
  const int kt_end = min(k_tiles_total, kt_begin + tiles_per_split);
  const int nkt = kt_end - kt_begin;
  if (nkt <= 0) return;
  // chunk-level bound along the contiguous dimension: extents rounded up to 4 (allocation is zero padded)
  const int Kend_A = A_KMAJ ? ((g.K + 3) & ~3) : g.K;
  const int Kend_B = B_KMAJ ? ((g.K + 3) & ~3) : g.K;
  const int Mr = A_KMAJ ? g.M : ((g.M + 3) & ~3);
  const int Nr = B_KMAJ ? g.N : ((g.N + 3) & ~3);

  float acc[WM / 16][WN / 8][4];
#pragma unroll
  for (int i = 0; i < WM / 16; ++i)
#pragma unroll
    for (int j = 0; j < WN / 8; ++j)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.f;

  auto issue = [&](int kt, int stage) {
    const int k0 = (kt_begin + kt) * BK;
    load_tile<A_KMAJ, BM>(sA + stage * TILE_FLOATS, g.A, g.lda, m0, k0, Mr, Kend_A, tid);
    load_tile<B_KMAJ, BN>(sB + stage * TILE_FLOATS, g.B, g.ldb, n0, k0, Nr, Kend_B, tid);
  };

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkt) issue(s, s);
    cp_async_commit();
  }

  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {   // prefetch tile kt + STAGES - 1 into the stage consumed at iteration kt - 1
      const int nk = kt + STAGES - 1;
      if (nk < nkt) issue(nk, nk % STAGES);
      cp_async_commit();
    }
    const float* a_s = sA + (kt % STAGES) * TILE_FLOATS;
    const float* b_s = sB + (kt % STAGES) * TILE_FLOATS;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 8) {
      uint32_t ah[WM / 16][4], al[WM / 16][4], bh[WN / 8][2], bl[WN / 8][2];
#pragma unroll
      for (int i = 0; i < WM / 16; ++i) {
        const int r = wm + i * 16 + grp;
        split_tf32(lds_elem<A_KMAJ, BM>(a_s, r, kk + tig), ah[i][0], al[i][0]);
        split_tf32(lds_elem<A_KMAJ, BM>(a_s, r + 8, kk + tig), ah[i][1], al[i][1]);
        split_tf32(lds_elem<A_KMAJ, BM>(a_s, r, kk + tig + 4), ah[i][2], al[i][2]);
        split_tf32(lds_elem<A_KMAJ, BM>(a_s, r + 8, kk + tig + 4), ah[i][3], al[i][3]);
      }
#pragma unroll
      for (int j = 0; j < WN / 8; ++j) {
        const int c = wn + j * 8 + grp;
        split_tf32(lds_elem<B_KMAJ, BN>(b_s, c, kk + tig), bh[j][0], bl[j][0]);
        split_tf32(lds_elem<B_KMAJ, BN>(b_s, c, kk + tig + 4), bh[j][1], bl[j][1]);
      }
#pragma unroll
      for (int i = 0; i < WM / 16; ++i)
#pragma unroll
        for (int j = 0; j < WN / 8; ++j) {
          mma_tf32(acc[i][j], al[i], bh[j]);      // small terms first
          mma_tf32(acc[i][j], ah[i], bl[j]);
          mma_tf32(acc[i][j], ah[i], bh[j]);
        }
    }
  }
  cp_async_wait<0>();

  // ---- epilogue ----
#pragma unroll
  for (int i = 0; i < WM / 16; ++i)
#pragma unroll
    for (int j = 0; j < WN / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + wm + i * 16 + grp + 8 * h;
        const int n = n0 + wn + j * 8 + 2 * tig;
        if (m >= g.M) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (n + e >= g.N) continue;
          float v = g.alpha * acc[i][j][2 * h + e];
          if (g.bias && blockIdx.z == 0) v += g.bias[n + e];
          float* aux = g.mask ? g.mask + (int64_t)m * g.ldmask + n + e : nullptr;
          if (g.relu == PHC_ACT_RELU) v = fmaxf(v, 0.f);
          if (g.relu == PHC_ACT_SILU) {
            if (aux) *aux = v;                                   // pre-activation, read back by PHC_ACT_SILU_BWD
            v = silu_f(v);
          } else if (aux) {
            v = (g.relu == PHC_ACT_SILU_BWD) ? v * silu_grad_f(*aux) : ((*aux > 0.f) ? v : 0.f);
          }
          float* dst = g.C + (int64_t)m * g.ldc + n + e;
          if (g.accumulate) atomicAdd(dst, v);
          else *dst = v;
        }
      }
}

// column sums: out[n] (+)= sum_m X[m, n]  (bias gradients).  One block per 32 columns, rows strided over threadIdx.y; one block
// owns a column, so the sum does not depend on scheduling.
__global__ void __launch_bounds__(1024) colsum_kernel(const float* __restrict__ X, int64_t ld, int M, int N,
                                                      float alpha, float* __restrict__ out, int accumulate) {
  __shared__ float s[32][33];
  const int n = blockIdx.x * 32 + threadIdx.x;
  float v = 0.f;
  if (n < N)
    for (int m = blockIdx.y * 32 + threadIdx.y; m < M; m += 32 * gridDim.y) v += X[(int64_t)m * ld + n];
  s[threadIdx.y][threadIdx.x] = v;
  __syncthreads();
  if (threadIdx.y == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) t += s[i][threadIdx.x];
    t *= alpha;
    out[n] = accumulate ? out[n] + t : t;
  }
}

// grouped column sums: up to PHC_GEMM_GROUP_MAX matrices in one launch (the bias gradients of every stack at one layer depth).
// A block is 8 rows x 32 lanes, each lane owns 4 consecutive columns (one 16-byte load per row): 128 columns x 256 rows per block,
// 8 independent loads in flight per thread; the 8 row partials meet in shared memory and leave as one partial per column and block.
// The last block of a column chunk to finish adds the partials of the chunk's row blocks in row order: the result does not depend on
// which block finishes first.
struct ColsumGroup {
  const float* X[PHC_GEMM_GROUP_MAX];
  float* out[PHC_GEMM_GROUP_MAX];
  int64_t ld[PHC_GEMM_GROUP_MAX];
  int32_t M[PHC_GEMM_GROUP_MAX], N[PHC_GEMM_GROUP_MAX], block_begin[PHC_GEMM_GROUP_MAX + 1], col_chunks[PHC_GEMM_GROUP_MAX];
  int32_t rows[PHC_GEMM_GROUP_MAX], row_chunks[PHC_GEMM_GROUP_MAX], chunk_begin[PHC_GEMM_GROUP_MAX];
  float alpha[PHC_GEMM_GROUP_MAX];
  int32_t count;
  float* part;              // [blocks][128] partial sums
  unsigned int* tickets;    // [column chunks] blocks of the chunk done so far (zero between launches)
};
constexpr int CS_MAX_ROW_CHUNKS = 32, CS_SLOTS = 8, CS_MAX_BLOCKS = 4096, CS_MAX_CHUNKS = 1024;
__device__ float g_cs_part[CS_SLOTS][CS_MAX_BLOCKS][128];
__device__ unsigned int g_cs_tickets[CS_SLOTS][CS_MAX_CHUNKS];

__global__ void __launch_bounds__(256) colsum_group_kernel(const __grid_constant__ ColsumGroup G) {
  __shared__ float4 part[8][32];
  int g = 0;
  while (g + 1 < G.count && (int)blockIdx.x >= G.block_begin[g + 1]) ++g;
  const int b = blockIdx.x - G.block_begin[g];
  const int cc = b % G.col_chunks[g], rc = b / G.col_chunks[g];
  const int lane = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c0 = cc * 128 + lane * 4;
  const int N = G.N[g], M = G.M[g];
  const int64_t ld = G.ld[g];
  const float* __restrict__ X = G.X[g];
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c0 < N) {
    const int r_end = min(M, (rc + 1) * G.rows[g]);
    int r = rc * G.rows[g] + ry;
    for (; r + 56 < r_end; r += 64) {
      float4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __ldg(reinterpret_cast<const float4*>(X + (int64_t)(r + 8 * u) * ld + c0));
#pragma unroll
      for (int u = 0; u < 8; ++u) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
    }
    for (; r < r_end; r += 8) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(X + (int64_t)r * ld + c0));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  part[ry][lane] = acc;
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x < 128) {
    const float* p = reinterpret_cast<const float*>(&part[0][0]) + threadIdx.x;
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += p[i * 128];
    G.part[(int64_t)blockIdx.x * 128 + threadIdx.x] = t;
    __threadfence();
  }
  __syncthreads();
  unsigned int* ticket = G.tickets + G.chunk_begin[g] + cc;
  if (threadIdx.x == 0) {
    last = atomicAdd(ticket, 1u) == (unsigned)(G.row_chunks[g] - 1);
    if (last) *ticket = 0u;                                   // back to zero for the next launch
  }
  __syncthreads();
  if (last && threadIdx.x < 128) {
    __threadfence();
    const int c = cc * 128 + threadIdx.x;
    if (c < N) {
      float t = 0.f;
      for (int i = 0; i < G.row_chunks[g]; ++i)
        t += __ldcg(G.part + ((int64_t)G.block_begin[g] + (int64_t)i * G.col_chunks[g] + cc) * 128 + threadIdx.x) * G.alpha[g];
      G.out[g][c] += t;
    }
  }
}

}  // namespace phc

extern "C" int phc_colsum_group(const PhcColsumDesc* d, int32_t count, void* stream) {
  if (!d || count < 1 || count > PHC_GEMM_GROUP_MAX) { phc_set_error("phc_colsum_group: 1 <= count <= PHC_GEMM_GROUP_MAX problems"); return PHC_ERR_INVALID_ARG; }
  phc::ColsumGroup G;
  int n = 0, blocks = 0, chunks = 0;
  for (int i = 0; i < count; ++i) {
    const PhcColsumDesc& q = d[i];
    if (!q.X || !q.out || q.M < 0 || q.N < 0) { phc_set_error("phc_colsum_group: bad problem (NULL pointer or negative size)"); return PHC_ERR_INVALID_ARG; }
    if ((q.ld & 3) || q.ld < ((q.N + 3) & ~3) || (reinterpret_cast<uintptr_t>(q.X) & 15)) {
      phc_set_error("phc_colsum_group: X must be 16-byte aligned with a leading dimension that is a multiple of 4 floats and >= N rounded up to 4");
      return PHC_ERR_INVALID_ARG;
    }
    if (q.M == 0 || q.N == 0) continue;
    for (int j = 0; j < n; ++j)                                 // the last block of a chunk adds without atomics: one writer per column
      if (q.out < G.out[j] + G.N[j] && G.out[j] < q.out + q.N) { phc_set_error("phc_colsum_group: the problems' out ranges overlap"); return PHC_ERR_INVALID_ARG; }
    G.X[n] = q.X; G.out[n] = q.out; G.ld[n] = q.ld; G.M[n] = q.M; G.N[n] = q.N; G.alpha[n] = q.alpha;
    G.col_chunks[n] = (q.N + 127) / 128;
    int rows = (q.M + phc::CS_MAX_ROW_CHUNKS - 1) / phc::CS_MAX_ROW_CHUNKS;
    rows = rows < 256 ? 256 : (rows + 63) / 64 * 64;
    G.rows[n] = rows;
    G.row_chunks[n] = (q.M + rows - 1) / rows;
    G.chunk_begin[n] = chunks;
    chunks += G.col_chunks[n];
    G.block_begin[n] = blocks;
    blocks += G.col_chunks[n] * G.row_chunks[n];
    ++n;
  }
  if (n == 0) return PHC_OK;
  if (blocks > phc::CS_MAX_BLOCKS || chunks > phc::CS_MAX_CHUNKS) { phc_set_error("phc_colsum_group: problems too large for one launch"); return PHC_ERR_UNSUPPORTED; }
  static float* part_base = nullptr;
  static unsigned int* ticket_base = nullptr;
  static unsigned int launch_no = 0;
  if (!part_base) {
    void* p = nullptr;
    cudaError_t e = cudaGetSymbolAddress(&p, phc::g_cs_part);
    if (e != cudaSuccess) return phc_check_cuda(e, "cudaGetSymbolAddress(g_cs_part)");
    part_base = static_cast<float*>(p);
    e = cudaGetSymbolAddress(&p, phc::g_cs_tickets);
    if (e != cudaSuccess) return phc_check_cuda(e, "cudaGetSymbolAddress(g_cs_tickets)");
    ticket_base = static_cast<unsigned int*>(p);
  }
  const unsigned int slot = launch_no++ % phc::CS_SLOTS;      // launches in flight on different streams use different slots
  G.part = part_base + (size_t)slot * phc::CS_MAX_BLOCKS * 128;
  G.tickets = ticket_base + (size_t)slot * phc::CS_MAX_CHUNKS;
  G.block_begin[n] = blocks; G.count = n;
  phc::colsum_group_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(G); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "colsum_group_kernel launch");
}

extern "C" int phc_gemm(const float* A, int64_t lda, int32_t a_kmajor, const float* B, int64_t ldb, int32_t b_kmajor,
                        float* C, int64_t ldc, int32_t M, int32_t N, int32_t K, float alpha, const float* bias,
                        int32_t relu, float* mask, int64_t ldmask, int32_t accumulate, int32_t k_splits,
                        void* stream) {
  using namespace phc;
  if (!A || !B || !C || M < 0 || N < 0 || K < 0) { phc_set_error("phc_gemm: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (M == 0 || N == 0) return PHC_OK;
  if ((lda & 3) || (ldb & 3) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) {
    phc_set_error("phc_gemm: A/B must be 16-byte aligned with leading dimensions that are multiples of 4 floats");
    return PHC_ERR_INVALID_ARG;
  }
  const int a_ext = a_kmajor ? K : M, b_ext = b_kmajor ? K : N;
  if (lda < ((a_ext + 3) & ~3) || ldb < ((b_ext + 3) & ~3) || ldc < N) {
    phc_set_error("phc_gemm: leading dimension smaller than the (4-padded) contiguous extent"); return PHC_ERR_INVALID_ARG;
  }
  if (k_splits < 1) k_splits = 1;
  if (k_splits > 1 && !accumulate) { phc_set_error("phc_gemm: split-K needs accumulate=1 (C pre-zeroed)"); return PHC_ERR_INVALID_ARG; }
  if (k_splits > 1 && (relu || mask)) { phc_set_error("phc_gemm: split-K cannot be combined with a non-linear epilogue"); return PHC_ERR_INVALID_ARG; }
  if (relu < 0 || relu > PHC_ACT_SILU_BWD || (relu == PHC_ACT_SILU_BWD && !mask)) { phc_set_error("phc_gemm: bad activation code"); return PHC_ERR_INVALID_ARG; }
  if (K == 0) { if (!accumulate) cudaMemset2DAsync(C, ldc * 4, 0, (size_t)N * 4, M, static_cast<cudaStream_t>(stream)); return PHC_OK; }
  GemmArgs g;
  g.A = A; g.B = B; g.C = C; g.bias = bias; g.mask = mask; g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldb; g.ldc = ldc;
  g.ldmask = ldmask; g.alpha = alpha; g.relu = relu; g.accumulate = accumulate; g.k_splits = k_splits;
  const dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, k_splits);
  const size_t smem = (size_t)2 * STAGES * TILE_FLOATS * sizeof(float);     // 80 KB
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
#define PHC_GEMM_LAUNCH(AK, BK_)                                                                             \
  do {                                                                                                       \
    static bool done = false;                                                                                \
    if (!done) {                                                                                             \
      e = cudaFuncSetAttribute(gemm_3xtf32_kernel<AK, BK_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
      if (e != cudaSuccess) return phc_check_cuda(e, "cudaFuncSetAttribute(gemm)");                          \
      done = true;                                                                                           \
    }                                                                                                        \
    gemm_3xtf32_kernel<AK, BK_><<<grid, GEMM_THREADS, smem, st>>>(g); phc_count_launches(1);                                        \
  } while (0)
  if (a_kmajor && b_kmajor) PHC_GEMM_LAUNCH(true, true);
  else if (a_kmajor && !b_kmajor) PHC_GEMM_LAUNCH(true, false);
  else if (!a_kmajor && b_kmajor) PHC_GEMM_LAUNCH(false, true);
  else PHC_GEMM_LAUNCH(false, false);
#undef PHC_GEMM_LAUNCH
  return phc_check_cuda(cudaGetLastError(), "gemm_3xtf32_kernel launch");
}

extern "C" int phc_colsum(const float* X, int64_t ld, int32_t M, int32_t N, float alpha, float* out, int32_t accumulate,
                          void* stream) {
  if (!X || !out || M < 0 || N < 0) { phc_set_error("phc_colsum: bad arguments"); return PHC_ERR_INVALID_ARG; }
  if (N == 0) return PHC_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  phc::colsum_kernel<<<dim3((N + 31) / 32, 1), dim3(32, 32), 0, st>>>(X, ld, M, N, alpha, out, accumulate); phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "colsum_kernel launch");
}
