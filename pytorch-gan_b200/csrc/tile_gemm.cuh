// tile_gemm.cuh -- the 32x32 fp32 FFMA tile GEMM of the cooperative MLP kernels (mlp_critic.cu,
// mlp_generator/mlp_generator.cu).
// Each phase of those kernels spreads the 32x32 output tiles of one or two small GEMMs over a persistent grid.
#pragma once
#include <cuda_runtime.h>

namespace b200gan {

constexpr int GT = 32;  // tile edge

// C(m,n) = sum_k A(m,k) B(k,n) for tile `tile` of an M x N problem; A(m,k) = A[m*sam + k*sak],
// B(k,n) = B[k*sbk + n*sbn].  256 threads, 2x2 outputs per thread.
template <class Epi>
__device__ __forceinline__ void tile_gemm(const float *__restrict__ A, int sam, int sak, const float *__restrict__ B,
                                          int sbk, int sbn, int M, int N, int K, int tile, Epi epi,
                                          float (*As)[GT + 1], float (*Bs)[GT + 1]) {
  const int tilesN = (N + GT - 1) / GT;
  const int m0 = (tile / tilesN) * GT, n0 = (tile % tilesN) * GT;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int k0 = 0; k0 < K; k0 += GT) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int e = tid + 256 * i;
      int k, m;
      if (sak == 1) { k = e & 31; m = e >> 5; } else { m = e & 31; k = e >> 5; }
      float v = 0.f;
      if (m0 + m < M && k0 + k < K) v = __ldg(A + (size_t)(m0 + m) * sam + (size_t)(k0 + k) * sak);
      As[k][m] = v;
      int kb, n;
      if (sbn == 1) { n = e & 31; kb = e >> 5; } else { kb = e & 31; n = e >> 5; }
      float w = 0.f;
      if (n0 + n < N && k0 + kb < K) w = __ldg(B + (size_t)(k0 + kb) * sbk + (size_t)(n0 + n) * sbn);
      Bs[kb][n] = w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GT; ++k) {
      float a0 = As[k][ty * 2], a1 = As[k][ty * 2 + 1];
      float b0 = Bs[k][tx * 2], b1 = Bs[k][tx * 2 + 1];
      acc[0][0] = fmaf(a0, b0, acc[0][0]);
      acc[0][1] = fmaf(a0, b1, acc[0][1]);
      acc[1][0] = fmaf(a1, b0, acc[1][0]);
      acc[1][1] = fmaf(a1, b1, acc[1][1]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      int m = m0 + ty * 2 + i, n = n0 + tx * 2 + j;
      if (m < M && n < N) epi(m, n, acc[i][j]);
    }
}

__device__ __forceinline__ int ntiles(int M, int N) { return ((M + GT - 1) / GT) * ((N + GT - 1) / GT); }

}  // namespace b200gan
