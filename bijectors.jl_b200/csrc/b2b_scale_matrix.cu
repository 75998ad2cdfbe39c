// Dense linear layer, B2B_SCALE_MATRIX (include/b2b.h): Scale(A) with a D x D matrix A (scale.jl:14,17,35-36):
//   forward   y = A x,    logjac = log|det A|          inverse   y = A⁻¹ x,   logjac = −log|det A|
//   reverse   (u the layer's input, M = A or A⁻¹, G = Σₙ ȳₙ uₙᵀ, s = Σₙ l̄ₙ, B = A⁻ᵀ)
//             forward layer: x̄ = Aᵀ ȳ,    Ā = G + s·B
//             inverse layer: x̄ = A⁻ᵀ ȳ,   Ā = −B G B − s·B
//
// factor_kernel (one CTA of 512 threads): blocked right-looking LU with partial pivoting of the fp32 A in fp64 (what
// logabsdet computes through getrf), column-major in the workspace.  A panel of kNB columns is factored in shared
// memory (pivot search by one warp, first maximum wins as in idamax), its row swaps are applied to the other columns
// one column per thread, the block row U12 is solved against the unit lower L11, and the trailing matrix takes the
// rank-kNB update A22 −= L21·U12 in one read and one write per element.  log|det A| = Σ log|Uᵢᵢ| in row order.  A zero
// pivot leaves its column unscaled (getrf's convention), so a singular A gives −Inf and finite y = A x.
// inv_kernel: A⁻¹ column by column from P A = L U; a warp solves kInvC columns, lanes own rows, and both substitutions
// step over k reading column k of L / U once (coalesced) for all of them.  M = A⁻¹ is rounded to fp32.
// map_kernel<DP, BN, TRANS>: Y = M X (or Mᵀ X) in exact fp32 FFMA.  A CTA owns all D rows of BN columns: it stages the
// x tile (rows padded to DP) in shared memory before anything is stored -- so y may alias x -- streams M through
// shared memory in k-blocks of kBK (double buffered through registers), and each thread keeps an 8 x 8 register tile.
// Every output is one fmaf chain in increasing k: results do not depend on N, the tile or the launch.
// Reverse mode: x̄ by map_kernel with the transposed operand; G by the chunked outer-product kernel of the full-covariance
// base (all tiles), its chunks and Σ l̄ summed in a fixed order in fp64, and the two D x D products of the inverse layer
// in fp64.  No atomics; every launch is graph-capturable.
//
// LU layer, B2B_SCALE_LU: y = P·L·U·x with L (unit lower) and U (upper) packed in one D x D F as getrf leaves them and P
// the permutation y[dst[r]] = (L U x)[r].  The dense layer's map and reverse mode on M = P·L·U (forward) or U⁻¹ L⁻¹ Pᵀ:
//   lu_prep_kernel (parallel over columns) writes M in fp32 from fp64 columns -- L·(U e_j) scattered to the rows dst[·],
//     or Pᵀ e_j solved against L and U as inv_kernel does -- and log|det U| in row order; the map is the dense one, so a
//     call is two launches.
//   reverse mode: M̄ = G (forward layer) or −M⁻ᵀ G M⁻ᵀ (inverse layer, the dense finalize without its s·B term), then
//     lu_bar_kernel takes M̄ through the factors: L̄ = 𝒮(Pᵀ M̄ Uᵀ), Ū = 𝒰(Lᵀ Pᵀ M̄) ± s·diag(1/Uᵢᵢ), packed like F.
//
// Triangular layer, B2B_SCALE_TRIANGULAR: Scale(T) with T lower or upper triangular, stored or unit diagonal.  The same
// launches with the structure made explicit, selected by the descriptor's kind in scale_prep:
//   tri_prep_kernel (parallel over columns, no serial step) writes M = T or T⁻¹ in fp32, zero outside the triangle and 1
//     on a unit diagonal, reading only the triangle of T; T⁻¹ column by column, a warp per kInvC columns with lanes over
//     rows, one fp64 substitution against identity columns.  An extra CTA sums log|Tᵢᵢ| in row order.
//   map_kernel<DP, BN, TRANS, TRI>: each warp owns contiguous row blocks -- one from the top and one from the bottom of
//     the tile, so the warps' work is balanced -- and skips the k-blocks that are zero for every row of a block.
//   reverse mode: T̄ = 𝒫(Ā) with 𝒫 the parameter's triangle (strict for the unit forms).  G is needed on 𝒫 only for the
//     forward layer (the outer-product kernel's lower tiles; for an upper T with the operands swapped, giving Gᵀ), in full
//     for the inverse layer; the finalize kernels take 𝒫 as an output mask ("full" for the dense layer).
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

#include "b2b_internal.h"

namespace b2b_scale {

constexpr int kFactorThreads = 512;
constexpr int kNB = 16;     // LU panel width
constexpr int kInvC = 4;    // columns of A⁻¹ per warp
constexpr int kInvWarps = 4;
constexpr int kBK = 16;     // k-block of the map GEMM
constexpr unsigned kFull = 0xffffffffu;

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

// factor storage: [LU (D x D fp64, column-major)][M = A⁻¹ (D x D fp32)][perm (D int32)][log|det A| (fp64)]
struct Factor {
  double* lu;
  float* minv;
  int* perm;
  double* logdet;
};

size_t factor_bytes(int D) {
  return al256(sizeof(double) * (size_t)D * D) + al256(sizeof(float) * (size_t)D * D) + al256(sizeof(int) * (size_t)D) +
         al256(sizeof(double)) + 256;
}

Factor carve(void* ws, int D) {
  char* p = b2b_align256(ws);
  Factor f;
  f.lu = reinterpret_cast<double*>(p);
  p += al256(sizeof(double) * (size_t)D * D);
  f.minv = reinterpret_cast<float*>(p);
  p += al256(sizeof(float) * (size_t)D * D);
  f.perm = reinterpret_cast<int*>(p);
  p += al256(sizeof(int) * (size_t)D);
  f.logdet = reinterpret_cast<double*>(p);
  return f;
}

// triangular storage: [M = T or T⁻¹ (D x D fp32, column-major)][log|det T| (fp64)]
struct TriFactor {
  float* m;
  double* logdet;
};

size_t tri_bytes(int D) { return al256(sizeof(float) * (size_t)D * D) + al256(sizeof(double)) + 256; }

TriFactor carve_tri(void* ws, int D) {
  char* p = b2b_align256(ws);
  TriFactor f;
  f.m = reinterpret_cast<float*>(p);
  f.logdet = reinterpret_cast<double*>(p + al256(sizeof(float) * (size_t)D * D));
  return f;
}

size_t factor_smem(int D) { return sizeof(double) * 2 * (size_t)kNB * D + sizeof(int) * ((size_t)D + kNB + 4); }

__global__ void __launch_bounds__(kFactorThreads, 1)
    factor_kernel(const float* __restrict__ A, int D, double* __restrict__ lu, int* __restrict__ perm_out,
                  double* __restrict__ logdet) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* Ps = reinterpret_cast<double*>(smem_raw);  // panel: Ps[c * D + i], column c of the panel, row i
  double* Us = Ps + (size_t)kNB * D;                 // block row U12: Us[r * D + j]
  int* perm = reinterpret_cast<int*>(Us + (size_t)kNB * D);
  int* pivs = perm + D;
  int* sp = pivs + kNB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (long long idx = tid; idx < (long long)D * D; idx += kFactorThreads) lu[idx] = (double)__ldg(A + idx);
  for (int i = tid; i < D; i += kFactorThreads) perm[i] = i;
  double ld = 0.0;  // thread 0
  __syncthreads();
  for (int k0 = 0; k0 < D; k0 += kNB) {
    const int nb = D - k0 < kNB ? D - k0 : kNB;
    for (int idx = tid; idx < nb * D; idx += kFactorThreads) {
      const int c = idx / D, i = idx - c * D;
      if (i >= k0) Ps[c * D + i] = lu[(size_t)(k0 + c) * D + i];
    }
    __syncthreads();
    // unblocked LU of the panel (rows k0..D-1)
    for (int c = 0; c < nb; ++c) {
      const int kk = k0 + c;
      if (warp == 0) {
        double best = -1.0;
        int bi = D;
        for (int i = kk + lane; i < D; i += 32) {
          const double v = fabs(Ps[c * D + i]);
          if (v > best) {
            best = v;
            bi = i;
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const double ov = __shfl_xor_sync(kFull, best, o);
          const int oi = __shfl_xor_sync(kFull, bi, o);
          if (ov > best || (ov == best && oi < bi)) {
            best = ov;
            bi = oi;
          }
        }
        if (lane == 0) {
          *sp = bi < D ? bi : kk;  // NaN column: no swap
          pivs[c] = *sp;
        }
      }
      __syncthreads();
      const int p = *sp;
      if (p != kk && tid < nb) {
        const double t = Ps[tid * D + kk];
        Ps[tid * D + kk] = Ps[tid * D + p];
        Ps[tid * D + p] = t;
      }
      __syncthreads();
      const double piv = Ps[c * D + kk];
      if (tid == 0) ld += log(fabs(piv));
      for (int i = kk + 1 + tid; i < D; i += kFactorThreads)
        if (piv != 0.0) Ps[c * D + i] /= piv;
      __syncthreads();
      const int m = D - kk - 1;
      for (int idx = tid; idx < (nb - c - 1) * m; idx += kFactorThreads) {
        const int c2 = c + 1 + idx / m, i = kk + 1 + idx % m;
        Ps[c2 * D + i] = fma(-Ps[c * D + i], Ps[c2 * D + kk], Ps[c2 * D + i]);
      }
      __syncthreads();
    }
    // the panel back to global; its row swaps applied to every other column (one column per thread, in order)
    for (int idx = tid; idx < nb * D; idx += kFactorThreads) {
      const int c = idx / D, i = idx - c * D;
      if (i >= k0) lu[(size_t)(k0 + c) * D + i] = Ps[c * D + i];
    }
    for (int j = tid; j < D; j += kFactorThreads) {
      if (j >= k0 && j < k0 + nb) continue;
      double* col = lu + (size_t)j * D;
      for (int c = 0; c < nb; ++c) {
        const int p = pivs[c];
        if (p != k0 + c) {
          const double t = col[k0 + c];
          col[k0 + c] = col[p];
          col[p] = t;
        }
      }
    }
    if (tid == 0)
      for (int c = 0; c < nb; ++c) {
        const int p = pivs[c], t = perm[k0 + c];
        perm[k0 + c] = perm[p];
        perm[p] = t;
      }
    __syncthreads();
    const int j0 = k0 + nb;
    if (j0 >= D) break;
    // U12 = L11⁻¹ A12, one column per thread, worked on in shared memory
    for (int j = j0 + tid; j < D; j += kFactorThreads) {
      double* col = lu + (size_t)j * D + k0;
      for (int r = 0; r < nb; ++r) Us[r * D + j] = col[r];
      for (int r = 0; r < nb; ++r) {
        const double ur = Us[r * D + j];
        for (int r2 = r + 1; r2 < nb; ++r2) Us[r2 * D + j] = fma(-Ps[r * D + k0 + r2], ur, Us[r2 * D + j]);
        col[r] = ur;
      }
    }
    __syncthreads();
    // A22 −= L21 · U12
    const int m = D - j0;
    for (int idx = tid; idx < m * m; idx += kFactorThreads) {
      const int j = j0 + idx / m, i = j0 + idx % m;
      double* a = lu + (size_t)j * D + i;
      double v = *a;
      for (int r = 0; r < nb; ++r) v = fma(-Ps[r * D + i], Us[r * D + j], v);
      *a = v;
    }
    __syncthreads();
  }
  for (int i = tid; i < D; i += kFactorThreads) perm_out[i] = perm[i];
  if (tid == 0) *logdet = ld;
}

// z := U⁻¹ L⁻¹ z for the kInvC columns of a warp (lanes own rows), L unit lower and U upper packed in `lu` (column-major,
// getrf's layout, fp64 or fp32 entries): forward substitution against L (right-looking), then back substitution against U.
// Reads L strictly below the diagonal and U on and above it; column k is read once (coalesced) for all the columns.
template <int R, class TF>
__device__ __forceinline__ void lu_solve_cols(double (&z)[R][kInvC], const TF* __restrict__ lu, int D, int lane) {
  // forward substitution, unit lower L (right-looking)
#pragma unroll
  for (int kb = 0; kb < R; ++kb) {
    for (int jj = 0; jj < 32; ++jj) {
      const int k = kb * 32 + jj;
      if (k >= D) break;
      double v[kInvC];
#pragma unroll
      for (int c = 0; c < kInvC; ++c) v[c] = __shfl_sync(kFull, z[kb][c], jj);
      const TF* Lk = lu + (size_t)k * D;
#pragma unroll
      for (int r = kb; r < R; ++r) {
        const int i = lane + 32 * r;
        if (i > k && i < D) {
          const double l = (double)Lk[i];
#pragma unroll
          for (int c = 0; c < kInvC; ++c) z[r][c] = fma(-l, v[c], z[r][c]);
        }
      }
    }
  }
  // back substitution, upper U
#pragma unroll
  for (int kb = R - 1; kb >= 0; --kb) {
    for (int jj = 31; jj >= 0; --jj) {
      const int k = kb * 32 + jj;
      if (k >= D) continue;
      const TF* Uk = lu + (size_t)k * D;
      const double ukk = (double)Uk[k];
      double v[kInvC];
#pragma unroll
      for (int c = 0; c < kInvC; ++c) {
        v[c] = __shfl_sync(kFull, z[kb][c], jj) / ukk;
        if (lane == jj) z[kb][c] = v[c];
      }
#pragma unroll
      for (int r = 0; r <= kb; ++r) {
        const int i = lane + 32 * r;
        if (i < k) {
          const double u = (double)Uk[i];
#pragma unroll
          for (int c = 0; c < kInvC; ++c) z[r][c] = fma(-u, v[c], z[r][c]);
        }
      }
    }
  }
}

// columns of M = A⁻¹ (fp32, column-major): solve L U z = P e_j
template <int R>
__global__ void __launch_bounds__(kInvWarps * 32)
    inv_kernel(const double* __restrict__ lu, const int* __restrict__ perm, float* __restrict__ minv, int D) {
  const int lane = threadIdx.x & 31;
  const int col0 = (blockIdx.x * kInvWarps + (threadIdx.x >> 5)) * kInvC;
  if (col0 >= D) return;
  double z[R][kInvC];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int i = lane + 32 * r;
    const int pi = i < D ? perm[i] : -1;
#pragma unroll
    for (int c = 0; c < kInvC; ++c) z[r][c] = (pi == col0 + c) ? 1.0 : 0.0;
  }
  lu_solve_cols<R>(z, lu, D, lane);
#pragma unroll
  for (int c = 0; c < kInvC; ++c) {
    const int j = col0 + c;
    if (j >= D) break;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int i = lane + 32 * r;
      if (i < D) minv[(size_t)j * D + i] = (float)z[r][c];
    }
  }
}

// *logdet = Σᵢ log|Tᵢᵢ| in row order (0 for unit), by the first warp of the calling CTA
template <int R>
__device__ __forceinline__ void diag_logdet(const float* __restrict__ T, int D, int unit, double* __restrict__ logdet) {
  __shared__ double lg[32 * R];
  const int lane = threadIdx.x & 31;
  if (threadIdx.x >= 32) return;
  for (int i = lane; i < D; i += 32) lg[i] = unit ? 0.0 : log(fabs((double)T[(size_t)i * D + i]));
  __syncwarp();
  if (lane == 0) {
    double s = 0.0;
    for (int i = 0; i < D; ++i) s += lg[i];
    *logdet = s;
  }
}

// M = T (inv == 0) or T⁻¹ of a triangular T (lower: upper == 0), fp32, zero outside the triangle; only the triangle of T
// is read, and not its diagonal when unit != 0.  T⁻¹ column j: the substitution of T z = e_j in fp64 (right-looking: z_k is
// final once steps before k ran, then the rows beyond k take −T(i, k)·z_k), rows owned by lanes.  The last CTA writes
// log|det T| = Σ log|Tᵢᵢ| in row order (0 for unit).
template <int R>
__global__ void __launch_bounds__(kInvWarps * 32)
    tri_prep_kernel(const float* __restrict__ T, int D, int upper, int unit, int inv, float* __restrict__ M,
                    double* __restrict__ logdet) {
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == gridDim.x - 1) {
    diag_logdet<R>(T, D, unit, logdet);
    return;
  }
  const int col0 = (blockIdx.x * kInvWarps + (threadIdx.x >> 5)) * kInvC;
  if (col0 >= D) return;
  auto in_tri = [&](int i, int j) { return upper ? i <= j : i >= j; };
  double z[R][kInvC];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int i = lane + 32 * r;
#pragma unroll
    for (int c = 0; c < kInvC; ++c) {
      const int j = col0 + c;
      double v = 0.0;
      if (i < D && j < D && in_tri(i, j)) {
        if (i == j) v = (unit || inv) ? 1.0 : (double)T[(size_t)j * D + i];
        else if (!inv) v = (double)T[(size_t)j * D + i];
      }
      z[r][c] = v;
    }
  }
  if (inv && !upper) {  // forward substitution from the warp's first column down
#pragma unroll
    for (int kb = 0; kb < R; ++kb) {
      for (int jj = 0; jj < 32; ++jj) {
        const int k = kb * 32 + jj;
        if (k >= D) break;
        if (k < col0) continue;
        const float* Tk = T + (size_t)k * D;
        const double tkk = unit ? 1.0 : (double)Tk[k];
        double v[kInvC];
#pragma unroll
        for (int c = 0; c < kInvC; ++c) {
          v[c] = __shfl_sync(kFull, z[kb][c], jj) / tkk;
          if (lane == jj) z[kb][c] = v[c];
        }
#pragma unroll
        for (int r = kb; r < R; ++r) {
          const int i = lane + 32 * r;
          if (i > k && i < D) {
            const double l = (double)Tk[i];
#pragma unroll
            for (int c = 0; c < kInvC; ++c) z[r][c] = fma(-l, v[c], z[r][c]);
          }
        }
      }
    }
  } else if (inv) {  // back substitution from the warp's last column up
    const int klast = col0 + kInvC - 1;
#pragma unroll
    for (int kb = R - 1; kb >= 0; --kb) {
      for (int jj = 31; jj >= 0; --jj) {
        const int k = kb * 32 + jj;
        if (k >= D || k > klast) continue;
        const float* Tk = T + (size_t)k * D;
        const double tkk = unit ? 1.0 : (double)Tk[k];
        double v[kInvC];
#pragma unroll
        for (int c = 0; c < kInvC; ++c) {
          v[c] = __shfl_sync(kFull, z[kb][c], jj) / tkk;
          if (lane == jj) z[kb][c] = v[c];
        }
#pragma unroll
        for (int r = 0; r <= kb; ++r) {
          const int i = lane + 32 * r;
          if (i < k) {
            const double u = (double)Tk[i];
#pragma unroll
            for (int c = 0; c < kInvC; ++c) z[r][c] = fma(-u, v[c], z[r][c]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < kInvC; ++c) {
    const int j = col0 + c;
    if (j >= D) break;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int i = lane + 32 * r;
      if (i < D) M[(size_t)j * D + i] = (float)z[r][c];
    }
  }
}

// M = P·L·U (inv == 0) or U⁻¹ L⁻¹ Pᵀ of an LU layer, fp32: F packs L (strictly below the diagonal, unit diagonal implied)
// and U (on and above it); y[dst[r]] = (L U x)[r], dst == NULL the identity.  Forward column j: u = U e_j, then L u
// right-looking from the last row up (step k adds L(i, k)·u_k to the rows below k while u_k is still U's), scattered to
// the rows dst[·].  Inverse column j: Pᵀ e_j (the 1 in the row r with dst[r] = j) solved against L and U as inv_kernel does.
// Each entry is computed in fp64 and rounded once.  The last CTA writes log|det U| = Σ log|Uᵢᵢ| in row order.
template <int R>
__global__ void __launch_bounds__(kInvWarps * 32)
    lu_prep_kernel(const float* __restrict__ F, const int* __restrict__ dst, int D, int inv, float* __restrict__ M,
                   double* __restrict__ logdet) {
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == gridDim.x - 1) {
    diag_logdet<R>(F, D, 0, logdet);
    return;
  }
  const int col0 = (blockIdx.x * kInvWarps + (threadIdx.x >> 5)) * kInvC;
  if (col0 >= D) return;
  double z[R][kInvC];
  int row[R];  // where row i of the warp's result goes: i (inverse) or dst[i] (forward)
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int i = lane + 32 * r;
    const int pi = i < D ? (dst ? dst[i] : i) : -1;
    row[r] = inv ? i : pi;
#pragma unroll
    for (int c = 0; c < kInvC; ++c) {
      const int j = col0 + c;
      z[r][c] = inv ? (pi == j ? 1.0 : 0.0) : (i < D && j < D && i <= j ? (double)F[(size_t)j * D + i] : 0.0);
    }
  }
  if (inv) {
    lu_solve_cols<R>(z, F, D, lane);
  } else {
    const int klast = col0 + kInvC - 1;  // u_k = 0 beyond the warp's last column
#pragma unroll
    for (int kb = R - 1; kb >= 0; --kb) {
      for (int jj = 31; jj >= 0; --jj) {
        const int k = kb * 32 + jj;
        if (k >= D || k > klast) continue;
        const float* Lk = F + (size_t)k * D;
        double v[kInvC];
#pragma unroll
        for (int c = 0; c < kInvC; ++c) v[c] = __shfl_sync(kFull, z[kb][c], jj);
#pragma unroll
        for (int r = kb; r < R; ++r) {
          const int i = lane + 32 * r;
          if (i > k && i < D) {
            const double l = (double)Lk[i];
#pragma unroll
            for (int c = 0; c < kInvC; ++c) z[r][c] = fma(l, v[c], z[r][c]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < kInvC; ++c) {
    const int j = col0 + c;
    if (j >= D) break;
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (lane + 32 * r < D) M[(size_t)j * D + row[r]] = (float)z[r][c];
  }
}

template <int DP, int BN>
__host__ __device__ constexpr int map_threads() {
  return (DP / 8) * (BN / 8);
}
template <int DP, int BN>
constexpr size_t map_smem() {
  return sizeof(float) * ((size_t)DP * (BN + 4) + 2 * (size_t)kBK * DP);
}

// acc[u][v] += a[u]·b[v] over one k-block for the rows u in [U0, U1) of a thread of the triangular map: rows u < 4 from
// the low block (first row r0), u >= 4 from the high block (r1)
template <int U0, int U1, int DP, int BN>
__device__ __forceinline__ void map_block(float (&acc)[8][8], const float* Mb, const float* Xb, int r0, int r1, int tx) {
  constexpr int XS = BN + 4;
#pragma unroll
  for (int kk = 0; kk < kBK; ++kk) {
    float a[8];
    if (U0 == 0) {
      const float4 a0 = *reinterpret_cast<const float4*>(Mb + kk * DP + r0);
      a[0] = a0.x, a[1] = a0.y, a[2] = a0.z, a[3] = a0.w;
    }
    if (U1 == 8) {
      const float4 a1 = *reinterpret_cast<const float4*>(Mb + kk * DP + r1);
      a[4] = a1.x, a[5] = a1.y, a[6] = a1.z, a[7] = a1.w;
    }
    const float4 b0 = *reinterpret_cast<const float4*>(Xb + kk * XS + tx * 4);
    const float4 b1 = *reinterpret_cast<const float4*>(Xb + kk * XS + BN / 2 + tx * 4);
    const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int u = U0; u < U1; ++u)
#pragma unroll
      for (int v = 0; v < 8; ++v) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
  }
}

// Y = op(M) X with op(M) = M (TRANS = false) or Mᵀ; logjac[n] = lj (+ logjac[n]) when logjac != NULL.  TRI = 0: dense M;
// TRI = 1 / 2: op(M) is lower / upper triangular, and row i reads k <= i / k >= i only.  Then warp w owns the low row
// block [w·H, (w+1)·H) and the high block [DP − (w+1)·H, DP − w·H), H = DP / (2·warps), so every warp has the same share
// of the triangle, and a block is skipped on the k-blocks that are zero for all its rows.  A skipped k-block would only
// add ±0 products to each chain, so the results are those of the dense map on the same M.
template <int DP, int BN, bool TRANS, int TRI = 0>
__global__ void __launch_bounds__(map_threads<DP, BN>(), 1)
    map_kernel(const float* __restrict__ M, const float* x, long long ldx, float* y, long long ldy, float* logjac,
               int accumulate, const double* __restrict__ logdet, float lj_sign, int D, long long N) {
  constexpr int T = map_threads<DP, BN>(), XS = BN + 4, PER = DP * kBK / T;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* Xs = reinterpret_cast<float*>(smem_raw);  // Xs[k * XS + n]
  float* Ms = Xs + (size_t)DP * XS;                // Ms[buf][kk * DP + i] = op(M)(i, k0 + kk)
  constexpr int H = DP / (2 * (T / 32));  // rows of a warp's block (TRI)
  static_assert(TRI == 0 || H == 4 * (32 / (BN / 8)), "a warp's row block is its thread groups' 4 rows each");
  const int tid = threadIdx.x, ty = TRI ? tid % 32 / (BN / 8) : tid % (DP / 8), tx = TRI ? tid % (BN / 8) : tid / (DP / 8);
  const int lo_base = TRI ? tid / 32 * H : 0, hi_base = TRI ? DP - (tid / 32 + 1) * H : 0;  // the warp's row blocks
  const long long n0 = (long long)blockIdx.x * BN;
  const int Kp = (D + kBK - 1) / kBK * kBK, KB = Kp / kBK;
  float pre[PER];
  auto fetch = [&](int kb) {
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int idx = tid + e * T;
      int i, kk;
      if (TRANS) {
        kk = idx % kBK;
        i = idx / kBK;
      } else {
        i = idx % DP;
        kk = idx / DP;
      }
      const int k = kb * kBK + kk;
      float v = 0.f;
      if (i < D && k < D) v = TRANS ? __ldg(M + (size_t)i * D + k) : __ldg(M + (size_t)k * D + i);
      pre[e] = v;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int idx = tid + e * T;
      const int i = TRANS ? idx / kBK : idx % DP, kk = TRANS ? idx % kBK : idx / DP;
      Ms[buf * kBK * DP + kk * DP + i] = pre[e];
    }
  };
  fetch(0);
  // the whole x tile is read before any y of it is written (y may alias x)
  for (int idx = tid; idx < BN * Kp; idx += T) {
    const int n = idx / Kp, k = idx - n * Kp;
    const long long col = n0 + n;
    Xs[k * XS + n] = (col < N && k < D) ? x[col * ldx + k] : 0.f;
  }
  stash(0);
  __syncthreads();
  float acc[8][8];
#pragma unroll
  for (int u = 0; u < 8; ++u)
#pragma unroll
    for (int v = 0; v < 8; ++v) acc[u][v] = 0.f;
  for (int kb = 0; kb < KB; ++kb) {
    if (kb + 1 < KB) fetch(kb + 1);
    const float* Mb = Ms + (kb & 1) * kBK * DP;
    const float* Xb = Xs + (size_t)kb * kBK * XS;
    if constexpr (TRI == 0) {
#pragma unroll
      for (int kk = 0; kk < kBK; ++kk) {
        const float4 a0 = *reinterpret_cast<const float4*>(Mb + kk * DP + ty * 4);
        const float4 a1 = *reinterpret_cast<const float4*>(Mb + kk * DP + DP / 2 + ty * 4);
        const float4 b0 = *reinterpret_cast<const float4*>(Xb + kk * XS + tx * 4);
        const float4 b1 = *reinterpret_cast<const float4*>(Xb + kk * XS + BN / 2 + tx * 4);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int u = 0; u < 8; ++u)
#pragma unroll
          for (int v = 0; v < 8; ++v) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
      }
    } else {  // warp-uniform: whether each row block meets a non-zero of this k-block
      const int k0 = kb * kBK, k1 = k0 + kBK - 1;
      const bool lo = lo_base < D && (TRI == 1 ? k0 <= lo_base + H - 1 : k1 >= lo_base);
      const bool hi = hi_base < D && (TRI == 1 ? k0 <= hi_base + H - 1 : k1 >= hi_base);
      const int r0 = lo_base + ty * 4, r1 = hi_base + ty * 4;
      if (lo && hi) map_block<0, 8, DP, BN>(acc, Mb, Xb, r0, r1, tx);
      else if (lo) map_block<0, 4, DP, BN>(acc, Mb, Xb, r0, r1, tx);
      else if (hi) map_block<4, 8, DP, BN>(acc, Mb, Xb, r0, r1, tx);
    }
    if (kb + 1 < KB) stash((kb + 1) & 1);
    __syncthreads();
  }
#pragma unroll
  for (int v = 0; v < 8; ++v) {
    const long long col = n0 + (v < 4 ? tx * 4 + v : BN / 2 + tx * 4 + v - 4);
    if (col >= N) continue;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = TRI ? (u < 4 ? lo_base : hi_base) + ty * 4 + (u & 3) : (u < 4 ? ty * 4 + u : DP / 2 + ty * 4 + u - 4);
      if (i < D) y[col * ldy + i] = acc[u][v];
    }
  }
  if (logjac) {
    const float lj = (float)(lj_sign * *logdet);
    for (int c = tid; c < BN && n0 + c < N; c += T) {
      const long long col = n0 + c;
      logjac[col] = accumulate ? logjac[col] + lj : lj;
    }
  }
}

// logjac only (y == NULL)
__global__ void logjac_kernel(float* __restrict__ logjac, int accumulate, const double* __restrict__ logdet,
                              float lj_sign, long long N) {
  const float lj = (float)(lj_sign * *logdet);
  for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (long long)gridDim.x * blockDim.x)
    logjac[n] = accumulate ? logjac[n] + lj : lj;
}

// Σₙ l̄ₙ in fp64: strided per-thread sums, then a fixed tree over the block
__global__ void __launch_bounds__(1024) ljsum_kernel(const float* __restrict__ ljbar, long long N, double* __restrict__ out) {
  __shared__ double red[1024];
  double s = 0.0;
  if (ljbar)
    for (long long n = threadIdx.x; n < N; n += 1024) s += (double)ljbar[n];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = red[0];
}

// Output masks of the finalize kernels: kMaskFull (the dense layer) or kMaskTri | upper·kMaskUpper | unit·kMaskStrict, the
// triangle 𝒫 of a triangular T's parameters (strict for a unit diagonal).
constexpr int kMaskFull = 0, kMaskTri = 1, kMaskUpper = 2, kMaskStrict = 4;

__device__ __forceinline__ bool in_mask(int mask, int i, int j) {
  if (mask == kMaskFull) return true;
  if (mask & kMaskUpper) return (mask & kMaskStrict) ? i < j : i <= j;
  return (mask & kMaskStrict) ? i > j : i >= j;
}

// forward layer: Ā = Σ_p part[p] + s·B;  inverse layer: Gd = Σ_p part[p] (fp64).  B(i, j) = A⁻¹(j, i) = minv[i·D + j].
// Triangular forward layer (mask != kMaskFull): T̄ = 𝒫(Σ_p part[p] + s·B), 0 elsewhere, with minv = T, so B's diagonal is
// 1/Tᵢᵢ and 𝒫 keeps nothing else of it; for an upper T the chunks hold Gᵀ and are read transposed.
__global__ void __launch_bounds__(256) gsum_kernel(const float* __restrict__ part, int P, const double* __restrict__ ljs,
                                                   const float* __restrict__ minv, int D, int mask, float* __restrict__ Abar,
                                                   double* __restrict__ Gd) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x, DD = (long long)D * D;
  if (idx >= DD) return;
  const int j = (int)(idx / D), i = (int)(idx - (long long)j * D);
  if (!Gd && !in_mask(mask, i, j)) {
    Abar[idx] = 0.f;
    return;
  }
  const long long src = (!Gd && (mask & kMaskUpper)) ? (long long)i * D + j : idx;
  double a = 0.0;
  for (int p = 0; p < P; ++p) a += (double)part[(size_t)p * DD + src];
  if (Gd) {
    Gd[idx] = a;
    return;
  }
  if (mask == kMaskFull) Abar[idx] = (float)(a + *ljs * (double)minv[(size_t)i * D + j]);
  else Abar[idx] = (float)(i == j && !(mask & kMaskStrict) ? a + *ljs / (double)minv[(size_t)i * D + i] : a);
}

// T = Gd · B (fp64, column-major).  With a triangular mask only the triangle the final product reads (𝒫 with its diagonal),
// zeros elsewhere.
__global__ void __launch_bounds__(256) prod_gb_kernel(const double* __restrict__ Gd, const float* __restrict__ minv, int D,
                                                      int mask, double* __restrict__ Tm) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)D * D) return;
  const int j = (int)(idx / D), i = (int)(idx - (long long)j * D);
  if (!in_mask(mask & ~kMaskStrict, i, j)) {
    Tm[idx] = 0.0;
    return;
  }
  double a = 0.0;
  for (int k = 0; k < D; ++k) a = fma(Gd[(size_t)k * D + i], (double)minv[(size_t)k * D + j], a);
  Tm[idx] = a;
}

// inverse layer: Ā = −B · T − s·B, on the mask (0 elsewhere).  With Ad != NULL (the LU layer): Ad = −B · T in fp64, in
// full and without the s·B term, for lu_bar_kernel.
__global__ void __launch_bounds__(256) final_inv_kernel(const double* __restrict__ Tm, const float* __restrict__ minv,
                                                        const double* __restrict__ ljs, int D, int mask,
                                                        float* __restrict__ Abar, double* __restrict__ Ad) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)D * D) return;
  const int j = (int)(idx / D), i = (int)(idx - (long long)j * D);
  if (!Ad && !in_mask(mask, i, j)) {
    Abar[idx] = 0.f;
    return;
  }
  double a = 0.0;
  for (int k = 0; k < D; ++k) a = fma((double)minv[(size_t)i * D + k], Tm[(size_t)j * D + k], a);
  if (Ad) {
    Ad[idx] = -a;
    return;
  }
  Abar[idx] = (float)(-a - *ljs * (double)minv[(size_t)i * D + j]);
}

// LU layer: F̄ from M̄ (fp64, column-major: G for the forward layer, −M⁻ᵀ G M⁻ᵀ for the inverse one) through M = P L U:
//   F̄(i, j) = (Pᵀ M̄ Uᵀ)(i, j) = Σ_{k≥j} M̄(dst[i], k)·U(j, k)                          i > j   (L̄)
//   F̄(i, j) = (Lᵀ Pᵀ M̄)(i, j) = M̄(dst[i], j) + Σ_{k>i} L(k, i)·M̄(dst[k], j) + sg·s/Uᵢᵢ   i ≤ j   (Ū, s/Uᵢᵢ on i = j)
// with sg = +1 for the forward layer and −1 for the inverse one, k increasing, one thread per entry.
__global__ void __launch_bounds__(256) lu_bar_kernel(const double* __restrict__ Mb, const float* __restrict__ F,
                                                     const int* __restrict__ dst, const double* __restrict__ ljs,
                                                     double sg, int D, float* __restrict__ Fbar) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)D * D) return;
  const int j = (int)(idx / D), i = (int)(idx - (long long)j * D);
  auto prow = [&](int r) { return dst ? dst[r] : r; };
  double a = 0.0;
  if (i > j) {
    const int pi = prow(i);
    for (int k = j; k < D; ++k) a = fma(Mb[(size_t)k * D + pi], (double)F[(size_t)k * D + j], a);
  } else {
    a = Mb[(size_t)j * D + prow(i)];
    for (int k = i + 1; k < D; ++k) a = fma((double)F[(size_t)i * D + k], Mb[(size_t)j * D + prow(k)], a);
    if (i == j) a += sg * *ljs / (double)F[(size_t)i * D + i];
  }
  Fbar[idx] = (float)a;
}

int launch_factor(const b2b_layer_desc& d, const Factor& f, int D, bool want_inverse, int* launches, cudaStream_t stream) {
  const size_t smem = factor_smem(D);
  cudaError_t e = cudaFuncSetAttribute(factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  factor_kernel<<<1, kFactorThreads, smem, stream>>>(d.p0, D, f.lu, f.perm, f.logdet);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*launches;
  if (!want_inverse) return B2B_OK;
  const int grid = (D + kInvWarps * kInvC - 1) / (kInvWarps * kInvC);
  if (D <= 32) inv_kernel<1><<<grid, kInvWarps * 32, 0, stream>>>(f.lu, f.perm, f.minv, D);
  else if (D <= 64) inv_kernel<2><<<grid, kInvWarps * 32, 0, stream>>>(f.lu, f.perm, f.minv, D);
  else if (D <= 128) inv_kernel<4><<<grid, kInvWarps * 32, 0, stream>>>(f.lu, f.perm, f.minv, D);
  else inv_kernel<8><<<grid, kInvWarps * 32, 0, stream>>>(f.lu, f.perm, f.minv, D);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*launches;
  return B2B_OK;
}

// M = P·L·U or U⁻¹ L⁻¹ Pᵀ and log|det U| of an LU layer, one launch
int launch_lu_prep(const b2b_layer_desc& d, const TriFactor& f, int D, int* launches, cudaStream_t stream) {
  const int grid = (D + kInvWarps * kInvC - 1) / (kInvWarps * kInvC) + 1;  // + the log|det U| CTA
  const int inv = d.inverse != 0;
  if (D <= 32) lu_prep_kernel<1><<<grid, kInvWarps * 32, 0, stream>>>(d.p0, d.i0, D, inv, f.m, f.logdet);
  else if (D <= 64) lu_prep_kernel<2><<<grid, kInvWarps * 32, 0, stream>>>(d.p0, d.i0, D, inv, f.m, f.logdet);
  else if (D <= 128) lu_prep_kernel<4><<<grid, kInvWarps * 32, 0, stream>>>(d.p0, d.i0, D, inv, f.m, f.logdet);
  else lu_prep_kernel<8><<<grid, kInvWarps * 32, 0, stream>>>(d.p0, d.i0, D, inv, f.m, f.logdet);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  ++*launches;
  return B2B_OK;
}

// M = T or T⁻¹ and log|det T| of a triangular layer, one launch
int launch_tri_prep(const b2b_layer_desc& d, const TriFactor& f, int D, int* launches, cudaStream_t stream) {
  const int grid = (D + kInvWarps * kInvC - 1) / (kInvWarps * kInvC) + 1;  // + the log|det T| CTA
  const int up = d.n0, unit = d.n1, inv = d.inverse != 0;
  if (D <= 32) tri_prep_kernel<1><<<grid, kInvWarps * 32, 0, stream>>>(d.p0, D, up, unit, inv, f.m, f.logdet);
  else if (D <= 64) tri_prep_kernel<2><<<grid, kInvWarps * 32, 0, stream>>>(d.p0, D, up, unit, inv, f.m, f.logdet);
  else if (D <= 128) tri_prep_kernel<4><<<grid, kInvWarps * 32, 0, stream>>>(d.p0, D, up, unit, inv, f.m, f.logdet);
  else tri_prep_kernel<8><<<grid, kInvWarps * 32, 0, stream>>>(d.p0, D, up, unit, inv, f.m, f.logdet);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  ++*launches;
  return B2B_OK;
}

template <int DP, int BN, bool TRANS, int TRI>
int launch_map_t(const float* M, const float* x, long long ldx, float* y, long long ldy, float* logjac, int accumulate,
                 const double* logdet, float sign, int D, long long N, cudaStream_t stream) {
  constexpr size_t smem = map_smem<DP, BN>();
  auto k = map_kernel<DP, BN, TRANS, TRI>;
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const long long grid = (N + BN - 1) / BN;
  k<<<(unsigned)grid, map_threads<DP, BN>(), smem, stream>>>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N);
  return (int)cudaGetLastError();
}

template <bool TRANS, int TRI>
int launch_map_d(const float* M, const float* x, long long ldx, float* y, long long ldy, float* logjac, int accumulate,
                 const double* logdet, float sign, int D, long long N, cudaStream_t stream) {
  if (D <= 32) return launch_map_t<32, 128, TRANS, TRI>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
  if (D <= 64) return launch_map_t<64, 128, TRANS, TRI>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
  if (D <= 128) return launch_map_t<128, 128, TRANS, TRI>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
  return launch_map_t<256, 64, TRANS, TRI>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
}

// Y = op(M) X with op(M) = M or (TRANS) Mᵀ, where M is dense (tri = 0) or lower / upper triangular (tri = 1 / 2)
template <bool TRANS>
int launch_map(int tri, const float* M, const float* x, long long ldx, float* y, long long ldy, float* logjac,
               int accumulate, const double* logdet, float sign, int D, long long N, cudaStream_t stream) {
  if (tri == 0) return launch_map_d<TRANS, 0>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
  if ((tri == 1) != TRANS) return launch_map_d<TRANS, 1>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
  return launch_map_d<TRANS, 2>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
}

// What the launches after the prep need, for any kind: the map operand M (A, A⁻¹, T, T⁻¹, P·L·U or U⁻¹ L⁻¹ Pᵀ), the
// B = M⁻ᵀ source of the finalize kernels, log|det|, the structure of M for the map, the output mask of the cotangent, and
// whether the cotangent goes through the LU factors (lu_bar_kernel).
struct ScaleOp {
  const float* M;
  const float* minv;
  double* logdet;
  int tri;   // 0 dense, 1 lower, 2 upper
  int mask;  // kMaskFull or the triangle 𝒫
  bool lu;
};

size_t prep_bytes(int kind, int D) { return kind == B2B_SCALE_MATRIX ? factor_bytes(D) : tri_bytes(D); }

// The prep launches of the layer `d` (the descriptor's kind decides them here, and nowhere else): the dense layer's LU, and
// A⁻¹ when `want_inverse`; the triangular layer's M (always: its map must not read the entries outside the triangle); the
// LU layer's M (always: the map needs the product of the factors).  For the inverse LU layer M = (P L U)⁻¹ is also the
// B = M⁻ᵀ source (minv) of final_inv_kernel.
int scale_prep(const b2b_layer_desc& d, void* ws, int D, bool want_inverse, ScaleOp* op, int* launches,
               cudaStream_t stream) {
  const bool inv = d.inverse != 0;
  if (d.kind == B2B_SCALE_TRIANGULAR) {
    const TriFactor f = carve_tri(ws, D);
    *op = ScaleOp{f.m, f.m, f.logdet, d.n0 ? 2 : 1, kMaskTri | (d.n0 ? kMaskUpper : 0) | (d.n1 ? kMaskStrict : 0), false};
    return launch_tri_prep(d, f, D, launches, stream);
  }
  if (d.kind == B2B_SCALE_LU) {
    const TriFactor f = carve_tri(ws, D);
    *op = ScaleOp{f.m, f.m, f.logdet, 0, kMaskFull, true};
    return launch_lu_prep(d, f, D, launches, stream);
  }
  const Factor f = carve(ws, D);
  *op = ScaleOp{inv ? f.minv : d.p0, f.minv, f.logdet, 0, kMaskFull, false};
  return launch_factor(d, f, D, want_inverse, launches, stream);
}

}  // namespace b2b_scale

using namespace b2b_scale;

size_t b2b_scale_workspace(int kind, int D) { return D >= 1 && D <= B2B_SCALE_MATRIX_MAX_D ? prep_bytes(kind, D) : 0; }

int b2b_fwd_scale(const B2BFwdSeg& s) {
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  if (D < 1 || D > B2B_SCALE_MATRIX_MAX_D) return B2B_EUNSUPPORTED;  // = B2B_SCALE_TRIANGULAR_MAX_D = B2B_SCALE_LU_MAX_D
  if (!s.workspace || s.workspace_bytes < prep_bytes(d.kind, D)) return B2B_EWORKSPACE;
  const bool inv = d.inverse != 0;
  ScaleOp op;
  int rc = scale_prep(d, s.workspace, D, inv && s.y, &op, s.launches, s.stream);
  if (rc != B2B_OK) return rc;
  const float sign = inv ? -1.f : 1.f;
  if (!s.y) {  // log-Jacobians only
    if (!s.logjac) return B2B_OK;
    long long g = (s.N + 255) / 256;
    logjac_kernel<<<(unsigned)(g < 1024 ? g : 1024), 256, 0, s.stream>>>(s.logjac, s.accumulate, op.logdet, sign, s.N);
    if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
    ++*s.launches;
    return B2B_OK;
  }
  rc = launch_map<false>(op.tri, op.M, s.x, s.ldx, s.y, s.ldy, s.logjac, s.accumulate, op.logdet, sign, D, s.N, s.stream);
  if (rc != B2B_OK) return rc;
  ++*s.launches;
  return B2B_OK;
}

// workspace: [factor storage][chunk partials of G (P x D x D fp32)][Gd, T (D x D fp64 each)][Σ l̄ (fp64)]
size_t b2b_scale_vjp_workspace(int kind, int D, long long N) {
  if (D < 1 || D > B2B_SCALE_MATRIX_MAX_D || N < 0) return 0;
  const long long clen = b2b_outer_chunk_len(N), P = N > 0 ? (N + clen - 1) / clen : 1;
  return prep_bytes(kind, D) + al256(sizeof(float) * (size_t)P * D * D) + 2 * al256(sizeof(double) * (size_t)D * D) +
         al256(sizeof(double));
}

int b2b_vjp_scale(const B2BVjpSeg& s) {
  const b2b_layer_desc& d = s.layers[0];
  const float *x = s.x, *ybar = s.ybar, *ljbar = s.ljbar;
  const long long ldx = s.ldx, ldyb = s.ldyb, ldxb = s.ldxb, N = s.N;
  float* const xbar = s.xbar;
  float* const Abar = s.bars[0];
  void* const workspace = s.workspace;
  const int D = s.D;
  int* const launches = s.launches;
  const cudaStream_t stream = s.stream;
  if (D < 1 || D > B2B_SCALE_MATRIX_MAX_D) return B2B_EUNSUPPORTED;
  if (!workspace || s.workspace_bytes < b2b_scale_vjp_workspace(d.kind, D, N)) return B2B_EWORKSPACE;
  const bool inv = d.inverse != 0, tri = d.kind == B2B_SCALE_TRIANGULAR, lu = d.kind == B2B_SCALE_LU;
  char* ws = static_cast<char*>(workspace) + prep_bytes(d.kind, D);
  const long long clen = b2b_outer_chunk_len(N), P = (N + clen - 1) / clen;
  float* part = reinterpret_cast<float*>(ws);
  ws += al256(sizeof(float) * (size_t)P * D * D);
  double* Gd = reinterpret_cast<double*>(ws);
  ws += al256(sizeof(double) * (size_t)D * D);
  double* Tm = reinterpret_cast<double*>(ws);
  ws += al256(sizeof(double) * (size_t)D * D);
  double* ljs = reinterpret_cast<double*>(ws);
  int rc = B2B_OK;
  ScaleOp op{};
  if (tri || lu || inv || Abar) {
    rc = scale_prep(d, workspace, D, true, &op, launches, stream);
    if (rc != B2B_OK) return rc;
  } else {
    op.M = d.p0;  // the dense forward layer's x̄ needs A only
  }
  // x̄ = op(M)ᵀ ȳ
  if (ybar) {
    rc = launch_map<true>(op.tri, op.M, ybar, ldyb, xbar, ldxb, nullptr, 0, nullptr, 0.f, D, N, stream);
    if (rc != B2B_OK) return rc;
  } else {
    rc = (int)cudaMemset2DAsync(xbar, (size_t)ldxb * sizeof(float), 0, (size_t)D * sizeof(float), (size_t)N, stream);
    if (rc != cudaSuccess) return rc;
  }
  ++*launches;
  if (!Abar) return B2B_OK;
  if (ybar) {
    if (tri && !inv)  // G on 𝒫 only: the lower tiles of G, or of Gᵀ (operands swapped) for an upper T
      rc = d.n0 ? b2b_launch_outer_chunks(x, ldx, ybar, ldyb, part, nullptr, D, N, true, stream)
                : b2b_launch_outer_chunks(ybar, ldyb, x, ldx, part, nullptr, D, N, true, stream);
    else
      rc = b2b_launch_outer_chunks(ybar, ldyb, x, ldx, part, nullptr, D, N, false, stream);
    if (rc != B2B_OK) return rc;
    ++*launches;
  }
  ljsum_kernel<<<1, 1024, 0, stream>>>(ljbar, N, ljs);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  ++*launches;
  const long long DD = (long long)D * D;
  const unsigned g = (unsigned)((DD + 255) / 256);
  gsum_kernel<<<g, 256, 0, stream>>>(part, ybar ? (int)P : 0, ljs, op.minv, D, op.mask, Abar, inv || lu ? Gd : nullptr);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  ++*launches;
  if (inv) {  // the LU layer's M̄ = −B G B goes back to Gd (prod_gb_kernel has read it)
    prod_gb_kernel<<<g, 256, 0, stream>>>(Gd, op.minv, D, op.mask, Tm);
    if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
    final_inv_kernel<<<g, 256, 0, stream>>>(Tm, op.minv, ljs, D, op.mask, Abar, lu ? Gd : nullptr);
    if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
    *launches += 2;
  }
  if (!lu) return B2B_OK;
  lu_bar_kernel<<<g, 256, 0, stream>>>(Gd, d.p0, d.i0, ljs, inv ? -1.0 : 1.0, D, Abar);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  ++*launches;
  return B2B_OK;
}
