// kge_tiles.cu -- fp32 CUDA-core tile kernels for the chunked negative contraction
// (engine 0; the wgmma engine in kge_umma.cu replaces the bilinear cases).
//
//   k_score  : S[c,i,j] = pair(a_i, b_j)                  create_neg fns, score_fun.py:26-38,91-108,
//                                                         268-286,345-376,427-449,512-554
//   k_grad<A>: GA[i,:]  = sum_j V_ij * dpair/da            autograd of the above (loss.backward())
//   k_grad<B>: G_neg[j,:] = sum_i V_ij * dpair/db (+reg)   written in place over the gathered rows
//
// Tiling: 64x64 outputs per CTA, 256 threads, 4x4 register micro-tile, 16-deep smem slabs stored
// transposed ([k][row]) so the inner loop reads two conflict-free float4 per 16 FMAs.
#include "kge_common.cuh"

namespace kge {


enum { OP_DOT = 0, OP_L1 = 1, OP_ROT = 2 };
constexpr int T = 64;      // tile edge
constexpr int BK = 16;     // slab depth
constexpr int LD = T + 4;  // padded leading dimension (keeps float4 alignment)

__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// column of the q-th float4 of a slab starting at k0 (OP_ROT: first half of the slab = real parts,
// second half = the matching imaginary parts)
template <int OP, int NQ>   // NQ float4 per row in the slab
__device__ __forceinline__ int slab_col(int k0, int q, int D, bool& valid) {
  if (OP == OP_ROT) {
    const int half = D >> 1, hq = NQ / 2;
    int within = k0 + (q % hq) * 4;
    valid = within < half;
    return (q < hq) ? within : half + within;
  }
  int col = k0 + q * 4;
  valid = col < D;
  return col;
}

// ------------------------------------------------------------------------------------------
template <int OP>
__global__ void __launch_bounds__(256) k_score(StepParams p, const float* __restrict__ A, const float* __restrict__ Bn,
                                               const float* __restrict__ a2, const float* __restrict__ b2,
                                               float* __restrict__ S, float* __restrict__ Vdist) {
  __shared__ __align__(16) float As[BK][LD];
  __shared__ __align__(16) float Bs[BK][LD];
  const int c = blockIdx.z, i0 = blockIdx.y * T, j0 = blockIdx.x * T;
  const int D = p.D;
  const float* Ac = A + ((long long)c * p.Cs) * D;
  const float* Bc = Bn + ((long long)c * p.Ns) * D;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int lr = threadIdx.x >> 2, lq = threadIdx.x & 3;
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;

  const int kend = (OP == OP_ROT) ? (D >> 1) : D;
  const int kstep = (OP == OP_ROT) ? BK / 2 : BK;
  for (int k0 = 0; k0 < kend; k0 += kstep) {
    bool valid;
    int col = slab_col<OP, 4>(k0, lq, D, valid);
    float4 av = (valid && i0 + lr < p.Cs) ? ld4(Ac + (long long)(i0 + lr) * D + col) : zero4();
    float4 bv = (valid && j0 + lr < p.Ns) ? ld4(Bc + (long long)(j0 + lr) * D + col) : zero4();
    As[lq * 4 + 0][lr] = av.x; As[lq * 4 + 1][lr] = av.y; As[lq * 4 + 2][lr] = av.z; As[lq * 4 + 3][lr] = av.w;
    Bs[lq * 4 + 0][lr] = bv.x; Bs[lq * 4 + 1][lr] = bv.y; Bs[lq * 4 + 2][lr] = bv.z; Bs[lq * 4 + 3][lr] = bv.w;
    __syncthreads();
    if (OP == OP_ROT) {
#pragma unroll
      for (int kk = 0; kk < BK / 2; ++kk) {
        float4 ar = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        float4 ai = *reinterpret_cast<const float4*>(&As[kk + BK / 2][ty * 4]);
        float4 br = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        float4 bi = *reinterpret_cast<const float4*>(&Bs[kk + BK / 2][tx * 4]);
        const float arr[4] = {ar.x, ar.y, ar.z, ar.w}, aii[4] = {ai.x, ai.y, ai.z, ai.w};
        const float brr[4] = {br.x, br.y, br.z, br.w}, bii[4] = {bi.x, bi.y, bi.z, bi.w};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float dre = arr[r] - brr[q], dim = aii[r] - bii[q];
            acc[r][q] += sqrtf(fmaf(dre, dre, dim * dim));
          }
      }
    } else {
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        const float aa[4] = {a4.x, a4.y, a4.z, a4.w}, bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (OP == OP_DOT) acc[r][q] = fmaf(aa[r], bb[q], acc[r][q]);
            else acc[r][q] += fabsf(aa[r] - bb[q]);
          }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + ty * 4 + r;
    if (i >= p.Cs) continue;
    const long long gi = (long long)c * p.Cs + i;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + tx * 4 + q;
      if (j >= p.Ns) continue;
      float s;
      if (p.model == KGE_TRANSE_L2) {
        // batched_l2_dist (score_fun.py:26-34): (|b|^2 - 2 a.b) + |a|^2, clamp 1e-30, sqrt
        float sq = fmaf(-2.f, acc[r][q], b2[(long long)c * p.Ns + j]) + a2[gi];
        float d = sqrtf(fmaxf(sq, 1e-30f));
        Vdist[gi * p.Ns + j] = d;
        s = p.gamma - d;
      } else if (OP == OP_DOT) {
        s = acc[r][q];
      } else {
        s = p.gamma - acc[r][q];
      }
      S[gi * p.Ns + j] = s;
    }
  }
}


// ------------------------------------------------------------------------------------------
// RotatE pair kernels (score_fun.py:512-554).  A complex dimension is one (re, im) float2; Hopper has no packed fp32x2
// arithmetic, so the pair operations below are two scalar FADD / FMUL / FFMA each (same rounding per component), next
// to one MUFU (sqrt / rsqrt) per complex pair per pass.
constexpr int RT = 64;             // tile edge (rows)
constexpr int RKS = 16;            // complex dims per slab (score)
constexpr int RLD = RT + 2;        // float2 per smem row: 528 B, 16-byte aligned, breaks the 4-way store conflict

__device__ __forceinline__ float2 pair_sub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 pair_mul(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 pair_fma(float2 a, float s, float2 c) { return make_float2(fmaf(a.x, s, c.x), fmaf(a.y, s, c.y)); }
__device__ __forceinline__ float sqrt_approx(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

__global__ void __launch_bounds__(256) k_rot_score(StepParams p, const float* __restrict__ A, const float* __restrict__ Bn,
                                                    float* __restrict__ S) {
  __shared__ __align__(16) float2 As[RKS][RLD];
  __shared__ __align__(16) float2 Bs[RKS][RLD];
  const int c = blockIdx.z, i0 = blockIdx.y * RT, j0 = blockIdx.x * RT;
  const int D = p.D, half = D >> 1;
  const float* Ac = A + ((long long)c * p.Cs) * D;
  const float* Bc = Bn + ((long long)c * p.Ns) * D;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int lr = threadIdx.x >> 2, lq = (threadIdx.x & 3) * 4;
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;
  for (int k0 = 0; k0 < half; k0 += RKS) {
    const int k = k0 + lq;
    const bool kv = k < half;                       // half % 4 == 0: a float4 is entirely valid or entirely padding
    float4 are = zero4(), aim = zero4(), bre = zero4(), bim = zero4();
    if (kv && i0 + lr < p.Cs) { are = ld4(Ac + (long long)(i0 + lr) * D + k); aim = ld4(Ac + (long long)(i0 + lr) * D + half + k); }
    if (kv && j0 + lr < p.Ns) { bre = ld4(Bc + (long long)(j0 + lr) * D + k); bim = ld4(Bc + (long long)(j0 + lr) * D + half + k); }
    As[lq + 0][lr] = make_float2(are.x, aim.x); As[lq + 1][lr] = make_float2(are.y, aim.y);
    As[lq + 2][lr] = make_float2(are.z, aim.z); As[lq + 3][lr] = make_float2(are.w, aim.w);
    Bs[lq + 0][lr] = make_float2(bre.x, bim.x); Bs[lq + 1][lr] = make_float2(bre.y, bim.y);
    Bs[lq + 2][lr] = make_float2(bre.z, bim.z); Bs[lq + 3][lr] = make_float2(bre.w, bim.w);
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < RKS; ++kk) {
      float2 a[4], b[4];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      *reinterpret_cast<float4*>(&a[2]) = *reinterpret_cast<const float4*>(&As[kk][ty * 4 + 2]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      *reinterpret_cast<float4*>(&b[2]) = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4 + 2]);
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 d = pair_sub(a[r], b[q]);
          const float2 sq = pair_mul(d, d);
          acc[r][q] += sqrt_approx(sq.x + sq.y);       // one MUFU; ~1e-7 relative on a sum of D/2 terms
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + ty * 4 + r;
    if (i >= p.Cs) continue;
    const long long gi = (long long)c * p.Cs + i;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + tx * 4 + q;
      if (j < p.Ns) S[gi * p.Ns + j] = p.gamma - acc[r][q];
    }
  }
}

// gradient of one side: x = "mine" rows (SIDE_B: negatives j, written in place over Bn with the regulariser; else
// positives i -> GA), y = the other side's rows.  A thread owns 4 x-rows x 4 complex dims and streams all y:
//   g[x, k] = sum_y -V[x,y] (mine - other) / |mine - other|        (complex modulus; d/d mine of gamma - |mine - other|)
template <bool SIDE_B>
__global__ void __launch_bounds__(256, 4) k_rot_grad(StepParams p, const float* __restrict__ V, const float* __restrict__ A,
                                                      float* __restrict__ Bn, float* __restrict__ GA) {
  constexpr int KW = 2;                                  // complex dims per thread (4 x-rows x 2 dims: 32 live float2)
  constexpr int KT = 16 * KW;                            // complex dims per block
  __shared__ __align__(16) float Vs[16][RT + 4];         // [y][x]
  __shared__ __align__(16) float2 Ys[16][KT + 2];        // [y][k]
  const int c = blockIdx.z, x0 = blockIdx.y * RT, k0 = blockIdx.x * KT;     // k0: first complex dim of this block
  const int D = p.D, half = D >> 1;
  const int X = SIDE_B ? p.Ns : p.Cs, Y = SIDE_B ? p.Cs : p.Ns;
  const float* mine = SIDE_B ? (Bn + ((long long)c * p.Ns) * D) : (A + ((long long)c * p.Cs) * D);
  const float* other = SIDE_B ? (A + ((long long)c * p.Cs) * D) : (Bn + ((long long)c * p.Ns) * D);
  const float* Vc = V + ((long long)c * p.Cs) * p.Ns;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int kk0 = k0 + tx * KW;                                      // this thread's complex dims (half % 4 == 0: both or none)
  const bool kok = kk0 < half;
  float2 m[4][KW], acc[4][KW];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int x = x0 + ty * 4 + r;
    float2 re = make_float2(0.f, 0.f), im = re;
    if (kok && x < X) {
      re = *reinterpret_cast<const float2*>(mine + (long long)x * D + kk0);
      im = *reinterpret_cast<const float2*>(mine + (long long)x * D + half + kk0);
    }
    m[r][0] = make_float2(re.x, im.x); m[r][1] = make_float2(re.y, im.y);
    acc[r][0] = make_float2(0.f, 0.f); acc[r][1] = acc[r][0];
  }
  for (int y0 = 0; y0 < Y; y0 += 16) {
    if (SIDE_B) {      // V[y = i][x = j]: rows of V are contiguous in x
      const int yy = threadIdx.x >> 4, xq = (threadIdx.x & 15) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int x = x0 + xq + e, y = y0 + yy;
        Vs[yy][xq + e] = (x < X && y < Y) ? Vc[(long long)y * p.Ns + x] : 0.f;
      }
    } else {           // V[x = i][y = j]
      const int x = threadIdx.x >> 2, yq = (threadIdx.x & 3) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int xx = x0 + x, y = y0 + yq + e;
        Vs[yq + e][x] = (xx < X && y < Y) ? Vc[(long long)xx * p.Ns + y] : 0.f;
      }
    }
    {  // other-rows slab: 16 rows x 32 complex dims, interleaved (re, im): 2 complex dims per thread
      const int yy = threadIdx.x >> 4, q = (threadIdx.x & 15) * 2;
      float2 re = make_float2(0.f, 0.f), im = re;
      if (k0 + q < half && y0 + yy < Y) {
        re = *reinterpret_cast<const float2*>(other + (long long)(y0 + yy) * D + k0 + q);
        im = *reinterpret_cast<const float2*>(other + (long long)(y0 + yy) * D + half + k0 + q);
      }
      *reinterpret_cast<float4*>(&Ys[yy][q]) = make_float4(re.x, im.x, re.y, im.y);
    }
    __syncthreads();
#pragma unroll 8
    for (int yy = 0; yy < 16; ++yy) {
      const float4 v4 = *reinterpret_cast<const float4*>(&Vs[yy][ty * 4]);
      const float vv[4] = {v4.x, v4.y, v4.z, v4.w};
      float2 o[KW];
      *reinterpret_cast<float4*>(&o[0]) = *reinterpret_cast<const float4*>(&Ys[yy][tx * KW]);
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int u = 0; u < KW; ++u) {
          const float2 d = pair_sub(m[r][u], o[u]);
          const float2 sq = pair_mul(d, d);
          // |d| = 0 (identical complex numbers): d itself is 0, so the finite rsqrt of the floor contributes nothing
          const float s = -vv[r] * rsqrtf(fmaxf(sq.x + sq.y, 1e-36f));
          acc[r][u] = pair_fma(d, s, acc[r][u]);
        }
    }
    __syncthreads();
  }
  if (!kok) return;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int x = x0 + ty * 4 + r;
    if (x >= X) continue;
    float2 gre = make_float2(acc[r][0].x, acc[r][1].x), gim = make_float2(acc[r][0].y, acc[r][1].y);
    if (SIDE_B) {
      float* row = Bn + ((long long)c * p.Ns + x) * D;
      gre.x += reg_grad(m[r][0].x, p.reg_norm, p.reg_coef); gre.y += reg_grad(m[r][1].x, p.reg_norm, p.reg_coef);
      gim.x += reg_grad(m[r][0].y, p.reg_norm, p.reg_coef); gim.y += reg_grad(m[r][1].y, p.reg_norm, p.reg_coef);
      *reinterpret_cast<float2*>(row + kk0) = gre;
      *reinterpret_cast<float2*>(row + half + kk0) = gim;
    } else {
      float* row = GA + ((long long)c * p.Cs + x) * D;
      *reinterpret_cast<float2*>(row + kk0) = gre;
      *reinterpret_cast<float2*>(row + half + kk0) = gim;
    }
  }
}

void launch_score(const LaunchCtx& c, const StepParams& p, const StepWs& w) {
  dim3 grid(ceil_div(p.Ns, T), ceil_div(p.Cs, T), p.C);
  if (p.model == KGE_TRANSE_L1) KGE_LAUNCH(c, k_score<OP_L1>, grid, 256, 0, p, w.A, w.Bn, w.a2, w.b2, w.S, w.V);
  else if (p.model == KGE_ROTATE) KGE_LAUNCH(c, k_rot_score, grid, 256, 0, p, w.A, w.Bn, w.S);
  else KGE_LAUNCH(c, k_score<OP_DOT>, grid, 256, 0, p, w.A, w.Bn, w.a2, w.b2, w.S, w.V);
}

// ------------------------------------------------------------------------------------------
// SIDE_A: x = positive i (mine = A rows, other = negative rows)  -> GA
// SIDE_B: x = negative j (mine = negative rows, other = A rows)  -> gradient written over Bn
template <int OP, bool SIDE_B>
__global__ void __launch_bounds__(256) k_grad(StepParams p, const float* __restrict__ V, const float* __restrict__ A,
                                              float* __restrict__ Bn, float* __restrict__ GA,
                                              const float* __restrict__ colsum) {
  __shared__ __align__(16) float Vs[BK][LD];   // [y][x]
  __shared__ __align__(16) float Ys[BK][LD];   // [y][k]
  const int c = blockIdx.z, x0 = blockIdx.y * T;
  const int D = p.D;
  const int k0 = blockIdx.x * ((OP == OP_ROT) ? T / 2 : T);   // first column (OP_ROT: first pair index)
  const int X = SIDE_B ? p.Ns : p.Cs, Y = SIDE_B ? p.Cs : p.Ns;
  const float* mine = SIDE_B ? (Bn + ((long long)c * p.Ns) * D) : (A + ((long long)c * p.Cs) * D);
  const float* other = SIDE_B ? (A + ((long long)c * p.Cs) * D) : (Bn + ((long long)c * p.Ns) * D);
  const float* Vc = V + ((long long)c * p.Cs) * p.Ns;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int half = D >> 1;

  // columns owned by this thread: OP_DOT/L1: k0 + tx*4 + q ; OP_ROT: re pairs k0+tx*2+{0,1}, im = half + same
  int colq[4];
  bool colok[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (OP == OP_ROT) {
      int pr = k0 + tx * 2 + (q & 1);
      colok[q] = pr < half;
      colq[q] = (q < 2) ? pr : half + pr;
    } else {
      colq[q] = k0 + tx * 4 + q;
      colok[q] = colq[q] < D;
    }
  }
  float m[4][4];
  if (OP != OP_DOT) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        int x = x0 + ty * 4 + r;
        m[r][q] = (x < X && colok[q]) ? mine[(long long)x * D + colq[q]] : 0.f;
      }
  }
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;

  for (int y0 = 0; y0 < Y; y0 += BK) {
    // V slab: Vs[yy][x] = coef(x0+x, y0+yy)
    if (SIDE_B) {
      const int yy = threadIdx.x >> 4, xq = (threadIdx.x & 15) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int x = x0 + xq + e, y = y0 + yy;
        Vs[yy][xq + e] = (x < X && y < Y) ? Vc[(long long)y * p.Ns + x] : 0.f;
      }
    } else {
      const int x = threadIdx.x >> 2, yq = (threadIdx.x & 3) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int xx = x0 + x, y = y0 + yq + e;
        Vs[yq + e][x] = (xx < X && y < Y) ? Vc[(long long)xx * p.Ns + y] : 0.f;
      }
    }
    {  // other-rows slab: 16 rows x 64 floats
      const int yy = threadIdx.x >> 4, q = threadIdx.x & 15;
      bool valid;
      int col;
      if (OP == OP_ROT) {
        int pr = k0 + (q & 7) * 4;
        valid = pr < half;
        col = (q < 8) ? pr : half + pr;
      } else {
        col = k0 + q * 4;
        valid = col < D;
      }
      float4 v = (valid && y0 + yy < Y) ? ld4(other + (long long)(y0 + yy) * D + col) : zero4();
      *reinterpret_cast<float4*>(&Ys[yy][q * 4]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int yy = 0; yy < BK; ++yy) {
      float4 v4 = *reinterpret_cast<const float4*>(&Vs[yy][ty * 4]);
      const float vv[4] = {v4.x, v4.y, v4.z, v4.w};
      float o[4];
      if (OP == OP_ROT) {
        float2 re = *reinterpret_cast<const float2*>(&Ys[yy][tx * 2]);
        float2 im = *reinterpret_cast<const float2*>(&Ys[yy][T / 2 + tx * 2]);
        o[0] = re.x; o[1] = re.y; o[2] = im.x; o[3] = im.y;
      } else {
        float4 y4 = *reinterpret_cast<const float4*>(&Ys[yy][tx * 4]);
        o[0] = y4.x; o[1] = y4.y; o[2] = y4.z; o[3] = y4.w;
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (OP == OP_DOT) {
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[r][q] = fmaf(vv[r], o[q], acc[r][q]);
        } else if (OP == OP_L1) {
          // d(gamma - |mine - other|_1)/d mine = -sign(mine - other)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[r][q] -= vv[r] * sgnf(m[r][q] - o[q]);
        } else {
          // d(gamma - |mine - other|)/d mine = -(mine - other)/|mine - other|   (complex modulus)
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            float dre = m[r][u] - o[u], dim = m[r][2 + u] - o[2 + u];
            float m2 = fmaf(dre, dre, dim * dim);
            float s = (m2 > 0.f) ? vv[r] * rsqrtf(m2) : 0.f;
            acc[r][u] = fmaf(-s, dre, acc[r][u]);
            acc[r][2 + u] = fmaf(-s, dim, acc[r][2 + u]);
          }
        }
      }
    }
    __syncthreads();
  }
  // epilogue
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int x = x0 + ty * 4 + r;
    if (x >= X) continue;
    if (SIDE_B) {
      float* row = Bn + ((long long)c * p.Ns + x) * D;
      const float cs = (p.model == KGE_TRANSE_L2) ? colsum[(long long)c * p.Ns + x] : 0.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (!colok[q]) continue;
        float b = (OP == OP_DOT) ? row[colq[q]] : m[r][q];
        float g = acc[r][q];
        if (p.model == KGE_TRANSE_L2) g = fmaf(-cs, b, g);     // sum_i V_ij a_i - (sum_i V_ij) b_j
        g += reg_grad(b, p.reg_norm, p.reg_coef);
        row[colq[q]] = g;
      }
    } else {
      float* row = GA + ((long long)c * p.Cs + x) * D;
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (colok[q]) row[colq[q]] = acc[r][q];
    }
  }
}

template <bool SIDE_B>
static void launch_grad_side(const LaunchCtx& c, const StepParams& p, const StepWs& w) {
  const int X = SIDE_B ? p.Ns : p.Cs;
  if (p.model == KGE_ROTATE) {
    dim3 grid(ceil_div(p.D / 2, 32), ceil_div(X, RT), p.C);
    KGE_LAUNCH(c, (k_rot_grad<SIDE_B>), grid, 256, 0, p, w.V, w.A, w.Bn, w.GA);
  } else if (p.model == KGE_TRANSE_L1) {
    dim3 grid(ceil_div(p.D, T), ceil_div(X, T), p.C);
    KGE_LAUNCH(c, (k_grad<OP_L1, SIDE_B>), grid, 256, 0, p, w.V, w.A, w.Bn, w.GA, w.colsum);
  } else {
    dim3 grid(ceil_div(p.D, T), ceil_div(X, T), p.C);
    KGE_LAUNCH(c, (k_grad<OP_DOT, SIDE_B>), grid, 256, 0, p, w.V, w.A, w.Bn, w.GA, w.colsum);
  }
}
void launch_grad_a(const LaunchCtx& c, const StepParams& p, const StepWs& w) { launch_grad_side<false>(c, p, w); }
void launch_grad_b(const LaunchCtx& c, const StepParams& p, const StepWs& w) { launch_grad_side<true>(c, p, w); }

}  // namespace kge
