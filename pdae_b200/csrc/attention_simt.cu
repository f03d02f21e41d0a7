// fp32 CUDA-core QKV attention ("parity mode"): S = (Q K^T) * ch^-1/2, softmax over keys, O = P V.
// Three launches per call: batched GEMM (NT) -> row softmax -> batched GEMM (NN).  Token-major
// (NHWC) operands, so Q/K/V are strided column blocks of the [B][T][3C] qkv tensor.
#include "common.cuh"

namespace pdae {

constexpr int GM = 64, GN = 64, GK = 16;

struct GemmArgs {
  const float* A; const float* Bm; float* C;
  int M, N, K;
  long long lda, ldb, ldc;
  // batch z = (b, h): offset = b * *_bs + h * *_hs
  long long a_bs, a_hs, b_bs, b_hs, c_bs, c_hs;
  int heads;
  int transB;  // 1: B given as [N][K] (row n, k contiguous) ; 0: [K][N]
  int transA;  // 1: A given as [K][M] (row k, m contiguous)
  float alpha;
};

__global__ void __launch_bounds__(256) gemm_batched_kernel(GemmArgs p) {
  __shared__ float As[GK][GM + 4];
  __shared__ float Bs[GK][GN + 4];
  const int z = blockIdx.z, bb = z / p.heads, hh = z % p.heads;
  const float* __restrict__ A = p.A + bb * p.a_bs + hh * p.a_hs;
  const float* __restrict__ Bm = p.Bm + bb * p.b_bs + hh * p.b_hs;
  float* __restrict__ C = p.C + bb * p.c_bs + hh * p.c_hs;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * GM, n0 = blockIdx.y * GN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += GK) {
    // A: 64 rows x 16 k ; thread -> (row = tid/4, k = (tid%4)*4 + i)
    {
      const int r = tid >> 2, kq = (tid & 3) * 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = m0 + r, k = k0 + kq + i;
        As[kq + i][r] = (m < p.M && k < p.K) ? (p.transA ? A[(long long)k * p.lda + m] : A[(long long)m * p.lda + k]) : 0.f;
      }
    }
    if (p.transB) {
      const int r = tid >> 2, kq = (tid & 3) * 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int n = n0 + r, k = k0 + kq + i;
        Bs[kq + i][r] = (n < p.N && k < p.K) ? Bm[(long long)n * p.ldb + k] : 0.f;
      }
    } else {
      const int k = tid >> 4, nq = (tid & 15) * 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int n = n0 + nq + i, kk = k0 + k;
        Bs[k][nq + i] = (n < p.N && kk < p.K) ? Bm[(long long)kk * p.ldb + n] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[k][ty * 4 + i]; bv[i] = Bs[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < p.N) C[(long long)m * p.ldc + n] = p.alpha * acc[i][j];
    }
  }
}

// one warp per row, cols <= 4096
__global__ void softmax_rows_kernel(float* __restrict__ S, long long rows, int cols) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float* r = S + row * cols;
  float mx = -INFINITY;
  for (int j = lane; j < cols; j += 32) mx = fmaxf(mx, r[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < cols; j += 32) {
    const float e = expf(r[j] - mx);
    r[j] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  for (int j = lane; j < cols; j += 32) r[j] *= inv;
}

// softmax(alpha * S) over rows of fp32 scores, written as bf16 probabilities (one warp per row)
__global__ void softmax_rows_bf16_kernel(const float* __restrict__ S, __nv_bfloat16* __restrict__ P, long long rows, int cols,
                                         float alpha) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* r = S + row * cols;
  __nv_bfloat16* o = P + row * cols;
  float mx = -INFINITY;
  for (int j = lane * 4; j < cols; j += 128) {
    const float4 v = *reinterpret_cast<const float4*>(r + j);
    mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, d));
  float sum = 0.f;
  for (int j = lane * 4; j < cols; j += 128) {
    const float4 v = *reinterpret_cast<const float4*>(r + j);
    sum += __expf(alpha * (v.x - mx)) + __expf(alpha * (v.y - mx)) + __expf(alpha * (v.z - mx)) + __expf(alpha * (v.w - mx));
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
  const float inv = 1.0f / sum;
  for (int j = lane * 4; j < cols; j += 128) {
    const float4 v = *reinterpret_cast<const float4*>(r + j);
    store4<__nv_bfloat16>(o + j, make_float4(__expf(alpha * (v.x - mx)) * inv, __expf(alpha * (v.y - mx)) * inv,
                                             __expf(alpha * (v.z - mx)) * inv, __expf(alpha * (v.w - mx)) * inv));
  }
}

// vT[z][c][t] = qkv[b][t][voff + h*hs + c]   (z = b*heads + h): 64x64 shared-memory tile transpose, bf16 pairs:
// every warp access is 32 x 4 B = 128 contiguous bytes on both the read (channel pairs) and the write (token pairs) side.
// T, ch even; the per-head channel offset even (host checks).
__global__ void __launch_bounds__(256) transpose_v_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ vT,
                                                          int T, int C3, int ch, int heads, long long voff, long long hs) {
  __shared__ uint32_t tile[64][33];   // [t][channel pair]
  const int z = blockIdx.z, b = z / heads, h = z % heads;
  const int t0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const __nv_bfloat16* src = qkv + (long long)b * T * C3 + voff + h * hs;
#pragma unroll
  for (int i = ty; i < 64; i += 8) {
    const int t = t0 + i, c = c0 + 2 * tx;
    uint32_t w = 0;
    if (t < T && c < ch) w = *reinterpret_cast<const uint32_t*>(src + (long long)t * C3 + c);
    tile[i][tx] = w;
  }
  __syncthreads();
  __nv_bfloat16* dst = vT + (long long)z * ch * T;
#pragma unroll
  for (int i = ty; i < 64; i += 8) {
    const int c = c0 + i, t = t0 + 2 * tx;
    if (c < ch && t < T) {
      const uint32_t w0 = tile[2 * tx][i >> 1], w1 = tile[2 * tx + 1][i >> 1];
      const uint32_t lo = (i & 1) ? (w0 >> 16) : (w0 & 0xffffu), hi = (i & 1) ? (w1 & 0xffff0000u) : (w1 << 16);
      *reinterpret_cast<uint32_t*>(dst + (long long)c * T + t) = lo | hi;
    }
  }
}

// ---- split-operand ("bf16x3") attention on the tensor cores -----------------------------------------------------------
// The fp32 qkv rows are re-laid-out as bf16 operand blocks so that the two attention GEMMs run on conv_tc2's batched-GEMM
// mode with fp32-grade products:  S = [q_hi|q_lo|q_hi] * [k_hi|k_hi|k_lo]^T  and  A = [p_hi|p_lo|p_hi] * [vT_hi|vT_hi|vT_lo]^T.
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// Q3 / K3: [B*heads][T][3*ch] ; one thread per (z, t, 8 channels): 2 x 32 B loads, 6 x 16 B stores
__device__ __forceinline__ void split8(const float* src, uint4& hi, uint4& lo) {
  const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
  const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint32_t h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    __nv_bfloat162 hh = __floats2bfloat162_rn(v[2 * e], v[2 * e + 1]);
    const float2 hf = __bfloat1622float2(hh);
    __nv_bfloat162 ll = __floats2bfloat162_rn(v[2 * e] - hf.x, v[2 * e + 1] - hf.y);
    h[e] = *reinterpret_cast<uint32_t*>(&hh);
    l[e] = *reinterpret_cast<uint32_t*>(&ll);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
__global__ void __launch_bounds__(256) qk_split3_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ Q3,
                                                        __nv_bfloat16* __restrict__ K3, int T, int C3, int ch, int heads,
                                                        long long koff, long long hs, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // over (z, t, ch / 8)
  if (i >= total) return;
  const int c8 = ch >> 3;
  const int c = (int)(i % c8) * 8;
  const long long zt = i / c8;
  const int t = (int)(zt % T);
  const int z = (int)(zt / T), b = z / heads, h = z % heads;
  const float* row = qkv + ((long long)b * T + t) * C3 + h * hs;
  uint4 qh, ql, kh, kl;
  split8(row + c, qh, ql);
  split8(row + koff + c, kh, kl);
  __nv_bfloat16* q = Q3 + zt * 3 * ch + c;
  __nv_bfloat16* k = K3 + zt * 3 * ch + c;
  *reinterpret_cast<uint4*>(q) = qh; *reinterpret_cast<uint4*>(q + ch) = ql; *reinterpret_cast<uint4*>(q + 2 * ch) = qh;
  *reinterpret_cast<uint4*>(k) = kh; *reinterpret_cast<uint4*>(k + ch) = kh; *reinterpret_cast<uint4*>(k + 2 * ch) = kl;
}

// VT3: [B*heads][ch][3*T] = [vT_hi | vT_hi | vT_lo]  (32 x 32 shared-memory transpose)
__global__ void __launch_bounds__(256) v_split3_transpose_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ VT3,
                                                                 int T, int C3, int ch, int heads, long long voff, long long hs) {
  __shared__ float tile[64][33];   // [t][c]
  const int z = blockIdx.z, b = z / heads, h = z % heads;
  const int t0 = blockIdx.x * 64, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  const float* src = qkv + (long long)b * T * C3 + voff + h * hs;
#pragma unroll
  for (int i = ty; i < 64; i += 8) {
    const int t = t0 + i, c = c0 + tx;
    tile[i][tx] = (t < T && c < ch) ? src[(long long)t * C3 + c] : 0.f;
  }
  __syncthreads();
  __nv_bfloat16* dst = VT3 + (long long)z * ch * 3 * T;
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, t = t0 + 2 * tx;     // two consecutive tokens per thread: 4-byte stores, 128 B per warp
    if (c < ch && t < T) {
      const float v0 = tile[2 * tx][i], v1 = tile[2 * tx + 1][i];
      __nv_bfloat162 hh = __floats2bfloat162_rn(v0, v1);
      const float2 hf = __bfloat1622float2(hh);
      __nv_bfloat162 ll = __floats2bfloat162_rn(v0 - hf.x, v1 - hf.y);
      __nv_bfloat16* r = dst + (long long)c * 3 * T + t;
      *reinterpret_cast<__nv_bfloat162*>(r) = hh;
      *reinterpret_cast<__nv_bfloat162*>(r + T) = hh;
      *reinterpret_cast<__nv_bfloat162*>(r + 2 * T) = ll;
    }
  }
}

// P3[row] = [p_hi | p_lo | p_hi],  p = softmax(alpha * S[row])  -- one warp per row, fp32 arithmetic (module.py:452-455)
__global__ void __launch_bounds__(256) softmax_split3_kernel(const float* __restrict__ S, __nv_bfloat16* __restrict__ P3,
                                                             long long rows, int cols, float alpha) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* s = S + row * cols;
  float mx = -3.0e38f;
  for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, s[c] * alpha);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int c = lane; c < cols; c += 32) sum += expf(s[c] * alpha - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  __nv_bfloat16* p = P3 + row * 3 * cols;
  for (int c = lane; c < cols; c += 32) {
    __nv_bfloat16 hi, lo;
    split_bf16(expf(s[c] * alpha - mx) * inv, hi, lo);
    p[c] = hi; p[cols + c] = lo; p[2 * cols + c] = hi;
  }
}

}  // namespace pdae

using namespace pdae;

extern "C" int pdae_softmax_bf16(const float* S, void* P_bf16, int64_t rows, int cols, float alpha, pdae_stream_t stream) {
  PDAE_REQUIRE(S && P_bf16 && cols % 4 == 0, "softmax_bf16: bad args");
  softmax_rows_bf16_kernel<<<cdiv(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(S, (__nv_bfloat16*)P_bf16, rows, cols, alpha);
  PDAE_LAUNCH_CHECK("softmax_rows_bf16_kernel");
  return PDAE_OK;
}


// fp32 qkv [B][T][3C] (channel order per `legacy`, model/module.py:440-447 / 469-477) -> the split-operand GEMM inputs
extern "C" int pdae_qkv_split3(const float* qkv, void* Q3, void* K3, void* VT3, int B, int T, int C, int heads, int legacy,
                               pdae_stream_t stream) {
  PDAE_REQUIRE(qkv && Q3 && K3 && VT3 && heads > 0 && C % heads == 0, "qkv_split3: bad args");
  const int ch = C / heads;
  const long long hs = legacy ? 3LL * ch : ch, ko = legacy ? ch : C, vo = legacy ? 2LL * ch : 2LL * C;
  PDAE_REQUIRE((long long)B * heads <= 65535, "qkv_split3: B*heads too large");
  PDAE_REQUIRE(ch % 8 == 0 && C % 4 == 0, "qkv_split3: C/heads=%d must be a multiple of 8", ch);
  PDAE_REQUIRE(T % 2 == 0, "qkv_split3: T must be even");
  const long long total = (long long)B * heads * T * (ch / 8);
  cudaStream_t s = (cudaStream_t)stream;
  qk_split3_kernel<<<cdiv(total, 256), 256, 0, s>>>(qkv, (__nv_bfloat16*)Q3, (__nv_bfloat16*)K3, T, 3 * C, ch, heads, ko, hs, total);
  PDAE_LAUNCH_CHECK("qk_split3_kernel");
  dim3 grid(cdiv(T, 64), cdiv(ch, 32), B * heads);
  v_split3_transpose_kernel<<<grid, 256, 0, s>>>(qkv, (__nv_bfloat16*)VT3, T, 3 * C, ch, heads, vo, hs);
  PDAE_LAUNCH_CHECK("v_split3_transpose_kernel");
  return PDAE_OK;
}

extern "C" int pdae_softmax_split3(const float* S, void* P3_bf16, int64_t rows, int cols, float alpha, pdae_stream_t stream) {
  PDAE_REQUIRE(S && P3_bf16 && rows > 0 && cols > 0, "softmax_split3: bad args");
  softmax_split3_kernel<<<cdiv(rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(S, (__nv_bfloat16*)P3_bf16, rows, cols, alpha);
  PDAE_LAUNCH_CHECK("softmax_split3_kernel");
  return PDAE_OK;
}

extern "C" int pdae_transpose_v(const void* qkv_bf16, void* vT_bf16, int B, int T, int C, int heads, int legacy,
                                pdae_stream_t stream) {
  PDAE_REQUIRE(qkv_bf16 && vT_bf16 && heads > 0 && C % heads == 0, "transpose_v: bad args");
  const int ch = C / heads;
  const long long voff = legacy ? 2LL * ch : 2LL * C, hs = legacy ? 3LL * ch : ch;
  PDAE_REQUIRE(T % 2 == 0 && ch % 2 == 0, "transpose_v: T=%d and C/heads=%d must be even", T, ch);
  dim3 grid(cdiv(T, 64), cdiv(ch, 64), B * heads);
  PDAE_REQUIRE(grid.z <= 65535, "transpose_v: B*heads too large");
  transpose_v_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)qkv_bf16, (__nv_bfloat16*)vT_bf16, T, 3 * C,
                                                            ch, heads, voff, hs);
  PDAE_LAUNCH_CHECK("transpose_v_kernel");
  return PDAE_OK;
}

// C[z] = alpha * op(A[z]) * op(B[z]),  z = (b, h) with offsets b * *_bs + h * *_hs  (attention backward GEMMs)
extern "C" int pdae_gemm_batched_simt(const float* A, int64_t lda, int64_t a_bs, int64_t a_hs, int transA, const float* Bm,
                                      int64_t ldb, int64_t b_bs, int64_t b_hs, int transB, float* C, int64_t ldc, int64_t c_bs,
                                      int64_t c_hs, int M, int N, int K, int batch, int heads, float alpha,
                                      pdae_stream_t stream) {
  PDAE_REQUIRE(A && Bm && C && heads > 0 && (long long)batch * heads <= 65535, "gemm_batched_simt: bad args");
  GemmArgs g;
  g.A = A; g.Bm = Bm; g.C = C; g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldb; g.ldc = ldc;
  g.a_bs = a_bs; g.a_hs = a_hs; g.b_bs = b_bs; g.b_hs = b_hs; g.c_bs = c_bs; g.c_hs = c_hs;
  g.heads = heads; g.transA = transA; g.transB = transB; g.alpha = alpha;
  dim3 grid(cdiv(M, GM), cdiv(N, GN), batch * heads);
  gemm_batched_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(g);
  PDAE_LAUNCH_CHECK("gemm_batched_kernel");
  return PDAE_OK;
}

extern "C" int pdae_attention_simt(const float* qkv, float* out, float* scratch, int B, int T, int C, int heads,
                                   int legacy, pdae_stream_t stream) {
  PDAE_REQUIRE(qkv && out && scratch, "attention_simt: null pointer");
  PDAE_REQUIRE(heads > 0 && C % heads == 0, "attention_simt: C %% heads != 0");
  PDAE_REQUIRE((long long)B * heads <= 65535, "attention_simt: B*heads too large for grid.z");
  const int ch = C / heads;
  cudaStream_t s = (cudaStream_t)stream;
  const long long row = 3LL * C;
  // channel offsets of q, k, v for head h: legacy -> h*3ch + {0, ch, 2ch} ; new -> {0, C, 2C} + h*ch
  const long long hs = legacy ? 3LL * ch : ch;
  const long long qo = 0, ko = legacy ? ch : C, vo = legacy ? 2LL * ch : 2LL * C;
  GemmArgs g;
  g.heads = heads;
  // S[z] = alpha * Q K^T
  g.A = qkv + qo; g.Bm = qkv + ko; g.C = scratch;
  g.M = T; g.N = T; g.K = ch; g.lda = row; g.ldb = row; g.ldc = T;
  g.a_bs = (long long)T * row; g.a_hs = hs; g.b_bs = (long long)T * row; g.b_hs = hs;
  g.c_bs = (long long)heads * T * T; g.c_hs = (long long)T * T;
  g.transB = 1;
  g.transA = 0;
  g.alpha = 1.0f / sqrtf((float)ch);
  dim3 grid1(cdiv(T, GM), cdiv(T, GN), B * heads);
  gemm_batched_kernel<<<grid1, 256, 0, s>>>(g);
  PDAE_LAUNCH_CHECK("gemm_batched_kernel(QK)");
  const long long rows = (long long)B * heads * T;
  softmax_rows_kernel<<<cdiv(rows * 32, 256), 256, 0, s>>>(scratch, rows, T);
  PDAE_LAUNCH_CHECK("softmax_rows_kernel");
  // O[z] = P V  -> out[b][t][h*ch + c]
  g.A = scratch; g.Bm = qkv + vo; g.C = out;
  g.M = T; g.N = ch; g.K = T; g.lda = T; g.ldb = row; g.ldc = C;
  g.a_bs = (long long)heads * T * T; g.a_hs = (long long)T * T; g.b_bs = (long long)T * row; g.b_hs = hs;
  g.c_bs = (long long)T * C; g.c_hs = ch;
  g.transB = 0;
  g.alpha = 1.0f;
  dim3 grid2(cdiv(T, GM), cdiv(ch, GN), B * heads);
  gemm_batched_kernel<<<grid2, 256, 0, s>>>(g);
  PDAE_LAUNCH_CHECK("gemm_batched_kernel(PV)");
  return PDAE_OK;
}
