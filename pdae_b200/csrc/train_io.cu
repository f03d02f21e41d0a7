// Caller-side steps either side of the hot path (SURVEY.md §8(f) rows 1, 3 and 4):
//   - fused multi-tensor Adam + EMA step  (trainer/train_representation_learning.py:57-69 Adam groups,
//     :192-212 the per-parameter python EMA loop `ema.mul_(decay).add_(p, alpha=1-decay)`)
//   - wire formats: fp32 NCHW [-1,1] -> uint8 NHWC (train_representation_learning.py:173-174 and every sampler),
//     uint8 NHWC -> normalised fp32 NCHW (dataset/ffhq.py:27-31 ToTensor + Normalize(0.5, 0.5))
//   - per-image MSE and SSIM (metric/utils.py:35-63)
// All HBM-bound; none of this is GEMM-shaped.
#include "common.cuh"

namespace pdae {

// ---------------------------------------------------------------------------------------------
// Adam + EMA.  One launch for ALL tensors: blockIdx.x -> (tensor, chunk) through a device-resident map.
// Arithmetic follows torch.optim.Adam's single-tensor path (non-amsgrad, coupled weight decay):
//   g += wd*p;  m = lerp(m, g, 1-b1);  v = b2*v + (1-b2)*g*g;  p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps)
// then, when ema_decay >= 0:  ema = ema*decay + (1-decay)*p   (the reference runs `accumulate` after optimizer.step()).
__global__ void __launch_bounds__(256) adam_ema_kernel(const pdae_adam_tensor* __restrict__ tab,
                                                       const int2* __restrict__ block_map, int chunk, float step_size,
                                                       float beta1, float beta2, float eps, float weight_decay,
                                                       float inv_sqrt_bc2, float grad_scale, float ema_decay) {
  const int2 tc = block_map[blockIdx.x];
  const pdae_adam_tensor T = tab[tc.x];
  const long long lo = (long long)tc.y * chunk;
  long long hi = lo + chunk;
  if (hi > T.n) hi = T.n;
  const float omb1 = 1.0f - beta1, omb2 = 1.0f - beta2, omd = 1.0f - ema_decay;
  auto upd = [&](float& p, float g, float& m, float& v) {
    g *= grad_scale;
    if (weight_decay != 0.0f) g = fmaf(weight_decay, p, g);
    m = fmaf(g - m, omb1, m);                       // lerp_
    v = fmaf(omb2 * g, g, beta2 * v);               // mul_(b2).addcmul_(g, g, 1-b2)
    const float denom = sqrtf(v) * inv_sqrt_bc2 + eps;
    p = p - step_size * (m / denom);
  };
  const bool vec = (((uintptr_t)T.p | (uintptr_t)T.g | (uintptr_t)T.m | (uintptr_t)T.v | (uintptr_t)T.ema) & 15) == 0 &&
                   (lo & 3) == 0;
  long long i = lo + (long long)threadIdx.x * 4;
  if (vec) {
    for (; i + 3 < hi; i += 256 * 4) {
      float4 p = *reinterpret_cast<float4*>(T.p + i);
      const float4 g = *reinterpret_cast<const float4*>(T.g + i);
      float4 m = *reinterpret_cast<float4*>(T.m + i), v = *reinterpret_cast<float4*>(T.v + i);
      upd(p.x, g.x, m.x, v.x); upd(p.y, g.y, m.y, v.y); upd(p.z, g.z, m.z, v.z); upd(p.w, g.w, m.w, v.w);
      *reinterpret_cast<float4*>(T.p + i) = p;
      *reinterpret_cast<float4*>(T.m + i) = m;
      *reinterpret_cast<float4*>(T.v + i) = v;
      if (T.ema && ema_decay >= 0.0f) {
        float4 e = *reinterpret_cast<float4*>(T.ema + i);
        e.x = fmaf(omd, p.x, e.x * ema_decay); e.y = fmaf(omd, p.y, e.y * ema_decay);
        e.z = fmaf(omd, p.z, e.z * ema_decay); e.w = fmaf(omd, p.w, e.w * ema_decay);
        *reinterpret_cast<float4*>(T.ema + i) = e;
      }
    }
    // tail (n % 4) of this chunk: first threads, scalar
    const long long tail0 = lo + ((hi - lo) & ~3LL);
    i = tail0 + threadIdx.x;
    if (i < hi) {
      float p = T.p[i], m = T.m[i], v = T.v[i];
      upd(p, T.g[i], m, v);
      T.p[i] = p; T.m[i] = m; T.v[i] = v;
      if (T.ema && ema_decay >= 0.0f) T.ema[i] = fmaf(omd, p, T.ema[i] * ema_decay);
    }
  } else {
    for (i = lo + threadIdx.x; i < hi; i += 256) {
      float p = T.p[i], m = T.m[i], v = T.v[i];
      upd(p, T.g[i], m, v);
      T.p[i] = p; T.m[i] = m; T.v[i] = v;
      if (T.ema && ema_decay >= 0.0f) T.ema[i] = fmaf(omd, p, T.ema[i] * ema_decay);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// fp32 NCHW in [-1,1] -> uint8 NHWC, the reference's op sequence with every fp32 rounding kept:
//   x.mul(0.5).add(0.5).mul(255).add(0.5).clamp(0,255) -> .to(uint8) (truncation)
__global__ void __launch_bounds__(256) images_to_u8_kernel(const float* __restrict__ x, uint8_t* __restrict__ out, int C, int HW,
                                                           long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    // i indexes the OUTPUT (b, pix, c): coalesced byte stores; the C strided reads hit the same lines across c
    const int c = (int)(i % C);
    const long long bp = i / C;
    const int pix = (int)(bp % HW);
    const long long b = bp / HW;
    float v = x[(b * C + c) * HW + pix];
    v = __fadd_rn(__fmul_rn(v, 0.5f), 0.5f);
    v = __fadd_rn(__fmul_rn(v, 255.0f), 0.5f);
    v = fminf(fmaxf(v, 0.0f), 255.0f);
    out[i] = (uint8_t)(int)v;   // NaN -> 0 like a saturating cast would not matter: inputs are finite
  }
}

// uint8 NHWC -> fp32 NCHW: ToTensor (x / 255) then Normalize(0.5, 0.5): (v - 0.5) / 0.5
__global__ void __launch_bounds__(256) u8_to_images_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int C, int HW,
                                                           long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    // i indexes the OUTPUT (b, c, pix)
    const int pix = (int)(i % HW);
    const long long bc = i / HW;
    const int c = (int)(bc % C);
    const long long b = bc / C;
    const float v = __fdiv_rn((float)in[(b * HW + pix) * C + c], 255.0f);
    out[i] = __fdiv_rn(__fsub_rn(v, 0.5f), 0.5f);
  }
}

// ---------------------------------------------------------------------------------------------
// per-image mean squared error (metric/utils.py:62-63), fp64 accumulation.  DET: each block stores its sum in its own slot
// acc[image][blockIdx.x] instead of adding it atomically (finish_parts_kernel adds the slots in order).
template <bool DET = false>
__global__ void __launch_bounds__(256) mse_kernel(const float* __restrict__ a, const float* __restrict__ b, long long per_image,
                                                  double* __restrict__ acc) {
  const long long base = (long long)blockIdx.y * per_image;
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_image; i += (long long)gridDim.x * blockDim.x) {
    const float d = a[base + i] - b[base + i];
    s += (double)(d * d);
  }
  __shared__ double red[8];
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    if (DET) acc[(long long)blockIdx.y * gridDim.x + blockIdx.x] = t;
    else atomicAdd(acc + blockIdx.y, t);
  }
}

__global__ void finish_mean_kernel(const double* __restrict__ acc, float* __restrict__ out, int B, double inv_n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) out[i] = (float)(acc[i] * inv_n);
}

// the nparts slots of image i, added in slot order
__global__ void finish_parts_kernel(const double* __restrict__ acc, long long nparts, float* __restrict__ out, int B,
                                    double inv_n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  double t = 0.0;
  for (long long k = 0; k < nparts; ++k) t += acc[(long long)i * nparts + k];
  out[i] = (float)(t * inv_n);
}

// SSIM (metric/utils.py:35-56): 11x11 Gaussian window (sigma 1.5, outer product of the normalised 1-D window, fp32),
// zero padding 5, depthwise; C1 = 0.01^2, C2 = 0.03^2; mean over (C,H,W).  One CTA = one 16x16 tile of one (b,c) plane.
// DET: each CTA stores its sum in its own slot acc[plane][tile y][tile x]; an image's slots are contiguous.
constexpr int SSIM_T = 16, SSIM_R = 5, SSIM_S = SSIM_T + 2 * SSIM_R;
template <bool DET = false>
__global__ void __launch_bounds__(256) ssim_kernel(const float* __restrict__ img1, const float* __restrict__ img2,
                                                   const float* __restrict__ win2d, int C, int H, int W,
                                                   double* __restrict__ acc) {
  __shared__ float t1[SSIM_S][SSIM_S + 1], t2[SSIM_S][SSIM_S + 1], wsm[121];
  __shared__ double red[8];
  const int plane = blockIdx.z;           // b*C + c
  const int b = plane / C;
  const int x0 = blockIdx.x * SSIM_T, y0 = blockIdx.y * SSIM_T;
  const float* p1 = img1 + (long long)plane * H * W;
  const float* p2 = img2 + (long long)plane * H * W;
  if (threadIdx.x < 121) wsm[threadIdx.x] = win2d[threadIdx.x];
  for (int i = threadIdx.x; i < SSIM_S * SSIM_S; i += 256) {
    const int ly = i / SSIM_S, lx = i % SSIM_S;
    const int gy = y0 + ly - SSIM_R, gx = x0 + lx - SSIM_R;
    const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
    t1[ly][lx] = in ? p1[(long long)gy * W + gx] : 0.0f;
    t2[ly][lx] = in ? p2[(long long)gy * W + gx] : 0.0f;
  }
  __syncthreads();
  const int lx = threadIdx.x % SSIM_T, ly = threadIdx.x / SSIM_T;
  double contrib = 0.0;
  if (y0 + ly < H && x0 + lx < W) {
    float mu1 = 0.f, mu2 = 0.f, s11 = 0.f, s22 = 0.f, s12 = 0.f;
#pragma unroll 1
    for (int ky = 0; ky < 11; ++ky)
#pragma unroll
      for (int kx = 0; kx < 11; ++kx) {
        const float w = wsm[ky * 11 + kx], a = t1[ly + ky][lx + kx], c = t2[ly + ky][lx + kx];
        mu1 = fmaf(w, a, mu1); mu2 = fmaf(w, c, mu2);
        s11 = fmaf(w, a * a, s11); s22 = fmaf(w, c * c, s22); s12 = fmaf(w, a * c, s12);
      }
    const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
    const float sg1 = s11 - mu1_sq, sg2 = s22 - mu2_sq, sg12 = s12 - mu12;
    const float c1 = 0.01f * 0.01f, c2 = 0.03f * 0.03f;
    contrib = (double)(((2.f * mu12 + c1) * (2.f * sg12 + c2)) / ((mu1_sq + mu2_sq + c1) * (sg1 + sg2 + c2)));
  }
  for (int o = 16; o; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = contrib;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    if (DET) acc[((long long)plane * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = t;
    else atomicAdd(acc + b, t);
  }
}


// Gather every weight-gradient accumulator of a backward plan (packed layouts, e.g. conv [k*k][Cin][Cout]) into ONE flat buffer
// in the parameters' own layouts: item i copies a <=4-D strided view to a contiguous run of `g` (dst linear order = row-major
// order of the view).  One launch replaces the per-parameter permute / contiguous / clone chain.
__global__ void __launch_bounds__(256) unpack_grads_kernel(const pdae_unpack_item* __restrict__ items, const int2* __restrict__ blocks,
                                                           int chunk, float* __restrict__ g) {
  const int2 bc = blocks[blockIdx.x];
  const pdae_unpack_item it = items[bc.x];
  const long long numel = (long long)it.shape[0] * it.shape[1] * it.shape[2] * it.shape[3];
  const long long lo = (long long)bc.y * chunk, hi = lo + chunk < numel ? lo + chunk : numel;
  float* dst = g + it.dst_off;
  for (long long i = lo + threadIdx.x; i < hi; i += 256) {
    long long r = i;
    const int i3 = (int)(r % it.shape[3]); r /= it.shape[3];
    const int i2 = (int)(r % it.shape[2]); r /= it.shape[2];
    const int i1 = (int)(r % it.shape[1]);
    const int i0 = (int)(r / it.shape[1]);
    const float v = it.src[i0 * it.stride[0] + i1 * it.stride[1] + i2 * it.stride[2] + i3 * it.stride[3]];
    dst[i] = it.add ? dst[i] + v : v;
  }
}

}  // namespace pdae

using namespace pdae;

extern "C" int pdae_adam_ema_step(const pdae_adam_tensor* table, const int32_t* block_map, int n_blocks, int chunk, float lr,
                                  float beta1, float beta2, float eps, float weight_decay, int64_t step, float grad_scale,
                                  float ema_decay, pdae_stream_t stream) {
  PDAE_REQUIRE(table && block_map && n_blocks > 0, "adam_ema_step: null table / empty block map");
  PDAE_REQUIRE(chunk > 0 && chunk % 4 == 0, "adam_ema_step: chunk=%d must be a positive multiple of 4", chunk);
  PDAE_REQUIRE(step >= 1, "adam_ema_step: step=%lld must be >= 1", (long long)step);
  // bias corrections in fp64 like python floats in torch.optim.adam._single_tensor_adam
  const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
  const float step_size = (float)((double)lr / bc1);
  const float inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
  adam_ema_kernel<<<n_blocks, 256, 0, (cudaStream_t)stream>>>(table, reinterpret_cast<const int2*>(block_map), chunk, step_size,
                                                              beta1, beta2, eps, weight_decay, inv_sqrt_bc2, grad_scale,
                                                              ema_decay);
  PDAE_LAUNCH_CHECK("adam_ema_kernel");
  return PDAE_OK;
}

extern "C" int pdae_unpack_grads(const pdae_unpack_item* items, const int32_t* block_map, int n_blocks, int chunk, float* g,
                                 pdae_stream_t stream) {
  PDAE_REQUIRE(items && block_map && g && n_blocks > 0 && chunk > 0, "unpack_grads: bad arguments");
  unpack_grads_kernel<<<n_blocks, 256, 0, (cudaStream_t)stream>>>(items, reinterpret_cast<const int2*>(block_map), chunk, g);
  PDAE_LAUNCH_CHECK("unpack_grads_kernel");
  return PDAE_OK;
}

static inline int io_grid(long long total) {
  int g = cdiv(total, 256);
  return g > 148 * 16 ? 148 * 16 : (g < 1 ? 1 : g);
}

extern "C" int pdae_images_to_u8_nhwc(const float* x_nchw, uint8_t* out_nhwc, int B, int C, int H, int W,
                                      pdae_stream_t stream) {
  PDAE_REQUIRE(x_nchw && out_nhwc && B > 0 && C > 0 && H > 0 && W > 0, "images_to_u8_nhwc: bad args");
  const long long total = (long long)B * C * H * W;
  images_to_u8_kernel<<<io_grid(total), 256, 0, (cudaStream_t)stream>>>(x_nchw, out_nhwc, C, H * W, total);
  PDAE_LAUNCH_CHECK("images_to_u8_kernel");
  return PDAE_OK;
}

extern "C" int pdae_u8_nhwc_to_images(const uint8_t* in_nhwc, float* out_nchw, int B, int C, int H, int W,
                                      pdae_stream_t stream) {
  PDAE_REQUIRE(in_nhwc && out_nchw && B > 0 && C > 0 && H > 0 && W > 0, "u8_nhwc_to_images: bad args");
  const long long total = (long long)B * C * H * W;
  u8_to_images_kernel<<<io_grid(total), 256, 0, (cudaStream_t)stream>>>(in_nhwc, out_nchw, C, H * W, total);
  PDAE_LAUNCH_CHECK("u8_to_images_kernel");
  return PDAE_OK;
}

extern "C" int pdae_mse_per_image(const float* a, const float* b, int B, int64_t per_image, double* workspace, float* out,
                                  pdae_stream_t stream) {
  PDAE_REQUIRE(a && b && workspace && out && B > 0 && per_image > 0, "mse_per_image: bad args");
  cudaStream_t s = (cudaStream_t)stream;
  PDAE_CUDA(cudaMemsetAsync(workspace, 0, sizeof(double) * B, s));
  int gx = cdiv(per_image, 256 * 8);
  if (gx > 64) gx = 64;
  mse_kernel<false><<<dim3(gx, B), 256, 0, s>>>(a, b, per_image, workspace);
  PDAE_LAUNCH_CHECK("mse_kernel");
  finish_mean_kernel<<<cdiv(B, 256), 256, 0, s>>>(workspace, out, B, 1.0 / (double)per_image);
  PDAE_LAUNCH_CHECK("finish_mean_kernel");
  return PDAE_OK;
}

extern "C" int pdae_ssim_per_image(const float* img1, const float* img2, const float* window_11x11, int B, int C, int H, int W,
                                   double* workspace, float* out, pdae_stream_t stream) {
  PDAE_REQUIRE(img1 && img2 && window_11x11 && workspace && out && B > 0 && C > 0 && H > 0 && W > 0, "ssim_per_image: bad args");
  PDAE_REQUIRE((long long)B * C <= 65535, "ssim_per_image: B*C=%lld exceeds the grid z limit", (long long)B * C);
  cudaStream_t s = (cudaStream_t)stream;
  PDAE_CUDA(cudaMemsetAsync(workspace, 0, sizeof(double) * B, s));
  ssim_kernel<false><<<dim3(cdiv(W, SSIM_T), cdiv(H, SSIM_T), B * C), 256, 0, s>>>(img1, img2, window_11x11, C, H, W, workspace);
  PDAE_LAUNCH_CHECK("ssim_kernel");
  finish_mean_kernel<<<cdiv(B, 256), 256, 0, s>>>(workspace, out, B, 1.0 / ((double)C * H * W));
  PDAE_LAUNCH_CHECK("finish_mean_kernel");
  return PDAE_OK;
}

// Deterministic per-image MSE / SSIM: every block's sum has its own workspace slot, and an image's slots are added in order.
static inline int mse_blocks(int64_t per_image) {
  const int gx = cdiv(per_image, 256 * 8);
  return gx > 64 ? 64 : gx;
}

extern "C" int64_t pdae_mse_det_workspace_bytes(int B, int64_t per_image) {
  if (B <= 0 || per_image <= 0) {
    ::pdae::set_error("mse_det_workspace_bytes: B=%d per_image=%lld must be > 0", B, (long long)per_image);
    return PDAE_EINVAL;
  }
  return (int64_t)B * mse_blocks(per_image) * (int64_t)sizeof(double);
}

extern "C" int pdae_mse_per_image_det(const float* a, const float* b, int B, int64_t per_image, double* workspace,
                                      int64_t workspace_bytes, float* out, pdae_stream_t stream) {
  PDAE_REQUIRE(a && b && workspace && out && B > 0 && B <= 65535 && per_image > 0, "mse_per_image_det: bad args");
  const int gx = mse_blocks(per_image);
  const long long need = (long long)B * gx * (long long)sizeof(double);
  PDAE_REQUIRE(workspace_bytes >= need, "mse_per_image_det: workspace of %lld bytes, %lld needed (pdae_mse_det_workspace_bytes)",
               (long long)workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  mse_kernel<true><<<dim3(gx, B), 256, 0, s>>>(a, b, per_image, workspace);
  PDAE_LAUNCH_CHECK("mse_kernel<det>");
  finish_parts_kernel<<<cdiv(B, 256), 256, 0, s>>>(workspace, gx, out, B, 1.0 / (double)per_image);
  PDAE_LAUNCH_CHECK("finish_parts_kernel");
  return PDAE_OK;
}

extern "C" int64_t pdae_ssim_det_workspace_bytes(int B, int C, int H, int W) {
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0) {
    ::pdae::set_error("ssim_det_workspace_bytes: B=%d C=%d H=%d W=%d must be > 0", B, C, H, W);
    return PDAE_EINVAL;
  }
  return (int64_t)B * C * cdiv(H, SSIM_T) * cdiv(W, SSIM_T) * (int64_t)sizeof(double);
}

extern "C" int pdae_ssim_per_image_det(const float* img1, const float* img2, const float* window_11x11, int B, int C, int H, int W,
                                       double* workspace, int64_t workspace_bytes, float* out, pdae_stream_t stream) {
  PDAE_REQUIRE(img1 && img2 && window_11x11 && workspace && out && B > 0 && C > 0 && H > 0 && W > 0,
               "ssim_per_image_det: bad args");
  PDAE_REQUIRE((long long)B * C <= 65535, "ssim_per_image_det: B*C=%lld exceeds the grid z limit", (long long)B * C);
  const long long parts = (long long)C * cdiv(H, SSIM_T) * cdiv(W, SSIM_T);
  PDAE_REQUIRE(workspace_bytes >= (long long)B * parts * (long long)sizeof(double),
               "ssim_per_image_det: workspace of %lld bytes, %lld needed (pdae_ssim_det_workspace_bytes)", (long long)workspace_bytes,
               (long long)B * parts * (long long)sizeof(double));
  cudaStream_t s = (cudaStream_t)stream;
  ssim_kernel<true><<<dim3(cdiv(W, SSIM_T), cdiv(H, SSIM_T), B * C), 256, 0, s>>>(img1, img2, window_11x11, C, H, W, workspace);
  PDAE_LAUNCH_CHECK("ssim_kernel<det>");
  finish_parts_kernel<<<cdiv(B, 256), 256, 0, s>>>(workspace, parts, out, B, 1.0 / ((double)C * H * W));
  PDAE_LAUNCH_CHECK("finish_parts_kernel");
  return PDAE_OK;
}
