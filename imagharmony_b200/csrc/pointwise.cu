// Small / bandwidth-bound kernels of the denoise step: small-M linear (time embeddings), sinusoidal embedding,
// nearest 2x upsample, channel concat, conv_in / conv_out (4-channel ends of the UNet, NCHW <-> NHWC), and the fused
// CFG-combine + Euler update + next-step input scaling (custom_pipelines.py:332-334,348-357).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>

#include "../../include/ih_api.h"
#include "host_util.h"
#include "ptx.cuh"

namespace ih {

__device__ __forceinline__ void ld8(const __half* p, float (&x)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = unpack_half2(w[e]);
    x[2 * e] = f.x;
    x[2 * e + 1] = f.y;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// out[m, n] = act_out( W[n, :] . act_in(x[m, :]) + b[n] ),  M <= 8.  One warp per output column; W is read once.
// ---------------------------------------------------------------------------------------------------------------
constexpr int SL_MAXM = 8;
__global__ void linear_small_kernel(const __half* __restrict__ x, long long ldx, const __half* __restrict__ w,
                                    const __half* __restrict__ bias, const __half* __restrict__ addend,
                                    long long ld_add, __half* __restrict__ out, long long ldo, int M, int N, int K,
                                    int act_in, int act_out, float out_scale) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float acc[SL_MAXM];
#pragma unroll
  for (int m = 0; m < SL_MAXM; ++m) acc[m] = 0.f;
  const __half* wr = w + (long long)n * K;
  for (int k = lane * 8; k < K; k += 256) {
    float wv[8];
    ld8(wr + k, wv);
#pragma unroll
    for (int m = 0; m < SL_MAXM; ++m) {
      if (m < M) {
        float xv[8];
        ld8(x + m * ldx + k, xv);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float xe = xv[e];
          if (act_in == 1) xe = __half2float(__float2half_rn(silu_f(xe)));  // SiLU output is fp16 in the reference
          acc[m] += wv[e] * xe;
        }
      }
    }
  }
#pragma unroll
  for (int m = 0; m < SL_MAXM; ++m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], o);
  }
  if (lane == 0) {
    const float b = bias ? __half2float(bias[n]) : 0.f;
    for (int m = 0; m < M; ++m) {
      float y = __half2float(__float2half_rn(acc[m] + b));  // nn.Linear output is fp16 before the activation
      if (act_out == 1) y = silu_f(y);
      if (out_scale != 1.f) y = __half2float(__float2half_rn(y)) * out_scale;  // `module(x) * scale` on an fp16 tensor
      if (addend) y = __half2float(__float2half_rn(y)) + __half2float(addend[m * ld_add + n]);  // fp16 tensor add
      out[m * ldo + n] = __float2half_rn(y);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// sinusoid(t, dim) = [cos(t f_j), sin(t f_j)], f_j = exp(-ln(10000) j / half)   (flip_sin_to_cos=True, shift 0)
// ---------------------------------------------------------------------------------------------------------------
__global__ void sinusoid_kernel(const float* __restrict__ t, const int* __restrict__ step, __half* __restrict__ out,
                                long long ldo, int n, int dim) {
  pdl_launch_dependents();
  pdl_wait();
  const int half_dim = dim >> 1;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half_dim) return;
  const int i = idx / half_dim, j = idx - i * half_dim;
  const float tv = step ? t[*step] : t[i];
  const float f = expf(-9.210340371976184f * (float)j / (float)half_dim);
  const float a = tv * f;
  out[i * ldo + j] = __float2half_rn(cosf(a));
  out[i * ldo + half_dim + j] = __float2half_rn(sinf(a));
}

__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int H, int W, int CV) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)B * 2 * H * 2 * W * CV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    long long r = i / CV;
    const int ox = (int)(r % (2 * W));
    r /= (2 * W);
    const int oy = (int)(r % (2 * H));
    const int b = (int)(r / (2 * H));
    out[i] = x[(((long long)b * H + (oy >> 1)) * W + (ox >> 1)) * CV + cv];
  }
}

__global__ void concat_kernel(const uint4* __restrict__ x0, int CV0, const uint4* __restrict__ x1, int CV1,
                              uint4* __restrict__ out, long long rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int CV = CV0 + CV1;
  const long long total = rows * CV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    const long long r = i / CV;
    out[i] = cv < CV0 ? x0[r * CV0 + cv] : x1[r * CV1 + (cv - CV0)];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// CFG + Euler. Rounding points follow the reference's fp16 tensor arithmetic (custom_pipelines.py:348-350) and
// diffusers' EulerDiscreteScheduler.step (fp32 inside, result cast back to fp16).
// ---------------------------------------------------------------------------------------------------------------
__global__ void euler_cfg_kernel(const __half* __restrict__ noise, __half* __restrict__ latents,
                                 __half* __restrict__ model_in, const float* __restrict__ sigmas,
                                 const int* __restrict__ step, float guidance, long long per_image, int n_images) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = *step;
  const float sigma = sigmas[i], sigma_next = sigmas[i + 1];
  const float den_next = sqrtf(sigma_next * sigma_next + 1.f);
  const long long total = per_image * n_images;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const float u = __half2float(noise[idx]);
    const float c = __half2float(noise[total + idx]);
    const float d1 = __half2float(__float2half_rn(c - u));
    const float d2 = __half2float(__float2half_rn(guidance * d1));
    const float eps = __half2float(__float2half_rn(u + d2));
    const float x = __half2float(latents[idx]);
    // [3P] diffusers: `sample - sigma_hat * model_output` multiplies a 0-dim fp32 sigma with the fp16 model output,
    // so the product is an fp16 tensor (type promotion keeps the dimensioned tensor's dtype)
    const float x0 = x - __half2float(__float2half_rn(sigma * eps));
    const float deriv = (x - x0) / sigma;
    const float xn = x + deriv * (sigma_next - sigma);
    const __half xh = __float2half_rn(xn);
    latents[idx] = xh;
    const __half mi = __float2half_rn(__half2float(xh) / den_next);
    model_in[idx] = mi;
    model_in[total + idx] = mi;
  }
}
// General form of the step (custom_pipelines.py:346-357): classifier-free guidance on or off (:223,332,348) and the
// optional guidance rescale of :352-354 ([3P] diffusers rescale_noise_cfg: per-image unbiased std of the text branch
// and of the guided prediction over all non-batch elements, fp16 tensors -> fp16 rounding points).  ONE block per
// image: a first sweep forms the guided prediction and its statistics (double accumulators, fixed reduction order:
// deterministic), a second sweep -- the image is L1/L2 resident -- applies rescale + Euler.  n_images blocks of
// 1024 threads; a 4 x 128 x 128 latent is 64 elements per thread.
__global__ void __launch_bounds__(1024) euler_ex_kernel(const __half* __restrict__ noise, __half* __restrict__ latents,
                                                         __half* __restrict__ model_in,
                                                         const float* __restrict__ sigmas, const int* __restrict__ step,
                                                         float guidance, float rescale, long long per_image,
                                                         int n_images, int cfg) {
  pdl_launch_dependents();
  pdl_wait();
  const int img = blockIdx.x;
  const int i = *step;
  const float sigma = sigmas[i], sigma_next = sigmas[i + 1];
  const float den_next = sqrtf(sigma_next * sigma_next + 1.f);
  const long long total = per_image * n_images;
  const long long base = (long long)img * per_image;
  auto guided = [&](long long idx, float& c_out) -> float {
    if (!cfg) {
      c_out = __half2float(noise[idx]);
      return c_out;
    }
    const float u = __half2float(noise[idx]);
    const float c = __half2float(noise[total + idx]);
    c_out = c;
    const float d1 = __half2float(__float2half_rn(c - u));
    const float d2 = __half2float(__float2half_rn(guidance * d1));
    return __half2float(__float2half_rn(u + d2));
  };
  float factor = 1.f;   // fp16(std_text / std_cfg)
  if (cfg && rescale > 0.f) {
    double s_t = 0.0, q_t = 0.0, s_g = 0.0, q_g = 0.0;
    for (long long e = threadIdx.x; e < per_image; e += blockDim.x) {
      float c;
      const float g = guided(base + e, c);
      s_t += c;
      q_t += (double)c * c;
      s_g += g;
      q_g += (double)g * g;
    }
    __shared__ double red[4][32];
    __shared__ float s_factor;
    double v[4] = {s_t, q_t, s_g, q_g};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
      if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double t[4] = {0, 0, 0, 0};
      const int nw = (blockDim.x + 31) >> 5;
      for (int k = 0; k < 4; ++k)
        for (int w = 0; w < nw; ++w) t[k] += red[k][w];
      const double n = (double)per_image;
      const double var_t = fmax((t[1] - t[0] * t[0] / n) / (n - 1.0), 0.0);
      const double var_g = fmax((t[3] - t[2] * t[2] / n) / (n - 1.0), 0.0);
      const float std_t = __half2float(__float2half_rn((float)sqrt(var_t)));   // torch.std of an fp16 tensor -> fp16
      const float std_g = __half2float(__float2half_rn((float)sqrt(var_g)));
      s_factor = __half2float(__float2half_rn(std_t / std_g));
    }
    __syncthreads();
    factor = s_factor;
  }
  for (long long e = threadIdx.x; e < per_image; e += blockDim.x) {
    const long long idx = base + e;
    float c;
    float eps = guided(idx, c);
    if (cfg && rescale > 0.f) {
      const float resc = __half2float(__float2half_rn(eps * factor));                  // noise_cfg * (std_text / std_cfg)
      const float a = __half2float(__float2half_rn(rescale * resc));
      const float b = __half2float(__float2half_rn((1.f - rescale) * eps));
      eps = __half2float(__float2half_rn(a + b));
    }
    const float x = __half2float(latents[idx]);
    const float x0 = x - __half2float(__float2half_rn(sigma * eps));
    const float deriv = (x - x0) / sigma;
    const float xn = x + deriv * (sigma_next - sigma);
    const __half xh = __float2half_rn(xn);
    latents[idx] = xh;
    const __half mi = __float2half_rn(__half2float(xh) / den_next);
    model_in[idx] = mi;
    if (cfg) model_in[total + idx] = mi;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Inpainting step ([3P] diffusers==0.30.0 StableDiffusionXLInpaintPipeline, 4-channel UNet): the transition of
// euler_cfg_kernel / euler_ex_kernel (same rounding points), then, before the next step's input is formed, the blend
//   proper = i + 1 < blend_end ? fp16(img + fp16(noise * fp16(sigma[i+1]))) : img     (add_noise after step())
//   x      = fp16(fp16(fp16(1 - m) * proper) + fp16(m * x_euler))                      (fp16 tensor arithmetic)
// with m = mask[b, pixel] broadcast over the 4 latent channels.  The last step of the loop blends with the clean
// image latents even when sigma[blend_end] is not 0 (denoising_end).  image_latents / noise: [n,4,h,w], mask [n,1,h,w].
// ---------------------------------------------------------------------------------------------------------------
struct InpaintArgs {
  const __half* image_latents;
  const __half* noise;
  const __half* mask;
  long long hw;          // pixels per image: n_per_image / 4
  bool renoise;          // i + 1 < blend_end
  float sig_next16;      // fp16(sigma[i+1])
};

// One element: Euler update of the guided prediction `eps`, mask blend, latents and next-step input written.
__device__ __forceinline__ void euler_inpaint_elem(long long idx, float eps, float sigma, float sigma_next, float den_next,
                                                   const InpaintArgs& ia, long long per_image, long long total, int cfg,
                                                   __half* __restrict__ latents, __half* __restrict__ model_in) {
  const float x = __half2float(latents[idx]);
  const float x0 = x - __half2float(__float2half_rn(sigma * eps));
  const float deriv = (x - x0) / sigma;
  const float xn = x + deriv * (sigma_next - sigma);
  const float xe = __half2float(__float2half_rn(xn));
  const long long b = idx / per_image;
  const float m = __half2float(ia.mask[b * ia.hw + (idx - b * per_image) % ia.hw]);
  float proper = __half2float(ia.image_latents[idx]);
  if (ia.renoise) proper = __half2float(__float2half_rn(proper + __half2float(__float2half_rn(__half2float(ia.noise[idx]) * ia.sig_next16))));
  const float keep = __half2float(__float2half_rn(__half2float(__float2half_rn(1.f - m)) * proper));
  const float gen = __half2float(__float2half_rn(m * xe));
  const __half xh = __float2half_rn(keep + gen);
  latents[idx] = xh;
  const __half mi = __float2half_rn(__half2float(xh) / den_next);
  model_in[idx] = mi;
  if (cfg) model_in[total + idx] = mi;
}

// Without guidance_rescale: grid-stride over all elements.  With it: one block per image (blockIdx.x = image), the
// per-image std ratio first, reduced in the order of euler_ex_kernel so both forms give the same factor.
__global__ void __launch_bounds__(1024) euler_inpaint_kernel(const __half* __restrict__ noise, __half* __restrict__ latents,
                                                             __half* __restrict__ model_in, const float* __restrict__ sigmas,
                                                             const int* __restrict__ step, float guidance, float rescale,
                                                             long long per_image, int n_images, int cfg,
                                                             const __half* __restrict__ image_latents,
                                                             const __half* __restrict__ blend_noise,
                                                             const __half* __restrict__ mask,
                                                             const int* __restrict__ blend_end) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = *step;
  const float sigma = sigmas[i], sigma_next = sigmas[i + 1];
  const float den_next = sqrtf(sigma_next * sigma_next + 1.f);
  const long long total = per_image * n_images;
  const InpaintArgs ia{image_latents, blend_noise, mask, per_image / 4, i + 1 < *blend_end,
                       __half2float(__float2half_rn(sigma_next))};
  auto guided = [&](long long idx, float& c_out) -> float {
    if (!cfg) {
      c_out = __half2float(noise[idx]);
      return c_out;
    }
    const float u = __half2float(noise[idx]);
    const float c = __half2float(noise[total + idx]);
    c_out = c;
    const float d1 = __half2float(__float2half_rn(c - u));
    const float d2 = __half2float(__float2half_rn(guidance * d1));
    return __half2float(__float2half_rn(u + d2));
  };
  const bool resc = cfg && rescale > 0.f;
  if (!resc) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
      float c;
      euler_inpaint_elem(idx, guided(idx, c), sigma, sigma_next, den_next, ia, per_image, total, cfg, latents, model_in);
    }
    return;
  }
  const long long base = (long long)blockIdx.x * per_image;
  double s_t = 0.0, q_t = 0.0, s_g = 0.0, q_g = 0.0;
  for (long long e = threadIdx.x; e < per_image; e += blockDim.x) {
    float c;
    const float g = guided(base + e, c);
    s_t += c;
    q_t += (double)c * c;
    s_g += g;
    q_g += (double)g * g;
  }
  __shared__ double red[4][32];
  __shared__ float s_factor;
  double v[4] = {s_t, q_t, s_g, q_g};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[4] = {0, 0, 0, 0};
    const int nw = (blockDim.x + 31) >> 5;
    for (int k = 0; k < 4; ++k)
      for (int w = 0; w < nw; ++w) t[k] += red[k][w];
    const double n = (double)per_image;
    const double var_t = fmax((t[1] - t[0] * t[0] / n) / (n - 1.0), 0.0);
    const double var_g = fmax((t[3] - t[2] * t[2] / n) / (n - 1.0), 0.0);
    const float std_t = __half2float(__float2half_rn((float)sqrt(var_t)));
    const float std_g = __half2float(__float2half_rn((float)sqrt(var_g)));
    s_factor = __half2float(__float2half_rn(std_t / std_g));
  }
  __syncthreads();
  const float factor = s_factor;
  for (long long e = threadIdx.x; e < per_image; e += blockDim.x) {
    float c;
    const float eps = guided(base + e, c);
    const float r = __half2float(__float2half_rn(eps * factor));
    const float a = __half2float(__float2half_rn(rescale * r));
    const float b = __half2float(__float2half_rn((1.f - rescale) * eps));
    euler_inpaint_elem(base + e, __half2float(__float2half_rn(a + b)), sigma, sigma_next, den_next, ia, per_image, total,
                       cfg, latents, model_in);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// DPM-Solver++ 2M step ([3P] diffusers==0.30.0 DPMSolverMultistepScheduler, dpmsolver++ / midpoint / epsilon).  The
// guided prediction is formed as in euler_cfg_kernel / euler_ex_kernel; every per-step scalar comes from the host
// table coeffs[i, IH_DPM_COEFFS] (torch fp32 0-dim arithmetic, the diffusers expressions), so the kernel has no exp /
// log and reproduces the fp16 / fp32 tensor arithmetic of convert_model_output + step:
//   x0  = fp16(fp16(x - fp16(sigma_s * eps)) * inv_alpha_s)       (ATen divides by a CPU scalar as a * (1 / b))
//   out = fp32(ratio * x) - fp16(c * x0)                            first order
//       - fp16(c_half * fp16(inv_r0 * fp16(x0 - prev_x0)))          second order (midpoint), prev_x0 = last step's x0
//   latents = model_in = prev... = fp16(out); prev_x0 <- x0
// Products and differences use explicit _rn intrinsics so that nvcc cannot contract them into FMAs that torch does not
// form.  A step is first order iff i == *loop_begin or coeffs[i].first != 0; both are read-only here.
// ---------------------------------------------------------------------------------------------------------------
struct DpmCoeffs {
  float sigma_s, inv_alpha_s, ratio, c, c_half, inv_r0;
  bool second;
};

__device__ __forceinline__ float cfg_guided(const __half* __restrict__ noise, long long idx, long long total, int cfg,
                                            float guidance, float& c_out) {
  if (!cfg) {
    c_out = __half2float(noise[idx]);
    return c_out;
  }
  const float u = __half2float(noise[idx]);
  const float c = __half2float(noise[total + idx]);
  c_out = c;
  const float d1 = __half2float(__float2half_rn(c - u));
  const float d2 = __half2float(__float2half_rn(guidance * d1));
  return __half2float(__float2half_rn(u + d2));
}

__device__ __forceinline__ float h16(float v) { return __half2float(__float2half_rn(v)); }

__device__ __forceinline__ void dpm_elem(long long idx, float eps, const DpmCoeffs& k, long long total, int cfg,
                                         __half* __restrict__ latents, __half* __restrict__ model_in,
                                         __half* __restrict__ prev_x0) {
  const float x = __half2float(latents[idx]);
  const float x0 = h16(__fmul_rn(h16(__fsub_rn(x, h16(__fmul_rn(k.sigma_s, eps)))), k.inv_alpha_s));
  float out = __fsub_rn(__fmul_rn(k.ratio, x), h16(__fmul_rn(k.c, x0)));
  if (k.second) {
    const float d1 = h16(__fmul_rn(k.inv_r0, h16(__fsub_rn(x0, __half2float(prev_x0[idx])))));
    out = __fsub_rn(out, h16(__fmul_rn(k.c_half, d1)));
  }
  const __half xh = __float2half_rn(out);
  latents[idx] = xh;
  prev_x0[idx] = __float2half_rn(x0);
  model_in[idx] = xh;                      // scale_model_input is the identity for this scheduler
  if (cfg) model_in[total + idx] = xh;
}

// Without guidance_rescale: grid-stride over all elements.  With it: one block per image, the std ratio reduced in the
// order of euler_ex_kernel.
__global__ void __launch_bounds__(1024) dpm_solver_kernel(const __half* __restrict__ noise, __half* __restrict__ latents,
                                                          __half* __restrict__ model_in, __half* __restrict__ prev_x0,
                                                          const float* __restrict__ coeffs, const int* __restrict__ step,
                                                          const int* __restrict__ loop_begin, float guidance,
                                                          float rescale, long long per_image, int n_images, int cfg) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = *step;
  const float* row = coeffs + (long long)i * IH_DPM_COEFFS;
  const DpmCoeffs k{row[0], row[1], row[2], row[3], row[4], row[5], !(i == *loop_begin || row[6] != 0.f)};
  const long long total = per_image * n_images;
  const bool resc = cfg && rescale > 0.f;
  if (!resc) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
      float c;
      dpm_elem(idx, cfg_guided(noise, idx, total, cfg, guidance, c), k, total, cfg, latents, model_in, prev_x0);
    }
    return;
  }
  const long long base = (long long)blockIdx.x * per_image;
  double s_t = 0.0, q_t = 0.0, s_g = 0.0, q_g = 0.0;
  for (long long e = threadIdx.x; e < per_image; e += blockDim.x) {
    float c;
    const float g = cfg_guided(noise, base + e, total, cfg, guidance, c);
    s_t += c;
    q_t += (double)c * c;
    s_g += g;
    q_g += (double)g * g;
  }
  __shared__ double red[4][32];
  __shared__ float s_factor;
  double v[4] = {s_t, q_t, s_g, q_g};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
    if ((threadIdx.x & 31) == 0) red[q][threadIdx.x >> 5] = v[q];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[4] = {0, 0, 0, 0};
    const int nw = (blockDim.x + 31) >> 5;
    for (int q = 0; q < 4; ++q)
      for (int w = 0; w < nw; ++w) t[q] += red[q][w];
    const double n = (double)per_image;
    const double var_t = fmax((t[1] - t[0] * t[0] / n) / (n - 1.0), 0.0);
    const double var_g = fmax((t[3] - t[2] * t[2] / n) / (n - 1.0), 0.0);
    const float std_t = h16((float)sqrt(var_t));
    const float std_g = h16((float)sqrt(var_g));
    s_factor = h16(std_t / std_g);
  }
  __syncthreads();
  const float factor = s_factor;
  for (long long e = threadIdx.x; e < per_image; e += blockDim.x) {
    float c;
    const float eps = cfg_guided(noise, base + e, total, cfg, guidance, c);
    const float r = h16(eps * factor);
    const float a = h16(rescale * r);
    const float b = h16((1.f - rescale) * eps);
    dpm_elem(base + e, h16(a + b), k, total, cfg, latents, model_in, prev_x0);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Euler Ancestral step ([3P] diffusers==0.30.0 EulerAncestralDiscreteScheduler, epsilon).  The guided prediction is
// formed as in euler_cfg_kernel / euler_ex_kernel; the per-step scalars come from the host table
// coeffs[i, IH_EULER_A_COEFFS] (torch fp32 0-dim arithmetic) and the step's Gaussian noise from row i of a buffer the
// host fills from the caller's torch generator before the graph replays:
//   x0   = x - fp16(sigma * eps)             (sample = x.float(); sigma * fp16 tensor is an fp16 tensor)
//   prev = fp32(fp32((x - x0) * inv_sigma) * dt) + x      (ATen divides by a CPU scalar as a * (1 / b))
//   prev = fp16(prev + fp16(noise * sigma_up))
// then, when image latents are given, the inpainting blend of euler_inpaint_elem, and the next model input
// fp16(x * inv_den_next).  Explicit _rn intrinsics keep nvcc from forming FMAs that torch does not form.
// ---------------------------------------------------------------------------------------------------------------
struct EulerACoeffs {
  float sigma, inv_sigma, dt, sigma_up, inv_den_next;
};

// ia.image_latents == nullptr: no blend (text-to-image, image-to-image).
__device__ __forceinline__ void euler_a_elem(long long idx, float eps, const EulerACoeffs& k,
                                             const __half* __restrict__ step_noise, const InpaintArgs& ia,
                                             long long per_image, long long total, int cfg,
                                             __half* __restrict__ latents, __half* __restrict__ model_in) {
  const float x = __half2float(latents[idx]);
  const float x0 = __fsub_rn(x, h16(__fmul_rn(k.sigma, eps)));
  const float d = __fmul_rn(__fsub_rn(x, x0), k.inv_sigma);
  const float prev = __fadd_rn(x, __fmul_rn(d, k.dt));
  float xa = h16(__fadd_rn(prev, h16(__fmul_rn(__half2float(step_noise[idx]), k.sigma_up))));
  if (ia.image_latents) {
    const long long b = idx / per_image;
    const float m = __half2float(ia.mask[b * ia.hw + (idx - b * per_image) % ia.hw]);
    float proper = __half2float(ia.image_latents[idx]);
    if (ia.renoise) proper = h16(__fadd_rn(proper, h16(__fmul_rn(__half2float(ia.noise[idx]), ia.sig_next16))));
    const float keep = h16(__fmul_rn(h16(__fsub_rn(1.f, m)), proper));
    xa = h16(__fadd_rn(keep, h16(__fmul_rn(m, xa))));
  }
  const __half xh = __float2half_rn(xa);
  latents[idx] = xh;
  const __half mi = __float2half_rn(__fmul_rn(xa, k.inv_den_next));
  model_in[idx] = mi;
  if (cfg) model_in[total + idx] = mi;
}

// fp16(std_text / std_guided) of image blockIdx.x (guidance_rescale), reduced in the order of euler_ex_kernel.
__device__ float cfg_rescale_factor(const __half* __restrict__ noise, long long base, long long per_image,
                                    long long total, float guidance) {
  double s_t = 0.0, q_t = 0.0, s_g = 0.0, q_g = 0.0;
  for (long long e = threadIdx.x; e < per_image; e += blockDim.x) {
    float c;
    const float g = cfg_guided(noise, base + e, total, 1, guidance, c);
    s_t += c;
    q_t += (double)c * c;
    s_g += g;
    q_g += (double)g * g;
  }
  __shared__ double red[4][32];
  __shared__ float s_factor;
  double v[4] = {s_t, q_t, s_g, q_g};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
    if ((threadIdx.x & 31) == 0) red[q][threadIdx.x >> 5] = v[q];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[4] = {0, 0, 0, 0};
    const int nw = (blockDim.x + 31) >> 5;
    for (int q = 0; q < 4; ++q)
      for (int w = 0; w < nw; ++w) t[q] += red[q][w];
    const double n = (double)per_image;
    const double var_t = fmax((t[1] - t[0] * t[0] / n) / (n - 1.0), 0.0);
    const double var_g = fmax((t[3] - t[2] * t[2] / n) / (n - 1.0), 0.0);
    s_factor = h16(h16((float)sqrt(var_t)) / h16((float)sqrt(var_g)));
  }
  __syncthreads();
  return s_factor;
}

// Without guidance_rescale: grid-stride over all elements.  With it: one block per image.
__global__ void __launch_bounds__(1024) euler_ancestral_kernel(
    const __half* __restrict__ noise, __half* __restrict__ latents, __half* __restrict__ model_in,
    const float* __restrict__ coeffs, const __half* __restrict__ step_noise, const int* __restrict__ step,
    float guidance, float rescale, long long per_image, int n_images, int cfg, const __half* __restrict__ image_latents,
    const __half* __restrict__ blend_noise, const __half* __restrict__ mask, const int* __restrict__ blend_end) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = *step;
  const float* row = coeffs + (long long)i * IH_EULER_A_COEFFS;
  const EulerACoeffs k{row[0], row[1], row[2], row[3], row[4]};
  const long long total = per_image * n_images;
  const __half* nz = step_noise + (long long)i * total;
  const InpaintArgs ia{image_latents, blend_noise, mask, per_image / 4, image_latents && i + 1 < *blend_end, row[5]};
  if (!(cfg && rescale > 0.f)) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
      float c;
      euler_a_elem(idx, cfg_guided(noise, idx, total, cfg, guidance, c), k, nz, ia, per_image, total, cfg, latents,
                   model_in);
    }
    return;
  }
  const long long base = (long long)blockIdx.x * per_image;
  const float factor = cfg_rescale_factor(noise, base, per_image, total, guidance);
  for (long long e = threadIdx.x; e < per_image; e += blockDim.x) {
    float c;
    const float eps = cfg_guided(noise, base + e, total, cfg, guidance, c);
    const float r = h16(eps * factor);
    const float a = h16(rescale * r);
    const float b = h16((1.f - rescale) * eps);
    euler_a_elem(base + e, h16(a + b), k, nz, ia, per_image, total, cfg, latents, model_in);
  }
}

// The loop's first model input in the convention of euler_ancestral_kernel: fp16(x * coeffs[*step, IN_SCALE]).
__global__ void euler_a_scale_input_kernel(const __half* __restrict__ latents, __half* __restrict__ model_in,
                                           const float* __restrict__ coeffs, const int* __restrict__ step,
                                           long long total, int duplicate) {
  pdl_launch_dependents();
  pdl_wait();
  const float s = coeffs[(long long)*step * IH_EULER_A_COEFFS + 6];
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const __half mi = __float2half_rn(__fmul_rn(__half2float(latents[idx]), s));
    model_in[idx] = mi;
    if (duplicate) model_in[total + idx] = mi;
  }
}

__global__ void step_inc_kernel(int* step) {
  pdl_launch_dependents();
  pdl_wait();
  *step += 1;
}

__global__ void scale_model_input_kernel(const __half* __restrict__ latents, __half* __restrict__ model_in,
                                         const float* __restrict__ sigmas, const int* __restrict__ step,
                                         long long total, int duplicate) {
  pdl_launch_dependents();
  pdl_wait();
  const float sigma = sigmas[*step];
  const float den = sqrtf(sigma * sigma + 1.f);
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const __half mi = __float2half_rn(__half2float(latents[idx]) / den);
    model_in[idx] = mi;
    if (duplicate) model_in[total + idx] = mi;   // CFG batch [uncond | cond] (custom_pipelines.py:332)
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Small generic attention (any head dims <= 128, few queries): one warp per (batch, head, query).
// HarmonyAttention's Cross_Attention (attention_processor.py:35-56): head_dim 40, value dim 64; scores are DIVIDED by
// `scale` = sqrt(head_dim) exactly like the reference (:45).
// ---------------------------------------------------------------------------------------------------------------
constexpr int SA_MAXK = 1024;
__global__ void attention_small_kernel(const __half* __restrict__ q, long long ldq, const __half* __restrict__ k,
                                       long long ldk, const __half* __restrict__ v, long long ldv,
                                       __half* __restrict__ out, long long ldo, int H, int Nq, int Nk, int dqk, int dv,
                                       float scale) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_p[];  // [warps][Nk]
  const int warp_in_block = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (blockDim.x >> 5) + warp_in_block;  // (b, h, iq)
  const int iq = gw % Nq;
  const int h = (gw / Nq) % H;
  const int b = gw / (Nq * H);
  float* p = s_p + warp_in_block * Nk;
  const __half* qr = q + ((long long)b * Nq + iq) * ldq + h * dqk;
  float mx = -INFINITY;
  for (int j = lane; j < Nk; j += 32) {
    const __half* kr = k + ((long long)b * Nk + j) * ldk + h * dqk;
    float acc = 0.f;
    for (int d = 0; d < dqk; ++d) acc += __half2float(qr[d]) * __half2float(kr[d]);
    // the reference rounds the fp16 matmul output before dividing by the scale (attention_processor.py:45)
    acc = __half2float(__float2half_rn(__half2float(__float2half_rn(acc)) / scale));
    p[j] = acc;
    mx = fmaxf(mx, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < Nk; j += 32) {
    const float e = __expf(p[j] - mx);
    p[j] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  __syncwarp();
  const float inv = 1.f / sum;
  for (int d = lane; d < dv; d += 32) {
    float acc = 0.f;
    for (int j = 0; j < Nk; ++j) {
      const float pj = __half2float(__float2half_rn(p[j] * inv));  // softmax output is an fp16 tensor
      acc += pj * __half2float(v[((long long)b * Nk + j) * ldv + h * dv + d]);
    }
    out[((long long)b * Nq + iq) * ldo + h * dv + d] = __float2half_rn(acc);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Generic SDPA for the CLIP towers (scope row f2: [3P] transformers CLIPAttention as the reference calls it through
// ip_adapter.py:81-84,163-164 (vision, head_dim 104 for ViT-bigG) and encode_prompt :292-319 (text, causal mask)):
// softmax(q k^T * scale [+ causal mask]) v with fp32 scores / softmax, one warp per (batch, head, query); keys are
// strided over the lanes with 16-byte loads, the PV sweep gives each lane dv/32 output channels.  head dims % 8 == 0.
// ---------------------------------------------------------------------------------------------------------------
__global__ void attention_generic_kernel(const __half* __restrict__ q, long long ldq, const __half* __restrict__ k,
                                         long long ldk, const __half* __restrict__ v, long long ldv,
                                         __half* __restrict__ out, long long ldo, int H, int Nq, int Nk, int dqk, int dv,
                                         float scale, int causal, long long total_warps) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_p[];  // [warps][Nk]
  const int warp_in_block = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const long long gw = (long long)blockIdx.x * (blockDim.x >> 5) + warp_in_block;  // (b, h, iq)
  if (gw >= total_warps) return;
  const int iq = (int)(gw % Nq);
  const int h = (int)((gw / Nq) % H);
  const int b = (int)(gw / ((long long)Nq * H));
  float* p = s_p + warp_in_block * Nk;
  const __half* qr = q + ((long long)b * Nq + iq) * ldq + h * dqk;
  const int nk_live = causal ? min(Nk, iq + 1 + (Nk - Nq)) : Nk;   // key j visible iff j <= iq (+ offset when Nk > Nq)
  float mx = -INFINITY;
  for (int j = lane; j < nk_live; j += 32) {
    const __half* kr = k + ((long long)b * Nk + j) * ldk + h * dqk;
    float acc = 0.f;
    for (int d = 0; d < dqk; d += 8) {
      float a[8], c[8];
      ld8(qr + d, a);
      ld8(kr + d, c);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc = fmaf(a[e], c[e], acc);
    }
    acc *= scale;
    p[j] = acc;
    mx = fmaxf(mx, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < nk_live; j += 32) {
    const float e = __expf(p[j] - mx);
    p[j] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  __syncwarp();
  const float inv = 1.f / sum;
  for (int d = lane; d < dv; d += 32) {
    float acc = 0.f;
    const __half* vc = v + (long long)b * Nk * ldv + h * dv + d;
    for (int j = 0; j < nk_live; ++j) acc = fmaf(p[j], __half2float(vc[(long long)j * ldv]), acc);
    out[((long long)b * Nq + iq) * ldo + h * dv + d] = __float2half_rn(acc * inv);
  }
}

// out[b, t, :] = tok_emb[ids[b, t], :] + pos_emb[t, :]   ([3P] CLIPTextEmbeddings; one 16-byte vector per thread)
__global__ void embed_tokens_kernel(const int* __restrict__ ids, const __half* __restrict__ tok, const __half* __restrict__ pos,
                                    __half* __restrict__ out, int rows, int T, int C8, int vocab) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)rows * C8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / C8), c = (int)(i - (long long)r * C8);
    int id = ids[r];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const uint4 a = reinterpret_cast<const uint4*>(tok)[(long long)id * C8 + c];
    const uint4 b = reinterpret_cast<const uint4*>(pos)[(long long)(r % T) * C8 + c];
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack_half2(aw[e]), g = unpack_half2(bw[e]);
      o[e] = pack_half2(f.x + g.x, f.y + g.y);
    }
    reinterpret_cast<uint4*>(out)[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// CLIP-scorer front end (PNS judge): decoded image NCHW fp16 in [-1, 1] -> area-averaged S x S image -> [0, 1] ->
// (v - mean[c]) / std[c] -> patch rows [B * (S/P)^2, Kpad] with k = c*P*P + py*P + px (the layout of the flattened
// CLIP patch_embedding conv weight), zero padded to Kpad.  One thread per output pixel and channel.
__global__ void resize_patchify_kernel(const __half* __restrict__ img, __half* __restrict__ out, int B, int C, int Hin,
                                       int Win, int S, int P, int Kpad, float m0, float m1, float m2, float s0, float s1,
                                       float s2) {
  pdl_launch_dependents();
  pdl_wait();
  const int G = S / P;
  const long long total = (long long)B * G * G * Kpad;
  const float fy = (float)Hin / (float)S, fx = (float)Win / (float)S;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int kk = (int)(i % Kpad);
    const long long row = i / Kpad;
    if (kk >= C * P * P) {
      out[i] = __float2half_rn(0.f);
      continue;
    }
    const int c = kk / (P * P), py = (kk / P) % P, px = kk % P;
    const int gx = (int)(row % G), gy = (int)((row / G) % G), b = (int)(row / ((long long)G * G));
    const int oy = gy * P + py, ox = gx * P + px;
    const float y0 = oy * fy, y1 = (oy + 1) * fy, x0 = ox * fx, x1 = (ox + 1) * fx;
    const int iy0 = (int)floorf(y0), iy1 = min(Hin, (int)ceilf(y1)), ix0 = (int)floorf(x0), ix1 = min(Win, (int)ceilf(x1));
    const __half* src = img + ((long long)b * C + c) * Hin * Win;
    float acc = 0.f, wsum = 0.f;
    for (int y = iy0; y < iy1; ++y) {
      const float wy = fminf(y1, (float)(y + 1)) - fmaxf(y0, (float)y);
      for (int x = ix0; x < ix1; ++x) {
        const float wx = fminf(x1, (float)(x + 1)) - fmaxf(x0, (float)x);
        acc = fmaf(wy * wx, __half2float(src[(long long)y * Win + x]), acc);
        wsum += wy * wx;
      }
    }
    float vpx = fminf(fmaxf(acc / wsum * 0.5f + 0.5f, 0.f), 1.f);
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
    out[i] = __float2half_rn((vpx - mean) / sd);
  }
}

// out[i] = a[i] + b[i % period]  (16-byte vectors; period in elements, multiple of 8)
__global__ void add_bcast_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ out,
                                 long long nvec, long long period_vec) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const uint4 x = a[i], y = b[i % period_vec];
    const uint32_t xw[4] = {x.x, x.y, x.z, x.w}, yw[4] = {y.x, y.y, y.z, y.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack_half2(xw[e]), g = unpack_half2(yw[e]);
      o[e] = pack_half2(f.x + g.x, f.y + g.y);
    }
    out[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// out[b, :] = mean over n of x[b, n, :]   (fp32 accumulation; one thread per 8 channels)
__global__ void mean_tokens_kernel(const __half* __restrict__ x, __half* __restrict__ out, int n, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (c >= D) return;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  for (int i = 0; i < n; ++i) {
    float v[8];
    ld8(x + ((long long)b * n + i) * D + c, v);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += v[e];
  }
  uint4 o;
  const float inv = 1.f / (float)n;
  o.x = pack_half2(acc[0] * inv, acc[1] * inv);
  o.y = pack_half2(acc[2] * inv, acc[3] * inv);
  o.z = pack_half2(acc[4] * inv, acc[5] * inv);
  o.w = pack_half2(acc[6] * inv, acc[7] * inv);
  *reinterpret_cast<uint4*>(out + (long long)b * D + c) = o;
}

// Row softmax in place: x[r, :] <- softmax(x[r, :]) over `cols` fp16 values (fp32 statistics), one block per row, the row
// held in registers (cols <= 256 threads x 16 vectors x 8 = 32768).  Used by the single-head, head_dim 512 attention
// of the VAE decoder's mid block (scores = (q / sqrt(d)) k^T from the tensor-core GEMM).
constexpr int SMX_THREADS = 256;
constexpr int SMX_MAXV = 16;
__global__ void __launch_bounds__(SMX_THREADS) softmax_rows_kernel(__half* __restrict__ x, long long ld, int cols,
                                                                   int valid) {
  __shared__ float s_red[SMX_THREADS / 32];
  __shared__ float s_bcast;
  pdl_launch_dependents();
  pdl_wait();
  __half* row = x + (long long)blockIdx.x * ld;
  const int nv = cols >> 3;
  float v[SMX_MAXV][8];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < SMX_MAXV; ++i) {
    const int vi = threadIdx.x + i * SMX_THREADS;
    if (vi < nv) {
      ld8(row + vi * 8, v[i]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (vi * 8 + e >= valid) v[i][e] = -INFINITY;   // padding columns (keys past the sequence end) get weight 0
        mx = fmaxf(mx, v[i][e]);
      }
    }
  }
  auto block_reduce = [&](float val, bool is_max) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float other = __shfl_xor_sync(0xffffffffu, val, o);
      val = is_max ? fmaxf(val, other) : val + other;
    }
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = val;
    __syncthreads();
    if (threadIdx.x == 0) {
      float r = s_red[0];
      for (int w = 1; w < SMX_THREADS / 32; ++w) r = is_max ? fmaxf(r, s_red[w]) : r + s_red[w];   // fixed order
      s_bcast = r;
    }
    __syncthreads();
    const float out = s_bcast;
    __syncthreads();
    return out;
  };
  mx = block_reduce(mx, true);
  const float ml2 = mx * 1.4426950408889634f;
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < SMX_MAXV; ++i) {
    const int vi = threadIdx.x + i * SMX_THREADS;
    if (vi < nv) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        v[i][e] = ex2_approx(fmaf(v[i][e], 1.4426950408889634f, -ml2));
        sum += v[i][e];
      }
    }
  }
  sum = block_reduce(sum, false);
  const float inv = 1.f / sum;
#pragma unroll
  for (int i = 0; i < SMX_MAXV; ++i) {
    const int vi = threadIdx.x + i * SMX_THREADS;
    if (vi < nv) {
      uint4 o;
      o.x = pack_half2(v[i][0] * inv, v[i][1] * inv);
      o.y = pack_half2(v[i][2] * inv, v[i][3] * inv);
      o.z = pack_half2(v[i][4] * inv, v[i][5] * inv);
      o.w = pack_half2(v[i][6] * inv, v[i][7] * inv);
      *reinterpret_cast<uint4*>(row + vi * 8) = o;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The 4-channel ends of the UNet on the tensor-core GEMM:
//   conv_in : im2col of the NCHW latent -> A [B*H*W, 64] (k = ci*9 + ky*3 + kx, zero padded from 36 to 64 columns),
//             then ih_gemm_f16 with the OIHW weight flattened to [320, 36->64]
//   conv_out: ih_conv2d_f16 with Cout padded 4 -> 16, then this gather NHWC[.., 16] -> NCHW[B, 4, H, W]
// ---------------------------------------------------------------------------------------------------------------
__global__ void im2col3x3_nchw_kernel(const __half* __restrict__ x, __half* __restrict__ out, int B, int Cin, int H,
                                      int W, int Kpad) {
  pdl_launch_dependents();
  pdl_wait();
  const long long npix = (long long)B * H * W;
  const int kv = Kpad >> 3;  // 16-byte vectors per row
  const long long total = npix * kv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % kv);
    const long long pix = i / kv;
    const int xw = (int)(pix % W);
    const int yh = (int)((pix / W) % H);
    const int b = (int)(pix / ((long long)W * H));
    __align__(16) __half vals[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = v * 8 + e;
      __half hv = __float2half_rn(0.f);
      if (k < Cin * 9) {
        const int ci = k / 9, t = k - ci * 9;
        const int yy = yh + t / 3 - 1, xx = xw + t % 3 - 1;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) hv = x[(((long long)b * Cin + ci) * H + yy) * W + xx];
      }
      vals[e] = hv;
    }
    *reinterpret_cast<uint4*>(out + pix * Kpad + v * 8) = *reinterpret_cast<const uint4*>(vals);
  }
}

__global__ void nhwc_to_nchw_kernel(const __half* __restrict__ x, long long ldc, __half* __restrict__ out, int B,
                                    long long HW, int C) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)B * C * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % HW;
    const int c = (int)((i / HW) % C);
    const int b = (int)(i / (HW * C));
    out[i] = x[((long long)b * HW + p) * ldc + c];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Image-to-image initial latents from the VAE encoder's moments: posterior sample, scaling and the scheduler's
// add_noise in one pass.  Rounding points of [3P] diffusers==0.30.0 StableDiffusionXLImg2ImgPipeline.prepare_latents
// (latents fp16) -> DiagonalGaussianDistribution.sample -> EulerDiscreteScheduler.add_noise:
//   eps fp32 (force_upcast: the posterior is fp32):
//     lv = clamp(logvar, -30, 20);  z = mean + exp(0.5 lv) * eps          (fp32, mul and add rounded separately)
//   eps fp16 (no upcast: every posterior op rounds to fp16):
//     lv = clamp(logvar, -30, 20);  sd = fp16(exp(fp16(0.5 lv)));  z = fp16(mean + fp16(sd * eps))
//   then  z = fp16(z);  z = fp16(scaling_factor * z);  x = fp16(z + fp16(noise * fp16(sigma)))
// moments: NHWC [Bm, HW, ldc], mean = channels [0, C), logvar = [C, 2C) (the padded conv_out of the encoder).
// Output image b uses moments[b % Bm] and eps[b % Be] (diffusers tiles a batch of encoded latents with torch.cat).
// eps, noise and out are NCHW; noise and out hold B images.
// ---------------------------------------------------------------------------------------------------------------
__global__ void vae_posterior_noise_kernel(const __half* __restrict__ moments, long long ldc, const void* __restrict__ eps,
                                           int eps_f32, const __half* __restrict__ noise, __half* __restrict__ out, int B,
                                           int Bm, int Be, long long HW, int C, float scaling_factor, float sigma) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)B * C * HW;
  const float sig16 = __half2float(__float2half_rn(sigma));
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % HW;
    const int c = (int)((i / HW) % C);
    const int b = (int)(i / (HW * C));
    const __half* mrow = moments + ((long long)(b % Bm) * HW + p) * ldc;
    const float mean = __half2float(mrow[c]);
    const float lv = fminf(fmaxf(__half2float(mrow[C + c]), -30.f), 20.f);
    const long long ei = ((long long)(b % Be) * C + c) * HW + p;
    float z;
    if (eps_f32) {
      z = __fadd_rn(mean, __fmul_rn(expf(0.5f * lv), static_cast<const float*>(eps)[ei]));
    } else {
      const float sd = __half2float(__float2half_rn(expf(__half2float(__float2half_rn(0.5f * lv)))));
      const float e = __half2float(static_cast<const __half*>(eps)[ei]);
      z = __half2float(__float2half_rn(mean + __half2float(__float2half_rn(sd * e))));
    }
    const float zs = __half2float(__float2half_rn(__fmul_rn(scaling_factor, __half2float(__float2half_rn(z)))));
    const float ns = __half2float(__float2half_rn(__half2float(noise[i]) * sig16));   // exact product of two fp16
    out[i] = __float2half_rn(zs + ns);
  }
}

static int grid_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace ih

using namespace ih;

extern "C" int ih_linear_small_f16(const void* x, long long ldx, const void* w, const void* bias, const void* addend,
                                   long long ld_add, void* out, long long ldo, int M, int N, int K, int act_in,
                                   int act_out, float out_scale, void* stream) {
  IH_CHECK(x && w && out, IH_ERR_ARG, "ih_linear_small_f16: null pointer");
  IH_CHECK(M >= 1 && M <= 64, IH_ERR_SHAPE, "ih_linear_small_f16: M=%d must be in [1,64] (use ih_gemm_f16)", M);
  IH_CHECK(K % 8 == 0 && ldx % 8 == 0, IH_ERR_ALIGN, "ih_linear_small_f16: K and ldx must be multiples of 8");
  const int warps = 8;
  for (int m0 = 0; m0 < M; m0 += SL_MAXM) {  // row chunks of 8 (W is re-read from L2 for the later chunks)
    const int mc = (M - m0) < SL_MAXM ? (M - m0) : SL_MAXM;
    IH_CUDA(launch_kernel(linear_small_kernel, dim3((N + warps - 1) / warps), dim3(warps * 32), (size_t)(0), (cudaStream_t)stream, 
        (const __half*)x + m0 * ldx, ldx, (const __half*)w, (const __half*)bias,
        addend ? (const __half*)addend + m0 * ld_add : nullptr, ld_add, (__half*)out + m0 * ldo, ldo, mc, N, K,
        act_in, act_out, out_scale));
  }
  return 0;
}

extern "C" int ih_sinusoid_f16(const void* t_f32, const void* step_i32, void* out, long long ldo, int n, int dim,
                               void* stream) {
  IH_CHECK(t_f32 && out && dim % 2 == 0, IH_ERR_ARG, "ih_sinusoid_f16: bad arguments");
  const int total = n * (dim / 2);
  IH_CUDA(launch_kernel(sinusoid_kernel, dim3((total + 255) / 256), dim3(256), (size_t)(0), (cudaStream_t)stream, (const float*)t_f32, (const int*)step_i32,
                                                                         (__half*)out, ldo, n, dim));
  return 0;
}

extern "C" int ih_upsample2x_f16(const void* x, void* out, int B, int H, int W, int C, void* stream) {
  IH_CHECK(x && out && C % 8 == 0, IH_ERR_ARG, "ih_upsample2x_f16: bad arguments");
  const long long total = (long long)B * 4 * H * W * (C / 8);
  IH_CUDA(launch_kernel(upsample2x_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, (const uint4*)x, (uint4*)out, B, H, W,
                                                                            C / 8));
  return 0;
}

extern "C" int ih_concat_f16(const void* x0, int C0, const void* x1, int C1, void* out, long long rows, void* stream) {
  IH_CHECK(x0 && x1 && out && C0 % 8 == 0 && C1 % 8 == 0, IH_ERR_ARG, "ih_concat_f16: bad arguments");
  const long long total = rows * ((C0 + C1) / 8);
  IH_CUDA(launch_kernel(concat_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, (const uint4*)x0, C0 / 8, (const uint4*)x1,
                                                                        C1 / 8, (uint4*)out, rows));
  return 0;
}

extern "C" int ih_euler_cfg_step(const void* noise_pred, void* latents, void* model_in, const void* sigmas, void* step,
                                 float guidance, long long n_per_image, int n_images, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  IH_CHECK(noise_pred && latents && model_in && sigmas && step, IH_ERR_ARG, "ih_euler_cfg_step: null pointer");
  const long long total = n_per_image * n_images;
  IH_CUDA(launch_kernel(euler_cfg_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)(0), stream, (const __half*)noise_pred, (__half*)latents,
                                                             (__half*)model_in, (const float*)sigmas,
                                                             (const int*)step, guidance, n_per_image, n_images));
  IH_CUDA(launch_kernel(step_inc_kernel, dim3(1), dim3(1), (size_t)(0), stream, (int*)step));
  return 0;
}

extern "C" int ih_euler_step_ex(const void* noise_pred, void* latents, void* model_in, const void* sigmas, void* step,
                                float guidance, float guidance_rescale, long long n_per_image, int n_images,
                                int use_cfg, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  IH_CHECK(noise_pred && latents && model_in && sigmas && step, IH_ERR_ARG, "ih_euler_step_ex: null pointer");
  IH_CHECK(n_per_image > 1 && n_images > 0, IH_ERR_SHAPE, "ih_euler_step_ex: bad shape");
  IH_CHECK(guidance_rescale >= 0.f && guidance_rescale <= 1.f, IH_ERR_ARG, "ih_euler_step_ex: guidance_rescale outside [0, 1]");
  IH_CUDA(launch_kernel(euler_ex_kernel, dim3(n_images), dim3(1024), (size_t)(0), stream, (const __half*)noise_pred,
                        (__half*)latents, (__half*)model_in, (const float*)sigmas, (const int*)step, guidance,
                        guidance_rescale, n_per_image, n_images, use_cfg ? 1 : 0));
  IH_CUDA(launch_kernel(step_inc_kernel, dim3(1), dim3(1), (size_t)(0), stream, (int*)step));
  return 0;
}

extern "C" int ih_euler_inpaint_step(const void* noise_pred, void* latents, void* model_in, const void* sigmas, void* step,
                                     float guidance, float guidance_rescale, long long n_per_image, int n_images,
                                     int use_cfg, const void* image_latents, const void* noise, const void* mask,
                                     const void* blend_end, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  IH_CHECK(noise_pred && latents && model_in && sigmas && step && image_latents && noise && mask && blend_end, IH_ERR_ARG,
           "ih_euler_inpaint_step: null pointer");
  IH_CHECK(n_per_image > 1 && n_per_image % 4 == 0 && n_images > 0, IH_ERR_SHAPE,
           "ih_euler_inpaint_step: n_per_image=%lld must be 4 latent channels x pixels", n_per_image);
  IH_CHECK(guidance_rescale >= 0.f && guidance_rescale <= 1.f, IH_ERR_ARG,
           "ih_euler_inpaint_step: guidance_rescale outside [0, 1]");
  const int cfg = use_cfg ? 1 : 0;
  const bool per_image = cfg && guidance_rescale > 0.f;
  const long long total = n_per_image * n_images;
  IH_CUDA(launch_kernel(euler_inpaint_kernel, dim3(per_image ? n_images : grid_for(total, 256)), dim3(per_image ? 1024 : 256),
                        (size_t)(0), stream, (const __half*)noise_pred, (__half*)latents, (__half*)model_in,
                        (const float*)sigmas, (const int*)step, guidance, guidance_rescale, n_per_image, n_images, cfg,
                        (const __half*)image_latents, (const __half*)noise, (const __half*)mask, (const int*)blend_end));
  IH_CUDA(launch_kernel(step_inc_kernel, dim3(1), dim3(1), (size_t)(0), stream, (int*)step));
  return 0;
}

extern "C" int ih_dpm_solver_step(const void* noise_pred, void* latents, void* model_in, void* prev_x0,
                                  const void* coeffs, void* step, const void* loop_begin, float guidance,
                                  float guidance_rescale, long long n_per_image, int n_images, int use_cfg,
                                  void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  IH_CHECK(noise_pred && latents && model_in && prev_x0 && coeffs && step && loop_begin, IH_ERR_ARG,
           "ih_dpm_solver_step: null pointer");
  IH_CHECK(n_per_image > 1 && n_images > 0, IH_ERR_SHAPE, "ih_dpm_solver_step: bad shape");
  IH_CHECK(guidance_rescale >= 0.f && guidance_rescale <= 1.f, IH_ERR_ARG,
           "ih_dpm_solver_step: guidance_rescale outside [0, 1]");
  const int cfg = use_cfg ? 1 : 0;
  const bool per_image = cfg && guidance_rescale > 0.f;
  const long long total = n_per_image * n_images;
  IH_CUDA(launch_kernel(dpm_solver_kernel, dim3(per_image ? n_images : grid_for(total, 256)), dim3(per_image ? 1024 : 256),
                        (size_t)(0), stream, (const __half*)noise_pred, (__half*)latents, (__half*)model_in,
                        (__half*)prev_x0, (const float*)coeffs, (const int*)step, (const int*)loop_begin, guidance,
                        guidance_rescale, n_per_image, n_images, cfg));
  IH_CUDA(launch_kernel(step_inc_kernel, dim3(1), dim3(1), (size_t)(0), stream, (int*)step));
  return 0;
}

extern "C" int ih_euler_ancestral_step(const void* noise_pred, void* latents, void* model_in, const void* coeffs,
                                       const void* step_noise, void* step, float guidance, float guidance_rescale,
                                       long long n_per_image, int n_images, int use_cfg, const void* image_latents,
                                       const void* blend_noise, const void* mask, const void* blend_end,
                                       void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  IH_CHECK(noise_pred && latents && model_in && coeffs && step_noise && step, IH_ERR_ARG,
           "ih_euler_ancestral_step: null pointer");
  const bool blend = image_latents != nullptr;
  IH_CHECK(blend == (blend_noise != nullptr) && blend == (mask != nullptr) && blend == (blend_end != nullptr),
           IH_ERR_ARG, "ih_euler_ancestral_step: image_latents, blend_noise, mask and blend_end go together");
  IH_CHECK(n_per_image > 1 && n_images > 0 && (!blend || n_per_image % 4 == 0), IH_ERR_SHAPE,
           "ih_euler_ancestral_step: bad shape");
  IH_CHECK(guidance_rescale >= 0.f && guidance_rescale <= 1.f, IH_ERR_ARG,
           "ih_euler_ancestral_step: guidance_rescale outside [0, 1]");
  const int cfg = use_cfg ? 1 : 0;
  const bool per_image = cfg && guidance_rescale > 0.f;
  const long long total = n_per_image * n_images;
  IH_CUDA(launch_kernel(euler_ancestral_kernel, dim3(per_image ? n_images : grid_for(total, 256)),
                        dim3(per_image ? 1024 : 256), (size_t)(0), stream, (const __half*)noise_pred, (__half*)latents,
                        (__half*)model_in, (const float*)coeffs, (const __half*)step_noise, (const int*)step, guidance,
                        guidance_rescale, n_per_image, n_images, cfg, (const __half*)image_latents,
                        (const __half*)blend_noise, (const __half*)mask, (const int*)blend_end));
  IH_CUDA(launch_kernel(step_inc_kernel, dim3(1), dim3(1), (size_t)(0), stream, (int*)step));
  return 0;
}

extern "C" int ih_euler_ancestral_scale_input(const void* latents, void* model_in, const void* coeffs, const void* step,
                                              long long total, int duplicate, void* stream) {
  IH_CHECK(latents && model_in && coeffs && step, IH_ERR_ARG, "ih_euler_ancestral_scale_input: null pointer");
  IH_CUDA(launch_kernel(euler_a_scale_input_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)(0),
                        (cudaStream_t)stream, (const __half*)latents, (__half*)model_in, (const float*)coeffs,
                        (const int*)step, total, duplicate ? 1 : 0));
  return 0;
}

extern "C" int ih_scale_model_input_ex(const void* latents, void* model_in, const void* sigmas, const void* step,
                                       long long total, int duplicate, void* stream) {
  IH_CHECK(latents && model_in && sigmas && step, IH_ERR_ARG, "ih_scale_model_input_ex: null pointer");
  IH_CUDA(launch_kernel(scale_model_input_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)(0), (cudaStream_t)stream, 
      (const __half*)latents, (__half*)model_in, (const float*)sigmas, (const int*)step, total, duplicate ? 1 : 0));
  return 0;
}

extern "C" int ih_attention_small_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                      long long ldv, void* out, long long ldo, int B, int H, int Nq, int Nk, int dqk,
                                      int dv, float scale, void* stream) {
  IH_CHECK(q && k && v && out, IH_ERR_ARG, "ih_attention_small_f16: null pointer");
  IH_CHECK(Nk >= 1 && Nk <= SA_MAXK && dqk >= 1 && dqk <= 128 && dv >= 1 && dv <= 128 && Nq >= 1, IH_ERR_SHAPE,
           "ih_attention_small_f16: Nk<=%d, head dims <= 128 required", SA_MAXK);
  const int warps = 4;
  const long long total = (long long)B * H * Nq;
  IH_CHECK(total % warps == 0 || true, IH_ERR_SHAPE, "unreachable");
  const int blocks = (int)((total + warps - 1) / warps);
  // pad the grid so every warp index is valid: the kernel indexes (b,h,iq) from the global warp id
  IH_CHECK(total == (long long)blocks * warps, IH_ERR_SHAPE,
           "ih_attention_small_f16: B*H*Nq = %lld must be a multiple of %d", total, warps);
  IH_CUDA(launch_kernel(attention_small_kernel, dim3(blocks), dim3(warps * 32), (size_t)(warps * Nk * sizeof(float)), (cudaStream_t)stream, 
      (const __half*)q, ldq, (const __half*)k, ldk, (const __half*)v, ldv, (__half*)out, ldo, H, Nq, Nk, dqk, dv,
      scale));
  return 0;
}

extern "C" int ih_attention_generic_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                        long long ldv, void* out, long long ldo, int B, int H, int Nq, int Nk, int dqk,
                                        int dv, float scale, int causal, void* stream) {
  IH_CHECK(q && k && v && out, IH_ERR_ARG, "ih_attention_generic_f16: null pointer");
  IH_CHECK(Nk >= 1 && Nk <= 4096 && Nq >= 1 && dqk >= 8 && dqk <= 256 && dv >= 1 && dv <= 256 && dqk % 8 == 0 &&
               ldq % 8 == 0 && ldk % 8 == 0, IH_ERR_SHAPE,
           "ih_attention_generic_f16: Nk <= 4096, head dims <= 256, dqk / ldq / ldk multiples of 8 required");
  IH_CHECK(!causal || Nk >= Nq, IH_ERR_SHAPE, "ih_attention_generic_f16: causal needs Nk >= Nq");
  const int warps = 4;
  const long long total = (long long)B * H * Nq;
  const int blocks = (int)((total + warps - 1) / warps);
  const size_t smem = (size_t)warps * Nk * sizeof(float);
  static bool configured = false;
  if (!configured) {
    IH_CUDA(cudaFuncSetAttribute(attention_generic_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 4096 * 4));
    configured = true;
  }
  IH_CUDA(launch_kernel(attention_generic_kernel, dim3(blocks), dim3(warps * 32), smem, (cudaStream_t)stream,
                        (const __half*)q, ldq, (const __half*)k, ldk, (const __half*)v, ldv, (__half*)out, ldo, H, Nq, Nk,
                        dqk, dv, scale, causal ? 1 : 0, total));
  return 0;
}

extern "C" int ih_embed_tokens_f16(const void* ids_i32, const void* tok_emb, const void* pos_emb, void* out, int rows,
                                   int T, int C, int vocab, void* stream) {
  IH_CHECK(ids_i32 && tok_emb && pos_emb && out, IH_ERR_ARG, "ih_embed_tokens_f16: null pointer");
  IH_CHECK(rows > 0 && T > 0 && C % 8 == 0 && vocab > 0, IH_ERR_SHAPE, "ih_embed_tokens_f16: bad shape");
  const long long total = (long long)rows * (C / 8);
  IH_CUDA(launch_kernel(embed_tokens_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream,
                        (const int*)ids_i32, (const __half*)tok_emb, (const __half*)pos_emb, (__half*)out, rows, T, C / 8,
                        vocab));
  return 0;
}

extern "C" int ih_resize_patchify_f16(const void* img_nchw, void* out, int B, int C, int Hin, int Win, int S, int P,
                                      int Kpad, const float* mean3, const float* std3, void* stream) {
  IH_CHECK(img_nchw && out && mean3 && std3, IH_ERR_ARG, "ih_resize_patchify_f16: null pointer");
  IH_CHECK(C == 3 && S % P == 0 && Kpad % 8 == 0 && Kpad >= C * P * P && Hin > 0 && Win > 0, IH_ERR_SHAPE,
           "ih_resize_patchify_f16: 3 channels, S %% P == 0, Kpad >= 3*P*P (multiple of 8) required");
  const long long total = (long long)B * (S / P) * (S / P) * Kpad;
  IH_CUDA(launch_kernel(resize_patchify_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream,
                        (const __half*)img_nchw, (__half*)out, B, C, Hin, Win, S, P, Kpad, mean3[0], mean3[1], mean3[2],
                        std3[0], std3[1], std3[2]));
  return 0;
}

extern "C" int ih_add_bcast_f16(const void* a, const void* b, void* out, long long n, long long period, void* stream) {
  IH_CHECK(a && b && out && n % 8 == 0 && period % 8 == 0 && period > 0, IH_ERR_ARG, "ih_add_bcast_f16: bad arguments");
  IH_CUDA(launch_kernel(add_bcast_kernel, dim3(grid_for(n / 8, 256)), dim3(256), (size_t)0, (cudaStream_t)stream,
                        (const uint4*)a, (const uint4*)b, (uint4*)out, n / 8, period / 8));
  return 0;
}

extern "C" int ih_mean_tokens_f16(const void* x, void* out, int B, int n, int D, void* stream) {
  IH_CHECK(x && out && D % 8 == 0 && n > 0, IH_ERR_ARG, "ih_mean_tokens_f16: bad arguments");
  IH_CUDA(launch_kernel(mean_tokens_kernel, dim3((D / 8 + 127) / 128, B), dim3(128), (size_t)0, (cudaStream_t)stream,
                        (const __half*)x, (__half*)out, n, D));
  return 0;
}

extern "C" int ih_softmax_rows_masked_f16(void* x, long long ld, long long rows, int cols, int valid_cols, void* stream) {
  IH_CHECK(x && rows > 0 && cols > 0 && valid_cols > 0 && valid_cols <= cols, IH_ERR_ARG,
           "ih_softmax_rows_masked_f16: bad arguments");
  IH_CHECK(cols % 8 == 0 && ld % 8 == 0 && cols <= SMX_THREADS * SMX_MAXV * 8, IH_ERR_SHAPE,
           "ih_softmax_rows_masked_f16: cols must be a multiple of 8 and <= %d", SMX_THREADS * SMX_MAXV * 8);
  IH_CHECK(rows <= 0x7fffffffLL, IH_ERR_SHAPE, "ih_softmax_rows_masked_f16: too many rows");
  IH_CUDA(launch_kernel(softmax_rows_kernel, dim3((unsigned)rows), dim3(SMX_THREADS), (size_t)0, (cudaStream_t)stream,
                        (__half*)x, ld, cols, valid_cols));
  return 0;
}

extern "C" int ih_im2col3x3_nchw_f16(const void* x_nchw, void* out, int B, int Cin, int H, int W, int Kpad,
                                     void* stream) {
  IH_CHECK(x_nchw && out && Kpad % 8 == 0 && Kpad >= Cin * 9, IH_ERR_ARG, "ih_im2col3x3_nchw_f16: bad arguments");
  const long long total = (long long)B * H * W * (Kpad / 8);
  IH_CUDA(launch_kernel(im2col3x3_nchw_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream,
                        (const __half*)x_nchw, (__half*)out, B, Cin, H, W, Kpad));
  return 0;
}


extern "C" int ih_nhwc_to_nchw_f16(const void* x, long long ldc, void* out, int B, long long HW, int C, void* stream) {
  IH_CHECK(x && out && C >= 1, IH_ERR_ARG, "ih_nhwc_to_nchw_f16: bad arguments");
  const long long total = (long long)B * C * HW;
  IH_CUDA(launch_kernel(nhwc_to_nchw_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream,
                        (const __half*)x, ldc, (__half*)out, B, HW, C));
  return 0;
}

extern "C" int ih_vae_posterior_noise_f16(const void* moments, long long ldc, const void* eps, int eps_f32,
                                          const void* noise, void* out, int B, int B_moments, int B_eps, long long HW,
                                          int C, float scaling_factor, float sigma, void* stream) {
  IH_CHECK(moments && eps && noise && out, IH_ERR_ARG, "ih_vae_posterior_noise_f16: null pointer");
  IH_CHECK(B >= 1 && B_moments >= 1 && B_eps >= 1 && HW >= 1 && C >= 1, IH_ERR_SHAPE,
           "ih_vae_posterior_noise_f16: empty shape (B=%d, B_moments=%d, B_eps=%d, C=%d)", B, B_moments, B_eps, C);
  IH_CHECK(B % B_moments == 0 && B % B_eps == 0, IH_ERR_SHAPE,
           "ih_vae_posterior_noise_f16: B=%d must be a multiple of B_moments=%d and B_eps=%d", B, B_moments, B_eps);
  IH_CHECK(ldc >= 2 * C, IH_ERR_SHAPE, "ih_vae_posterior_noise_f16: ldc=%lld cannot hold mean and logvar of %d channels",
           ldc, C);
  IH_CHECK(eps_f32 == 0 || eps_f32 == 1, IH_ERR_ARG, "ih_vae_posterior_noise_f16: eps_f32 must be 0 or 1");
  const long long total = (long long)B * C * HW;
  IH_CUDA(launch_kernel(vae_posterior_noise_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream,
                        (const __half*)moments, ldc, eps, eps_f32, (const __half*)noise, (__half*)out, B, B_moments, B_eps,
                        HW, C, scaling_factor, sigma));
  return 0;
}

namespace ih {

// conv_in of the 9-channel inpainting UNet: the same patch matrix for the channel concatenation [x0 | x1] of two NCHW
// tensors (x0 [B, C0, H, W] the per-step latents, x1 [B, C1, H, W] the static mask | masked-image latents), read from
// the two sources directly so the 9-channel input is never materialised.  Column k = ci*9 + ky*3 + kx, ci < C0 from x0.
__global__ void im2col3x3_nchw_cat_kernel(const __half* __restrict__ x0, int C0, const __half* __restrict__ x1, int C1,
                                          __half* __restrict__ out, int B, int H, int W, int Kpad) {
  pdl_launch_dependents();
  pdl_wait();
  const long long npix = (long long)B * H * W;
  const int kv = Kpad >> 3;  // 16-byte vectors per row
  const long long total = npix * kv;
  const int kvalid = (C0 + C1) * 9;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % kv);
    const long long pix = i / kv;
    const int xw = (int)(pix % W);
    const int yh = (int)((pix / W) % H);
    const int b = (int)(pix / ((long long)W * H));
    __align__(16) __half vals[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = v * 8 + e;
      __half hv = __float2half_rn(0.f);
      if (k < kvalid) {
        const int ci = k / 9, t = k - ci * 9;
        const int yy = yh + t / 3 - 1, xx = xw + t % 3 - 1;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
          hv = ci < C0 ? x0[(((long long)b * C0 + ci) * H + yy) * W + xx]
                       : x1[(((long long)b * C1 + (ci - C0)) * H + yy) * W + xx];
        }
      }
      vals[e] = hv;
    }
    *reinterpret_cast<uint4*>(out + pix * Kpad + v * 8) = *reinterpret_cast<const uint4*>(vals);
  }
}

}  // namespace ih

extern "C" int ih_im2col3x3_nchw_cat_f16(const void* x0, int C0, const void* x1, int C1, void* out, int B, int H, int W,
                                         int Kpad, void* stream) {
  IH_CHECK(x0 && x1 && out, IH_ERR_ARG, "ih_im2col3x3_nchw_cat_f16: null pointer");
  IH_CHECK(B >= 1 && H >= 1 && W >= 1 && C0 >= 1 && C1 >= 1, IH_ERR_SHAPE,
           "ih_im2col3x3_nchw_cat_f16: empty shape (B=%d, H=%d, W=%d, C0=%d, C1=%d)", B, H, W, C0, C1);
  IH_CHECK(Kpad % 8 == 0 && Kpad >= (C0 + C1) * 9, IH_ERR_ARG,
           "ih_im2col3x3_nchw_cat_f16: Kpad=%d must be a multiple of 8 and >= (C0 + C1) * 9 = %d", Kpad, (C0 + C1) * 9);
  const long long total = (long long)B * H * W * (Kpad / 8);
  IH_CUDA(launch_kernel(im2col3x3_nchw_cat_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0,
                        (cudaStream_t)stream, (const __half*)x0, C0, (const __half*)x1, C1, (__half*)out, B, H, W, Kpad));
  return 0;
}

namespace ih {

// ControlNet conditioning embedding ([3P] diffusers ControlNetConditioningEmbedding): 3x3 convs, pad 1, stride 1 or 2,
// over the 3/16/32/96 channel widths that the implicit-GEMM conv cannot take (it needs whole 64-wide K blocks per tap).
// One thread per output element (pixel, cout), cout fastest; fp32 accumulation over the 9 * Cin products in tap order,
// then + bias, optional SiLU, one fp16 rounding.  The input is read through element strides, so the NCHW control image
// and the NHWC intermediate activations take the same kernel; the weight is tap-major [Cout, 9 * Cin].  It runs once
// per pipeline call, so the simple form is kept.
__global__ void conv3x3_small_kernel(const __half* __restrict__ x, long long sb, long long sh, long long sw, long long sc,
                                     const __half* __restrict__ w, const __half* __restrict__ bias,
                                     __half* __restrict__ out, int B, int H, int W, int Cin, int Cout, int stride,
                                     int Ho, int Wo, int silu) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)B * Ho * Wo * Cout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % Cout);
    const long long pix = i / Cout;
    const int xo = (int)(pix % Wo);
    const int yo = (int)((pix / Wo) % Ho);
    const int b = (int)(pix / ((long long)Wo * Ho));
    const __half* wr = w + (long long)co * 9 * Cin;
    float acc = 0.f;
#pragma unroll 1
    for (int t = 0; t < 9; ++t) {
      const int yy = yo * stride + t / 3 - 1, xx = xo * stride + t % 3 - 1;
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      const __half* xp = x + b * sb + yy * sh + xx * sw;
      const __half* wp = wr + t * Cin;
      for (int ci = 0; ci < Cin; ++ci) acc = fmaf(__half2float(xp[ci * sc]), __half2float(wp[ci]), acc);
    }
    if (bias) acc += __half2float(bias[co]);
    if (silu) acc = acc / (1.f + __expf(-acc));
    out[i] = __float2half_rn(acc);
  }
}

// ControlNet residual injection: for every entry k, rows [0, rows) of residual k are added to rows
// [skip_row0, skip_row0 + rows) of skip tensor k in place, skip = fp16(skip + fp16(res * scale[k])) -- diffusers'
// rounding points (the ControlNet scales its fp16 outputs, the UNet adds them).  The entry table is a kernel argument,
// so a captured CUDA graph keeps it with the launch; the scales are read from device memory, so one graph serves every
// conditioning scale.  blockIdx.y selects the entry; 8 halves per thread.
struct CnTable {
  IhCnResidual e[IH_CN_MAX_RESIDUALS];
};

__global__ void controlnet_add_residuals_kernel(const __grid_constant__ CnTable tab, const float* __restrict__ scale) {
  pdl_launch_dependents();
  pdl_wait();
  const IhCnResidual en = tab.e[blockIdx.y];
  const float s = scale[blockIdx.y];
  const long long nvec = en.rows * (en.channels / 8);
  const uint4* r = reinterpret_cast<const uint4*>(en.residual);
  uint4* d = reinterpret_cast<uint4*>(en.skip) + en.skip_row0 * (en.channels / 8);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    uint4 rv = r[i], dv = d[i];
    __half2* rh = reinterpret_cast<__half2*>(&rv);
    __half2* dh = reinterpret_cast<__half2*>(&dv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 rf = __half22float2(rh[j]), df = __half22float2(dh[j]);
      const float a = __half2float(__float2half_rn(__fmul_rn(rf.x, s)));
      const float b = __half2float(__float2half_rn(__fmul_rn(rf.y, s)));
      dh[j] = __floats2half2_rn(__fadd_rn(df.x, a), __fadd_rn(df.y, b));
    }
    d[i] = dv;
  }
}

// Multi-ControlNet residual injection: for every entry e, rows [0, rows) of the K nets' residuals are added to rows
// [skip_row0, skip_row0 + rows) of skip tensor e in place,
//   acc = fp16(r_0 * s_0[e]);  acc = fp16(acc + fp16(r_k * s_k[e])) for k = 1 .. K-1;  skip = fp16(skip + acc)
// -- diffusers' rounding points: each ControlNet scales its fp16 outputs, MultiControlNetModel sums them in net order,
// the UNet adds the sum.  One pass over the skips instead of K read-modify-write passes, which would also round the
// skip after every net.  With K = 1 it computes exactly controlnet_add_residuals_kernel, but measured 1-4% slower on
// the SDXL 1024^2 skips (the scale-vector table and the net loop), so single-net steps keep that kernel.  Table, scales
// and grid as there.
struct CnMultiTable {
  IhCnMultiResidual e[IH_CN_MAX_RESIDUALS];
  const float* scale[IH_CN_MAX_NETS];
  int n_nets;
};
// 4 KB is the kernel-parameter limit of every sm_90 launch path (larger needs the CUDA 12.1 large-parameter opt-in)
static_assert(sizeof(CnMultiTable) <= 4096, "the ControlNet injection table must fit the 4 KB kernel-parameter limit");

__device__ __forceinline__ float cn_scaled(__half r, float s) {
  return __half2float(__float2half_rn(__fmul_rn(__half2float(r), s)));
}

__global__ void controlnet_add_residuals_multi_kernel(const __grid_constant__ CnMultiTable tab) {
  pdl_launch_dependents();
  pdl_wait();
  const IhCnMultiResidual& en = tab.e[blockIdx.y];
  const int K = tab.n_nets;
  float s[IH_CN_MAX_NETS];
#pragma unroll
  for (int k = 0; k < IH_CN_MAX_NETS; ++k) s[k] = k < K ? tab.scale[k][blockIdx.y] : 0.f;
  const long long nvec = en.rows * (en.channels / 8);
  uint4* d = reinterpret_cast<uint4*>(en.skip) + en.skip_row0 * (en.channels / 8);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    uint4 rv = reinterpret_cast<const uint4*>(en.residual[0])[i], dv = d[i];
    const __half* rh = reinterpret_cast<const __half*>(&rv);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = cn_scaled(rh[j], s[0]);
#pragma unroll
    for (int k = 1; k < IH_CN_MAX_NETS; ++k) {
      if (k >= K) break;
      rv = reinterpret_cast<const uint4*>(en.residual[k])[i];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = __half2float(__float2half_rn(__fadd_rn(acc[j], cn_scaled(rh[j], s[k]))));
    }
    __half2* dh = reinterpret_cast<__half2*>(&dv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 df = __half22float2(dh[j]);
      dh[j] = __floats2half2_rn(__fadd_rn(df.x, acc[2 * j]), __fadd_rn(df.y, acc[2 * j + 1]));
    }
    d[i] = dv;
  }
}

static int controlnet_add_residuals_multi(const IhCnMultiResidual* entries, int n_entries, const void* const* scales,
                                          int n_nets, cudaStream_t stream) {
  const char* fn = "ih_controlnet_add_residuals_multi_f16";
  IH_CHECK(entries && scales, IH_ERR_ARG, "%s: null pointer", fn);
  IH_CHECK(n_entries >= 1 && n_entries <= IH_CN_MAX_RESIDUALS, IH_ERR_SHAPE, "%s: n_entries=%d outside [1, %d]", fn,
           n_entries, IH_CN_MAX_RESIDUALS);
  IH_CHECK(n_nets >= 1 && n_nets <= IH_CN_MAX_NETS, IH_ERR_SHAPE, "%s: n_nets=%d outside [1, %d]", fn, n_nets,
           IH_CN_MAX_NETS);
  CnMultiTable tab{};
  tab.n_nets = n_nets;
  for (int k = 0; k < n_nets; ++k) {
    IH_CHECK(scales[k], IH_ERR_ARG, "%s: scale vector %d is a null pointer", fn, k);
    tab.scale[k] = (const float*)scales[k];
  }
  long long most = 0;
  for (int k = 0; k < n_entries; ++k) {
    const IhCnMultiResidual& e = entries[k];
    IH_CHECK(e.skip, IH_ERR_ARG, "%s: entry %d has a null skip pointer", fn, k);
    IH_CHECK(e.rows >= 1 && e.skip_row0 >= 0 && e.channels >= 8 && e.channels % 8 == 0, IH_ERR_SHAPE,
             "%s: entry %d: rows=%lld, skip_row0=%lld, channels=%d (a multiple of 8)", fn, k, e.rows, e.skip_row0,
             e.channels);
    unsigned long long addr = (unsigned long long)e.skip;
    for (int j = 0; j < n_nets; ++j) {
      IH_CHECK(e.residual[j], IH_ERR_ARG, "%s: entry %d has a null residual pointer for net %d", fn, k, j);
      addr |= (unsigned long long)e.residual[j];
    }
    IH_CHECK(addr % 16 == 0, IH_ERR_ALIGN, "%s: entry %d is not 16-byte aligned", fn, k);
    tab.e[k] = e;
    most = e.rows * (e.channels / 8) > most ? e.rows * (e.channels / 8) : most;
  }
  IH_CUDA(launch_kernel(controlnet_add_residuals_multi_kernel, dim3(grid_for(most, 256), n_entries), dim3(256), (size_t)0,
                        stream, tab));
  return 0;
}

}  // namespace ih

extern "C" int ih_conv3x3_small_f16(const void* x, long long sb, long long sh, long long sw, long long sc, const void* w,
                                    const void* bias, void* out, int B, int H, int W, int Cin, int Cout, int stride,
                                    int silu, void* stream) {
  IH_CHECK(x && w && out, IH_ERR_ARG, "ih_conv3x3_small_f16: null pointer");
  IH_CHECK(B >= 1 && H >= 1 && W >= 1 && Cin >= 1 && Cout >= 1, IH_ERR_SHAPE,
           "ih_conv3x3_small_f16: empty shape (B=%d, H=%d, W=%d, Cin=%d, Cout=%d)", B, H, W, Cin, Cout);
  IH_CHECK(stride == 1 || stride == 2, IH_ERR_ARG, "ih_conv3x3_small_f16: stride must be 1 or 2, got %d", stride);
  IH_CHECK(silu == 0 || silu == 1, IH_ERR_ARG, "ih_conv3x3_small_f16: silu must be 0 or 1");
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long total = (long long)B * Ho * Wo * Cout;
  IH_CUDA(launch_kernel(conv3x3_small_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, (cudaStream_t)stream,
                        (const __half*)x, sb, sh, sw, sc, (const __half*)w, (const __half*)bias, (__half*)out, B, H, W,
                        Cin, Cout, stride, Ho, Wo, silu));
  return 0;
}

extern "C" int ih_controlnet_add_residuals_f16(const IhCnResidual* entries, int n_entries, const void* scale,
                                               void* stream) {
  IH_CHECK(entries && scale, IH_ERR_ARG, "ih_controlnet_add_residuals_f16: null pointer");
  IH_CHECK(n_entries >= 1 && n_entries <= IH_CN_MAX_RESIDUALS, IH_ERR_SHAPE,
           "ih_controlnet_add_residuals_f16: n_entries=%d outside [1, %d]", n_entries, IH_CN_MAX_RESIDUALS);
  ih::CnTable tab{};
  long long most = 0;
  for (int k = 0; k < n_entries; ++k) {
    const IhCnResidual& e = entries[k];
    IH_CHECK(e.skip && e.residual, IH_ERR_ARG, "ih_controlnet_add_residuals_f16: entry %d has a null pointer", k);
    IH_CHECK(e.rows >= 1 && e.skip_row0 >= 0 && e.channels >= 8 && e.channels % 8 == 0, IH_ERR_SHAPE,
             "ih_controlnet_add_residuals_f16: entry %d: rows=%lld, skip_row0=%lld, channels=%d (a multiple of 8)", k,
             e.rows, e.skip_row0, e.channels);
    IH_CHECK(((unsigned long long)e.skip | (unsigned long long)e.residual) % 16 == 0, IH_ERR_ALIGN,
             "ih_controlnet_add_residuals_f16: entry %d is not 16-byte aligned", k);
    tab.e[k] = e;
    most = e.rows * (e.channels / 8) > most ? e.rows * (e.channels / 8) : most;
  }
  IH_CUDA(launch_kernel(ih::controlnet_add_residuals_kernel, dim3(grid_for(most, 256), n_entries), dim3(256), (size_t)0,
                        (cudaStream_t)stream, tab, (const float*)scale));
  return 0;
}

extern "C" int ih_controlnet_add_residuals_multi_f16(const IhCnMultiResidual* entries, int n_entries,
                                                     const void* const* scales, int n_nets, void* stream) {
  return ih::controlnet_add_residuals_multi(entries, n_entries, scales, n_nets, (cudaStream_t)stream);
}
