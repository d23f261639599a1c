// GroupNorm (NHWC, fp32/double statistics, optional SiLU, optional two-source channel concat) and LayerNorm.
// HBM-bound: every element is read twice (statistics + apply) and written once with 16-byte vector accesses.
// Replaces nn.GroupNorm / nn.SiLU / nn.LayerNorm of the diffusers UNet the reference drives
// (custom_pipelines.py:338-345); LayerNorm also serves ImageProjModel.norm (ip_adapter.py:47) and Resampler norms.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdlib.h>

#include "../../include/ih_api.h"
#include "host_util.h"
#include "ptx.cuh"

namespace ih {

__device__ __forceinline__ void load8(const __half* p, float (&x)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = unpack_half2(w[e]);
    x[2 * e] = f.x;
    x[2 * e + 1] = f.y;
  }
}
__device__ __forceinline__ void store8(__half* p, const float (&x)[8]) {
  uint4 o;
  o.x = pack_half2(x[0], x[1]);
  o.y = pack_half2(x[2], x[3]);
  o.z = pack_half2(x[4], x[5]);
  o.w = pack_half2(x[6], x[7]);
  *reinterpret_cast<uint4*>(p) = o;
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm statistics.  grid = (G row-chunks, B); block = CV * R threads (CV = C/8 channel vectors, R row lanes).
// Each block writes fp32 partial (sum, sumsq) per group -- no atomics on the data path -- and the last block of an
// image to finish (one atomic ticket per block) reduces the G partials in double and publishes mean / rstd.
// workspace layout: [GN_MAXB] uint32 tickets at a FIXED offset (so calls with different B never scribble over them;
// zero once, self-resetting) | floats: [B][GN_MAXG][2*groups] partials | [B][2*groups] mean,rstd
// ---------------------------------------------------------------------------------------------------------------
constexpr int GN_MAXG = 512;
constexpr int GN_MAXB = 1024;
constexpr int GN_SYNC_WORDS = 3 * GN_MAXB;   // per image: ticket (statistics), ready flag and departure counter (fused kernel)
// The R*2*C-float statistics buffer (8*C bytes once R = 1) plus the kernels' static shared memory must fit the 48 KiB
// a kernel gets without an opt-in; SDXL needs at most 2560 channels.
constexpr int GN_MAXC = 4096;

// The last block of an image sums the G partials of each of the 2*groups values in `slices` interleaved chains (a fixed
// order: deterministic), keeping 2*groups*slices doubles in the statistics buffer.
__host__ __device__ __forceinline__ int gn_slices(int threads, int groups) {
  const int s = threads / (2 * groups);
  return s < 1 ? 1 : (s > 4 ? 4 : s);
}

__global__ void gn_stats_kernel(const __half* __restrict__ x0, int C0, const __half* __restrict__ x1, int C1, int HW,
                                int groups, int R, int rows_per_block, float eps, float* __restrict__ ws, int B) {
  extern __shared__ float s_acc[];  // [R][2][C] per-row-lane partials (summed in a fixed order: deterministic)
  __shared__ bool s_last;
  pdl_launch_dependents();
  pdl_wait();
  const int C = C0 + C1;
  const int CV = C >> 3;
  const int b = blockIdx.y;
  const int cv = threadIdx.x % CV;
  const int rl = threadIdx.x / CV;
  const int c = cv << 3;
  const __half* src;
  long long stride;
  if (c < C0) {
    src = x0 + (long long)b * HW * C0 + c;
    stride = C0;
  } else {
    src = x1 + (long long)b * HW * C1 + (c - C0);
    stride = C1;
  }
  float s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
  const int row_begin = blockIdx.x * rows_per_block;
  const int row_end = min(HW, row_begin + rows_per_block);
  int row = row_begin + rl;
  for (; row + 3 * R < row_end; row += 4 * R) {  // 4 independent 16-byte loads in flight per thread
    float v0[8], v1[8], v2[8], v3[8];
    load8(src + (long long)row * stride, v0);
    load8(src + (long long)(row + R) * stride, v1);
    load8(src + (long long)(row + 2 * R) * stride, v2);
    load8(src + (long long)(row + 3 * R) * stride, v3);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      s[e] += (v0[e] + v1[e]) + (v2[e] + v3[e]);
      q[e] += (v0[e] * v0[e] + v1[e] * v1[e]) + (v2[e] * v2[e] + v3[e] * v3[e]);
    }
  }
  for (; row < row_end; row += R) {
    float v[8];
    load8(src + (long long)row * stride, v);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      s[e] += v[e];
      q[e] += v[e] * v[e];
    }
  }
  {
    float* mine = s_acc + (long long)rl * 2 * C;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      mine[c + e] = s[e];
      mine[C + c + e] = q[e];
    }
  }
  __syncthreads();
  const int cpg = C / groups;
  float* part = ws + ((long long)b * GN_MAXG + blockIdx.x) * 2 * groups;
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float ds = 0.f, dq = 0.f;
    for (int rr = 0; rr < R; ++rr) {
      const float* pr = s_acc + (long long)rr * 2 * C;
      for (int i = 0; i < cpg; ++i) {
        ds += pr[g * cpg + i];
        dq += pr[C + g * cpg + i];
      }
    }
    part[g] = ds;
    part[groups + g] = dq;
  }
  __threadfence();
  __syncthreads();
  unsigned int* tickets = reinterpret_cast<unsigned int*>(ws) - GN_SYNC_WORDS;  // ws points just past the sync arrays
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(&tickets[b], 1u);
    s_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    // all threads reduce the G partials: value index v = t % (2*groups), slice = t / (2*groups); L2 (ld.cg) loads
    // are independent so they pipeline; fixed summation order keeps the result deterministic.
    double* s_red = reinterpret_cast<double*>(s_acc);  // reuse: 2*groups*slices doubles fit (checked on the host)
    const int nv = 2 * groups;
    const int slices = gn_slices(blockDim.x, groups);
    const float* pp = ws + (long long)b * GN_MAXG * nv;
    __syncthreads();
    for (int t = threadIdx.x; t < nv * slices; t += blockDim.x) {  // 2*groups may exceed the block: loop
      const int v = t % nv, sl = t / nv;
      double a = 0.0;
#pragma unroll 8
      for (int k = sl; k < (int)gridDim.x; k += slices) a += (double)__ldcg(pp + (long long)k * nv + v);
      s_red[sl * nv + v] = a;
    }
    __syncthreads();
    float* fin = ws + (long long)B * GN_MAXG * nv + (long long)b * nv;
    const double n = (double)HW * cpg;
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
      double ds = 0.0, dq = 0.0;
      for (int sl = 0; sl < slices; ++sl) {
        ds += s_red[sl * nv + g];
        dq += s_red[sl * nv + groups + g];
      }
      const double mean = ds / n;
      double var = dq / n - mean * mean;
      if (var < 0.0) var = 0.0;
      fin[g] = (float)mean;
      fin[groups + g] = (float)(1.0 / sqrt(var + (double)eps));
    }
    if (threadIdx.x == 0) tickets[b] = 0u;  // self-reset for the next call
  }
}

__global__ void gn_apply_kernel(const __half* __restrict__ x0, int C0, const __half* __restrict__ x1, int C1, int HW,
                                int groups, int R, int rows_per_block, const float* __restrict__ fin_all,
                                const __half* __restrict__ gamma, const __half* __restrict__ beta, int silu,
                                __half* __restrict__ out) {
  extern __shared__ float s_ss[];  // scale[C], shift[C]
  pdl_launch_dependents();
  pdl_wait();
  const int C = C0 + C1;
  const int CV = C >> 3;
  const int b = blockIdx.y;
  const int cpg = C / groups;
  const float* fin = fin_all + (long long)b * 2 * groups;
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    const int g = ch / cpg;
    const float mean = fin[g], rstd = fin[groups + g];
    const float ga = __half2float(gamma[ch]), be = __half2float(beta[ch]);
    s_ss[ch] = ga * rstd;
    s_ss[C + ch] = be - mean * ga * rstd;
  }
  __syncthreads();
  const int cv = threadIdx.x % CV;
  const int rl = threadIdx.x / CV;
  const int c = cv << 3;
  const __half* src;
  long long stride;
  if (c < C0) {
    src = x0 + (long long)b * HW * C0 + c;
    stride = C0;
  } else {
    src = x1 + (long long)b * HW * C1 + (c - C0);
    stride = C1;
  }
  float sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    sc[e] = s_ss[c + e];
    sh[e] = s_ss[C + c + e];
  }
  __half* dst = out + (long long)b * HW * C + c;
  const int row_begin = blockIdx.x * rows_per_block;
  const int row_end = min(HW, row_begin + rows_per_block);
  int row = row_begin + rl;
  for (; row + 3 * R < row_end; row += 4 * R) {
    float v[4][8];
#pragma unroll
    for (int u = 0; u < 4; ++u) load8(src + (long long)(row + u * R) * stride, v[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float y = v[u][e] * sc[e] + sh[e];
        if (silu) y = silu_f(y);
        v[u][e] = y;
      }
      store8(dst + (long long)(row + u * R) * C, v[u]);
    }
  }
  for (; row < row_end; row += R) {
    float v[8];
    load8(src + (long long)row * stride, v);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float y = v[e] * sc[e] + sh[e];
      if (silu) y = silu_f(y);
      v[e] = y;
    }
    store8(dst + (long long)row * C, v);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm in ONE launch: statistics pass, image-wide hand-over, apply pass.  Same decomposition as the two kernels
// above (grid = (G row-chunks, B), every block owns a row range of one image).  After its partial sums are published,
// the last block of an image finalises mean / rstd and raises `ready[b]`; all blocks of the image wait for that flag,
// then normalise THEIR OWN rows (second read: L1 / L2 hits).  The host caps the grid at the number of co-resident
// blocks (occupancy query), so the wait cannot deadlock; a bounded spin traps instead of hanging.  The last block to
// leave an image resets the flags, so the workspace is reusable by the next launch (and by CUDA-graph replays).
// ---------------------------------------------------------------------------------------------------------------
__global__ void gn_fused_kernel(const __half* __restrict__ x0, int C0, const __half* __restrict__ x1, int C1, int HW,
                                int groups, int R, int rows_per_block, float eps, float* __restrict__ ws, int B,
                                const __half* __restrict__ gamma, const __half* __restrict__ beta, int silu,
                                __half* __restrict__ out) {
  extern __shared__ float s_acc[];  // statistics: [R][2][C] per-row-lane partials; apply: scale[C], shift[C]
  __shared__ bool s_last;
  pdl_launch_dependents();
  pdl_wait();
  const int C = C0 + C1;
  const int CV = C >> 3;
  const int b = blockIdx.y;
  const int cv = threadIdx.x % CV;
  const int rl = threadIdx.x / CV;
  const int c = cv << 3;
  const __half* src;
  long long stride;
  if (c < C0) {
    src = x0 + (long long)b * HW * C0 + c;
    stride = C0;
  } else {
    src = x1 + (long long)b * HW * C1 + (c - C0);
    stride = C1;
  }
  const int row_begin = blockIdx.x * rows_per_block;
  const int row_end = min(HW, row_begin + rows_per_block);
  const int cpg = C / groups;
  unsigned int* tickets = reinterpret_cast<unsigned int*>(ws) - GN_SYNC_WORDS;
  unsigned int* ready = tickets + GN_MAXB;
  unsigned int* done = ready + GN_MAXB;
  float* fin = ws + (long long)B * GN_MAXG * 2 * groups + (long long)b * 2 * groups;
  // ---- statistics of my rows ----
  {
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    int row = row_begin + rl;
    for (; row + 3 * R < row_end; row += 4 * R) {
      float v0[8], v1[8], v2[8], v3[8];
      load8(src + (long long)row * stride, v0);
      load8(src + (long long)(row + R) * stride, v1);
      load8(src + (long long)(row + 2 * R) * stride, v2);
      load8(src + (long long)(row + 3 * R) * stride, v3);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s[e] += (v0[e] + v1[e]) + (v2[e] + v3[e]);
        q[e] += (v0[e] * v0[e] + v1[e] * v1[e]) + (v2[e] * v2[e] + v3[e] * v3[e]);
      }
    }
    for (; row < row_end; row += R) {
      float v[8];
      load8(src + (long long)row * stride, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s[e] += v[e];
        q[e] += v[e] * v[e];
      }
    }
    float* mine = s_acc + (long long)rl * 2 * C;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      mine[c + e] = s[e];
      mine[C + c + e] = q[e];
    }
  }
  __syncthreads();
  float* part = ws + ((long long)b * GN_MAXG + blockIdx.x) * 2 * groups;
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float ds = 0.f, dq = 0.f;
    for (int rr = 0; rr < R; ++rr) {
      const float* pr = s_acc + (long long)rr * 2 * C;
      for (int i = 0; i < cpg; ++i) {
        ds += pr[g * cpg + i];
        dq += pr[C + g * cpg + i];
      }
    }
    part[g] = ds;
    part[groups + g] = dq;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(&tickets[b], 1u);
    s_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    double* s_red = reinterpret_cast<double*>(s_acc);  // reuse: 2*groups*slices doubles fit (checked on the host)
    const int nv = 2 * groups;
    const int slices = gn_slices(blockDim.x, groups);
    const float* pp = ws + (long long)b * GN_MAXG * nv;
    __syncthreads();
    for (int t = threadIdx.x; t < nv * slices; t += blockDim.x) {  // 2*groups may exceed the block: loop
      const int v = t % nv, sl = t / nv;
      double a = 0.0;
#pragma unroll 8
      for (int k = sl; k < (int)gridDim.x; k += slices) a += (double)__ldcg(pp + (long long)k * nv + v);
      s_red[sl * nv + v] = a;
    }
    __syncthreads();
    const double n = (double)HW * cpg;
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
      double ds = 0.0, dq = 0.0;
      for (int sl = 0; sl < slices; ++sl) {
        ds += s_red[sl * nv + g];
        dq += s_red[sl * nv + groups + g];
      }
      const double mean = ds / n;
      double var = dq / n - mean * mean;
      if (var < 0.0) var = 0.0;
      fin[g] = (float)mean;
      fin[groups + g] = (float)(1.0 / sqrt(var + (double)eps));
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      tickets[b] = 0u;            // self-reset for the next call
      __threadfence();
      atomicExch(&ready[b], 1u);  // mean / rstd of image b are published
    }
  }
  // ---- image-wide hand-over ----
  if (threadIdx.x == 0) {
    unsigned int spins = 0;
    while (atomicAdd(&ready[b], 0u) == 0u) {
      __nanosleep(32);
      if (++spins > IH_SPIN_LIMIT) __trap();
    }
    __threadfence();
  }
  __syncthreads();
  // ---- apply to my rows ----
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    const int g = ch / cpg;
    const float mean = __ldcg(fin + g), rstd = __ldcg(fin + groups + g);
    const float ga = __half2float(gamma[ch]), be = __half2float(beta[ch]);
    s_acc[ch] = ga * rstd;
    s_acc[C + ch] = be - mean * ga * rstd;
  }
  __syncthreads();
  {
    float sc[8], sh[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      sc[e] = s_acc[c + e];
      sh[e] = s_acc[C + c + e];
    }
    __half* dst = out + (long long)b * HW * C + c;
    int row = row_begin + rl;
    for (; row + 3 * R < row_end; row += 4 * R) {
      float v[4][8];
#pragma unroll
      for (int u = 0; u < 4; ++u) load8(src + (long long)(row + u * R) * stride, v[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float y = v[u][e] * sc[e] + sh[e];
          if (silu) y = silu_f(y);
          v[u][e] = y;
        }
        store8(dst + (long long)(row + u * R) * C, v[u]);
      }
    }
    for (; row < row_end; row += R) {
      float v[8];
      load8(src + (long long)row * stride, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float y = v[e] * sc[e] + sh[e];
        if (silu) y = silu_f(y);
        v[e] = y;
      }
      store8(dst + (long long)row * C, v);
    }
  }
  // ---- departure: the last block of the image to get here re-arms the flags ----
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int d = atomicAdd(&done[b], 1u);
    if (d == gridDim.x - 1) {
      done[b] = 0u;
      ready[b] = 0u;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm: one 16-byte vector per thread, TPR (multiple of 32) threads per row, several rows per block.
// two-pass (mean, then centred variance) in registers.
// ---------------------------------------------------------------------------------------------------------------
__global__ void layernorm_kernel(const __half* __restrict__ x, const __half* __restrict__ gamma,
                                 const __half* __restrict__ beta, __half* __restrict__ out, int rows, int C, int TPR,
                                 float eps) {
  __shared__ float s_red[2][32];
  pdl_launch_dependents();
  pdl_wait();
  const int rpb = blockDim.x / TPR;
  const int rl = threadIdx.x / TPR;
  const int tr = threadIdx.x - rl * TPR;
  const int row = blockIdx.x * rpb + rl;
  const int CV = C >> 3;
  const bool active = (row < rows) && (tr < CV);
  const int wpr = TPR >> 5;                 // warps per row
  const int wrow = (threadIdx.x >> 5);      // this thread's warp index in the block
  const int w0 = rl * wpr;                  // first warp of this row
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  if (active) load8(x + (long long)row * C + tr * 8, v);
  float sum = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) s_red[0][wrow] = sum;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < wpr; ++w) tot += s_red[0][w0 + w];
  const float mean = tot / (float)C;
  float sq = 0.f;
  if (active) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float d = v[e] - mean;
      sq += d * d;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  if ((threadIdx.x & 31) == 0) s_red[1][wrow] = sq;
  __syncthreads();
  float tq = 0.f;
  for (int w = 0; w < wpr; ++w) tq += s_red[1][w0 + w];
  const float rstd = rsqrtf(tq / (float)C + eps);
  if (active) {
    float g[8], bt[8], y[8];
    load8(gamma + tr * 8, g);
    load8(beta + tr * 8, bt);
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = (v[e] - mean) * rstd * g[e] + bt[e];
    store8(out + (long long)row * C + tr * 8, y);
  }
}

}  // namespace ih

using namespace ih;

extern "C" long long ih_groupnorm_workspace_bytes(int B, int groups) {
  return ((long long)B * GN_MAXG * 2 * groups + (long long)B * 2 * groups) * (long long)sizeof(float) +
         (long long)GN_SYNC_WORDS * (long long)sizeof(unsigned int);
}

extern "C" int ih_groupnorm_f16(const void* x0, int C0, const void* x1, int C1, const void* gamma, const void* beta,
                                void* out, void* stats_ws, int B, int HW, int groups, float eps, int silu,
                                void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  IH_CHECK(x0 && gamma && beta && out && stats_ws, IH_ERR_ARG, "ih_groupnorm_f16: null pointer");
  if (!x1) C1 = 0;
  const int C = C0 + C1;
  IH_CHECK(C0 % 8 == 0 && C1 % 8 == 0 && groups >= 1 && C > 0 && C % groups == 0, IH_ERR_SHAPE,
           "ih_groupnorm_f16: C0=%d C1=%d groups=%d unsupported", C0, C1, groups);
  IH_CHECK(C <= GN_MAXC, IH_ERR_SHAPE, "ih_groupnorm_f16: C=%d exceeds %d", C, GN_MAXC);
  IH_CHECK(B >= 1 && B <= GN_MAXB && HW >= 1, IH_ERR_SHAPE, "ih_groupnorm_f16: B=%d (max %d) HW=%d", B, GN_MAXB, HW);
  const int CV = C / 8;
  int R = 256 / CV;
  if (R < 1) R = 1;
  const int threads = CV * R;
  // the last block's reduction reuses the statistics buffer: C > 1024 (one row lane) needs groups <= C / 2
  IH_CHECK((size_t)2 * groups * gn_slices(threads, groups) * sizeof(double) <= (size_t)R * 2 * C * sizeof(float),
           IH_ERR_SHAPE, "ih_groupnorm_f16: groups=%d too many for C=%d", groups, C);
  // row chunks per image: about `bps` blocks per SM overall, at most GN_MAXG per image.  Measured (tools/gn_probe.py):
  // at UNet batch 2 the kernels are launch/latency bound and 2 blocks per SM is best; from batch 16 on they are
  // bandwidth bound and 4 blocks per SM (more loads in flight) is 1.6x faster (64.5 -> 40.6 us at B16 32^2 C1280).
  const int bps = B >= 8 ? 4 : 2;
  int G = (bps * num_sms() + B - 1) / B;
  if (G > GN_MAXG) G = GN_MAXG;
  int rows_per_block = (HW + G - 1) / G;
  if (rows_per_block < 4 * R) rows_per_block = 4 * R;
  G = (HW + rows_per_block - 1) / rows_per_block;
  float* ws = (float*)((unsigned int*)stats_ws + GN_SYNC_WORDS);
  // One launch (statistics -> hand-over -> apply) when every block of the grid can be resident at once; IH_GN_FUSED=0
  // keeps the two-kernel form.
  static const bool fused_env = [] {
    const char* e = getenv("IH_GN_FUSED");
    return !(e && e[0] == '0');
  }();
  if (fused_env) {
    const size_t smem = (size_t)R * 2 * C * sizeof(float);
    int occ = 0;
    IH_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_fused_kernel, threads, smem));
    const long long capacity = (long long)occ * num_sms();
    int Gf = G;
    if ((long long)Gf * B > capacity) Gf = (int)(capacity / B);
    if (Gf >= 1) {
      int rpb = (HW + Gf - 1) / Gf;
      if (rpb < 4 * R) rpb = 4 * R;
      Gf = (HW + rpb - 1) / rpb;
      IH_CUDA(launch_kernel(gn_fused_kernel, dim3(Gf, B), dim3(threads), smem, stream, (const __half*)x0, C0,
                            (const __half*)x1, C1, HW, groups, R, rpb, eps, ws, B, (const __half*)gamma,
                            (const __half*)beta, silu, (__half*)out));
      return 0;
    }
  }
  dim3 grid(G, B);
  IH_CUDA(launch_kernel(gn_stats_kernel, dim3(grid), dim3(threads), (size_t)((size_t)R * 2 * C * sizeof(float)), stream, (const __half*)x0, C0, (const __half*)x1, C1, HW,
                                                                     groups, R, rows_per_block, eps, ws, B));
  const float* fin = ws + (long long)B * GN_MAXG * 2 * groups;
  IH_CUDA(launch_kernel(gn_apply_kernel, dim3(grid), dim3(threads), (size_t)(2 * C * sizeof(float)), stream, (const __half*)x0, C0, (const __half*)x1, C1, HW,
                                                                     groups, R, rows_per_block, fin,
                                                                     (const __half*)gamma, (const __half*)beta, silu,
                                                                     (__half*)out));
  return 0;
}

extern "C" int ih_layernorm_f16(const void* x, const void* gamma, const void* beta, void* out, int rows, int C,
                                float eps, void* stream) {
  IH_CHECK(x && gamma && beta && out, IH_ERR_ARG, "ih_layernorm_f16: null pointer");
  IH_CHECK(C % 8 == 0 && C <= 8 * 1024 && rows > 0, IH_ERR_SHAPE, "ih_layernorm_f16: C=%d unsupported", C);
  const int CV = C / 8;
  const int TPR = ((CV + 31) / 32) * 32;
  int rpb = 256 / TPR;
  if (rpb < 1) rpb = 1;
  const int blocks = (rows + rpb - 1) / rpb;
  IH_CUDA(launch_kernel(layernorm_kernel, dim3(blocks), dim3(TPR * rpb), (size_t)(0), (cudaStream_t)stream, (const __half*)x, (const __half*)gamma,
                                                                   (const __half*)beta, (__half*)out, rows, C, TPR, eps));
  return 0;
}
