// Softmax on wgmma accumulator fragments (layout: see ptx.cuh).  A query row lives in the four threads of a quad;
// thread column pair cq = 2 (lane % 4) of every 8-column group.  Used by the attention kernels of attn.cu.
#pragma once
#include "ptx.cuh"

namespace ih {

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// One key block holding every key: columns [0, n_text) text, [n_text, valid) image prompt (n_ip of them), the rest
// padding.  Replaces the scores in place by [P_t / l_t | ip_scale * P_ip / l_ip] (0 in the padding).
template <int NI>
__device__ __forceinline__ void softmax_two_segment(float (&sc)[4 * NI], int cq, int valid, int n_text, int n_ip,
                                                    float sl2, float ip_scale) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float mx_t = -INFINITY, mx_i = -INFINITY;
#pragma unroll
    for (int i = 0; i < NI; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * i + cq + e;
        const float s = sc[4 * i + 2 * h + e];
        if (col < n_text) mx_t = fmaxf(mx_t, s);
        else if (col < valid) mx_i = fmaxf(mx_i, s);
      }
    const float m_t = quad_max(mx_t) * sl2, m_i = quad_max(mx_i) * sl2;
    float l_t = 0.f, l_i = 0.f;
#pragma unroll
    for (int i = 0; i < NI; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * i + cq + e;
        float& s = sc[4 * i + 2 * h + e];
        float pv = 0.f;
        if (col < n_text) {
          pv = ex2_approx(fmaf(s, sl2, -m_t));
          l_t += pv;
        } else if (col < valid) {
          pv = ex2_approx(fmaf(s, sl2, -m_i));
          l_i += pv;
        }
        s = pv;
      }
    const float inv_t = 1.f / quad_sum(l_t);
    const float l_i_all = quad_sum(l_i);
    const float inv_i = (n_ip > 0) ? ip_scale / l_i_all : 0.f;
#pragma unroll
    for (int i = 0; i < NI; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * i + cq + e;
        sc[4 * i + 2 * h + e] *= (col < n_text) ? inv_t : inv_i;
      }
  }
}

// Online-softmax update for one 128-key block of the two rows (h = 0, 1) a thread holds: masks the columns >= valid
// (MASK: only the clipped last block has any), raises the running max, replaces the scores in place by
// 2^(s sl2 - m_new) and folds their sum into the running sum.  alpha[h] is the factor the O rows must be rescaled by
// (online_softmax_rescale); the caller applies it once no MMA into O is in flight.  Every attention kernel that walks
// key blocks uses this one sequence of operations, so a row's result does not depend on which kernel computed it.
template <bool MASK>
__device__ __forceinline__ void online_softmax_block(float (&sc)[64], float (&m_run)[2], float (&l_run)[2],
                                                     float (&alpha)[2], int cq, int valid, float sl2) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int col = 8 * i + cq;
      if (MASK && col >= valid) sc[4 * i + 2 * h] = -INFINITY;
      if (MASK && col + 1 >= valid) sc[4 * i + 2 * h + 1] = -INFINITY;
      mx = fmaxf(mx, fmaxf(sc[4 * i + 2 * h], sc[4 * i + 2 * h + 1]));
    }
    mx = quad_max(mx);
    const float m_new = fmaxf(m_run[h], mx * sl2);
    alpha[h] = ex2_approx(m_run[h] - m_new);
    m_run[h] = m_new;
    float ls = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      sc[4 * i + 2 * h] = ex2_approx(fmaf(sc[4 * i + 2 * h], sl2, -m_new));
      sc[4 * i + 2 * h + 1] = ex2_approx(fmaf(sc[4 * i + 2 * h + 1], sl2, -m_new));
      ls += sc[4 * i + 2 * h] + sc[4 * i + 2 * h + 1];
    }
    l_run[h] = l_run[h] * alpha[h] + ls;
  }
}

// O rows (accumulator fragment of 64 head columns) *= alpha of their row
__device__ __forceinline__ void online_softmax_rescale(float (&o)[32], const float (&alpha)[2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i + 2 * h] *= alpha[h];
      o[4 * i + 2 * h + 1] *= alpha[h];
    }
}

// fp32 probabilities (accumulator fragment of KS16 x 16 keys) -> fp16 A-operand fragments of KS16 k16 steps
template <int KS16>
__device__ __forceinline__ void pack_p_frags(const float (&sc)[8 * KS16], uint32_t (&pf)[4 * KS16]) {
#pragma unroll
  for (int kk = 0; kk < KS16; ++kk) {
    pf[4 * kk + 0] = pack_half2(sc[8 * kk + 0], sc[8 * kk + 1]);
    pf[4 * kk + 1] = pack_half2(sc[8 * kk + 2], sc[8 * kk + 3]);
    pf[4 * kk + 2] = pack_half2(sc[8 * kk + 4], sc[8 * kk + 5]);
    pf[4 * kk + 3] = pack_half2(sc[8 * kk + 6], sc[8 * kk + 7]);
  }
}

}  // namespace ih
