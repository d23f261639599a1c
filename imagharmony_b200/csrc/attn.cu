// wgmma attention for sm_90a, head_dim 64, no mask, softmax scale 1/8 (folded into exp2).
//
// One CTA = 128 query rows of one (batch, head): warpgroups 0 and 1 own 64 rows each; thread 0 issues the TMA loads
// (Q once, K/V double-buffered per 128-key block, a stage refilled as soon as both warpgroups have released it).  Per block: S = Q K^T (wgmma, Q and K from shared memory) into
// registers; the row softmax runs on the accumulator fragment (a row lives in the four threads of a quad: two shuffles
// per reduction); the fp32 probabilities are packed in place into the fp16 A-register fragment of O += P V (wgmma with
// A from registers, V as the MN-major B operand).  Two CTAs are co-resident per SM.
//
// Nk <= 128 (cross-attention, one key block): two independent softmaxes over the text columns [0, Nk - n_ip) and the
// image-prompt columns [Nk - n_ip, Nk) give P = [P_t / l_t | ip_scale * P_ip / l_ip], and the single PV MMA yields
//   softmax(q k_t^T) v_t + ip_scale * softmax(q k_ip^T) v_ip  -- attention_processor.py:423-450 (n_ip = 0: plain SDPA).
// Longer key axes use the online softmax; the last partial wave of query tiles can be cut into KV parts whose
// un-normalised partial results (fp32 O rows, running max, running sum) are merged by attn_combine_kernel.  By default
// they run on attn_ws_f16_kernel (persistent, warp-specialised, one CTA per SM: see there); attn_f16_kernel serves
// Nk <= 128 and, through ih_attention_set_kernel(1), the long shapes too, with bit-identical whole rows.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdlib.h>
#include <math.h>

#include "../../include/ih_api.h"
#include "host_util.h"
#include "ptx.cuh"
#include "softmax_frag.cuh"

namespace ih {

constexpr int ATT_THREADS = 256;        // warpgroups 0-1: MMA + softmax (thread 0 also issues the TMA loads)
constexpr int ATT_TILE = 128 * 64 * 2;  // 16 KiB: 128 rows x 64 fp16
constexpr int ATT_KS = 2;               // K / V stages
constexpr int ATT_SMEM_TILES = ATT_TILE * (1 + 2 * ATT_KS);  // Q | (K, V)[KS]
constexpr int ATT_SMEM_BYTES = ATT_SMEM_TILES + 128 + 1024;  // + barriers + alignment slack

struct AttnParams {
  int Nq, Nk, n_ip;
  int num_kv_blocks;
  float scale_log2;  // softmax scale * log2(e)
  float ip_scale;
  __half* out;
  long long ldo;
  // work decomposition: a unit is `rows` query rows of one (batch, head).  CTAs [0, n_whole) process a whole unit; CTA
  // n_whole + i processes KV part (i % split) of unit n_whole + i / split and writes an un-normalised partial result
  // (fp32 O rows, running max, running sum) to the workspace, merged by attn_combine_kernel.
  int rows;      // query rows per unit: 128 (attn_f16_kernel) or ATW_ROWS (attn_ws_f16_kernel)
  int H, qtiles, n_whole, split;
  float* ws_o;   // [slots][rows][64]
  float* ws_ml;  // [slots][rows][2]
  int n_items;   // n_whole + (units - n_whole) * split
};

// Work item -> KV blocks [jb, je) of query tile q0 of (b, head); slot >= 0: a KV part written to workspace slot `slot`.
struct AttnItem {
  int q0, head, b, jb, je, slot;
};
__device__ __forceinline__ AttnItem attn_item(const AttnParams& p, int item) {
  AttnItem w;
  int unit = item;
  w.jb = 0;
  w.je = p.num_kv_blocks;
  w.slot = -1;
  if (unit >= p.n_whole) {
    w.slot = unit - p.n_whole;
    const int su = w.slot / p.split;
    const int part = w.slot - su * p.split;
    unit = p.n_whole + su;
    w.jb = part * p.num_kv_blocks / p.split;          // balanced contiguous partition of the KV blocks
    w.je = (part + 1) * p.num_kv_blocks / p.split;
  }
  w.q0 = (unit % p.qtiles) * p.rows;
  w.head = (unit / p.qtiles) % p.H;
  w.b = unit / (p.qtiles * p.H);
  return w;
}

// Rows r0 and r0 + 8 of the item (the two rows of the thread's accumulator fragment): normalised fp16 output, or
// for a KV part the un-normalised fp32 O rows and (running max, running sum) in the workspace.
__device__ __forceinline__ void attn_store_rows(const AttnParams& p, const AttnItem& w, int r0, int cq,
                                                const float (&o)[32], const float (&m_run)[2],
                                                const float (&l_run)[2], bool single) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 8 * h;                      // row inside the unit
    const int qrow = w.q0 + r;
    const float l = quad_sum(l_run[h]);
    if (w.slot >= 0) {
      float2* dst = reinterpret_cast<float2*>(p.ws_o + ((long long)w.slot * p.rows + r) * 64);
#pragma unroll
      for (int i = 0; i < 8; ++i) dst[(8 * i + cq) >> 1] = make_float2(o[4 * i + 2 * h], o[4 * i + 2 * h + 1]);
      if (cq == 0) reinterpret_cast<float2*>(p.ws_ml)[(long long)w.slot * p.rows + r] = make_float2(m_run[h], l);
    } else if (qrow < p.Nq) {
      const float inv = single ? 1.f : 1.f / l;
      __half* dst = p.out + ((long long)w.b * p.Nq + qrow) * p.ldo + w.head * 64;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + 8 * i + cq) = pack_half2(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
    }
  }
}

__global__ void __launch_bounds__(ATT_THREADS, 2) attn_f16_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                   const __grid_constant__ CUtensorMap tmK,
                                                                   const __grid_constant__ CUtensorMap tmV,
                                                                   const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + ATT_TILE;                  // [KS]
  uint8_t* sV = sK + ATT_KS * ATT_TILE;           // [KS]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ATT_SMEM_TILES);
  uint64_t* q_full = bars;                        // [1]
  uint64_t* kv_full = bars + 1;                   // [KS]
  uint64_t* kv_empty = kv_full + ATT_KS;          // [KS]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const AttnItem w = attn_item(p, blockIdx.x);
  const int q0 = w.q0, head = w.head, b = w.b, jb = w.jb;
  const int nb = w.je - w.jb;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < ATT_KS; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 8);   // lane 0 of every MMA warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  auto load_kv = [&](int j, int st) {
    mbar_arrive_expect_tx(&kv_full[st], 2 * ATT_TILE);
    tma_load_3d(sK + st * ATT_TILE, &tmK, &kv_full[st], head * 64, (jb + j) * 128, b);
    tma_load_3d(sV + st * ATT_TILE, &tmV, &kv_full[st], head * 64, (jb + j) * 128, b);
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(q_full, ATT_TILE);
    tma_load_3d(sQ, &tmQ, q_full, head * 64, q0, b);
    for (int j = 0; j < nb && j < ATT_KS; ++j) load_kv(j, j);
  }

  const int wg = warp >> 2;
  const int rw = ((warp & 3) << 4) + (lane >> 2);   // my rows inside the warpgroup's 64: rw, rw + 8
  const int cq = (lane & 3) << 1;
  const float sl2 = p.scale_log2;
  const bool single = (p.num_kv_blocks == 1);
  const uint64_t q_desc = wgmma_desc_sw128(smem_u32(sQ) + wg * (64 * 128));
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(q_full, 0);

  int s = 0;
  uint32_t ph = 0;
  for (int j = 0; j < nb; ++j) {
    mbar_wait(&kv_full[s], ph);
    float sc[64];
    const uint64_t k_desc = wgmma_desc_sw128(smem_u32(sK + s * ATT_TILE));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss<128>(sc, q_desc + 2 * k, k_desc + 2 * k, k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sc);
    const int valid = p.Nk - (jb + j) * 128;   // valid keys of this block (>= 1)
    if (single) {
      softmax_two_segment<16>(sc, cq, valid, p.Nk - p.n_ip, p.n_ip, sl2, p.ip_scale);
    } else {
      float alpha[2];
      online_softmax_block<true>(sc, m_run, l_run, alpha, cq, valid, sl2);
      online_softmax_rescale(o, alpha);
    }
    uint32_t pf[32];
    pack_p_frags<8>(sc, pf);
    const uint32_t v_addr = smem_u32(sV + s * ATT_TILE);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)   // V: MN-major, 16 keys = 16 rows of 128 B = 2048 B per step
      wgmma_rs<64, 1>(o, *reinterpret_cast<const uint32_t(*)[4]>(pf + 4 * kk), wgmma_desc_sw128(v_addr + kk * 2048), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[s]);
    if (threadIdx.x == 0 && j + ATT_KS < nb) {   // refill the stage once every warp has released block j
      mbar_wait(&kv_empty[s], ph);
      load_kv(j + ATT_KS, s);
    }
    if (++s == ATT_KS) {
      s = 0;
      ph ^= 1;
    }
  }

  attn_store_rows(p, w, wg * 64 + rw, cq, o, m_run, l_run, single);
}

// Persistent, warp-specialised kernel for the multi-block path (Nk > 128, n_ip == 0).  One CTA per SM walks the work
// items blockIdx.x, blockIdx.x + gridDim.x, ...  Warpgroup 0 is the producer: one warp issues every TMA load (Q into a
// 2-deep ring, K and V into an ATW_KS-deep ring with separate "full" barriers) and is the only thread that waits on
// "empty" barriers, so it runs ahead into the next item while the current one finishes.  Warpgroups 1..ATW_CONSUMERS
// own 64 query rows each of a unit of ATW_ROWS rows; they never wait on each other's data, only take turns issuing
// MMAs (ping-pong, below).  Inside a warpgroup the QK^T of block j is issued before the PV of block j-1, and the
// softmax of block j runs while that PV is still on the tensor cores; O is rescaled once it lands.
// The per-row arithmetic (MMA shapes and k order, online_softmax_block, pack_p_frags) is that of attn_f16_kernel.
// Three MMA warpgroups (192-row units) rather than two: at head dim 64 the softmax (MUFU ex2, fp16 packing) of a
// block takes about as long as its MMAs, so with three warpgroups taking turns two of them have softmax work to
// overlap each one's MMAs, and the units per (batch, head) drop by a third.  On an H100 (400 W) this was 1.33x the
// old kernel at (2,10,4096^2) and 1.43x at (2,20,1024^2); two warpgroups gave 1.0-1.15x.
#ifndef ATW_CONSUMERS
#define ATW_CONSUMERS 3                                         // MMA warpgroups (64 query rows each)
#endif
constexpr int ATW_ROWS = 64 * ATW_CONSUMERS;                    // query rows per unit
constexpr int ATW_THREADS = 128 * (1 + ATW_CONSUMERS);
constexpr int ATW_KS = 4;                                       // K / V stages
constexpr int ATW_Q_TILE = ATW_ROWS * 64 * 2;
constexpr int ATW_SMEM_TILES = 2 * ATW_Q_TILE + ATT_TILE * 2 * ATW_KS;   // Q[2] | K[KS] | V[KS]
// register split (multiples of 8, 64K registers per SM): the producer keeps what TMA issue needs
constexpr int ATW_PRODUCER_REGS = ATW_CONSUMERS == 2 ? 40 : 32;
constexpr int ATW_CONSUMER_REGS = ATW_CONSUMERS == 2 ? 232 : 160;
static_assert(128 * ATW_PRODUCER_REGS + 128 * ATW_CONSUMERS * ATW_CONSUMER_REGS <= 65536, "register budget");
constexpr int ATW_SMEM_BYTES = ATW_SMEM_TILES + 256 + 1024;     // + barriers + alignment slack

#ifndef ATW_PINGPONG
#define ATW_PINGPONG 1   // order the MMA warpgroups' tensor-core work (see the consumer loop)
#endif

// keep the compiler from reusing registers that an asynchronous MMA still reads
template <int N>
__device__ __forceinline__ void fence_regs_u32(uint32_t (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

__global__ void __launch_bounds__(ATW_THREADS, 1) attn_ws_f16_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                     const __grid_constant__ CUtensorMap tmK,
                                                                     const __grid_constant__ CUtensorMap tmV,
                                                                     const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                             // [2]
  uint8_t* sK = smem + 2 * ATW_Q_TILE;            // [KS]
  uint8_t* sV = sK + ATW_KS * ATT_TILE;           // [KS]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ATW_SMEM_TILES);
  uint64_t* q_full = bars;                        // [2]
  uint64_t* q_empty = bars + 2;                   // [2]
  uint64_t* k_full = bars + 4;                    // [KS]
  uint64_t* v_full = k_full + ATW_KS;             // [KS]
  uint64_t* kv_empty = v_full + ATW_KS;           // [KS]
  constexpr uint32_t CONSUMER_WARPS = ATW_CONSUMERS * 4;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&q_full[s], 1);
      mbar_init(&q_empty[s], CONSUMER_WARPS);    // lane 0 of every MMA warp
    }
    for (int s = 0; s < ATW_KS; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&kv_empty[s], CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp < 4) {
    // ------------------------------ producer warpgroup ------------------------------
    setmaxnreg_dec<ATW_PRODUCER_REGS>();
    if (warp == 0) {
      int s = 0, qs = 0;
      uint32_t ph = 0, qph = 0;
      for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
        const AttnItem w = attn_item(p, item);
        mbar_wait(&q_empty[qs], qph ^ 1);
        if (elect_one()) {
          mbar_arrive_expect_tx(&q_full[qs], ATW_Q_TILE);
          tma_load_3d(sQ + qs * ATW_Q_TILE, &tmQ, &q_full[qs], w.head * 64, w.q0, w.b);
        }
        __syncwarp();
        if (++qs == 2) {
          qs = 0;
          qph ^= 1;
        }
        for (int j = w.jb; j < w.je; ++j) {
          mbar_wait(&kv_empty[s], ph ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(&k_full[s], ATT_TILE);
            tma_load_3d(sK + s * ATT_TILE, &tmK, &k_full[s], w.head * 64, j * 128, w.b);
            mbar_arrive_expect_tx(&v_full[s], ATT_TILE);
            tma_load_3d(sV + s * ATT_TILE, &tmV, &v_full[s], w.head * 64, j * 128, w.b);
          }
          __syncwarp();
          if (++s == ATW_KS) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    }
    return;
  }

  // ------------------------------ MMA + softmax warpgroups ------------------------------
  setmaxnreg_inc<ATW_CONSUMER_REGS>();
  const int wg = (threadIdx.x >> 7) - 1;            // rows [64 wg, 64 wg + 64) of the unit
  const int rw = ((warp & 3) << 4) + (lane >> 2);   // my rows inside the warpgroup's 64: rw, rw + 8
  const int cq = (lane & 3) << 1;
  const float sl2 = p.scale_log2;
  // Ping-pong: a warpgroup issues its MMAs of a block (QK^T of block j and PV of block j - 1) only after the previous
  // one in round-robin order has issued its own, through named barriers (1 + wg: "my turn").  The tensor cores then
  // take the warpgroups in turn, and each one's softmax runs under the others' MMAs.  Warpgroup 0 goes first; the
  // last warpgroup skips its very last hand-over so that every barrier phase is complete when the CTA exits.
  auto mma_turn = [&]() {
    if (ATW_PINGPONG) named_bar_sync(1 + wg, 2 * 128);
  };
  auto mma_pass = [&](bool last) {
    if (ATW_PINGPONG && !(last && wg == ATW_CONSUMERS - 1)) named_bar_arrive(1 + (wg + 1) % ATW_CONSUMERS, 2 * 128);
  };
  if (ATW_PINGPONG && wg == ATW_CONSUMERS - 1) named_bar_arrive(1, 2 * 128);
  int s = 0, qs = 0;
  uint32_t ph = 0, qph = 0;
  for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
    const AttnItem w = attn_item(p, item);
    const int nb = w.je - w.jb;
    const bool last_item = item + (int)gridDim.x >= p.n_items;
    const uint64_t q_desc = wgmma_desc_sw128(smem_u32(sQ + qs * ATW_Q_TILE) + wg * (64 * 128));
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, alpha[2];
    float sc[64];
    uint32_t pf[32];
    mbar_wait(&q_full[qs], qph);

    // block jb: S = Q K^T and its softmax (O is still zero: no rescale)
    mbar_wait(&k_full[s], ph);
    {
      const uint64_t k_desc = wgmma_desc_sw128(smem_u32(sK + s * ATT_TILE));
      mma_turn();
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<128>(sc, q_desc + 2 * k, k_desc + 2 * k, k != 0);
      wgmma_commit();
      mma_pass(false);
      wgmma_wait<0>();
      fence_regs(sc);
    }
    if (nb == 1) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&q_empty[qs]);
    }
    {
      const int valid = p.Nk - w.jb * 128;
      if (valid < 128) online_softmax_block<true>(sc, m_run, l_run, alpha, cq, valid, sl2);
      else online_softmax_block<false>(sc, m_run, l_run, alpha, cq, valid, sl2);
    }
    pack_p_frags<8>(sc, pf);
    int sp = s;                                      // stage of the block whose P V is pending
    uint32_t php = ph;
    if (++s == ATW_KS) {
      s = 0;
      ph ^= 1;
    }

    for (int j = 1; j < nb; ++j) {
      mbar_wait(&k_full[s], ph);
      mbar_wait(&v_full[sp], php);
      const uint64_t k_desc = wgmma_desc_sw128(smem_u32(sK + s * ATT_TILE));
      const uint32_t v_addr = smem_u32(sV + sp * ATT_TILE);
      mma_turn();
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<128>(sc, q_desc + 2 * k, k_desc + 2 * k, k != 0);
      wgmma_commit();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)   // V: MN-major, 16 keys = 16 rows of 128 B = 2048 B per step
        wgmma_rs<64, 1>(o, *reinterpret_cast<const uint32_t(*)[4]>(pf + 4 * kk), wgmma_desc_sw128(v_addr + kk * 2048), 1);
      wgmma_commit();
      mma_pass(false);
      wgmma_wait<1>();                               // S of block j is in; P V of block j - 1 may still run
      fence_regs(sc);
      if (j == nb - 1) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&q_empty[qs]);
      }
      const int valid = p.Nk - (w.jb + j) * 128;
      if (valid < 128) online_softmax_block<true>(sc, m_run, l_run, alpha, cq, valid, sl2);
      else online_softmax_block<false>(sc, m_run, l_run, alpha, cq, valid, sl2);
      wgmma_wait<0>();
      fence_regs(o);
      fence_regs_u32(pf);
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[sp]);
      online_softmax_rescale(o, alpha);
      pack_p_frags<8>(sc, pf);
      sp = s;
      php = ph;
      if (++s == ATW_KS) {
        s = 0;
        ph ^= 1;
      }
    }

    mbar_wait(&v_full[sp], php);
    {
      const uint32_t v_addr = smem_u32(sV + sp * ATT_TILE);
      mma_turn();
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        wgmma_rs<64, 1>(o, *reinterpret_cast<const uint32_t(*)[4]>(pf + 4 * kk), wgmma_desc_sw128(v_addr + kk * 2048), 1);
      wgmma_commit();
      mma_pass(last_item);
      wgmma_wait<0>();
      fence_regs(o);
      fence_regs_u32(pf);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[sp]);
    attn_store_rows(p, w, wg * 64 + rw, cq, o, m_run, l_run, false);
    if (++qs == 2) {
      qs = 0;
      qph ^= 1;
    }
  }
}

// Merge the `split` KV parts of the units that attn_f16_kernel processed piecewise:
//   M = max_i m_i,  out = sum_i O_i 2^(m_i - M) / sum_i l_i 2^(m_i - M)   (fixed order: deterministic).
// grid = (#split units * rows / 64), block = 256: 64 rows per block, 4 threads (16 columns each) per row.
__global__ void __launch_bounds__(256) attn_combine_kernel(const AttnParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int per_unit = p.rows / 64;
  const int su = blockIdx.x / per_unit;
  const int row = (blockIdx.x - su * per_unit) * 64 + (threadIdx.x >> 2);
  const int c0 = (threadIdx.x & 3) * 16;
  const int unit = p.n_whole + su;
  const int qrow = (unit % p.qtiles) * p.rows + row;
  if (qrow >= p.Nq) return;
  const int head = (unit / p.qtiles) % p.H;
  const int b = unit / (p.qtiles * p.H);
  const float2* ml = reinterpret_cast<const float2*>(p.ws_ml);
  float mmax = -INFINITY;
  for (int i = 0; i < p.split; ++i) mmax = fmaxf(mmax, ml[((long long)su * p.split + i) * p.rows + row].x);
  float acc[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) acc[e] = 0.f;
  float l = 0.f;
  for (int i = 0; i < p.split; ++i) {
    const long long wrow = ((long long)su * p.split + i) * p.rows + row;
    const float2 v = ml[wrow];
    const float w = ex2_approx(v.x - mmax);
    l = fmaf(v.y, w, l);
    const float4* src = reinterpret_cast<const float4*>(p.ws_o + wrow * 64 + c0);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 o = src[g];
      acc[g * 4 + 0] = fmaf(o.x, w, acc[g * 4 + 0]);
      acc[g * 4 + 1] = fmaf(o.y, w, acc[g * 4 + 1]);
      acc[g * 4 + 2] = fmaf(o.z, w, acc[g * 4 + 2]);
      acc[g * 4 + 3] = fmaf(o.w, w, acc[g * 4 + 3]);
    }
  }
  const float inv = 1.f / l;
  __half* dst = p.out + ((long long)b * p.Nq + qrow) * p.ldo + head * 64 + c0;
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    uint4 o;
    o.x = pack_half2(acc[g * 8 + 0] * inv, acc[g * 8 + 1] * inv);
    o.y = pack_half2(acc[g * 8 + 2] * inv, acc[g * 8 + 3] * inv);
    o.z = pack_half2(acc[g * 8 + 4] * inv, acc[g * 8 + 5] * inv);
    o.w = pack_half2(acc[g * 8 + 6] * inv, acc[g * 8 + 7] * inv);
    *reinterpret_cast<uint4*>(dst + g * 8) = o;
  }
}

// KV-split plan: with U units on G resident CTA slots (SMs x CTAs per SM), the last U mod G units would run as a nearly
// empty extra wave; they are cut into `split` KV parts each so that (U mod G) * split <= G CTAs share that wave.
// Cost model in KV-block iterations (an estimate, not a measurement): a part pays ATT_SPLIT_OVERHEAD iterations for
// its partial write and the merge kernel.  Returns split (1 = none) and the number of units processed whole.
constexpr float ATT_SPLIT_OVERHEAD = 3.0f;
static int g_split_policy = 0;   // 0: cost model, 1: split every partial last wave of a multi-block shape (tests)
static int g_kernel = 0;         // multi-block path: 0 = attn_ws_f16_kernel, 1 = attn_f16_kernel (tests, A/B tools)

template <typename K>
static int attn_resident_ctas(K kernel, int threads, int smem) {
  int per_sm = 0;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1)
    per_sm = 1;
  return num_sms() * per_sm;
}

// resident CTA slots of the kernel that serves the multi-block path (also sets the shared-memory attributes once)
static int attn_slots() {
  static const int slots_old = attn_resident_ctas(attn_f16_kernel, ATT_THREADS, ATT_SMEM_BYTES);
  static const int slots_ws = attn_resident_ctas(attn_ws_f16_kernel, ATW_THREADS, ATW_SMEM_BYTES);
  return g_kernel == 1 ? slots_old : slots_ws;
}

// query rows per unit of the kernel that serves a shape (Nk > 128 is the multi-block path)
static int attn_rows(int Nk) { return (Nk > 128 && g_kernel == 0) ? ATW_ROWS : 128; }

static void attn_plan(int units, int nb, int* n_whole, int* split) {
  const int G = attn_slots();
  const int rem = units % G;
  *n_whole = units;
  *split = 1;
  if (rem == 0 || nb < 2) return;
  int s = G / rem;
  if (s > nb) s = nb;
  if (s < 2) {
    if (g_split_policy == 0) return;
    s = 2;   // policy 1: cut the partial wave even where its parts overflow into one more
  }
  const float t_whole = (float)nb, t_split = (float)((nb + s - 1) / s) + ATT_SPLIT_OVERHEAD;
  if (t_split >= t_whole && g_split_policy == 0) return;
  *n_whole = units - rem;
  *split = s;
}

}  // namespace ih

using namespace ih;

extern "C" void ih_attention_set_split_policy(int policy) { g_split_policy = policy; }
extern "C" void ih_attention_set_kernel(int kernel) { g_kernel = kernel == 1 ? 1 : 0; }

extern "C" long long ih_attention_workspace_bytes(int B, int H, int Nq, int Nk, int n_ip) {
  if (B <= 0 || H <= 0 || Nq <= 0 || Nk <= 128 || n_ip != 0) return 0;
  int n_whole, split;
  const int rows = attn_rows(Nk);
  const int units = B * H * ((Nq + rows - 1) / rows);
  attn_plan(units, (Nk + 127) / 128, &n_whole, &split);
  if (units == n_whole) return 0;
  return (long long)(units - n_whole) * split * rows * (64 + 2) * (long long)sizeof(float);
}

extern "C" int ih_attention_ws_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                   long long ldv, void* out, long long ldo, int B, int H, int Nq, int Nk, int n_ip,
                                   float ip_scale, void* workspace, long long workspace_bytes, void* stream) {
  IH_CHECK(q && k && v && out, IH_ERR_ARG, "ih_attention_ws_f16: null pointer");
  IH_CHECK(B > 0 && H > 0 && Nq > 0 && Nk > 0, IH_ERR_SHAPE, "ih_attention_ws_f16: bad shape");
  IH_CHECK(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, IH_ERR_ALIGN,
           "ih_attention_ws_f16: row strides must be multiples of 8 elements");
  IH_CHECK(n_ip >= 0 && n_ip < Nk, IH_ERR_ARG, "ih_attention_ws_f16: n_ip out of range");
  IH_CHECK(n_ip == 0 || Nk <= 128, IH_ERR_SHAPE, "ih_attention_ws_f16: decoupled IP path needs Nk <= 128");

  const int rows = n_ip == 0 ? attn_rows(Nk) : 128;
  CUtensorMap tq, tk, tv;
  const uint32_t box[3] = {64u, 128u, 1u};
  {
    const uint64_t dims[3] = {(uint64_t)H * 64, (uint64_t)Nq, (uint64_t)B};
    const uint64_t str[2] = {(uint64_t)ldq * 2, (uint64_t)Nq * ldq * 2};
    const uint32_t qbox[3] = {64u, (uint32_t)rows, 1u};
    int rc = get_tmap_f16(&tq, q, 3, dims, str, qbox);
    if (rc) return rc;
  }
  {
    const uint64_t dims[3] = {(uint64_t)H * 64, (uint64_t)Nk, (uint64_t)B};
    const uint64_t str[2] = {(uint64_t)ldk * 2, (uint64_t)Nk * ldk * 2};
    int rc = get_tmap_f16(&tk, k, 3, dims, str, box);
    if (rc) return rc;
  }
  {
    const uint64_t dims[3] = {(uint64_t)H * 64, (uint64_t)Nk, (uint64_t)B};
    const uint64_t str[2] = {(uint64_t)ldv * 2, (uint64_t)Nk * ldv * 2};
    int rc = get_tmap_f16(&tv, v, 3, dims, str, box);
    if (rc) return rc;
  }
  AttnParams p{};
  p.Nq = Nq;
  p.Nk = Nk;
  p.n_ip = n_ip;
  p.num_kv_blocks = (Nk + 127) / 128;
  p.scale_log2 = 0.125f * 1.4426950408889634f;
  p.ip_scale = ip_scale;
  p.out = (__half*)out;
  p.ldo = ldo;
  p.H = H;
  p.rows = rows;
  p.qtiles = (Nq + rows - 1) / rows;
  const int units = B * H * p.qtiles;
  attn_slots();   // sets the shared-memory attribute once
  p.n_whole = units;
  p.split = 1;
  if (n_ip == 0) attn_plan(units, p.num_kv_blocks, &p.n_whole, &p.split);
  const long long slots = (long long)(units - p.n_whole) * p.split;
  const long long need = slots * rows * 66 * (long long)sizeof(float);
  if (slots > 0 && (!workspace || workspace_bytes < need)) {
    p.n_whole = units;   // no (or too small a) workspace: every unit runs whole
    p.split = 1;
  }
  const int n_split_ctas = (units - p.n_whole) * p.split;
  p.n_items = p.n_whole + n_split_ctas;
  p.ws_o = reinterpret_cast<float*>(workspace);
  p.ws_ml = p.ws_o ? p.ws_o + (long long)n_split_ctas * rows * 64 : nullptr;
  if (rows != 128) {
    const int grid = p.n_items < num_sms() ? p.n_items : num_sms();
    IH_CUDA(launch_kernel(attn_ws_f16_kernel, dim3(grid), dim3(ATW_THREADS), (size_t)ATW_SMEM_BYTES,
                          (cudaStream_t)stream, tq, tk, tv, p));
  } else {
    IH_CUDA(launch_kernel(attn_f16_kernel, dim3(p.n_items), dim3(ATT_THREADS), (size_t)ATT_SMEM_BYTES,
                          (cudaStream_t)stream, tq, tk, tv, p));
  }
  if (n_split_ctas > 0)
    IH_CUDA(launch_kernel(attn_combine_kernel, dim3((units - p.n_whole) * (rows / 64)), dim3(256), (size_t)0, (cudaStream_t)stream,
                          p));
  return 0;
}
