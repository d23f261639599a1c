// wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
//   out[M,N] = epilogue( A[M,K] * W[N,K]^T )           fp16 in, fp32 accumulate in registers, fp16 out
//
// Persistent CTAs (one per SM) walk 128 x BN output tiles. Warpgroup 0 is the TMA producer (one elected lane of warp 0
// issues the loads; warp 1 may prefetch the next kernel's weights into L2), warpgroups 1 and 2 each own 64 rows of the
// tile: wgmma main loop over a STAGES-deep mbarrier ring of 128B-swizzled operand tiles (64 fp16 = one 128 B row per
// K-block), then the epilogue straight from the accumulator registers into swizzled staging slabs that leave by TMA
// store. While the MMA warpgroups run the epilogue of one tile the producer already fills the ring for the next.
//
// Convolution is the same kernel ("im2col-free"): the activation is NHWC, the A tile of tap (dy,dx) is a 4-D TMA box
// {64 channels, bw, bh, 1} at spatial offset (dx-1, dy-1) with out-of-bounds zero fill providing the padding; the
// weight is [Cout, taps*Cin] tap-major. Stride-2 convolutions read four parity-subsampled views of the input.
//
// Replaces (reference call sites): nn.Linear in attention_processor.py:292-320,396-453 (to_q/to_k/to_v/to_out,
// to_k_ip/to_v_ip) and, in the diffusers UNet the reference drives at custom_pipelines.py:338-345, every Linear
// (proj_in/out, FF GEGLU) and Conv2d.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdlib.h>

#include "../../include/ih_api.h"
#include "host_util.h"
#include "ptx.cuh"

namespace ih {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KiB

struct alignas(64) TmapSet4 {
  CUtensorMap m[4];
};

struct GemmParams {
  int M, N;     // logical output rows / cols (GEGLU: N = number of gated outputs)
  int m_tiles;  // number of 128-row output tiles
  int num_kb;   // K blocks of 64 (taps * cin_kb for conv)
  int mode;     // 0 = plain GEMM, 1 = conv (4-D A maps)
  int cin_kb;   // conv: K blocks per 3x3 tap
  // conv: cumulative K-block end of every tap.  Taps 0..8 are the 3x3 window; taps 9 / 10 (optional) are a fused 1x1
  // SHORTCUT convolution over one or two further NHWC sources (ResnetBlock2D conv_shortcut on the channel concat of the
  // hidden state and the skip connection): their K blocks accumulate into the same accumulator, so `conv2(h) +
  // shortcut(cat(x, skip))` is ONE launch and the concatenated tensor is never materialised.
  int n_taps;
  int tap_kb_end[12];
  int Ho, Wo;   // conv: output spatial size
  int bw, bh;   // conv: spatial tile (bw*bh == 128)
  int tiles_x, tiles_y;
  signed char tap_map[12], tap_ox[12], tap_oy[12];
  int gate_row_off;  // GEGLU: row offset of the gate half inside W
  const __half* bias;
  const __half* rowbias;
  int rows_per_group;
  long long ld_rowbias;
  const __half* residual;
  long long ldr;
  __half* out;
  long long ldo;
  int act;  // 0 none, 1 SiLU, 2 GELU(erf), 3 quick-GELU (applied after bias, before residual)
  int relu;  // IH_EPI_RELU: relu_nan_f AFTER the residual add (TAESD's fuse(conv(x) + skip(x)))
  unsigned long long* trace;  // optional: %globaltimer stamps of CTA 0 (ih_gemm_set_trace), nullptr in production
  // L2 prefetch of the NEXT kernel's weights (ih_gemm_prefetch_next): inside a denoise step every GEMM streams its weights
  // from HBM (5.2 GB per step >> L2), and a short launch cannot hide the first HBM round trips.  An otherwise idle
  // producer warp issues cp.async.bulk.prefetch.L2 for this CTA's slice while the main loop runs.
  const unsigned char* pf_ptr;
  unsigned long long pf_bytes;
  // LayerNorm folding (plain GEMM mode only).  A producer GEMM writes, per output row, the sum and the sum of squares
  // of the fp16-rounded values it stores as partial sums whose total over slots is the row's (stats_out
  // [ceil(N/64), M, 2] fp32, one writer per slot, every slot written: deterministic, nothing to zero).  The consumer
  // GEMM multiplies the RAW rows with gamma-scaled, row-CENTRED weights
  // Wc[n,k] = W[n,k] gamma[k] - mean_k(W[n,:] gamma) -- so x Wc^T = (x - mean(x)) (W gamma)^T -- and applies
  //   out = rstd[m] * acc + c[n],  c = W beta + b (passed as `bias`)   (= LayerNorm(x) W^T + b in real arithmetic)
  // with rstd rebuilt from the producer's slabs (ln_stats [ln_slabs, M, 2]).
  float alpha;   // out = alpha * acc (* rstd) + bias ...: power-of-two output scaling of the VAE's scaled residual stream
  float* stats_out;
  const float* ln_stats;
  int ln_slabs;
  float ln_inv_c;
  float ln_eps;
};

template <int BN, int STAGES, bool GEGLU>
struct GemmSmem {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int TILE_BYTES = STAGES * STAGE_BYTES;
  static constexpr int BN_OUT = GEGLU ? BN / 2 : BN;
  static constexpr int SLABS = (BN_OUT + 63) / 64;   // 64-column output slabs per tile
  static constexpr int SLAB_BYTES = BM * 64 * 2;     // one 128-row x 64-column fp16 staging slab (TMA store source)
  // BN_OUT = 64 k + 32 (the 160-column tile): the last slab is 32 columns wide, staged with 64-byte rows and stored
  // through the 32-column tensor maps, so that it never writes the next tile's columns
  static constexpr bool NARROW_LAST = (BN_OUT % 64) == 32;
  static constexpr int ALL_SLAB_BYTES = SLABS * SLAB_BYTES - (NARROW_LAST ? SLAB_BYTES / 2 : 0);
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_LIMIT = 232448;          // 227 KiB per CTA
  // one staging slab per output slab when that fits (no buffer reuse inside a tile), else two (ping-pong)
  static constexpr int STG_SLABS =
      (TILE_BYTES + ALL_SLAB_BYTES + BAR_BYTES + 1024 <= SMEM_LIMIT) ? SLABS : (SLABS < 2 ? SLABS : 2);
  static constexpr int STG_BYTES = STG_SLABS == SLABS ? ALL_SLAB_BYTES : STG_SLABS * SLAB_BYTES;
  static constexpr int TOTAL = TILE_BYTES + STG_BYTES + BAR_BYTES + 1024;  // + alignment slack
  static_assert(TOTAL <= SMEM_LIMIT, "GEMM shared-memory budget exceeded");
  static_assert(STG_SLABS <= 4, "residual barriers");
};

constexpr int GEMM_THREADS = 384;   // warpgroup 0 producer, warpgroups 1-2 MMA + epilogue (64 tile rows each)
constexpr int GEMM_MMA_THREADS = 256;

// Persistent kernel: grid = min(#tiles, #SMs); every CTA walks tiles blockIdx.x, +gridDim.x, ...  The stage ring runs
// continuously across tiles.
template <int BN, int STAGES, bool GEGLU>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_f16_kernel(const __grid_constant__ TmapSet4 amaps,
                                                                    const __grid_constant__ CUtensorMap bmap,
                                                                    const __grid_constant__ CUtensorMap omap,
                                                                    const __grid_constant__ CUtensorMap rmap,
                                                                    const __grid_constant__ CUtensorMap omap32,
                                                                    const __grid_constant__ CUtensorMap rmap32,
                                                                    const GemmParams p) {
  using S = GemmSmem<BN, STAGES, GEGLU>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stg = smem + S::TILE_BYTES;            // [STG_SLABS] epilogue staging slabs, 16 KiB each (1024-aligned)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::TILE_BYTES + S::STG_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* res_bar = empty_bar + STAGES;         // [4] residual slab landed (one per staging slab)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  auto stamp = [&](int slot) {
    if (p.trace && blockIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      p.trace[slot] = t;
    }
  };
  if (threadIdx.x == 0) stamp(0);
  constexpr int BN_OUT = GEGLU ? BN / 2 : BN;
  const int n_tiles = (p.N + BN_OUT - 1) / BN_OUT;
  const int num_tiles = n_tiles * p.m_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&amaps.m[0]);
    tma_prefetch_desc(&bmap);
    tma_prefetch_desc(&omap);
    if (S::NARROW_LAST) tma_prefetch_desc(&omap32);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], GEMM_MMA_THREADS / 32);   // lane 0 of every MMA warp
    }
    for (int a = 0; a < 4; ++a) mbar_init(&res_bar[a], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp(1);
  pdl_launch_dependents();  // the next kernel may begin its prologue now ...
  pdl_wait();               // ... and we may not touch global memory before our predecessor has finished
  if (threadIdx.x == 0) stamp(2);

  if (warp < 4) {
    // ------------------------------ producer warpgroup ------------------------------
    setmaxnreg_dec<40>();
    if (warp == 0) {
      // TMA: whole warp in uniform control flow; one elected lane arms the barrier and issues the loads
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n_tile = tile % n_tiles;
        const int m_tile = tile / n_tiles;
        const int n0 = n_tile * BN_OUT;
        const int m0 = m_tile * BM;
        int img = 0, x0 = 0, y0 = 0;
        if (p.mode == 1) {
          const int per_img = p.tiles_x * p.tiles_y;
          img = m_tile / per_img;
          const int t = m_tile - img * per_img;
          y0 = (t / p.tiles_x) * p.bh;
          x0 = (t % p.tiles_x) * p.bw;
        }
        // conv: the tap of a K block is tracked incrementally (warp-uniform registers): tap_lo <= kb < tap_hi
        int tap = 0, tap_lo = 0, tap_hi = p.mode == 1 ? p.tap_kb_end[0] : 0x7fffffff;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          if (kb == tap_hi) {
            ++tap;
            tap_lo = tap_hi;
            tap_hi = p.tap_kb_end[tap];
          }
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sA = smem + stage * S::STAGE_BYTES;
          uint8_t* sB = sA + A_STAGE_BYTES;
          if (elect_one()) {
            mbar_arrive_expect_tx(&full_bar[stage], S::STAGE_BYTES);
            if (p.mode == 0) {
              tma_load_2d(sA, &amaps.m[0], &full_bar[stage], kb * BK, m0);
            } else {
              const int ckb = kb - tap_lo;
              tma_load_4d(sA, &amaps.m[p.tap_map[tap]], &full_bar[stage], ckb * BK, x0 + p.tap_ox[tap],
                          y0 + p.tap_oy[tap], img);
            }
            if (GEGLU) {
              tma_load_2d(sB, &bmap, &full_bar[stage], kb * BK, n0);
              tma_load_2d(sB + (BN / 2) * BK * 2, &bmap, &full_bar[stage], kb * BK, p.gate_row_off + n0);
            } else {
              tma_load_2d(sB, &bmap, &full_bar[stage], kb * BK, n0);
            }
          }
          __syncwarp();
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    } else if (warp == 1 && lane == 0 && p.pf_ptr) {
      // my 1/gridDim slice of the next kernel's weights -> L2 (a hint: no completion to wait for)
      constexpr unsigned long long CH = 16384;
      const unsigned long long per = ((p.pf_bytes / gridDim.x) + CH - 1) / CH * CH;
      unsigned long long off = per * blockIdx.x;
      const unsigned long long end = off + per < p.pf_bytes ? off + per : p.pf_bytes;
      for (; off < end; off += CH) {
        const unsigned long long n = end - off < CH ? ((end - off) & ~15ull) : CH;
        if (n) l2_prefetch_bulk(p.pf_ptr + off, (uint32_t)n);
      }
    }
  } else {
    // ------------------------------ MMA + epilogue warpgroups ------------------------------
    setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;            // rows [64 wg, 64 wg + 64) of the tile
    const int ct = threadIdx.x - 128;                 // 0..255
    const int r0 = wg * 64 + ((warp & 3) << 4) + (lane >> 2);   // my accumulator rows: r0, r0 + 8
    const int cq = (lane & 3) << 1;                   // my column pair inside every 8-column group
    const bool issuer = (ct == 0);
    constexpr int SLABS = S::SLABS;
    constexpr int NBUF = S::STG_SLABS;
    // Epilogue latency cuts for every tile but the 256-row ones: the LayerNorm statistics of both rows in flight
    // together, each slab's bias columns loaded ahead of its stores, and the lazy store drain.  The 256-row tiles keep
    // the plain order: their 128 accumulator registers leave no room for the batched loads, and the GEGLU tile got
    // slower with the restructured epilogue even where it did not spill (DESIGN section 3).
    constexpr bool FAST_EPI = BN != 256;
    uint32_t res_par = 0;                             // bit b: parity of res_bar[b]
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    // slab sl of the tile: 64 columns in a 128 B-row staging buffer, or (the last slab of a 160-column tile) 32
    // columns in 64 B rows, fetched and stored through the 32-column tensor maps
    auto narrow = [](int sl) { return S::NARROW_LAST && sl == SLABS - 1; };
    auto load_residual = [&](int sl, uint8_t* dst, uint64_t* bar, int col0, int m_tile, int x0, int y0, int img) {
      const CUtensorMap* m = narrow(sl) ? &rmap32 : &rmap;
      mbar_arrive_expect_tx(bar, narrow(sl) ? BM * 64 : BM * 128);
      if (p.mode == 0) tma_load_2d(dst, m, bar, col0, m_tile * BM);
      else tma_load_4d(dst, m, bar, col0, x0, y0, img);
    };
    // byte offset of the 16-byte chunk c of row r inside a staging slab (the TMA swizzle of the slab's tensor map)
    auto stg_off = [&](int sl, int r, int c) {
      return narrow(sl) ? r * 64 + ((c ^ ((r >> 1) & 3)) << 4) : r * 128 + ((c ^ (r & 7)) << 4);
    };
    float carry_sum = 0.f, carry_sq = 0.f;            // row statistics of slab 0 of an odd 160-column tile
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int n_tile = tile % n_tiles;
      const int m_tile = tile / n_tiles;
      const int n0 = n_tile * BN_OUT;
      int img = 0, x0 = 0, y0 = 0;
      if (p.mode == 1) {
        const int per_img = p.tiles_x * p.tiles_y;
        img = m_tile / per_img;
        const int t = m_tile - img * per_img;
        y0 = (t / p.tiles_x) * p.bh;
        x0 = (t % p.tiles_x) * p.bw;
      }
      // residual slabs of the first NBUF slabs are fetched now, behind the main loop (the staging buffers are free:
      // the previous tile ended after its stores had read them)
      if (issuer && p.residual) {
#pragma unroll
        for (int sl = 0; sl < SLABS && sl < NBUF; ++sl) {
          const int col0 = n0 + sl * 64;
          if (col0 >= p.N) break;
          load_residual(sl, stg + sl * S::SLAB_BYTES, &res_bar[sl], col0, m_tile, x0, y0, img);
        }
      }

      // ---- main loop: one wgmma group per K block in flight; a stage is released once its group has completed
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (issuer && it == 0 && kb == 0) stamp(3);
        const uint32_t a_addr = smem_u32(smem + stage * S::STAGE_BYTES) + wg * (64 * 128);
        const uint32_t b_addr = smem_u32(smem + stage * S::STAGE_BYTES + A_STAGE_BYTES);
        const uint64_t a_desc = wgmma_desc_sw128(a_addr);
        const uint64_t b_desc = wgmma_desc_sw128(b_addr);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)   // +32 bytes per K=16 step inside the 128 B swizzle row
          wgmma_ss<BN>(acc, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0 ? 1 : 0);
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      if (issuer) stamp(4 + (it < 3 ? it : 3));

      // ---- epilogue: registers -> bias / LN-fold / activation / GEGLU / residual -> fp16 pairs in the 128B-swizzled
      // staging slab -> TMA store (clipped at the M / N / image edges by the tensor map)
      long long orow[2];
      float rstd[2];
      const __half* rb[2] = {nullptr, nullptr};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        if (p.mode == 0) {
          orow[h] = (long long)m_tile * BM + r;
        } else {
          const int hh = r / p.bw, ww = r - hh * p.bw;
          int y = y0 + hh, x = x0 + ww;
          if (y >= p.Ho) y = p.Ho - 1;   // clamped rows are clipped by the TMA store; keep the row-bias index in range
          if (x >= p.Wo) x = p.Wo - 1;
          orow[h] = ((long long)img * p.Ho + y) * p.Wo + x;
        }
        if (p.rowbias) {
          const long long max_grp = ((long long)p.M - 1) / p.rows_per_group;
          long long grp = orow[h] / p.rows_per_group;
          if (grp > max_grp) grp = max_grp;
          rb[h] = p.rowbias + grp * p.ld_rowbias;
        }
        // folded LayerNorm: 1 / std of the row from the producer's slabs
        rstd[h] = p.alpha;
        if (!FAST_EPI && p.ln_stats && orow[h] < p.M) {
          const float2* st = reinterpret_cast<const float2*>(p.ln_stats) + orow[h];   // [slab][row]
          float ssum = 0.f, ssq = 0.f;
          for (int i0 = 0; i0 < p.ln_slabs; i0 += 10) {   // 10 independent loads in flight
            float2 t[10];
#pragma unroll
            for (int i = 0; i < 10; ++i)
              t[i] = (i0 + i < p.ln_slabs) ? __ldg(st + (long long)(i0 + i) * p.M) : make_float2(0.f, 0.f);
#pragma unroll
            for (int i = 0; i < 10; ++i) {
              ssum += t[i].x;
              ssq += t[i].y;
            }
          }
          const float ln_mean = ssum * p.ln_inv_c;
          const float var = fmaxf(ssq * p.ln_inv_c - ln_mean * ln_mean, 0.f);
          rstd[h] = p.alpha * rsqrtf(var + p.ln_eps);
        }
      }
      if constexpr (FAST_EPI) {
        // the same per-row sums in the same slab order, with the loads of both rows in flight together
        if (p.ln_stats) {
          const bool ok[2] = {orow[0] < p.M, orow[1] < p.M};
          float ssum[2] = {0.f, 0.f}, ssq[2] = {0.f, 0.f};
          for (int i0 = 0; i0 < p.ln_slabs; i0 += 10) {
            float2 t[2][10];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float2* st = reinterpret_cast<const float2*>(p.ln_stats) + orow[h];   // [slab][row]
#pragma unroll
              for (int i = 0; i < 10; ++i)
                t[h][i] = (ok[h] && i0 + i < p.ln_slabs) ? __ldg(st + (long long)(i0 + i) * p.M) : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int i = 0; i < 10; ++i) {
                ssum[h] += t[h][i].x;
                ssq[h] += t[h][i].y;
              }
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (ok[h]) {
              const float ln_mean = ssum[h] * p.ln_inv_c;
              const float var = fmaxf(ssq[h] * p.ln_inv_c - ln_mean * ln_mean, 0.f);
              rstd[h] = p.alpha * rsqrtf(var + p.ln_eps);
            }
          }
        }
        // lazy store drain: without a residual nothing writes staging between the last slab of one tile and the first
        // slab of the next, so the previous tile's stores are waited for here, after this tile's main loop, rather
        // than before it; the barrier also keeps the previous tile's statistics readers ahead of the overwrite
        if (!p.residual && it > 0) {
          if (issuer) tma_store_wait_read0();
          named_bar_sync(1, GEMM_MMA_THREADS);
        }
      }
#pragma unroll
      for (int sl = 0; sl < SLABS; ++sl) {
        const int col0 = n0 + sl * 64;
        if (col0 < p.N) {
          // the slab's bias, gate-bias and row-bias columns, loaded ahead of the waits and stores below: loaded where
          // they are used, each would wait behind the staging stores before it (one global round trip per 8 columns)
          __half2 bh[8], gh[8], rh[2][8];
          if constexpr (FAST_EPI) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = col0 + j * 8 + cq;
              const bool ok = j < (narrow(sl) ? 4 : 8) && col < p.N;
              bh[j] = gh[j] = rh[0][j] = rh[1][j] = __float2half2_rn(0.f);
              if (p.bias && ok) {
                bh[j] = *reinterpret_cast<const __half2*>(p.bias + col);
                if (GEGLU) gh[j] = *reinterpret_cast<const __half2*>(p.bias + p.gate_row_off + col);
              }
#pragma unroll
              for (int h = 0; h < 2; ++h)
                if (rb[h] && ok) rh[h][j] = *reinterpret_cast<const __half2*>(rb[h] + col);
            }
          }
          const int buf = sl % NBUF;
          uint8_t* sbuf = stg + buf * S::SLAB_BYTES;
          if (sl >= NBUF) {
            // staging-buffer reuse: the store of slab sl - NBUF must have read the buffer out; then the residual slab
            // is fetched into it
            if (issuer) {
              tma_store_wait_read<(NBUF > 1 ? NBUF - 1 : 0)>();
              if (p.residual) load_residual(sl, sbuf, &res_bar[buf], col0, m_tile, x0, y0, img);
            }
            named_bar_sync(1, GEMM_MMA_THREADS);
          }
          if (p.residual) {
            mbar_wait(&res_bar[buf], (res_par >> buf) & 1u);
            res_par ^= 1u << buf;
          }
#pragma unroll
          for (int j = 0; j < (narrow(sl) ? 4 : 8); ++j) {
            const int i = sl * 8 + j;                // accumulator 8-column group (GEGLU: value half)
            const int lc = sl * 64 + j * 8 + cq;     // tile-local output column of my pair
            const int col = n0 + lc;
            const bool col_ok = col < p.N;
            float2 bv = make_float2(0.f, 0.f), bg = make_float2(0.f, 0.f);
            if constexpr (FAST_EPI) {
              bv = __half22float2(bh[j]);   // zero without a bias
              bg = __half22float2(gh[j]);
            } else if (p.bias && col_ok) {
              bv = __half22float2(*reinterpret_cast<const __half2*>(p.bias + col));
              if (GEGLU) bg = __half22float2(*reinterpret_cast<const __half2*>(p.bias + p.gate_row_off + col));
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = r0 + 8 * h;
              float x0v = fmaf(rstd[h], acc[4 * i + 2 * h], bv.x);
              float x1v = fmaf(rstd[h], acc[4 * i + 2 * h + 1], bv.y);
              if (GEGLU) {
                constexpr int G = BN / 16;           // the gate columns sit BN / 2 columns (BN / 16 groups) further
                x0v *= gelu_erf_f(fmaf(rstd[h], acc[4 * (i + G) + 2 * h], bg.x));
                x1v *= gelu_erf_f(fmaf(rstd[h], acc[4 * (i + G) + 2 * h + 1], bg.y));
              }
              if (rb[h] && col_ok) {
                const float2 f = FAST_EPI ? __half22float2(rh[h][j])
                                          : __half22float2(*reinterpret_cast<const __half2*>(rb[h] + col));
                x0v += f.x;
                x1v += f.y;
              }
              if (p.act == 1) {
                x0v = silu_f(x0v);
                x1v = silu_f(x1v);
              } else if (p.act == 2) {
                x0v = gelu_erf_f(x0v);
                x1v = gelu_erf_f(x1v);
              } else if (p.act == 3) {   // quick_gelu x * sigmoid(1.702 x) ([3P] CLIP-L text tower MLP)
                x0v = __fdividef(x0v, 1.f + __expf(-1.702f * x0v));
                x1v = __fdividef(x1v, 1.f + __expf(-1.702f * x1v));
              }
              uint32_t* slot = reinterpret_cast<uint32_t*>(sbuf + stg_off(sl, r, j) + cq * 2);
              if (p.residual) {
                const float2 f = unpack_half2(*slot);
                x0v += f.x;
                x1v += f.y;
              }
              if (p.relu) {
                x0v = relu_nan_f(x0v);
                x1v = relu_nan_f(x1v);
              }
              *slot = pack_half2(x0v, x1v);
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(2, GEMM_MMA_THREADS);      // the slab is complete in shared memory
          if (issuer) {
            const CUtensorMap* m = narrow(sl) ? &omap32 : &omap;
            if (p.mode == 0) tma_store_2d(m, sbuf, col0, m_tile * BM);
            else tma_store_4d(m, sbuf, col0, x0, y0, img);
            tma_store_commit();
          }
          // row statistics of exactly the fp16 values a later LayerNorm would read: one warpgroup per slab, one row
          // per thread, re-read from the staging buffer; one writer per (slot, row).  Each slot holds a partial sum
          // of the row's statistics and the total over all slots is the row's: 64-column tiles write slot col0 / 64; a pair
          // of 160-column tiles covers the 5 slots of its 320 columns -- the even tile writes its three slabs into the
          // first three, the odd tile its slabs 0 + 2 (96 columns) into the fourth and slab 1 into the fifth.
          if (p.stats_out && wg == (sl & 1)) {
            const int r = ct & 127;
            const long long srow = (long long)m_tile * BM + r;
            if (srow < p.M) {
              float st_sum = 0.f, st_sq = 0.f;
#pragma unroll
              for (int c = 0; c < (narrow(sl) ? 4 : 8); ++c) {
                if (col0 + c * 8 < p.N) {
                  const uint4 o = *reinterpret_cast<const uint4*>(sbuf + stg_off(sl, r, c));
                  const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 f = unpack_half2(ow[e]);
                    st_sum += f.x + f.y;
                    st_sq = fmaf(f.x, f.x, fmaf(f.y, f.y, st_sq));
                  }
                }
              }
              int slot = col0 >> 6;
              bool write = true;
              if (BN_OUT == 160) {
                const int base = (n_tile >> 1) * 5;
                if ((n_tile & 1) == 0) {
                  slot = base + sl;
                } else if (sl == 0) {
                  carry_sum = st_sum;
                  carry_sq = st_sq;
                  write = false;
                } else {
                  slot = base + (sl == 1 ? 4 : 3);
                  if (sl == 2) {
                    st_sum += carry_sum;
                    st_sq += carry_sq;
                  }
                }
              }
              if (write)
                reinterpret_cast<float2*>(p.stats_out)[(long long)slot * p.M + srow] = make_float2(st_sum, st_sq);
            }
          }
        }
      }
      // the staging buffers may be rewritten (next tile) / must stay valid (kernel end) until the bulk stores have read
      // them; global visibility is given by kernel completion (the next kernel's griddepcontrol.wait / stream order)
      if (!FAST_EPI || p.residual) {
        if (issuer) tma_store_wait_read0();
        named_bar_sync(1, GEMM_MMA_THREADS);        // statistics readers are done with the staging buffers too
      }
    }
    if (FAST_EPI && issuer) tma_store_wait_read0();   // lazy drain: the last tile's stores read out before exit
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp(8);
}

// ------------------------------------------------------------------------------------------------
// Ping-pong GEMM for the LayerNorm-folded GEGLU-in and q|k|v launches (plain GEMM mode; bias, LN fold and GEGLU only).
//
// In gemm_f16_kernel both MMA warpgroups share every tile, so the tensor cores idle through each epilogue; with the
// 10-20 k-blocks of a transformer GEMM that is about half of a multi-round launch.  Here each MMA warpgroup owns WHOLE
// 128 x 128 tiles (two m64n128 blocks, 128 accumulator registers): CTA c walks tiles c, c + grid, ... (numbered as in
// pp_tile_coords) and hands them to warpgroup 1, 2, 1, 2, ..., so one warpgroup's epilogue runs under the other's main
// loop.  One producer warp fills one stage ring with the k-blocks of all the CTA's tiles in that order, and the two MMA
// warpgroups consume it in turn (as CUTLASS's ping-pong does): the running main loop has the whole ring of loads in
// flight ahead of it, instead of half of it while the idle warpgroup's half sits full.  The main loops take turns
// through two named barriers, so the two warpgroups' epilogues do not fall together.
// The epilogue is gemm_f16_kernel's expressions in the same order -- the LayerNorm statistics summed in slab order,
// fmaf(rstd, acc, bias), gelu_erf_f on the gate, pack_half2 -- so the outputs are bitwise equal to it.  The LayerNorm
// statistics of the tile's rows and its bias columns are fetched during the main loop.
// ------------------------------------------------------------------------------------------------
constexpr int PP_STAGES = 6;      // one ring, shared by both MMA warpgroups
constexpr int PP_BN = 128;        // B-tile rows (GEGLU: 64 value + 64 gate rows, 64 outputs)
// named barriers (gemm_f16_kernel uses 1 and 2): 3 + wg lets warpgroup wg start its next main loop, 5 + wg is its
// epilogue barrier
constexpr int PP_BAR_ORDER = 3;
constexpr int PP_BAR_EPI = 5;

// Tile order: bands of PP_BAND row tiles, M fastest inside a band.  The 132 tiles in flight then share 16 A row
// blocks and about 8 weight column blocks, instead of (N fastest) reading the whole weight -- 26 MB for a 1024^2
// GEGLU-in -- for every 1.6 rows of tiles, or (M fastest) the whole of a tall A for every column.  A permutation of
// whole tiles: each output element is computed as before.  The last band may be narrower.
constexpr int PP_BAND = 16;

__device__ __forceinline__ void pp_tile_coords(int tile, int n_tiles, int m_tiles, int& m_tile, int& n_tile) {
  const int first = tile / (PP_BAND * n_tiles) * PP_BAND;
  const int rows = min(PP_BAND, m_tiles - first);
  const int r = tile - first * n_tiles;
  m_tile = first + r % rows;
  n_tile = r / rows;
}

struct PpOperands {   // one MMA warpgroup's epilogue operands of its current tile
  float rstd[BM];      // alpha (LayerNorm folded: alpha / std) of every tile row
  __half2 bias[64];    // bias pairs of the tile's columns (GEGLU: 32 value pairs, then 32 gate pairs)
};

template <bool GEGLU>
struct PpSmem {
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + PP_BN * BK * 2;   // 32 KiB
  static constexpr int RING_BYTES = PP_STAGES * STAGE_BYTES;
  static constexpr int BN_OUT = GEGLU ? PP_BN / 2 : PP_BN;
  static constexpr int SLABS = BN_OUT / 64;
  static constexpr int SLAB_BYTES = BM * 64 * 2;
  static constexpr int STG_BYTES = 2 * SLAB_BYTES;   // one staging slab per MMA warpgroup
  static constexpr int BAR_BYTES = 128;              // full and empty barriers of the ring
  static constexpr int TOTAL = RING_BYTES + STG_BYTES + BAR_BYTES + 2 * sizeof(PpOperands) + 1024;   // + alignment slack
  static_assert(2 * PP_STAGES * 8 <= BAR_BYTES, "ping-pong GEMM barriers");
  static_assert(TOTAL <= GemmSmem<128, 6, false>::SMEM_LIMIT, "ping-pong GEMM shared-memory budget exceeded");
};

template <bool GEGLU>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_pp_f16_kernel(const __grid_constant__ CUtensorMap amap,
                                                                       const __grid_constant__ CUtensorMap bmap,
                                                                       const __grid_constant__ CUtensorMap omap,
                                                                       const GemmParams p) {
  using S = PpSmem<GEGLU>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stg = smem + S::RING_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::RING_BYTES + S::STG_BYTES);
  uint64_t* empty_bar = full_bar + PP_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  auto stamp = [&](int slot) {
    if (p.trace && blockIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      p.trace[slot] = t;
    }
  };
  if (threadIdx.x == 0) stamp(0);
  constexpr int BN_OUT = S::BN_OUT;
  const int n_tiles = (p.N + BN_OUT - 1) / BN_OUT;
  const int num_tiles = n_tiles * p.m_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&amap);
    tma_prefetch_desc(&bmap);
    tma_prefetch_desc(&omap);
    for (int s = 0; s < PP_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);   // lane 0 of the four warps of the MMA warpgroup that consumed the stage
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp(1);
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) stamp(2);

  if (warp < 4) {
    // ------------------------------ producer warpgroup ------------------------------
    setmaxnreg_dec<40>();
    if (warp == 0) {
      // every k-block of the CTA's tiles, in the order the two MMA warpgroups take them
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_tile, n_tile;
        pp_tile_coords(tile, n_tiles, p.m_tiles, m_tile, n_tile);
        const int n0 = n_tile * BN_OUT;
        const int m0 = m_tile * BM;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sA = smem + stage * S::STAGE_BYTES;
          uint8_t* sB = sA + A_STAGE_BYTES;
          if (elect_one()) {
            mbar_arrive_expect_tx(&full_bar[stage], S::STAGE_BYTES);
            tma_load_2d(sA, &amap, &full_bar[stage], kb * BK, m0);
            tma_load_2d(sB, &bmap, &full_bar[stage], kb * BK, n0);
            if (GEGLU) tma_load_2d(sB + (PP_BN / 2) * BK * 2, &bmap, &full_bar[stage], kb * BK, p.gate_row_off + n0);
          }
          __syncwarp();
          if (++stage == PP_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    } else if (warp == 1 && lane == 0 && p.pf_ptr) {
      constexpr unsigned long long CH = 16384;
      const unsigned long long per = ((p.pf_bytes / gridDim.x) + CH - 1) / CH * CH;
      unsigned long long off = per * blockIdx.x;
      const unsigned long long end = off + per < p.pf_bytes ? off + per : p.pf_bytes;
      for (; off < end; off += CH) {
        const unsigned long long n = end - off < CH ? ((end - off) & ~15ull) : CH;
        if (n) l2_prefetch_bulk(p.pf_ptr + off, (uint32_t)n);
      }
    }
  } else {
    // ------------------------------ MMA + epilogue warpgroups, one whole tile each ------------------------------
    setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int rw = ((warp & 3) << 4) + (lane >> 2);   // my accumulator rows: 64 mb + rw + 8 h
    const int cq = (lane & 3) << 1;                   // my column pair inside every 8-column group
    const int t = threadIdx.x & 127;
    const bool issuer = t == 0;
    uint8_t* my_stg = stg + wg * S::SLAB_BYTES;
    PpOperands* my_ops = reinterpret_cast<PpOperands*>(smem + S::RING_BYTES + S::STG_BYTES + S::BAR_BYTES) + wg;
    const int ln_n = p.ln_stats ? p.ln_slabs : 0;
    const float2* ln_st = reinterpret_cast<const float2*>(p.ln_stats);   // [slab][row]
    float acc[2][PP_BN / 2];
    int j = wg;   // index of the tile among this CTA's tiles
    for (int tile = blockIdx.x + wg * gridDim.x; tile < num_tiles; tile += 2 * gridDim.x, j += 2) {
      int m_tile, n_tile;
      pp_tile_coords(tile, n_tiles, p.m_tiles, m_tile, n_tile);
      const int n0 = n_tile * BN_OUT;
      // epilogue operands, fetched behind the main loop and handed over in shared memory: the warpgroup's thread t
      // sums the LayerNorm statistics of tile row t, the load of slab kb + 1 in flight behind k-block kb, and threads
      // 0..63 fetch one bias pair each (GEGLU: 32 value pairs, then 32 gate pairs)
      const long long ln_row = (long long)m_tile * BM + t;
      const bool ln_ok = ln_row < p.M;
      auto ln_load = [&](int s) {
        return ln_ok && s < ln_n ? __ldg(ln_st + (long long)s * p.M + ln_row) : make_float2(0.f, 0.f);
      };
      float ssum = 0.f, ssq = 0.f;
      float2 st = ln_load(0);
      auto ln_step = [&](int s) {   // add slab s (in st) to the row's sums, then fetch slab s + 1
        ssum += st.x;
        ssq += st.y;
        st = ln_load(s + 1);
      };
      __half2 bias_pair = __float2half2_rn(0.f);
      {
        const int col = n0 + 2 * (GEGLU ? (t & 31) : t);
        if (t < 64 && p.bias && col < p.N)
          bias_pair = *reinterpret_cast<const __half2*>(p.bias + ((GEGLU && t >= 32) ? p.gate_row_off : 0) + col);
      }

      // ---- main loop, after the other warpgroup has issued all of the CTA's previous tile
      if (j > 0) named_bar_sync(PP_BAR_ORDER + wg, 256);
      // The tile's k-blocks are the ring's k-blocks g = j num_kb, j num_kb + 1, ...; k-block g fills stage g % STAGES in
      // the stage's phase g / STAGES.  A parity wait cannot tell phase n from phase n - 2, so it is only sound if the
      // stage's full barrier has completed at least g / STAGES phases when the wait starts, i.e. if k-block g - STAGES
      // has landed.  The turn-taking above gives that: every k-block before g belongs to an earlier tile of this CTA,
      // and the main loop of that tile (this warpgroup's, or the other's, which passed the named barrier only after its
      // last wait) has waited for it.  Nor can the barrier be a phase further on: the producer refills a stage only
      // after the warpgroup that waits on it has freed it.
      const int g = j * p.num_kb;
      int stage = g % PP_STAGES;
      uint32_t phase = (g / PP_STAGES) & 1;
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (issuer && j == 0 && kb == 0) stamp(3);
        const uint32_t a_addr = smem_u32(smem + stage * S::STAGE_BYTES);
        const uint64_t a_desc0 = wgmma_desc_sw128(a_addr);
        const uint64_t a_desc1 = wgmma_desc_sw128(a_addr + 64 * 128);
        const uint64_t b_desc = wgmma_desc_sw128(a_addr + A_STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          wgmma_ss<PP_BN>(acc[0], a_desc0 + 2 * k, b_desc + 2 * k, (kb | k) != 0 ? 1 : 0);
          wgmma_ss<PP_BN>(acc[1], a_desc1 + 2 * k, b_desc + 2 * k, (kb | k) != 0 ? 1 : 0);
        }
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == PP_STAGES) {
          stage = 0;
          phase ^= 1;
        }
        if (kb == 0 && t < 64) my_ops->bias[t] = bias_pair;
        if (kb < ln_n) ln_step(kb);
      }
      // this tile's MMAs are issued: the other warpgroup may start the CTA's next tile
      if (tile + gridDim.x < num_tiles) named_bar_arrive(PP_BAR_ORDER + (wg ^ 1), 256);
      wgmma_wait<0>();
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      if (issuer) stamp(4 + (j < 3 ? j : 3));

      // ---- epilogue: the same expressions in the same order as gemm_f16_kernel
      for (int s = p.num_kb; s < ln_n; ++s) ln_step(s);   // statistics slabs past the k-blocks
      float rstd = p.alpha;
      if (ln_n && ln_ok) {
        const float ln_mean = ssum * p.ln_inv_c;
        const float var = fmaxf(ssq * p.ln_inv_c - ln_mean * ln_mean, 0.f);
        rstd = p.alpha * rsqrtf(var + p.ln_eps);
      }
      my_ops->rstd[t] = rstd;
      const uint32_t stg_row = smem_u32(my_stg) + rw * 128 + cq * 2;   // rows 64 mb + rw + 8 h: (row & 7) == lane >> 2
      const uint32_t ops_bias = smem_u32(my_ops->bias) + (cq >> 1) * 4;
#pragma unroll
      for (int sl = 0; sl < S::SLABS; ++sl) {
        // the staging slab is rewritten: the stores of my previous slab must have read it out; the first barrier of
        // the tile also publishes the operands above
        if (issuer) tma_store_wait_read0();
        named_bar_sync(PP_BAR_EPI + wg, 128);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int mb = q >> 1, h = q & 1;
          const float rs = __uint_as_float(ld_shared_u32(smem_u32(my_ops->rstd) + (64 * mb + rw + 8 * h) * 4));
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const int i = sl * 8 + c;   // accumulator 8-column group; its bias pair is 4 i + cq / 2 (GEGLU gate: + 32)
            const float2 bv = unpack_half2(ld_shared_u32(ops_bias + 16 * i));
            float x0v = fmaf(rs, acc[mb][4 * i + 2 * h], bv.x);
            float x1v = fmaf(rs, acc[mb][4 * i + 2 * h + 1], bv.y);
            if (GEGLU) {
              const float2 bg = unpack_half2(ld_shared_u32(ops_bias + 128 + 16 * i));
              x0v *= gelu_erf_f(fmaf(rs, acc[mb][4 * (i + 8) + 2 * h], bg.x));
              x1v *= gelu_erf_f(fmaf(rs, acc[mb][4 * (i + 8) + 2 * h + 1], bg.y));
            }
            st_shared_u32(stg_row + (64 * mb + 8 * h) * 128 + ((c ^ (lane >> 2)) << 4), pack_half2(x0v, x1v));
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(PP_BAR_EPI + wg, 128);   // the slab is complete in staging
        if (issuer) {
          if (n0 + sl * 64 < p.N) tma_store_2d(&omap, my_stg, n0 + sl * 64, m_tile * BM);
          tma_store_commit();
        }
      }
    }
    if (issuer) tma_store_wait_read0();   // staging stays valid until the last stores have read it
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp(8);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// The output (and residual) tensor as the epilogue's TMA stores and loads see it: 64-column slabs with a 128-byte
// swizzle, and, for the 160-column tile, its 32-column last slab with a 64-byte swizzle.
struct OutMaps {
  CUtensorMap o, r, o32, r32;
};
struct OutView {
  void* out;
  const void* residual;
  int rank;
  uint64_t dims[4];
  uint64_t ostr[3], rstr[3];
  uint32_t box[4];   // box[0] (the column count) is set per slab width
};

static int out_maps(const OutView& v, bool narrow_slab, OutMaps& m) {
  uint32_t box[4] = {64u, v.box[1], v.box[2], v.box[3]};
  int rc = get_tmap_f16(&m.o, v.out, v.rank, v.dims, v.ostr, box);
  if (rc) return rc;
  m.r = m.o;
  if (v.residual && (rc = get_tmap_f16(&m.r, v.residual, v.rank, v.dims, v.rstr, box))) return rc;
  m.o32 = m.o;
  m.r32 = m.r;
  if (narrow_slab) {
    box[0] = 32u;
    if ((rc = get_tmap_f16(&m.o32, v.out, v.rank, v.dims, v.ostr, box, 64))) return rc;
    if (v.residual && (rc = get_tmap_f16(&m.r32, v.residual, v.rank, v.dims, v.rstr, box, 64))) return rc;
  }
  return 0;
}

template <int BN, int STAGES, bool GEGLU>
static int launch_gemm(const TmapSet4& amaps, const CUtensorMap& bmap, const OutMaps& om, GemmParams& p, int m_tiles,
                       cudaStream_t stream) {
  using S = GemmSmem<BN, STAGES, GEGLU>;
  static bool configured = false;
  auto kern = gemm_f16_kernel<BN, STAGES, GEGLU>;
  if (!configured) {
    IH_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    configured = true;
  }
  constexpr int BN_OUT = GEGLU ? BN / 2 : BN;
  p.m_tiles = m_tiles;
  const long long n_tiles = (p.N + BN_OUT - 1) / BN_OUT;
  const long long tiles = n_tiles * m_tiles;
  const int grid = (int)(tiles < num_sms() ? tiles : num_sms());
  IH_CUDA(launch_kernel(kern, dim3(grid), dim3(GEMM_THREADS), (size_t)(S::TOTAL), stream, amaps, bmap, om.o, om.r,
                        om.o32, om.r32, p));
  return 0;
}

template <bool GEGLU>
static int launch_gemm_pp(const TmapSet4& amaps, const CUtensorMap& bmap, const OutMaps& om, GemmParams& p, int m_tiles,
                          cudaStream_t stream) {
  using S = PpSmem<GEGLU>;
  static bool configured = false;
  auto kern = gemm_pp_f16_kernel<GEGLU>;
  if (!configured) {
    IH_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    configured = true;
  }
  p.m_tiles = m_tiles;
  const long long tiles = (long long)((p.N + S::BN_OUT - 1) / S::BN_OUT) * m_tiles;
  const int grid = (int)(tiles < num_sms() ? tiles : num_sms());
  IH_CUDA(launch_kernel(kern, dim3(grid), dim3(GEMM_THREADS), (size_t)(S::TOTAL), stream, amaps.m[0], bmap, om.o, p));
  return 0;
}

// Cost model for the persistent kernel (one CTA per SM): a launch takes `rounds` tiles per SM one after the other,
// each costing num_kb k-blocks of main loop plus a fixed part (pipeline fill, epilogue, store drain).  Padded columns of
// a partially filled last N tile cost as much as real ones.  160-column tiles need N % 320 == 0 when the launch writes
// row statistics (see the epilogue).  `cost` receives the chosen tile's estimate (not set for the 64-column tile).
static int pick_bn(long long m_tiles, int N, int num_kb, bool allow160, double* cost = nullptr) {
  if (N <= 64) return 64;
  const int sms = num_sms();
  // 128x64 tiles for launches that cannot fill the SMs with wider ones (e.g. the 1280-channel level of a 512^2 edit,
  // M = 512): each SM then streams fewer bytes per k-block and drains one slab.
  if (m_tiles * ((N + 63) / 64) <= sms) return 64;
  // Measured with tools/ab_probe.py tile (M = 2048, 128 tiles in one round, K = 1280 vs 5120) on an NVIDIA H100 80GB
  // HBM3 at a 400 W power limit: per k-block 0.583 / 0.706 / 0.877 / 1.161 us and fixed 3.3 / 3.7 / 3.9 / 8.8 us for
  // the 128 / 160 / 192 / 256-column tiles, here in units of the 128-column tile's k-block.  The main loop is
  // MMA-bound (cost ~ BN), not L2-bound; the 256-column tile's fixed part is larger because its epilogue ping-pongs
  // two staging slabs.
  double best = 1e30;
  int best_bn = 256;
  const int cands[4] = {256, 192, 160, 128};
  const double kb_cost[4] = {1.99, 1.50, 1.21, 1.0};
  const double fixed_cost[4] = {15.1, 6.7, 6.3, 5.7};
  for (int i = 0; i < 4; ++i) {
    const int bn = cands[i];
    if (bn == 160 && !allow160) continue;
    const long long tiles = m_tiles * ((N + bn - 1) / bn);
    const long long rounds = (tiles + sms - 1) / sms;
    const double t = (double)rounds * (kb_cost[i] * num_kb + fixed_cost[i]);
    if (t < best - 1e-9) {
      best = t;
      best_bn = bn;
    }
  }
  if (cost) *cost = best;
  return best_bn;
}

// Whether the ping-pong kernel beats gemm_f16_kernel's choice.  Both are linear models of the launch time in us, fitted
// to tools/ab_probe.py pp (the LayerNorm-folded q|k|v and GEGLU launches of the SDXL base and refiner UNets at 512^2 -
// 1024^2, 1 and 4 images; H100 80GB HBM3 at a 700 W power limit; DESIGN section 3), in the rounds R of tiles per SM:
//   ping-pong, plain  0.491 R kb + 0.515 R + 1.88     (128 x 128 tiles; within 12 % of the table)
//   ping-pong, GEGLU  0.479 R kb + 1.49 R - 1.18      (64 outputs per tile; within 17 %)
//   old, plain        0.620 (pick_bn's cost) + 2.35   (within 18 %)
//   old, GEGLU        0.972 R kb + 7.03 R - 1.73      (the 256-row tile, 128 outputs; within 10 %)
// These least-squares fits pick the faster kernel at every shape of the table.  The ping-pong GEGLU tile costs half as
// much per k-block of output as the 256-row tile and little per round, so it wins at every GEGLU shape of the table,
// the refiner's K = 1536 included.
static bool pick_pp(long long m_tiles, int N, int num_kb, bool geglu) {
  const int sms = num_sms();
  auto rounds = [&](int cols) { return (double)((m_tiles * ((N + cols - 1) / cols) + sms - 1) / sms); };
  if (geglu) {
    const double pp = rounds(64) * (0.479 * num_kb + 1.49) - 1.18;
    const double old = rounds(128) * (0.972 * num_kb + 7.03) - 1.73;
    return pp < old;
  }
  double cost;
  if (pick_bn(m_tiles, N, num_kb, true, &cost) == 64) return false;   // one round of narrow tiles: not in the table
  return rounds(128) * (0.491 * num_kb + 0.515) + 1.88 < 0.620 * cost + 2.35;
}

static int dispatch(const TmapSet4& amaps, const OutView& ov, const void* w, int ldw_rows, long long K, GemmParams& p,
                    int m_tiles, int geglu, int force_bn, cudaStream_t stream) {
  // tile_n: 0 = the cost model's choice, 64 / 128 / 160 / 192 / 256 force that tile width; 512 and 384 (the widest
  // tiles a caller may ask for) are the 256- and 192-column tiles.  For GEGLU the width counts the B tile's rows
  // (value and gate halves: 128 / 192 / 256, i.e. 64 / 96 / 128 outputs per tile).
  if (force_bn == 512) force_bn = 256;
  if (force_bn == 384) force_bn = 192;
  // the ping-pong kernel: bias, LayerNorm fold and GEGLU only (the q|k|v and GEGLU-in launches of a transformer block)
  const bool pp_ok = p.mode == 0 && !p.residual && !p.rowbias && !p.stats_out && p.act == 0 && !p.relu && p.alpha == 1.f;
  IH_CHECK(force_bn != IH_TILE_PINGPONG || pp_ok, IH_ERR_ARG,
           "ih_gemm_f16: tile_n = IH_TILE_PINGPONG supports bias, LayerNorm folding and GEGLU only");
  const bool pp = force_bn == IH_TILE_PINGPONG || (force_bn == 0 && pp_ok && pick_pp(m_tiles, p.N, p.num_kb, geglu));
  int bn = PP_BN;   // the ping-pong tile: 128 B-tile rows
  if (!pp && geglu) {
    // 256 unless asked: it is the fastest GEGLU tile of this kernel at the UNet's shapes (tools/ab_probe.py geglu,
    // DESIGN section 3)
    bn = force_bn > 0 ? force_bn : 256;
    IH_CHECK(bn == 128 || bn == 192 || bn == 256, IH_ERR_ARG, "ih_gemm_f16: GEGLU tile_n must be 128, 192 or 256 (got %d)",
             bn);
    // the 96-output tile would split a 64-column statistics slot between two tiles
    IH_CHECK(bn != 192 || !p.stats_out, IH_ERR_SHAPE, "ih_gemm_ln_f16: the 192-row GEGLU tile cannot write stats_out");
  } else if (!pp) {
    const bool allow160 = !p.stats_out || p.N % 320 == 0;
    bn = force_bn > 0 ? force_bn : pick_bn(m_tiles, p.N, p.num_kb, allow160);
    IH_CHECK(bn != 160 || allow160, IH_ERR_SHAPE, "ih_gemm_ln_f16: 160-column tiles with stats_out need N %% 320 == 0");
  }
  const int bn_out = geglu ? bn / 2 : bn;
  CUtensorMap bmap;
  const uint64_t bdims[2] = {(uint64_t)K, (uint64_t)ldw_rows};
  const uint64_t bstr[1] = {(uint64_t)K * 2};
  const uint32_t bbox[2] = {(uint32_t)BK, (uint32_t)bn_out};   // GEGLU: the value and the gate half are loaded apart
  int rc = get_tmap_f16(&bmap, w, 2, bdims, bstr, bbox);
  if (rc) return rc;
  OutMaps om;
  if ((rc = out_maps(ov, bn_out % 64 == 32, om))) return rc;
  if (pp) return geglu ? launch_gemm_pp<true>(amaps, bmap, om, p, m_tiles, stream)
                       : launch_gemm_pp<false>(amaps, bmap, om, p, m_tiles, stream);
  if (geglu) {
    switch (bn) {
      case 256: return launch_gemm<256, 4, true>(amaps, bmap, om, p, m_tiles, stream);
      case 192: return launch_gemm<192, 5, true>(amaps, bmap, om, p, m_tiles, stream);
      default: return launch_gemm<128, 6, true>(amaps, bmap, om, p, m_tiles, stream);
    }
  }
  switch (bn) {
    case 256: return launch_gemm<256, 4, false>(amaps, bmap, om, p, m_tiles, stream);
    case 192: return launch_gemm<192, 4, false>(amaps, bmap, om, p, m_tiles, stream);
    case 160: return launch_gemm<160, 5, false>(amaps, bmap, om, p, m_tiles, stream);
    case 128: return launch_gemm<128, 6, false>(amaps, bmap, om, p, m_tiles, stream);
    case 64: return launch_gemm<64, 8, false>(amaps, bmap, om, p, m_tiles, stream);
    default: return set_error(IH_ERR_ARG, "unsupported BN %d", bn);
  }
}

static unsigned long long* g_trace = nullptr;
// one-shot hint consumed by the next GEMM / conv launch of this thread (ih_gemm_prefetch_next)
static thread_local const void* g_pf_ptr = nullptr;
static thread_local unsigned long long g_pf_bytes = 0;
// The hint is consumed by the FIRST launch attempt after it was set, whether or not that call gets as far as launching:
// a call that fails validation must not leave a pointer behind for an unrelated later launch.
struct PrefetchHint {
  const unsigned char* ptr;
  unsigned long long bytes;
};
static PrefetchHint take_prefetch_hint() {
  PrefetchHint h{(const unsigned char*)g_pf_ptr, g_pf_bytes};
  g_pf_ptr = nullptr;
  g_pf_bytes = 0;
  return h;
}
}  // namespace ih

using namespace ih;

// debugging aid: device buffer of >= 16 uint64 that CTA 0 of subsequent GEMM launches fills with %globaltimer stamps
// (0 kernel entry, 1 setup done, 2 predecessor finished, 3 first operands landed, 4..7 accumulator ready for tiles
// 0..3+, 8 CTA done); pass NULL to disable.
extern "C" void ih_gemm_set_trace(void* device_buffer) { ih::g_trace = (unsigned long long*)device_buffer; }

extern "C" void ih_gemm_prefetch_next(const void* weights, long long bytes) {
  ih::g_pf_ptr = (weights && bytes >= 16 && ((uintptr_t)weights & 15) == 0) ? weights : nullptr;
  ih::g_pf_bytes = ih::g_pf_ptr ? (unsigned long long)bytes : 0;
}

static int gemm_impl(const void* a, long long lda, const void* w, const void* bias, const void* rowbias,
                     int rows_per_group, long long ld_rowbias, const void* residual, long long ldr, void* out,
                     long long ldo, int M, int N, int K, int epilogue, int tile_n, const void* ln_stats,
                     int ln_slabs, float ln_eps, void* stats_out, float alpha, void* stream);

extern "C" int ih_gemm_f16(const void* a, long long lda, const void* w, const void* bias, const void* rowbias,
                           int rows_per_group, long long ld_rowbias, const void* residual, long long ldr, void* out,
                           long long ldo, int M, int N, int K, int epilogue, int tile_n, void* stream) {
  return gemm_impl(a, lda, w, bias, rowbias, rows_per_group, ld_rowbias, residual, ldr, out, ldo, M, N, K, epilogue,
                   tile_n, nullptr, 0, 0.f, nullptr, 1.f, stream);
}

extern "C" int ih_gemm_scaled_f16(const void* a, long long lda, const void* w, const void* bias, const void* residual,
                                  long long ldr, void* out, long long ldo, int M, int N, int K, int epilogue, float alpha,
                                  void* stream) {
  return gemm_impl(a, lda, w, bias, nullptr, 0, 0, residual, ldr, out, ldo, M, N, K, epilogue, 0, nullptr, 0, 0.f,
                   nullptr, alpha, stream);
}

extern "C" int ih_gemm_ln_f16(const void* a, long long lda, const void* w, const void* bias, const void* rowbias,
                              int rows_per_group, long long ld_rowbias, const void* residual, long long ldr, void* out,
                              long long ldo, int M, int N, int K, int epilogue, int tile_n, const void* ln_stats,
                              int ln_slabs, float ln_eps, void* stats_out, void* stream) {
  return gemm_impl(a, lda, w, bias, rowbias, rows_per_group, ld_rowbias, residual, ldr, out, ldo, M, N, K, epilogue,
                   tile_n, ln_stats, ln_slabs, ln_eps, stats_out, 1.f, stream);
}

static int gemm_impl(const void* a, long long lda, const void* w, const void* bias, const void* rowbias,
                     int rows_per_group, long long ld_rowbias, const void* residual, long long ldr, void* out,
                     long long ldo, int M, int N, int K, int epilogue, int tile_n, const void* ln_stats,
                     int ln_slabs, float ln_eps, void* stats_out, float alpha, void* stream) {
  const PrefetchHint hint = take_prefetch_hint();
  IH_CHECK(a && w && out, IH_ERR_ARG, "ih_gemm_f16: null pointer");
  IH_CHECK(M > 0 && N > 0 && K > 0, IH_ERR_SHAPE, "ih_gemm_f16: bad shape M=%d N=%d K=%d", M, N, K);
  IH_CHECK(K % 8 == 0 && N % 8 == 0 && lda % 8 == 0 && ldo % 8 == 0, IH_ERR_ALIGN,
           "ih_gemm_f16: K, N, lda, ldo must be multiples of 8 (16-byte rows)");
  const bool geglu = (epilogue & IH_EPI_GEGLU) != 0;
  IH_CHECK(!geglu || (N % 16 == 0), IH_ERR_SHAPE, "ih_gemm_f16: GEGLU needs even split of N");
  IH_CHECK(!(residual) || ldr % 8 == 0, IH_ERR_ALIGN, "ih_gemm_f16: ldr must be a multiple of 8");
  IH_CHECK(!(epilogue & IH_EPI_RELU) || epilogue == IH_EPI_RELU, IH_ERR_ARG,
           "ih_gemm_f16: IH_EPI_RELU cannot be combined with other epilogue flags");
  IH_CHECK(!rowbias || (rows_per_group > 0 && ld_rowbias % 8 == 0), IH_ERR_ARG,
           "ih_gemm_f16: rowbias needs rows_per_group > 0 and ld_rowbias %% 8 == 0");

  TmapSet4 amaps;
  const uint64_t adims[2] = {(uint64_t)K, (uint64_t)M};
  const uint64_t astr[1] = {(uint64_t)lda * 2};
  const uint32_t abox[2] = {(uint32_t)BK, (uint32_t)BM};
  int rc = get_tmap_f16(&amaps.m[0], a, 2, adims, astr, abox);
  if (rc) return rc;
  amaps.m[1] = amaps.m[2] = amaps.m[3] = amaps.m[0];

  GemmParams p{};
  p.M = M;
  p.N = geglu ? N / 2 : N;
  p.num_kb = (K + BK - 1) / BK;
  p.mode = 0;
  p.gate_row_off = geglu ? N / 2 : 0;
  p.bias = (const __half*)bias;
  p.rowbias = (const __half*)rowbias;
  p.rows_per_group = rows_per_group > 0 ? rows_per_group : 1;
  p.ld_rowbias = ld_rowbias;
  p.residual = (const __half*)residual;
  p.ldr = ldr;
  p.out = (__half*)out;
  p.ldo = ldo;
  p.act = (epilogue & IH_EPI_SILU) ? 1 : ((epilogue & IH_EPI_GELU) ? 2 : ((epilogue & IH_EPI_QUICK_GELU) ? 3 : 0));
  p.relu = epilogue == IH_EPI_RELU;
  p.trace = g_trace;
  p.pf_ptr = hint.ptr;
  p.pf_bytes = hint.bytes;
  IH_CHECK(!ln_stats || ln_slabs > 0, IH_ERR_ARG, "ih_gemm_ln_f16: ln_stats needs ln_slabs > 0");
  IH_CHECK(!stats_out || N % 64 == 0 || geglu, IH_ERR_SHAPE, "ih_gemm_ln_f16: stats_out needs N %% 64 == 0");
  p.stats_out = (float*)stats_out;
  p.ln_stats = (const float*)ln_stats;
  p.ln_slabs = ln_slabs;
  p.ln_inv_c = 1.0f / (float)K;
  p.ln_eps = ln_eps;
  p.alpha = alpha;
  const int m_tiles = (M + BM - 1) / BM;
  const OutView ov{out, residual, 2, {(uint64_t)p.N, (uint64_t)M}, {(uint64_t)ldo * 2}, {(uint64_t)ldr * 2},
                   {64u, (uint32_t)BM}};
  return dispatch(amaps, ov, w, N, K, p, m_tiles, geglu, tile_n, (cudaStream_t)stream);
}

static int conv_impl(const void* x, const void* w, const void* bias, const void* rowbias, long long ld_rowbias,
                     const void* residual, void* out, int B, int Hin, int Win, int Cin, int Cout, int ksize, int stride,
                     int tile_n, float alpha, void* stream, const void* sc0 = nullptr, int Csc0 = 0,
                     const void* sc1 = nullptr, int Csc1 = 0, bool pad_bottom_right = false,
                     int epilogue = IH_EPI_NONE);

extern "C" int ih_conv2d_f16(const void* x, const void* w, const void* bias, const void* rowbias,
                             long long ld_rowbias, const void* residual, void* out, int B, int Hin, int Win, int Cin,
                             int Cout, int ksize, int stride, int tile_n, void* stream) {
  return conv_impl(x, w, bias, rowbias, ld_rowbias, residual, out, B, Hin, Win, Cin, Cout, ksize, stride, tile_n, 1.f,
                   stream);
}

extern "C" int ih_conv2d_scaled_f16(const void* x, const void* w, const void* bias, const void* residual, void* out,
                                    int B, int Hin, int Win, int Cin, int Cout, int stride, float alpha, void* stream,
                                    int epilogue) {
  return conv_impl(x, w, bias, nullptr, 0, residual, out, B, Hin, Win, Cin, Cout, 3, stride, 0, alpha, stream, nullptr, 0,
                   nullptr, 0, false, epilogue);
}

extern "C" int ih_conv2d_shortcut_f16(const void* x, const void* w, const void* bias, const void* rowbias,
                                      long long ld_rowbias, const void* sc0, int Csc0, const void* sc1, int Csc1, void* out,
                                      int B, int H, int W, int Cin, int Cout, void* stream) {
  IH_CHECK(sc0 && Csc0 > 0 && Csc0 % BK == 0 && (!sc1 || (Csc1 > 0 && Csc1 % BK == 0)), IH_ERR_SHAPE,
           "ih_conv2d_shortcut_f16: shortcut sources need channel counts that are multiples of 64");
  return conv_impl(x, w, bias, rowbias, ld_rowbias, nullptr, out, B, H, W, Cin, Cout, 3, 1, 0, 1.f, stream, sc0, Csc0,
                   sc1 ? sc1 : nullptr, sc1 ? Csc1 : 0);
}

extern "C" int ih_conv2d_down_f16(const void* x, const void* w, const void* bias, void* out, int B, int Hin, int Win,
                                  int Cin, int Cout, int tile_n, float alpha, void* stream) {
  return conv_impl(x, w, bias, nullptr, 0, nullptr, out, B, Hin, Win, Cin, Cout, 3, 2, tile_n, alpha, stream, nullptr, 0,
                   nullptr, 0, true);
}

static int conv_impl(const void* x, const void* w, const void* bias, const void* rowbias, long long ld_rowbias,
                     const void* residual, void* out, int B, int Hin, int Win, int Cin, int Cout, int ksize, int stride,
                     int tile_n, float alpha, void* stream, const void* sc0, int Csc0, const void* sc1, int Csc1,
                     bool pad_bottom_right, int epilogue) {
  const PrefetchHint hint = take_prefetch_hint();
  IH_CHECK(x && w && out, IH_ERR_ARG, "ih_conv2d_f16: null pointer");
  IH_CHECK(epilogue == IH_EPI_NONE || epilogue == IH_EPI_RELU, IH_ERR_ARG,
           "ih_conv2d_scaled_f16: epilogue must be IH_EPI_NONE or IH_EPI_RELU (got %d)", epilogue);
  IH_CHECK(ksize == 3, IH_ERR_ARG, "ih_conv2d_f16: ksize must be 3 (1x1 convs are ih_gemm_f16)");
  IH_CHECK(stride == 1 || stride == 2, IH_ERR_ARG, "ih_conv2d_f16: stride must be 1 or 2");
  IH_CHECK(Cin % 8 == 0 && Cout % 8 == 0, IH_ERR_ALIGN, "ih_conv2d_f16: channels must be multiples of 8");
  IH_CHECK(stride == 1 || (Hin % 2 == 0 && Win % 2 == 0), IH_ERR_SHAPE, "ih_conv2d_f16: stride 2 needs even H, W");
  const int Ho = Hin / stride, Wo = Win / stride;

  // spatial tile: bw x bh = 128 output pixels, minimise padded tiles
  int best_bw = 128;
  long long best_tiles = -1;
  for (int bw = 128; bw >= 1; bw >>= 1) {
    const int bh = 128 / bw;
    const long long t = (long long)((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh);
    if (best_tiles < 0 || t < best_tiles) {
      best_tiles = t;
      best_bw = bw;
    }
  }
  GemmParams p{};
  p.bw = best_bw;
  p.bh = 128 / best_bw;
  p.tiles_x = (Wo + p.bw - 1) / p.bw;
  p.tiles_y = (Ho + p.bh - 1) / p.bh;
  p.Ho = Ho;
  p.Wo = Wo;
  p.mode = 1;
  p.cin_kb = (Cin + BK - 1) / BK;
  p.n_taps = 9;
  for (int t = 0; t < 9; ++t) p.tap_kb_end[t] = (t + 1) * p.cin_kb;
  if (sc0) {
    p.tap_kb_end[9] = p.tap_kb_end[8] + Csc0 / BK;
    p.n_taps = 10;
    if (sc1) {
      p.tap_kb_end[10] = p.tap_kb_end[9] + Csc1 / BK;
      p.n_taps = 11;
    }
  }
  for (int t = p.n_taps; t < 12; ++t) p.tap_kb_end[t] = 0x7fffffff;   // sentinel: the tap search always terminates
  p.num_kb = p.tap_kb_end[p.n_taps - 1];
  p.M = B * Ho * Wo;
  p.N = Cout;
  p.bias = (const __half*)bias;
  p.rowbias = (const __half*)rowbias;
  p.rows_per_group = Ho * Wo;
  p.ld_rowbias = ld_rowbias;
  p.residual = (const __half*)residual;
  p.ldr = Cout;
  p.out = (__half*)out;
  p.ldo = Cout;
  p.trace = g_trace;
  p.pf_ptr = hint.ptr;
  p.pf_bytes = hint.bytes;
  p.alpha = alpha;
  p.relu = epilogue == IH_EPI_RELU;

  TmapSet4 amaps;
  const uint32_t abox[4] = {(uint32_t)BK, (uint32_t)p.bw, (uint32_t)p.bh, 1u};
  if (stride == 1) {
    const uint64_t adims[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)B};
    const uint64_t astr[3] = {(uint64_t)Cin * 2, (uint64_t)Win * Cin * 2, (uint64_t)Hin * Win * Cin * 2};
    int rc = get_tmap_f16(&amaps.m[0], x, 4, adims, astr, abox);
    if (rc) return rc;
    amaps.m[1] = amaps.m[2] = amaps.m[3] = amaps.m[0];
    for (int t = 0; t < 9; ++t) {
      p.tap_map[t] = 0;
      p.tap_ox[t] = (signed char)(t % 3 - 1);
      p.tap_oy[t] = (signed char)(t / 3 - 1);
    }
    const void* srcs[2] = {sc0, sc1};
    const int chans[2] = {Csc0, Csc1};
    for (int i = 0; i < 2 && srcs[i]; ++i) {       // fused 1x1 shortcut sources: centre tap of their own tensor maps
      const uint64_t sdims[4] = {(uint64_t)chans[i], (uint64_t)Win, (uint64_t)Hin, (uint64_t)B};
      const uint64_t sstr[3] = {(uint64_t)chans[i] * 2, (uint64_t)Win * chans[i] * 2, (uint64_t)Hin * Win * chans[i] * 2};
      rc = get_tmap_f16(&amaps.m[1 + i], srcs[i], 4, sdims, sstr, abox);
      if (rc) return rc;
      p.tap_map[9 + i] = (signed char)(1 + i);
      p.tap_ox[9 + i] = p.tap_oy[9 + i] = 0;
    }
  } else {
    IH_CHECK(!sc0, IH_ERR_ARG, "ih_conv2d: a fused shortcut needs stride 1");
    // pad 1 on every side: input row 2*oy + dy - 1: dy=0 -> odd rows at oy-1, dy=1 -> even rows at oy, dy=2 -> odd rows
    // at oy.  Bottom/right pad only (VAE encoder Downsample2D: F.pad(x, (0,1,0,1)), pad 0): input row 2*oy + dy:
    // dy=0 -> even rows at oy, dy=1 -> odd rows at oy, dy=2 -> even rows at oy+1 (past the last row: TMA zero fill).
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        const __half* base = (const __half*)x + ((long long)py * Win + px) * Cin;
        const uint64_t adims[4] = {(uint64_t)Cin, (uint64_t)Win / 2, (uint64_t)Hin / 2, (uint64_t)B};
        const uint64_t astr[3] = {(uint64_t)2 * Cin * 2, (uint64_t)2 * Win * Cin * 2, (uint64_t)Hin * Win * Cin * 2};
        int rc = get_tmap_f16(&amaps.m[py * 2 + px], base, 4, adims, astr, abox);
        if (rc) return rc;
      }
    const int par[3] = {pad_bottom_right ? 0 : 1, pad_bottom_right ? 1 : 0, pad_bottom_right ? 0 : 1};
    const int off[3] = {pad_bottom_right ? 0 : -1, 0, pad_bottom_right ? 1 : 0};
    for (int t = 0; t < 9; ++t) {
      const int dy = t / 3, dx = t % 3;
      p.tap_map[t] = (signed char)(par[dy] * 2 + par[dx]);
      p.tap_ox[t] = (signed char)off[dx];
      p.tap_oy[t] = (signed char)off[dy];
    }
  }
  const int m_tiles = B * p.tiles_x * p.tiles_y;
  // weight is [Cout, 9*Cin] tap-major; when Cin is not a multiple of 64 each tap's K range is padded by TMA zero fill
  IH_CHECK(Cin % BK == 0, IH_ERR_SHAPE, "ih_conv2d_f16: Cin must be a multiple of 64 (got %d)", Cin);
  const uint64_t ostr[3] = {(uint64_t)Cout * 2, (uint64_t)Wo * Cout * 2, (uint64_t)Ho * Wo * Cout * 2};
  const OutView ov{out, residual, 4, {(uint64_t)Cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)B}, {ostr[0], ostr[1], ostr[2]},
                   {ostr[0], ostr[1], ostr[2]}, {64u, (uint32_t)p.bw, (uint32_t)p.bh, 1u}};
  return dispatch(amaps, ov, w, Cout, (long long)9 * Cin + Csc0 + Csc1, p, m_tiles, 0, tile_n, (cudaStream_t)stream);
}
