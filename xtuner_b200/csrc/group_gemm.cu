// Grouped expert GEMMs on wgmma (SURVEY.md §8a rows a6/a7, kernels K1-K3 of §2.3).
//
// One persistent, warp-specialised kernel template covers the three products of the expert FFN:
//   NT  out[M,N]    = x[M,Kd]  . w[e][N,Kd]^T      forward            (ragged M, groups = experts)
//   NN  out[M,Kd]   = dy[M,N]  . w[e][N,Kd]        backward dX        (ragged M)
//   TN  dw[e][N,Kd] = dy[rows_e]^T . x[rows_e]     backward dW        (ragged reduction dim)
//
// Structure per CTA (384 threads, 1 CTA/SM, grid = #SMs), output tile 128 x BLOCK_N (256, or 128 for narrow shapes):
//   warpgroup 0    TMA producer: cp.async.bulk.tensor 2-D tiles (128B swizzle) into a kStages-deep smem ring
//   warpgroups 1-2 consumers, 64 rows each: wgmma.mma_async m64 x BLOCK_N x 16 (bf16 -> fp32 in registers) from shared
//                  memory, one k-block in flight while the next is issued; then the epilogue fp32 -> bf16 -> global
// The tile list is derived on the device from tokens_per_expert (no host read, reference contract:
// SURVEY.md §8b "tokens_per_expert is a device tensor").  Ragged group boundaries: A tiles may over-read
// into the next group's rows (masked at the store); for TN the partial last k-block is zero-filled in
// shared memory before the MMA.
#include <cstdlib>

#include "common.cuh"
#include "sm100_ptx.cuh"

namespace xtb {

enum GemmMode { MODE_NT = 0, MODE_NN = 1, MODE_TN = 2 };

constexpr int BLOCK_M = 128;  // 64 rows per consumer warpgroup
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 bytes = one swizzle atom
constexpr int WGMMA_K = 16;
constexpr int kMaxExperts = 1024;
constexpr int kGemmThreads = 384;
constexpr int kConsumerWarps = 8;

// STORE = 1 (default): every consumer warp packs 16-row x 64-column bf16 boxes into its own 2 KiB staging buffer (128-byte
//            swizzle) and one lane issues a TMA store; boxes cut by a ragged expert boundary are copied out masked.
// STORE = 0: registers -> 4-byte global stores.  Kept as the bit-identity yardstick of the default (XTB_GEMM_EPI=0;
//            tests/test_gpu_group_gemm.py::test_tma_store_epilogue_is_bit_identical_to_direct_stores).
template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;  // 16 KiB
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;  // 16 / 32 KiB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (BLOCK_N == 128) ? 6 : 4;
  static constexpr int kBoxBytes = 16 * 128;  // one staging box: 16 rows x 64 bf16
  static constexpr int kStagingBytes = kConsumerWarps * kBoxBytes;
  // smem: [1024 align slack][stages * (A|B)][staging boxes][barriers + scheduler tables]
  static constexpr int kAuxBytes = 8 * (2 * kStages) + 2 * 4 * (kMaxExperts + 1);
  static constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kStagingBytes + kAuxBytes;
};
static_assert(GemmCfg<128>::kSmemBytes <= 232448 && GemmCfg<256>::kSmemBytes <= 232448, "shared memory budget (227 KiB)");

struct GemmArgs {
  const int64_t* tokens_per_expert;
  __nv_bfloat16* out;
  int E;
  int m_out_tiles;  // TN only: N / BLOCK_M
  int n_tiles;      // output-column tiles
  int k_red;        // reduction extent for NT/NN (Kd or N); unused for TN
  int ld_out;       // leading dimension of out (elements)
  int w_rows;       // rows of one expert's weight matrix (N) — row offset of expert e in the B tensor map
  __nv_bfloat16* out2;        // EPI_SWIGLU: activation output a[M, I]
  int inter;                  // EPI_SWIGLU: I (out = h[M, 2I], gate columns [0,I), up columns [I,2I))
  // TN only: a second product over the same token groups in the same launch (xtb_group_gemm_tn_pair): its tiles follow
  // the first product's in the persistent tile list, operands come from tmap_a2 / tmap_b2, the output goes through
  // tmap_o2.  n_prob = 2 enables it.
  int n_prob;
  __nv_bfloat16* out_b;
  int m_out_tiles_b, n_tiles_b, ld_out_b;
  // EPI_CE (lm_head logits, one group): for every row and column tile, (max, sum exp(z - max)) of the stored bf16 logits
  // z goes to ce_part[row * n_tiles + n_blk]
  float2* ce_part;
};

enum GemmEpilogue { EPI_PLAIN = 0, EPI_SWIGLU = 1, EPI_CE = 2 };

template <int BLOCK_N, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BLOCK_N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BLOCK_N == 256) ptx::wgmma_m64n256k16_bf16<TA, TB>(d, da, db, accumulate);
  else ptx::wgmma_m64n128k16_bf16<TA, TB>(d, da, db, accumulate);
}

template <int MODE, int BLOCK_N, int EPI, int STORE>
__global__ void __launch_bounds__(kGemmThreads, 1)
group_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_o, const __grid_constant__ CUtensorMap tmap_o2,
                  const __grid_constant__ CUtensorMap tmap_a2, const __grid_constant__ CUtensorMap tmap_b2,
                  const GemmArgs args) {
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr bool kAMn = (MODE == MODE_TN);                     // A is MN-major (contiguous along M)
  constexpr bool kBMn = (MODE == MODE_NN || MODE == MODE_TN);  // B is MN-major (contiguous along N)
  constexpr int kStages = Cfg::kStages;
  constexpr int kAcc = BLOCK_N / 2;  // fp32 accumulator registers per consumer thread

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* staging = smem + kStages * Cfg::kStageBytes;  // kConsumerWarps boxes of 2 KiB (1024-byte aligned)
  uint8_t* aux = staging + Cfg::kStagingBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
  uint64_t* empty_bar = full_bar + kStages;
  int* s_row_start = reinterpret_cast<int*>(empty_bar + kStages);  // [E+1]
  int* s_tile_start = s_row_start + (kMaxExperts + 1);             // [E+1]  (NT/NN)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int E = args.E;

  // programmatic dependent launch: barrier init and descriptor prefetch below touch nothing a predecessor wrote, so they
  // may run while it drains; tokens_per_expert (and everything after the block barrier) is read after the wait
  pdl_trigger();
  if (warp == 0) {
    if (lane == 0) {
      ptx::prefetch_tensormap(&tmap_a);
      ptx::prefetch_tensormap(&tmap_b);
      if constexpr (STORE) {
        ptx::prefetch_tensormap(&tmap_o);
        if constexpr (EPI == EPI_SWIGLU) ptx::prefetch_tensormap(&tmap_o2);
      }
      if constexpr (MODE == MODE_TN) {
        if (args.n_prob == 2) {
          ptx::prefetch_tensormap(&tmap_a2);
          ptx::prefetch_tensormap(&tmap_b2);
          if constexpr (STORE) ptx::prefetch_tensormap(&tmap_o2);
        }
      }
    }
    pdl_wait();
    // prefix sums of tokens_per_expert (rows) and of per-expert tile counts
    int run_rows = 0, run_tiles = 0;
    for (int e0 = 0; e0 < E; e0 += 32) {
      const int e = e0 + lane;
      const int cnt = (e < E) ? (int)args.tokens_per_expert[e] : 0;
      const int tl = ((cnt + BLOCK_M - 1) / BLOCK_M) * args.n_tiles;
      int ir = cnt, it = tl;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, ir, o);
        const int b = __shfl_up_sync(0xffffffffu, it, o);
        if (lane >= o) { ir += a; it += b; }
      }
      if (e < E) {
        s_row_start[e] = run_rows + ir - cnt;
        s_tile_start[e] = run_tiles + it - tl;
      }
      run_rows += __shfl_sync(0xffffffffu, ir, 31);
      run_tiles += __shfl_sync(0xffffffffu, it, 31);
    }
    if (lane == 0) {
      s_row_start[E] = run_rows;
      s_tile_start[E] = run_tiles;
    }
  } else if (warp == 1) {
    if (lane == 0) {
      for (int s = 0; s < kStages; ++s) {
        ptx::mbar_init(&full_bar[s], 1);
        ptx::mbar_init(&empty_bar[s], kConsumerWarps);
      }
      ptx::fence_mbar_init();
    }
  }
  pdl_wait();
  __syncthreads();

  // TN: the tile list of the first product, then (n_prob == 2) the second product's — equal cost per tile (same token
  // groups), so one list over both fills the last wave that each product alone would leave partly empty
  const int tiles0 = E * args.m_out_tiles * args.n_tiles;
  const int tiles1 = (MODE == MODE_TN && args.n_prob == 2) ? E * args.m_out_tiles_b * args.n_tiles_b : 0;
  const int total_tiles = (MODE == MODE_TN) ? tiles0 + tiles1 : s_tile_start[E];

  // tile decode shared by all roles (each role walks the same sequence)
  struct Tile {
    int e, m_blk, n_blk, row0, row_end, num_kb, prob;
  };
  auto decode = [&](int tile, int& e_hint) -> Tile {
    Tile t;
    t.prob = 0;
    if constexpr (MODE == MODE_TN) {
      int mt = args.m_out_tiles, nt = args.n_tiles;
      if (tile >= tiles0) {
        tile -= tiles0;
        t.prob = 1;
        mt = args.m_out_tiles_b;
        nt = args.n_tiles_b;
      }
      const int per_e = mt * nt;
      t.e = tile / per_e;
      const int local = tile - t.e * per_e;
      t.m_blk = local / nt;
      t.n_blk = local - t.m_blk * nt;
      t.row0 = s_row_start[t.e];
      t.row_end = s_row_start[t.e + 1];
      t.num_kb = (t.row_end - t.row0 + BLOCK_K - 1) / BLOCK_K;
    } else {
      while (tile >= s_tile_start[e_hint + 1]) ++e_hint;
      t.e = e_hint;
      const int local = tile - s_tile_start[t.e];
      t.m_blk = local / args.n_tiles;
      t.n_blk = local - t.m_blk * args.n_tiles;
      t.row0 = s_row_start[t.e] + t.m_blk * BLOCK_M;
      t.row_end = s_row_start[t.e + 1];
      t.num_kb = args.k_red / BLOCK_K;
    }
    return t;
  };

  if (warp < 4) {
    // ================================ TMA producer ================================================
    ptx::setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      int e_hint = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const Tile t = decode(tile, e_hint);
        for (int kb = 0; kb < t.num_kb; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          ptx::mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if constexpr (MODE == MODE_NT) {
            ptx::tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, t.row0);
            if constexpr (EPI == EPI_SWIGLU) {
              // B tile rows [0, BLOCK_N/2) = gate_proj rows, the rest = up_proj rows of the same BLOCK_N/2 output features
              constexpr int half = BLOCK_N / 2;
              ptx::tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, t.e * args.w_rows + t.n_blk * half);
              ptx::tma_load_2d(sb + half * 128, &tmap_b, &full_bar[stage], kb * BLOCK_K,
                               t.e * args.w_rows + args.inter + t.n_blk * half);
            } else {
              ptx::tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, t.e * args.w_rows + t.n_blk * BLOCK_N);
            }
          } else if constexpr (MODE == MODE_NN) {
            ptx::tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, t.row0);
#pragma unroll
            for (int a = 0; a < BLOCK_N / 64; ++a)
              ptx::tma_load_2d(sb + a * 8192, &tmap_b, &full_bar[stage], t.n_blk * BLOCK_N + a * 64,
                               t.e * args.w_rows + kb * BLOCK_K);
          } else {
            const CUtensorMap* ma = t.prob ? &tmap_a2 : &tmap_a;
            const CUtensorMap* mb = t.prob ? &tmap_b2 : &tmap_b;
#pragma unroll
            for (int a = 0; a < BLOCK_M / 64; ++a)
              ptx::tma_load_2d(sa + a * 8192, ma, &full_bar[stage], t.m_blk * BLOCK_M + a * 64, t.row0 + kb * BLOCK_K);
#pragma unroll
            for (int a = 0; a < BLOCK_N / 64; ++a)
              ptx::tma_load_2d(sb + a * 8192, mb, &full_bar[stage], t.n_blk * BLOCK_N + a * 64, t.row0 + kb * BLOCK_K);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ================================ consumers: wgmma + epilogue ==================================
    ptx::setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;  // consumer warpgroup: rows [64 wg, 64 wg + 64) of the tile
    const int cw = warp - 4;         // consumer warp: rows [16 cw, 16 cw + 16) of the tile
    const int r_lo = lane >> 2;      // this lane's rows inside the warp's 16: r_lo and r_lo + 8
    const int qc = lane & 3;         // ... and its column pair inside every 8-column chunk
    uint8_t* box = staging + cw * Cfg::kBoxBytes;
    const uint32_t box_u32 = ptx::smem_u32(box);

    // One 16 x 64 bf16 box of this warp (p0[j] / p1[j]: the lane's column pair of chunk j, rows r_lo / r_lo + 8) goes to
    // rows [grow, grow+16) x columns [gcol, gcol+64) of the tensor behind `map`; `valid` = rows of this expert.
    auto emit_box = [&](const CUtensorMap* map, __nv_bfloat16* gbase, int ld, int gcol, int grow, int valid,
                        const uint32_t (&p0)[8], const uint32_t (&p1)[8]) {
      if constexpr (STORE) {
        if (lane == 0) ptx::bulk_wait_read_all();  // the previous store has finished reading the box
        __syncwarp();
        // 128-byte swizzle: 16-byte chunk j of row r lives at chunk j ^ (r & 7)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t off = (uint32_t)r_lo * 128 + (uint32_t)((j ^ r_lo) << 4) + qc * 4;
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(box_u32 + off), "r"(p0[j]) : "memory");
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(box_u32 + off + 1024), "r"(p1[j]) : "memory");
        }
        ptx::fence_proxy_async_smem();
        __syncwarp();
        if (valid >= 16) {
          if (lane == 0) {
            ptx::tma_store_2d(map, box, gcol, grow);
            ptx::bulk_commit_group();
          }
        } else {
          // ragged boundary inside the box: masked copy of the valid rows, 8 lanes per 128-byte row
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int idx = i * 32 + lane;
            const int r = idx >> 3, c = idx & 7;
            if (r < valid) {
              const uint4 v = *reinterpret_cast<const uint4*>(box + r * 128 + ((c ^ (r & 7)) << 4));
              *reinterpret_cast<uint4*>(gbase + (size_t)(grow + r) * ld + gcol + c * 8) = v;
            }
          }
          __syncwarp();
        }
      } else {
        uint32_t* d0 = reinterpret_cast<uint32_t*>(gbase + (size_t)(grow + r_lo) * ld + gcol + qc * 2);
        uint32_t* d1 = reinterpret_cast<uint32_t*>(gbase + (size_t)(grow + r_lo + 8) * ld + gcol + qc * 2);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (r_lo < valid) d0[j * 4] = p0[j];
          if (r_lo + 8 < valid) d1[j * 4] = p1[j];
        }
      }
    };

    float acc[kAcc];
    int stage = 0;
    uint32_t phase = 0;
    int e_hint = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const Tile t = decode(tile, e_hint);
      // output of this tile's product (TN with two products: the second one's through tmap_o2)
      const bool second = (MODE == MODE_TN) && t.prob;
      __nv_bfloat16* const o_ptr = second ? args.out_b : args.out;
      const int o_ld = second ? args.ld_out_b : args.ld_out;
      const CUtensorMap* const o_map = second ? &tmap_o2 : &tmap_o;
      int grow, valid;
      if constexpr (MODE == MODE_TN) {  // dw viewed as [E * N, Kd]
        grow = (t.e * (second ? args.m_out_tiles_b : args.m_out_tiles) + t.m_blk) * BLOCK_M + cw * 16;
        valid = 16;
      } else {
        grow = t.row0 + cw * 16;
        valid = min(16, t.row_end - grow);
      }
      if (t.num_kb == 0) {
        // TN, empty expert: zero tile (reference semantics); rare, plain stores, two lanes per row
        __nv_bfloat16* zrow = o_ptr + (size_t)(grow + (lane >> 1)) * o_ld + (size_t)t.n_blk * BLOCK_N + (lane & 1) * (BLOCK_N / 2);
        const uint4 z = make_uint4(0, 0, 0, 0);
        for (int c = 0; c < BLOCK_N / 16; ++c) reinterpret_cast<uint4*>(zrow)[c] = z;
        continue;
      }
      for (int kb = 0; kb < t.num_kb; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        uint8_t* sa = smem + stage * Cfg::kStageBytes;
        uint8_t* sb = sa + Cfg::kABytes;
        if constexpr (MODE == MODE_TN) {
          // zero the token rows beyond this expert's range (they hold the next expert's data)
          const int valid_k = t.row_end - (t.row0 + kb * BLOCK_K);
          if (valid_k < BLOCK_K) {
            const uint4 z = make_uint4(0, 0, 0, 0);
            const int first = valid_k * 8;  // 16-byte chunk index inside a [64 rows][128 B] atom
            const int ct = threadIdx.x - 128;
#pragma unroll
            for (int a = 0; a < (BLOCK_M + BLOCK_N) / 64; ++a)  // the A atoms, then the B atoms (contiguous)
              for (int c = first + ct; c < 512; c += 32 * kConsumerWarps) reinterpret_cast<uint4*>(sa + a * 8192)[c] = z;
            ptx::fence_proxy_async_smem();
            ptx::named_barrier_sync(1, 32 * kConsumerWarps);
          }
        }
        const uint32_t a_addr = ptx::smem_u32(sa) + wg * 8192, b_addr = ptx::smem_u32(sb);
        ptx::fence_accumulator(acc);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
          // (this warpgroup's 64 A rows start wg * 8192 B into the A block)
          const uint64_t da = kAMn ? ptx::make_smem_desc_sw128(a_addr + k * 2048, 8192, 1024)
                                   : ptx::make_smem_desc_sw128(a_addr + k * 32, 16, 1024);
          const uint64_t db = kBMn ? ptx::make_smem_desc_sw128(b_addr + k * 2048, 8192, 1024)
                                   : ptx::make_smem_desc_sw128(b_addr + k * 32, 16, 1024);
          wgmma_bf16<BLOCK_N, kAMn ? 1 : 0, kBMn ? 1 : 0>(acc, da, db, (kb > 0 || k > 0) ? 1u : 0u);
        }
        ptx::wgmma_commit();
        if (kb > 0) {
          ptx::wgmma_wait<1>();
          if (lane == 0) ptx::mbar_arrive(&empty_bar[stage == 0 ? kStages - 1 : stage - 1]);
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::fence_accumulator(acc);
      if (lane == 0) ptx::mbar_arrive(&empty_bar[stage == 0 ? kStages - 1 : stage - 1]);

      // ---- epilogue: this warp's 16 rows, 64 columns at a time -------------------------------------
      if (valid <= 0) continue;
      if constexpr (EPI == EPI_SWIGLU) {
        // accumulator columns [0,half) = gate, [half,2*half) = up of output features n_blk*half + [0,half).
        // h = bf16(acc) is stored (saved for backward, as the reference's autograd does) and
        // a = bf16( bf16(silu(h_gate)) * h_up ) is produced in the same pass (ops/act_fn.py:7-9 roundings).
        constexpr int half = BLOCK_N / 2;
#pragma unroll
        for (int b = 0; b < half / 64; ++b) {
          const int fcol = t.n_blk * half + b * 64;
          uint32_t g0[8], g1[8], u0[8], u1[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int cg = 4 * (b * 8 + j), cu = 4 * (half / 8 + b * 8 + j);
            g0[j] = pack_bf16x2(acc[cg], acc[cg + 1]);
            g1[j] = pack_bf16x2(acc[cg + 2], acc[cg + 3]);
            u0[j] = pack_bf16x2(acc[cu], acc[cu + 1]);
            u1[j] = pack_bf16x2(acc[cu + 2], acc[cu + 3]);
          }
          emit_box(&tmap_o, args.out, args.ld_out, fcol, grow, valid, g0, g1);
          emit_box(&tmap_o, args.out, args.ld_out, args.inter + fcol, grow, valid, u0, u1);
          auto act = [](uint32_t g, uint32_t u) {
            float ga, gb, ua, ub;
            unpack_bf16x2(g, ga, gb);
            unpack_bf16x2(u, ua, ub);
            const float sa_ = __bfloat162float(__float2bfloat16_rn(silu_fast(ga)));
            const float sb_ = __bfloat162float(__float2bfloat16_rn(silu_fast(gb)));
            return pack_bf16x2(sa_ * ua, sb_ * ub);
          };
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            g0[j] = act(g0[j], u0[j]);
            g1[j] = act(g1[j], u1[j]);
          }
          emit_box(&tmap_o2, args.out2, args.inter, fcol, grow, valid, g0, g1);
        }
      } else {
#pragma unroll
        for (int b = 0; b < BLOCK_N / 64; ++b) {
          uint32_t p0[8], p1[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = 4 * (b * 8 + j);
            p0[j] = pack_bf16x2(acc[c], acc[c + 1]);
            p1[j] = pack_bf16x2(acc[c + 2], acc[c + 3]);
          }
          emit_box(o_map, o_ptr, o_ld, t.n_blk * BLOCK_N + b * 64, grow, valid, p0, p1);
        }
        if constexpr (EPI == EPI_CE) {
          // Statistics of the bf16 logits just stored, from the same rounded values.  Lane (r_lo, qc) holds columns
          // 8j + 2qc + {0, 1} of row r_lo in acc[4j], acc[4j+1] and of row r_lo + 8 in acc[4j+2], acc[4j+3]; the four
          // lanes of a quad hold a whole row of the tile.
          auto bf = [](float x) { return __bfloat162float(__float2bfloat16_rn(x)); };
          float m0 = __int_as_float(0xff800000), m1 = m0;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            m0 = fmaxf(m0, fmaxf(acc[4 * j], acc[4 * j + 1]));
            m1 = fmaxf(m1, fmaxf(acc[4 * j + 2], acc[4 * j + 3]));
          }
#pragma unroll
          for (int o = 1; o < 4; o <<= 1) {
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
          }
          m0 = bf(m0);  // rounding is monotonic: the max of the rounded row is the rounded max
          m1 = bf(m1);
          float s0 = 0.f, s1 = 0.f;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            s0 += expf(bf(acc[4 * j]) - m0);
            s0 += expf(bf(acc[4 * j + 1]) - m0);
            s1 += expf(bf(acc[4 * j + 2]) - m1);
            s1 += expf(bf(acc[4 * j + 3]) - m1);
          }
#pragma unroll
          for (int o = 1; o < 4; o <<= 1) {  // same sum on all four lanes (the two operands of each add commute)
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
          }
          if (qc == 0) {
            if (r_lo < valid) args.ce_part[(size_t)(grow + r_lo) * args.n_tiles + t.n_blk] = make_float2(m0, s0);
            if (r_lo + 8 < valid) args.ce_part[(size_t)(grow + r_lo + 8) * args.n_tiles + t.n_blk] = make_float2(m1, s1);
          }
        }
      }
    }
    if constexpr (STORE) {
      if (lane == 0) ptx::bulk_wait_all();  // stores performed before the CTA exits
    }
  }
}

// ---- host side: tensor maps ------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encode_tiled = nullptr;

// 2-D row-major bf16 tensor [rows, cols]; box = [box_rows, box_cols], 128-byte swizzle, OOB -> zeros.
static int make_tmap(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                     uint32_t box_cols) {
  if (!g_encode_tiled) {
    const int rc = xtb_init();
    if (rc != XTB_OK) return rc;
  }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUresult r = g_encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides,
                                    box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(XTB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d (rows=%llu cols=%llu box=%ux%u)", (int)r,
                (unsigned long long)rows, (unsigned long long)cols, box_rows, box_cols);
  return XTB_OK;
}

// XTB_GEMM_EPI=0 selects the direct-store epilogue (the bit-identity yardstick); default = TMA-store epilogue
static bool gemm_epi_store() {
  static const bool v = !(getenv("XTB_GEMM_EPI") && atoi(getenv("XTB_GEMM_EPI")) == 0);
  return v;
}

template <int MODE, int BLOCK_N, int EPI, int STORE>
static int launch_gemm_impl(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const CUtensorMap& to2,
                            const CUtensorMap& ta2, const CUtensorMap& tb2, const GemmArgs& args, cudaStream_t st) {
  using Cfg = GemmCfg<BLOCK_N>;
  static bool attr_set = false;
  auto kfn = group_gemm_kernel<MODE, BLOCK_N, EPI, STORE>;
  if (!attr_set) {
    XTB_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  XTB_CUDA(launch_pdl(kfn, dim3(sm_count()), dim3(kGemmThreads), (size_t)Cfg::kSmemBytes, st, ta, tb, to, to2, ta2, tb2, args));
  XTB_LAUNCH_OK();
  return XTB_OK;
}

// rows_out = rows of the 2-D view of `out` (and of `out2`, the SwiGLU epilogue's a[M, I]).  ta2 / tb2 / rows_out_b: the
// operands and output rows of the second product of a two-product TN launch (args.n_prob == 2), else unused.
template <int MODE, int BLOCK_N, int EPI = EPI_PLAIN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& args, uint64_t rows_out,
                       cudaStream_t st, const CUtensorMap* ta2 = nullptr, const CUtensorMap* tb2 = nullptr,
                       uint64_t rows_out_b = 0) {
  const CUtensorMap& a2 = ta2 ? *ta2 : ta;
  const CUtensorMap& b2 = tb2 ? *tb2 : tb;
  if (gemm_epi_store()) {
    CUtensorMap to, to2;
    int rc;
    if ((rc = make_tmap(&to, args.out, rows_out, (uint64_t)args.ld_out, 16, 64))) return rc;
    if constexpr (EPI == EPI_SWIGLU) {
      if ((rc = make_tmap(&to2, args.out2, rows_out, (uint64_t)args.inter, 16, 64))) return rc;
    } else if (MODE == MODE_TN && args.n_prob == 2) {
      if ((rc = make_tmap(&to2, args.out_b, rows_out_b, (uint64_t)args.ld_out_b, 16, 64))) return rc;
    } else {
      to2 = to;
    }
    return launch_gemm_impl<MODE, BLOCK_N, EPI, 1>(ta, tb, to, to2, a2, b2, args, st);
  }
  return launch_gemm_impl<MODE, BLOCK_N, EPI, 0>(ta, tb, ta, ta, a2, b2, args, st);
}

static int check_common(const void* a, const void* b, const int64_t* tpe, void* out, int64_t M_total, int N, int Kd,
                        int E, const char* name) {
  XTB_CHECK_ARG(a && b && tpe && out, "%s: null pointer", name);
  XTB_CHECK_ARG(M_total >= 0 && M_total < (1ll << 31), "%s: bad M_total=%lld", name, (long long)M_total);
  XTB_CHECK_ARG(E > 0 && E <= kMaxExperts, "%s: E=%d out of range (1..%d)", name, E, kMaxExperts);
  XTB_CHECK_ARG(N > 0 && Kd > 0 && N % 128 == 0 && Kd % 128 == 0, "%s: N=%d and Kd=%d must be multiples of 128", name,
                N, Kd);
  XTB_CHECK_ARG(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(out)) &
                 15) == 0,
                "%s: pointers must be 16-byte aligned", name);
  XTB_ENSURE_CTX(a);
  return XTB_OK;
}

// NT output tile width: 256 columns where N allows, else 128
static int nt_block_n(int N) { return (N % 256 == 0) ? 256 : 128; }

// The NT product of xtb_group_gemm_nt; `a` arrives with tokens_per_expert, out and the epilogue's own fields set.
template <int EPI>
static int launch_nt(const void* x, const void* w, int64_t M_total, int N, int Kd, int E, GemmArgs a, cudaStream_t st) {
  const int BN = nt_block_n(N);
  CUtensorMap ta, tb;
  int rc;
  if ((rc = make_tmap(&ta, x, (uint64_t)M_total, (uint64_t)Kd, BLOCK_M, BLOCK_K))) return rc;
  if ((rc = make_tmap(&tb, w, (uint64_t)E * N, (uint64_t)Kd, BN, BLOCK_K))) return rc;
  a.E = E;
  a.n_tiles = N / BN;
  a.k_red = Kd;
  a.ld_out = N;
  a.w_rows = N;
  if (BN == 256) return launch_gemm<MODE_NT, 256, EPI>(ta, tb, a, (uint64_t)M_total, st);
  return launch_gemm<MODE_NT, 128, EPI>(ta, tb, a, (uint64_t)M_total, st);
}

}  // namespace xtb

using namespace xtb;

extern "C" int xtb_tma_init_() {
  if (g_encode_tiled) return XTB_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  XTB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || !fn)
    return fail(XTB_ERR_CUDA, "driver does not export cuTensorMapEncodeTiled (query result %d)", (int)qres);
  g_encode_tiled = reinterpret_cast<PFN_encodeTiled>(fn);
  return XTB_OK;
}

extern "C" int xtb_group_gemm_nt(const void* x, const void* w, const int64_t* tokens_per_expert, int64_t M_total,
                                 int N, int Kd, int E, void* out, xtb_stream_t stream) {
  int rc = check_common(x, w, tokens_per_expert, out, M_total, N, Kd, E, "xtb_group_gemm_nt");
  if (rc) return rc;
  if (M_total == 0) return XTB_OK;
  GemmArgs a{};
  a.tokens_per_expert = tokens_per_expert;
  a.out = static_cast<__nv_bfloat16*>(out);
  return launch_nt<EPI_PLAIN>(x, w, M_total, N, Kd, E, a, as_stream(stream));
}

// The lm_head logits of xtb_lm_head_ce (csrc/lm_head_ce.cu): z[T, V] = bf16(h[T, H] . w[V, H]^T), the NT product with one
// group (tokens_per_expert = {T} on the device) and the EPI_CE epilogue.  ce_part holds lm_head_ce_vocab_tiles(V) entries
// per row.
int xtb::lm_head_ce_vocab_tiles(int V) { return V / nt_block_n(V); }

int xtb::lm_head_logits_ce(const void* h, const void* w, const int64_t* tokens_per_expert, int64_t T, int H, int V,
                           void* z, float2* ce_part, cudaStream_t st) {
  GemmArgs a{};
  a.tokens_per_expert = tokens_per_expert;
  a.out = static_cast<__nv_bfloat16*>(z);
  a.ce_part = ce_part;
  return launch_nt<EPI_CE>(h, w, T, V, H, 1, a, st);
}

extern "C" int xtb_group_gemm_nt_swiglu(const void* x, const void* w13, const int64_t* tokens_per_expert,
                                        int64_t M_total, int I, int Kd, int E, void* h_out, void* a_out,
                                        xtb_stream_t stream) {
  int rc = check_common(x, w13, tokens_per_expert, h_out, M_total, 2 * I, Kd, E, "xtb_group_gemm_nt_swiglu");
  if (rc) return rc;
  XTB_CHECK_ARG(a_out && (reinterpret_cast<uintptr_t>(a_out) & 15) == 0, "xtb_group_gemm_nt_swiglu: bad a_out");
  XTB_CHECK_ARG(I % 64 == 0, "xtb_group_gemm_nt_swiglu: I=%d must be a multiple of 64", I);
  if (M_total == 0) return XTB_OK;
  // a tile holds BN/2 gate_proj rows and the BN/2 up_proj rows of the same output features
  const int BN = (I % 128 == 0) ? 256 : 128;
  CUtensorMap ta, tb;
  if ((rc = make_tmap(&ta, x, (uint64_t)M_total, (uint64_t)Kd, BLOCK_M, BLOCK_K))) return rc;
  if ((rc = make_tmap(&tb, w13, (uint64_t)E * 2 * I, (uint64_t)Kd, BN / 2, BLOCK_K))) return rc;
  GemmArgs a{};
  a.tokens_per_expert = tokens_per_expert;
  a.out = static_cast<__nv_bfloat16*>(h_out);
  a.out2 = static_cast<__nv_bfloat16*>(a_out);
  a.inter = I;
  a.E = E;
  a.n_tiles = I / (BN / 2);
  a.k_red = Kd;
  a.ld_out = 2 * I;
  a.w_rows = 2 * I;
  if (BN == 256) return launch_gemm<MODE_NT, 256, EPI_SWIGLU>(ta, tb, a, (uint64_t)M_total, as_stream(stream));
  return launch_gemm<MODE_NT, 128, EPI_SWIGLU>(ta, tb, a, (uint64_t)M_total, as_stream(stream));
}

extern "C" int xtb_group_gemm_nn(const void* dy, const void* w, const int64_t* tokens_per_expert, int64_t M_total,
                                 int N, int Kd, int E, void* out, xtb_stream_t stream) {
  int rc = check_common(dy, w, tokens_per_expert, out, M_total, N, Kd, E, "xtb_group_gemm_nn");
  if (rc) return rc;
  if (M_total == 0) return XTB_OK;
  const int BN = (Kd % 256 == 0) ? 256 : 128;
  CUtensorMap ta, tb;
  if ((rc = make_tmap(&ta, dy, (uint64_t)M_total, (uint64_t)N, BLOCK_M, BLOCK_K))) return rc;
  // B(n'=column of w, k=row of w[e]) is MN-major: boxes of 64 columns x 64 rows
  if ((rc = make_tmap(&tb, w, (uint64_t)E * N, (uint64_t)Kd, BLOCK_K, 64))) return rc;
  GemmArgs a{};
  a.tokens_per_expert = tokens_per_expert;
  a.out = static_cast<__nv_bfloat16*>(out);
  a.E = E;
  a.n_tiles = Kd / BN;
  a.k_red = N;
  a.ld_out = Kd;
  a.w_rows = N;
  if (BN == 256) return launch_gemm<MODE_NN, 256>(ta, tb, a, (uint64_t)M_total, as_stream(stream));
  return launch_gemm<MODE_NN, 128>(ta, tb, a, (uint64_t)M_total, as_stream(stream));
}

// One or (dy_b != nullptr) two TN products over the same token groups in one launch.
static int launch_tn(const void* dy_a, const void* x_a, int N_a, int Kd_a, void* dw_a, const void* dy_b, const void* x_b,
                     int N_b, int Kd_b, void* dw_b, const int64_t* tokens_per_expert, int64_t M_total, int E, int BN,
                     cudaStream_t st) {
  int rc;
  CUtensorMap ta, tb, ta2, tb2;
  if ((rc = make_tmap(&ta, dy_a, (uint64_t)M_total, (uint64_t)N_a, BLOCK_K, 64))) return rc;
  if ((rc = make_tmap(&tb, x_a, (uint64_t)M_total, (uint64_t)Kd_a, BLOCK_K, 64))) return rc;
  GemmArgs a{};
  a.tokens_per_expert = tokens_per_expert;
  a.E = E;
  a.out = static_cast<__nv_bfloat16*>(dw_a);
  a.m_out_tiles = N_a / BLOCK_M;
  a.n_tiles = Kd_a / BN;
  a.ld_out = Kd_a;
  if (dy_b) {
    if ((rc = make_tmap(&ta2, dy_b, (uint64_t)M_total, (uint64_t)N_b, BLOCK_K, 64))) return rc;
    if ((rc = make_tmap(&tb2, x_b, (uint64_t)M_total, (uint64_t)Kd_b, BLOCK_K, 64))) return rc;
    a.n_prob = 2;
    a.out_b = static_cast<__nv_bfloat16*>(dw_b);
    a.m_out_tiles_b = N_b / BLOCK_M;
    a.n_tiles_b = Kd_b / BN;
    a.ld_out_b = Kd_b;
  }
  const CUtensorMap* pa2 = dy_b ? &ta2 : nullptr;
  const CUtensorMap* pb2 = dy_b ? &tb2 : nullptr;
  if (BN == 256) return launch_gemm<MODE_TN, 256>(ta, tb, a, (uint64_t)E * N_a, st, pa2, pb2, (uint64_t)E * N_b);
  return launch_gemm<MODE_TN, 128>(ta, tb, a, (uint64_t)E * N_a, st, pa2, pb2, (uint64_t)E * N_b);
}

extern "C" int xtb_group_gemm_tn(const void* dy, const void* x, const int64_t* tokens_per_expert, int64_t M_total,
                                 int N, int Kd, int E, void* dw, xtb_stream_t stream) {
  int rc = check_common(dy, x, tokens_per_expert, dw, M_total, N, Kd, E, "xtb_group_gemm_tn");
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  if (M_total == 0) {
    XTB_CUDA(cudaMemsetAsync(dw, 0, (size_t)E * N * Kd * 2, st));
    return XTB_OK;
  }
  return launch_tn(dy, x, N, Kd, dw, nullptr, nullptr, 0, 0, nullptr, tokens_per_expert, M_total, E,
                   (Kd % 256 == 0) ? 256 : 128, st);
}

// Both weight gradients of an expert MLP in ONE launch: dw_a[e] = dy_a[rows_e]^T @ x_a[rows_e] and
// dw_b[e] = dy_b[rows_e]^T @ x_b[rows_e] over the same token groups, one tile list over both.  Every tile is computed
// exactly as by xtb_group_gemm_tn: identical bits.
extern "C" int xtb_group_gemm_tn_pair(const void* dy_a, const void* x_a, int N_a, int Kd_a, void* dw_a, const void* dy_b,
                                      const void* x_b, int N_b, int Kd_b, void* dw_b, const int64_t* tokens_per_expert,
                                      int64_t M_total, int E, xtb_stream_t stream) {
  int rc = check_common(dy_a, x_a, tokens_per_expert, dw_a, M_total, N_a, Kd_a, E, "xtb_group_gemm_tn_pair");
  if (rc) return rc;
  if ((rc = check_common(dy_b, x_b, tokens_per_expert, dw_b, M_total, N_b, Kd_b, E, "xtb_group_gemm_tn_pair"))) return rc;
  // one launch serves both products when they take the same tile width
  const bool pair_ok = M_total > 0 && (Kd_a % 256 == 0) == (Kd_b % 256 == 0);
  if (!pair_ok) {  // the two launches it stands for
    if ((rc = xtb_group_gemm_tn(dy_a, x_a, tokens_per_expert, M_total, N_a, Kd_a, E, dw_a, stream))) return rc;
    return xtb_group_gemm_tn(dy_b, x_b, tokens_per_expert, M_total, N_b, Kd_b, E, dw_b, stream);
  }
  return launch_tn(dy_a, x_a, N_a, Kd_a, dw_a, dy_b, x_b, N_b, Kd_b, dw_b, tokens_per_expert, M_total, E,
                   (Kd_a % 256 == 0) ? 256 : 128, as_stream(stream));
}
