// RMSNorm fused with its neighbours on the path (SURVEY.md §8f-3: "RMSNorm -> gate -> router fusion" and the
// backward adds around it).  Reference: post_attention_layernorm in MoEDecoderLayer._pre_moe_forward
// (module/decoder_layer/moe_decoder_layer.py:664-679) = F.rms_norm (ops/rms_norm/__init__.py:8-11):
//   x = bf16( float(h) * rsqrt(mean(float(h)^2) + eps) * float(w) )
//
// forward  xtb_rmsnorm_gate : one pass over h produces x, rstd AND the fp32 gate logits of bf16-rounded x
//                             (a1), so the activations are read from HBM once instead of three times.
// backward xtb_moe_dispatch_bwd_rmsnorm : g_x = bf16(bf16(sum_k g_xperm[row(t,k)]) + g_x_gate)   (dispatch bwd +
//                             autograd's add), then RMSNorm backward, then "+ residual grad" — one kernel,
//                             warp per token with the whole row in registers.
#include <cstdlib>

#include "common.cuh"

namespace xtb {


// ---- forward: norm + gate logits.  A warp owns TW tokens whose rows stay in registers (ROW8 16-byte vectors per lane
// and token): one HBM read, all loads of the rows in flight at once, W_gate resident in smem ------------------------
template <int E_MAX, int TW, int ROW8>
__global__ void __launch_bounds__(256, 1) rmsnorm_gate_kernel(const __nv_bfloat16* __restrict__ h,
                                                              const float* __restrict__ norm_w,  // [H] fp32
                                                              const float* __restrict__ gate_w,  // [E,H] fp32
                                                              __nv_bfloat16* __restrict__ x_out,
                                                              float* __restrict__ rstd_out, float* __restrict__ logits,
                                                              int T, int H, int E, float eps) {
  extern __shared__ float s_w[];  // gate weight [E][H] followed by norm weight [H]
  float* s_nw = s_w + (size_t)E * H;
  const float4* src = reinterpret_cast<const float4*>(gate_w);
  float4* dst = reinterpret_cast<float4*>(s_w);
  for (int i = threadIdx.x; i < E * H / 4; i += blockDim.x) dst[i] = __ldg(src + i);
  for (int i = threadIdx.x; i < H; i += blockDim.x) s_nw[i] = norm_w[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const float inv_h = 1.f / (float)H;
  for (int t0 = warp_global * TW; t0 < T; t0 += n_warps * TW) {
    uint4 raw[TW][ROW8];
#pragma unroll
    for (int i = 0; i < TW; ++i)
#pragma unroll
      for (int c = 0; c < ROW8; ++c)
        raw[i][c] = ld_stream_16(h + (size_t)min(t0 + i, T - 1) * H + (c * 32 + lane) * 8);
    float xv[TW][ROW8][8];
    float rstd[TW];
#pragma unroll
    for (int i = 0; i < TW; ++i) {
      float ss = 0.f;
#pragma unroll
      for (int c = 0; c < ROW8; ++c) {
        unpack_bf16x8(raw[i][c], xv[i][c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss = fmaf(xv[i][c][j], xv[i][c][j], ss);
      }
      rstd[i] = rsqrtf(warp_sum(ss) * inv_h + eps);
      if (lane == 0 && t0 + i < T && rstd_out) rstd_out[t0 + i] = rstd[i];
    }
    float acc[TW][E_MAX];
#pragma unroll
    for (int i = 0; i < TW; ++i)
#pragma unroll
      for (int e = 0; e < E_MAX; ++e) acc[i][e] = 0.f;
#pragma unroll
    for (int c = 0; c < ROW8; ++c) {
      const int hh = (c * 32 + lane) * 8;
      const float4 nw0 = *reinterpret_cast<const float4*>(s_nw + hh);
      const float4 nw1 = *reinterpret_cast<const float4*>(s_nw + hh + 4);
      const float nw[8] = {nw0.x, nw0.y, nw0.z, nw0.w, nw1.x, nw1.y, nw1.z, nw1.w};
#pragma unroll
      for (int i = 0; i < TW; ++i) {
        uint32_t p[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          p[j] = pack_bf16x2(xv[i][c][2 * j] * rstd[i] * nw[2 * j], xv[i][c][2 * j + 1] * rstd[i] * nw[2 * j + 1]);
          unpack_bf16x2(p[j], xv[i][c][2 * j], xv[i][c][2 * j + 1]);  // logits use the bf16-rounded x
        }
        if (t0 + i < T) st_stream_16(x_out + (size_t)(t0 + i) * H + hh, make_uint4(p[0], p[1], p[2], p[3]));
      }
#pragma unroll
      for (int e = 0; e < E_MAX; ++e) {
        if (e < E) {
          const float4 w0 = *reinterpret_cast<const float4*>(s_w + (size_t)e * H + hh);
          const float4 w1 = *reinterpret_cast<const float4*>(s_w + (size_t)e * H + hh + 4);
#pragma unroll
          for (int i = 0; i < TW; ++i) {
            float a = acc[i][e];
            a = fmaf(xv[i][c][0], w0.x, a);
            a = fmaf(xv[i][c][1], w0.y, a);
            a = fmaf(xv[i][c][2], w0.z, a);
            a = fmaf(xv[i][c][3], w0.w, a);
            a = fmaf(xv[i][c][4], w1.x, a);
            a = fmaf(xv[i][c][5], w1.y, a);
            a = fmaf(xv[i][c][6], w1.z, a);
            a = fmaf(xv[i][c][7], w1.w, a);
            acc[i][e] = a;
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < TW; ++i)
#pragma unroll
      for (int e = 0; e < E_MAX; ++e) {
        const float s = warp_sum(acc[i][e]);
        if (lane == 0 && e < E && t0 + i < T) logits[(size_t)(t0 + i) * E + e] = s;
      }
  }
}

// ---- block-wide sum of TB values per thread (blockDim.x == 256): result broadcast to all threads ---------------
template <int TB>
__device__ __forceinline__ void block_sum(float (&v)[TB], float* s_red /* [8][TB] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < TB; ++i) v[i] = warp_sum(v[i]);
  __syncthreads();  // previous use of s_red is over
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < TB; ++i) s_red[warp * TB + i] = v[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < TB; ++i) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += s_red[w * TB + i];
    v[i] = t;
  }
}

// ---- norm-only forward, column-owned: thread j owns 8 columns per 2048-wide pass, a block handles TB tokens ----
template <int TB>
__global__ void __launch_bounds__(256) rmsnorm_cols_kernel(const __nv_bfloat16* __restrict__ h,
                                                           const float* __restrict__ norm_w,
                                                           __nv_bfloat16* __restrict__ x_out,
                                                           float* __restrict__ rstd_out, int T, int H, float eps) {
  pdl_sync();
  __shared__ float s_red[8 * TB];
  const int t0 = blockIdx.x * TB;
  const int col = threadIdx.x * 8;
  const int n_pass = (H + 2047) / 2048;
  float ss[TB];
#pragma unroll
  for (int i = 0; i < TB; ++i) ss[i] = 0.f;
  uint4 raw[TB];  // single-pass fast path keeps the row slice in registers
  for (int p = 0; p < n_pass; ++p) {
    const int c = p * 2048 + col;
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      raw[i] = (c < H && t0 + i < T) ? ld_stream_16(h + (size_t)(t0 + i) * H + c) : make_uint4(0, 0, 0, 0);
      float f[8];
      unpack_bf16x8(raw[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss[i] = fmaf(f[j], f[j], ss[i]);
    }
  }
  block_sum<TB>(ss, s_red);
  float rstd[TB];
#pragma unroll
  for (int i = 0; i < TB; ++i) {
    rstd[i] = rsqrtf(ss[i] / (float)H + eps);
    if (threadIdx.x == 0 && t0 + i < T && rstd_out) rstd_out[t0 + i] = rstd[i];
  }
  for (int p = 0; p < n_pass; ++p) {
    const int c = p * 2048 + col;
    if (c >= H) break;
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(norm_w + c));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(norm_w + c + 4));
    const float nw[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      if (t0 + i >= T) continue;
      const uint4 r = (n_pass == 1) ? raw[i] : ld_stream_16(h + (size_t)(t0 + i) * H + c);
      float f[8];
      unpack_bf16x8(r, f);
      uint4 o;
      o.x = pack_bf16x2(f[0] * rstd[i] * nw[0], f[1] * rstd[i] * nw[1]);
      o.y = pack_bf16x2(f[2] * rstd[i] * nw[2], f[3] * rstd[i] * nw[3]);
      o.z = pack_bf16x2(f[4] * rstd[i] * nw[4], f[5] * rstd[i] * nw[5]);
      o.w = pack_bf16x2(f[6] * rstd[i] * nw[6], f[7] * rstd[i] * nw[7]);
      st_stream_16(x_out + (size_t)(t0 + i) * H + c, o);
    }
  }
}

// ---- backward: dispatch-bwd (+gate grad) -> RMSNorm bwd -> + residual grad --------------------------------------
// g_x      = bf16( bf16(sum_k g_xp[row_k]) + g_x_gate )            (g_x_gate nullable)
// wg       = float(g_x) * w ;  c = mean_h(wg * h) * rstd^2
// g_h      = bf16( bf16((wg - h * c) * rstd) + g_res )             (g_res nullable)
// g_norm_w = sum_t float(g_x) * h * rstd                            (per-block partials, nullable)
// Column-owned and persistent: thread j owns columns [8j, 8j+8) (H == 2048 per pass of 256 threads), a block walks
// over groups of TB tokens; the per-token row reduction is a block reduction, the per-column weight gradient lives
// in 8 registers per thread for the whole kernel (no atomics).  H must be <= 2048 and a multiple of 8.
// The two kernels below differ only in how a token's rows reach registers; the arithmetic is these four functions.
// They keep no local arrays: their results go to arrays the caller owns, which also serve as their scratch.  A local
// array in an inlined helper changes how nvcc allocates the kernels' registers.

// the thread's 8 norm-weight columns (zeros past the end of the row)
__device__ __forceinline__ void load_norm_w8(const float* norm_w, int v, bool live, float (&nw)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) nw[j] = 0.f;
  if (live) {
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(norm_w + v * 8));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(norm_w + v * 8 + 4));
    nw[0] = w0.x; nw[1] = w0.y; nw[2] = w0.z; nw[3] = w0.w; nw[4] = w1.x; nw[5] = w1.y; nw[6] = w1.z; nw[7] = w1.w;
  }
}

// One token before the row reduction: acc = fp32 sum of its K gathered rows, hv / gv / rs = its h, gate grad and rstd.
// Adds the token's share of the norm-weight gradient to gw, returns wg in g (which holds the unpacked gate grad until
// then), float(h) in hf and this thread's part of the row dot sum(wg * h).  A token past T (tok_ok false) contributes
// zeros.
__device__ __forceinline__ float norm_bwd_token(const float (&acc)[8], const uint4& hv, const uint4& gv, float rs,
                                                bool has_gate, bool tok_ok, const float (&nw)[8], float (&gw)[8],
                                                float (&g)[8], float (&hf)[8]) {
  unpack_bf16x8(gv, g);
  unpack_bf16x8(hv, hf);
  float dot = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float gj = __bfloat162float(__float2bfloat16_rn(acc[j]));               // permute-bwd output (bf16)
    if (has_gate) gj = __bfloat162float(__float2bfloat16_rn(gj + g[j]));  // autograd's bf16 add
    if (!tok_ok) gj = 0.f;
    gw[j] = fmaf(gj * rs, hf[j], gw[j]);
    gj *= nw[j];
    g[j] = gj;
    dot = fmaf(gj, hf[j], dot);
  }
  return dot;
}

// One token after the row reduction (dot = the whole row's sum): the token's 8 g_h values in o, before the bf16 pack,
// with the residual grad rv added when has_res (o holds the unpacked rv until then)
__device__ __forceinline__ void norm_bwd_token_out(const float (&g)[8], const float (&hf)[8], float dot, float rs,
                                                   const uint4& rv, bool has_res, int H, float (&o)[8]) {
  const float cterm = dot * rs * rs / (float)H;
  unpack_bf16x8(rv, o);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float val = (g[j] - hf[j] * cterm) * rs;
    if (has_res) val = __bfloat162float(__float2bfloat16_rn(val)) + o[j];
    o[j] = val;
  }
}

// the block's row of norm-weight-gradient partials (reduced by reduce_partial_rows_kernel)
__device__ __forceinline__ void store_partial_gw(float* __restrict__ partial_gw, int H, int v, bool live,
                                                 const float (&gw)[8]) {
  if (partial_gw && live) {
    float* dst = partial_gw + (size_t)blockIdx.x * H + v * 8;
    *reinterpret_cast<float4*>(dst) = make_float4(gw[0], gw[1], gw[2], gw[3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(gw[4], gw[5], gw[6], gw[7]);
  }
}

// any K: a group's h / gate-grad / residual-grad vectors are loaded up front, the K rows of a token one after another
template <int TB>
__global__ void __launch_bounds__(256, 2) dispatch_bwd_rmsnorm_kernel(
    const uint4* __restrict__ g_xp, const int32_t* __restrict__ row_id_map, const uint4* __restrict__ g_x_gate,
    const uint4* __restrict__ h, const float* __restrict__ rstd, const float* __restrict__ norm_w,
    const uint4* __restrict__ g_res, uint4* __restrict__ g_h, float* __restrict__ partial_gw, int T, int K, int H) {
  pdl_sync();
  __shared__ float s_red[8 * TB];
  const int row_vec = H / 8;
  const int v = threadIdx.x;           // 16-byte vector index inside the row
  const bool live = v < row_vec;
  float nw[8];
  load_norm_w8(norm_w, v, live, nw);
  float gw[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int n_groups = (T + TB - 1) / TB;
  for (int grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    const int t0 = grp * TB;
    uint4 hv[TB], gv[TB], rv[TB];
    float rs[TB];
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      const int t = min(t0 + i, T - 1);
      hv[i] = live ? ld_stream_16(h + (size_t)t * row_vec + v) : make_uint4(0, 0, 0, 0);
      gv[i] = (live && g_x_gate) ? ld_stream_16(g_x_gate + (size_t)t * row_vec + v) : make_uint4(0, 0, 0, 0);
      rv[i] = (live && g_res) ? ld_stream_16(g_res + (size_t)t * row_vec + v) : make_uint4(0, 0, 0, 0);
      rs[i] = rstd[t];
    }
    float g[TB][8], hf[TB][8], dot[TB];
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      const int t = min(t0 + i, T - 1);
      for (int k = 0; k < K; ++k) {
        const int r = row_id_map[(size_t)t * K + k];
        if (!live || r < 0) continue;
        float f[8];
        unpack_bf16x8(ld_stream_16(g_xp + (size_t)r * row_vec + v), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
      }
      dot[i] = norm_bwd_token(acc, hv[i], gv[i], rs[i], g_x_gate != nullptr, t0 + i < T, nw, gw, g[i], hf[i]);
    }
    block_sum<TB>(dot, s_red);
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      if (!live || t0 + i >= T) continue;
      float o[8];
      norm_bwd_token_out(g[i], hf[i], dot[i], rs[i], rv[i], g_res != nullptr, H, o);
      st_stream_16(g_h + (size_t)(t0 + i) * row_vec + v, pack_bf16x8(o));
    }
  }
  store_partial_gw(partial_gw, H, v, live, gw);
}

// ---- the same backward with the loads of the NEXT token group in flight while the current one is reduced --------------
// The kernel above issues a group's loads, waits, reduces over the row (two block barriers), stores, and only then asks
// for the next group: with two resident CTAs per SM the memory system idles through every reduce/store phase (ncu: 50 %
// of DRAM peak, 24 % warps active).  Here every thread copies its own 16-byte pieces of group g+1 into a second
// shared-memory stage with cp.async (LDGSTS: no registers held, no barrier needed — a thread only ever reads back what it
// copied itself) before it touches group g; the row ids and rstd of group g+2 are fetched into registers at the same time so
// that the address of a gathered row is never a load away when its copy is issued.  The arithmetic is the kernel above's
// (the same functions, the same summation order): identical bits.  KT = top-k (compile time), TB tokens per group;
// dynamic smem = 2 stages x TB x (KT + 3) pieces x 4 KiB.
__device__ __forceinline__ void cp_async_16_zfill(void* smem_dst, const void* gsrc, bool pred) {
  const uint32_t dst = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int n = pred ? 16 : 0;  // src-size 0: nothing is read, 16 zero bytes are written
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(gsrc), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <int KT, int TB>
__global__ void __launch_bounds__(256, 2) dispatch_bwd_rmsnorm_pipe_kernel(
    const uint4* __restrict__ g_xp, const int32_t* __restrict__ row_id_map, const uint4* __restrict__ g_x_gate,
    const uint4* __restrict__ h, const float* __restrict__ rstd, const float* __restrict__ norm_w,
    const uint4* __restrict__ g_res, uint4* __restrict__ g_h, float* __restrict__ partial_gw, int T, int H) {
  pdl_sync();
  constexpr int P = KT + 3;             // pieces per token: KT gathered rows, h, gate grad, residual grad
  extern __shared__ uint4 s_stage[];    // [2][TB][P][256]
  __shared__ float s_red[8 * TB];
  const int row_vec = H / 8;
  const int v = threadIdx.x;
  const bool live = v < row_vec;
  float nw[8];
  load_norm_w8(norm_w, v, live, nw);
  float gw[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int n_groups = (T + TB - 1) / TB;
  auto slot = [&](int stage, int i, int p) -> uint4* { return s_stage + ((size_t)((stage * TB + i) * P + p)) * 256 + v; };
  auto load_ids = [&](int grp, int (&r)[TB][KT], float (&rs)[TB]) {
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      const int t = min(grp * TB + i, T - 1);
#pragma unroll
      for (int k = 0; k < KT; ++k) r[i][k] = row_id_map[(size_t)t * KT + k];
      rs[i] = rstd[t];
    }
  };
  auto issue = [&](int grp, int stage, const int (&r)[TB][KT]) {
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      const int t = min(grp * TB + i, T - 1);
#pragma unroll
      for (int k = 0; k < KT; ++k) {
        const bool ok = live && r[i][k] >= 0;
        cp_async_16_zfill(slot(stage, i, k), g_xp + (ok ? (size_t)r[i][k] * row_vec + v : 0), ok);
      }
      cp_async_16_zfill(slot(stage, i, KT), h + (live ? (size_t)t * row_vec + v : 0), live);
      const bool okg = live && g_x_gate != nullptr, okr = live && g_res != nullptr;
      cp_async_16_zfill(slot(stage, i, KT + 1), okg ? g_x_gate + (size_t)t * row_vec + v : h, okg);
      cp_async_16_zfill(slot(stage, i, KT + 2), okr ? g_res + (size_t)t * row_vec + v : h, okr);
    }
    cp_async_commit();
  };

  int grp = blockIdx.x;
  int r_nxt[TB][KT];
  float rs_cur[TB], rs_nxt[TB];
  if (grp < n_groups) {
    int r0[TB][KT];
    load_ids(grp, r0, rs_cur);
    issue(grp, 0, r0);
    if (grp + (int)gridDim.x < n_groups) load_ids(grp + gridDim.x, r_nxt, rs_nxt);
  }
  int stage = 0;
  while (grp < n_groups) {
    const int t0 = grp * TB;
    const int g1 = grp + gridDim.x, g2 = g1 + gridDim.x;
    const bool has1 = g1 < n_groups;
    if (has1) issue(g1, stage ^ 1, r_nxt);
    int r_n2[TB][KT];
    float rs_n2[TB];
    if (g2 < n_groups) load_ids(g2, r_n2, rs_n2);
    if (has1) cp_async_wait<1>();
    else cp_async_wait<0>();

    float g[TB][8], hf[TB][8], dot[TB];
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < KT; ++k) {
        float f[8];
        unpack_bf16x8(*slot(stage, i, k), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
      }
      const uint4 hv = *slot(stage, i, KT), gv = *slot(stage, i, KT + 1);
      dot[i] = norm_bwd_token(acc, hv, gv, rs_cur[i], g_x_gate != nullptr, t0 + i < T, nw, gw, g[i], hf[i]);
    }
    block_sum<TB>(dot, s_red);
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      if (!live || t0 + i >= T) continue;
      float o[8];
      norm_bwd_token_out(g[i], hf[i], dot[i], rs_cur[i], *slot(stage, i, KT + 2), g_res != nullptr, H, o);
      st_stream_16(g_h + (size_t)(t0 + i) * row_vec + v, pack_bf16x8(o));
    }
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      rs_cur[i] = rs_nxt[i];
      rs_nxt[i] = rs_n2[i];
#pragma unroll
      for (int k = 0; k < KT; ++k) r_nxt[i][k] = r_n2[i][k];
    }
    stage ^= 1;
    grp = g1;
  }
  store_partial_gw(partial_gw, H, v, live, gw);
}

static int norm_bwd_blocks(int T) { return max(1, min(sm_count() * 2, (T + 3) / 4)); }  // 2 resident CTAs per SM

}  // namespace xtb

using namespace xtb;

extern "C" int xtb_rmsnorm_gate(const void* h_bf16, const float* norm_w_f32, const float* gate_w_f32, float eps,
                                int T, int H, int E, void* x_out_bf16, float* rstd_out, float* logits,
                                xtb_stream_t stream) {
  XTB_CHECK_ARG(h_bf16 && norm_w_f32 && x_out_bf16, "xtb_rmsnorm_gate: null pointer");
  XTB_CHECK_ARG(T >= 0 && H > 0 && H % 8 == 0, "xtb_rmsnorm_gate: H=%d must be a multiple of 8", H);
  XTB_CHECK_ARG(!gate_w_f32 || (logits && E > 0 && E <= 8), "xtb_rmsnorm_gate: fused gate supports E <= 8 (got %d)", E);
  XTB_ENSURE_CTX(h_bf16);
  if (T == 0) return XTB_OK;
  cudaStream_t st = as_stream(stream);
  const auto* hp = static_cast<const __nv_bfloat16*>(h_bf16);
  auto* xp = static_cast<__nv_bfloat16*>(x_out_bf16);
  XTB_CHECK_ARG(H == 256 || H == 512 || H == 1024 || H == 2048,
                "xtb_rmsnorm_gate: unsupported H=%d (256, 512, 1024, 2048: the row lives in registers)", H);
  if (!gate_w_f32) {
    // norm only: column-owned streaming kernel, 4 tokens per 256-thread block (one 8-column vector per thread)
    XTB_LAUNCH(rmsnorm_cols_kernel<4>, dim3((T + 3) / 4), dim3(256), 0, st, true, hp, norm_w_f32, xp, rstd_out, T, H, eps);
    return XTB_OK;
  }
  const int blocks = min(sm_count(), (T + 15) / 16);
  const size_t smem = ((size_t)E * H + H) * sizeof(float);
  XTB_CHECK_ARG(smem <= 200 * 1024, "xtb_rmsnorm_gate: E*H too large for the fused gate (%zu bytes of smem)", smem);
  auto* kernel = H == 256 ? rmsnorm_gate_kernel<8, 2, 1>
               : H == 512 ? rmsnorm_gate_kernel<8, 2, 2>
               : H == 1024 ? rmsnorm_gate_kernel<8, 2, 4>
                           : rmsnorm_gate_kernel<8, 2, 8>;
  XTB_LAUNCH(kernel, dim3(blocks), dim3(256), smem, st, false, hp, norm_w_f32, gate_w_f32, xp, rstd_out, logits, T, H, E,
             eps);
  return XTB_OK;
}

extern "C" size_t xtb_moe_dispatch_bwd_rmsnorm_workspace_bytes(int T, int H) {
  return (size_t)norm_bwd_blocks(T) * H * sizeof(float);
}

extern "C" int xtb_moe_dispatch_bwd_rmsnorm(const void* g_xperm_bf16, const int32_t* row_id_map,
                                            const void* g_x_gate_bf16, const void* h_bf16, const float* rstd,
                                            const float* norm_w_f32, const void* g_res_bf16, int T, int K, int H,
                                            void* g_h_bf16, float* g_norm_w, void* workspace, xtb_stream_t stream) {
  XTB_CHECK_ARG(g_xperm_bf16 && row_id_map && h_bf16 && rstd && norm_w_f32 && g_h_bf16,
                "xtb_moe_dispatch_bwd_rmsnorm: null pointer");
  XTB_CHECK_ARG(T >= 0 && K > 0 && H > 0 && H % 8 == 0 && H <= 2048,
                "xtb_moe_dispatch_bwd_rmsnorm: H=%d must be a multiple of 8 and <= 2048 (one 16-byte vector per thread)", H);
  XTB_CHECK_ARG(!g_norm_w || workspace, "xtb_moe_dispatch_bwd_rmsnorm: workspace required for the weight gradient");
  XTB_ENSURE_CTX(h_bf16);
  if (T == 0) return XTB_OK;
  cudaStream_t st = as_stream(stream);
  const int blocks = norm_bwd_blocks(T);
  float* partial = g_norm_w ? static_cast<float*>(workspace) : nullptr;
  const auto* gx = static_cast<const uint4*>(g_xperm_bf16);
  const auto* gxg = static_cast<const uint4*>(g_x_gate_bf16);
  const auto* hv = static_cast<const uint4*>(h_bf16);
  const auto* gres = static_cast<const uint4*>(g_res_bf16);
  auto* gh = static_cast<uint4*>(g_h_bf16);
  if (K == 2 || K == 8) {
    // <KT, TB>: two stages of TB token groups, (KT + 3) 16-byte vectors per thread each
    auto* kernel = K == 2 ? dispatch_bwd_rmsnorm_pipe_kernel<2, 2> : dispatch_bwd_rmsnorm_pipe_kernel<8, 1>;
    const int TB = K == 2 ? 2 : 1;
    const size_t smem = (size_t)2 * TB * (K + 3) * 256 * sizeof(uint4);
    XTB_LAUNCH(kernel, dim3(blocks), dim3(256), smem, st, true, gx, row_id_map, gxg, hv, rstd, norm_w_f32, gres, gh,
               partial, T, H);
  } else {
    XTB_LAUNCH(dispatch_bwd_rmsnorm_kernel<4>, dim3(blocks), dim3(256), 0, st, true, gx, row_id_map, gxg, hv, rstd,
               norm_w_f32, gres, gh, partial, T, K, H);
  }
  if (g_norm_w) {
    // H outputs, up to 2 partial rows per SM: 32 warps per block put all of a lane's ~9 loads in flight at once
    XTB_LAUNCH(reduce_partial_rows_kernel<32>, dim3((H + 31) / 32), dim3(1024), 0, st, true, (const float*)partial,
               g_norm_w, blocks, (int64_t)H);
  }
  return XTB_OK;
}
