// q/k RMSNorm fused with the rotary embedding, the step in front of the attention kernel (SURVEY.md §8f-3: "RoPE/qk-norm
// before attention").  Reference: MultiHeadAttention.forward (module/attention/mha.py:353-363) runs q_norm / k_norm
// (F.rms_norm, ops/rms_norm/__init__.py:8-11), a transpose, and apply_rotary_pos_emb_cuda (ops/rotary_emb.py:18-49) as
// separate eager ops; here one kernel reads q, k, cos and sin once and writes the rotated q and k once, and one kernel does
// the same for the backward.  Formulas and rounding points: include/xtuner_b200.h.
//
// Mapping: a row is one (token, head) vector of D bf16 values, held by L = D/8 lanes as one 16-byte vector each, so a warp
// works on 32/L rows side by side.  Lane c of a row holds columns [8c, 8c+8); the rotate_half partner of column i lives in
// lane c ^ (L/2), one shfl.xor per 32-bit word, and the row's sums are a log2(L)-level butterfly inside the L lanes.  A CTA
// owns kQkTokens tokens and stages their cos/sin rows in shared memory once for all Hq + Hkv heads.
#include "common.cuh"

namespace xtb {

constexpr int kQkTokens = 4;   // tokens per CTA group
constexpr int kQkUnroll = 2;   // rows each lane has in flight

template <int D>
struct QkGeom {
  static constexpr int L = D / 8;      // lanes per row
  static constexpr int RPW = 32 / L;   // rows per warp and pass
  static constexpr int RPP = 8 * RPW;  // rows per 256-thread CTA and pass
};

__device__ __forceinline__ float bf16r(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

__device__ __forceinline__ void unpack8(const uint4& r, float (&f)[8]) {
  unpack_bf16x2(r.x, f[0], f[1]);
  unpack_bf16x2(r.y, f[2], f[3]);
  unpack_bf16x2(r.z, f[4], f[5]);
  unpack_bf16x2(r.w, f[6], f[7]);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}
template <int L>
__device__ __forceinline__ float row_sum(float v) {
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <int L>
__device__ __forceinline__ uint4 partner(const uint4& v) {
  return make_uint4(__shfl_xor_sync(0xffffffffu, v.x, L / 2), __shfl_xor_sync(0xffffffffu, v.y, L / 2),
                    __shfl_xor_sync(0xffffffffu, v.z, L / 2), __shfl_xor_sync(0xffffffffu, v.w, L / 2));
}

// q and k of one call, and where row r = tt * (Hq + Hkv) + h of a token group lives
struct QkOperands {
  const __nv_bfloat16* q;
  const __nv_bfloat16* k;
  int64_t q_st, q_sh, k_st, k_sh;  // token and head strides, elements
  int Hq, Hkv;
  __device__ __forceinline__ const __nv_bfloat16* row(int t, int h) const {
    return h < Hq ? q + (size_t)t * q_st + (size_t)h * q_sh : k + (size_t)t * k_st + (size_t)(h - Hq) * k_sh;
  }
};

// contiguous [T, Hq, D] / [T, Hkv, D] outputs (and [T, H] rstd)
__device__ __forceinline__ size_t qk_out_index(int t, int h, int Hq, int Hkv, bool& is_q) {
  is_q = h < Hq;
  return is_q ? (size_t)t * Hq + h : (size_t)t * Hkv + (h - Hq);
}

template <int D>
__device__ __forceinline__ void stage_cos_sin(uint4 (*s_cs)[kQkTokens][D / 8], const __nv_bfloat16* cos,
                                              const __nv_bfloat16* sin, int t0, int nt) {
  constexpr int L = D / 8;
  for (int i = threadIdx.x; i < 2 * kQkTokens * L; i += blockDim.x) {
    const int which = i / (kQkTokens * L), tt = (i / L) % kQkTokens, c = i % L;
    if (tt < nt) s_cs[which][tt][c] = ld_stream_16((which ? sin : cos) + (size_t)(t0 + tt) * D + c * 8);
  }
}

// ---- forward ------------------------------------------------------------------------------------------------------------
template <int D, bool NORM>
__global__ void __launch_bounds__(256) qk_norm_rope_kernel(QkOperands in, const __nv_bfloat16* __restrict__ cos,
                                                           const __nv_bfloat16* __restrict__ sin,
                                                           const float* __restrict__ w_q, const float* __restrict__ w_k,
                                                           __nv_bfloat16* __restrict__ out_q,
                                                           __nv_bfloat16* __restrict__ out_k, float* __restrict__ rstd_q,
                                                           float* __restrict__ rstd_k, int T, float eps) {
  using G = QkGeom<D>;
  constexpr int L = G::L;
  __shared__ uint4 s_cs[2][kQkTokens][L];
  pdl_sync();
  const int t0 = blockIdx.x * kQkTokens;
  const int nt = min(kQkTokens, T - t0);
  const int lane = threadIdx.x & 31, sub = lane / L, c = lane % L;
  const bool first = c < L / 2;
  float wq[8], wk[8];
  if (NORM) {
#pragma unroll
    for (int j = 0; j < 8; ++j) wq[j] = __ldg(w_q + c * 8 + j), wk[j] = __ldg(w_k + c * 8 + j);
  }
  stage_cos_sin<D>(s_cs, cos, sin, t0, nt);
  __syncthreads();
  const int H = in.Hq + in.Hkv;
  const int n_rows = nt * H;
  for (int rb = (threadIdx.x >> 5) * G::RPW; rb < n_rows; rb += kQkUnroll * G::RPP) {  // warp-uniform bound
    uint4 raw[kQkUnroll];
#pragma unroll
    for (int u = 0; u < kQkUnroll; ++u) {
      const int r = min(rb + u * G::RPP + sub, n_rows - 1);
      raw[u] = ld_stream_16(in.row(t0 + r / H, r % H) + c * 8);
    }
#pragma unroll
    for (int u = 0; u < kQkUnroll; ++u) {
      const int r_raw = rb + u * G::RPP + sub;
      const int r = min(r_raw, n_rows - 1), tt = r / H, h = r % H;
      bool is_q;
      const size_t o = qk_out_index(t0 + tt, h, in.Hq, in.Hkv, is_q);
      float x[8];
      unpack8(raw[u], x);
      if (NORM) {
        float ss = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) ss = fmaf(x[j], x[j], ss);
        const float rs = rsqrtf(row_sum<L>(ss) * (1.f / D) + eps);
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = bf16r(x[j] * rs * (is_q ? wq[j] : wk[j]));
        if (c == 0 && r_raw < n_rows) (is_q ? rstd_q : rstd_k)[o] = rs;
      }
      const uint4 pv = partner<L>(pack8(x));
      float p[8], cs[8], sn[8];
      unpack8(pv, p);
      unpack8(s_cs[0][tt][c], cs);
      unpack8(s_cs[1][tt][c], sn);
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] = bf16r(x[j] * cs[j]) + bf16r((first ? -p[j] : p[j]) * sn[j]);
      if (r_raw < n_rows) st_stream_16((is_q ? out_q : out_k) + o * D + c * 8, pack8(x));
    }
  }
}

// ---- backward -----------------------------------------------------------------------------------------------------------
// Persistent over token groups: a thread keeps the weight-gradient sums of its 8 columns of q and of k in registers; at the
// end the CTA adds its 8 * RPW row slots in slot order and writes one partial row [dw_q | dw_k] (2D floats).
template <int D, bool NORM>
__global__ void __launch_bounds__(256, 2) qk_norm_rope_bwd_kernel(QkOperands g, QkOperands in,
                                                               const __nv_bfloat16* __restrict__ cos,
                                                               const __nv_bfloat16* __restrict__ sin,
                                                               const float* __restrict__ w_q, const float* __restrict__ w_k,
                                                               const float* __restrict__ rstd_q,
                                                               const float* __restrict__ rstd_k,
                                                               __nv_bfloat16* __restrict__ dx_q,
                                                               __nv_bfloat16* __restrict__ dx_k,
                                                               float* __restrict__ partial, int T) {
  using G = QkGeom<D>;
  constexpr int L = G::L;
  __shared__ uint4 s_cs[2][kQkTokens][L];
  __shared__ float s_red[NORM ? G::RPP : 1][NORM ? 2 * D : 1];
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, sub = lane / L, c = lane % L;
  const bool first = c < L / 2;
  float wq[8], wk[8], dwq[8], dwk[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    dwq[j] = dwk[j] = 0.f;
    if (NORM) wq[j] = __ldg(w_q + c * 8 + j), wk[j] = __ldg(w_k + c * 8 + j);
  }
  const int H = in.Hq + in.Hkv;
  const int n_groups = (T + kQkTokens - 1) / kQkTokens;
  for (int grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    const int t0 = grp * kQkTokens;
    const int nt = min(kQkTokens, T - t0);
    __syncthreads();  // the previous group's cos/sin are no longer read
    stage_cos_sin<D>(s_cs, cos, sin, t0, nt);
    __syncthreads();
    const int n_rows = nt * H;
    for (int rb = warp * G::RPW; rb < n_rows; rb += kQkUnroll * G::RPP) {
      uint4 graw[kQkUnroll], xraw[kQkUnroll];
      float rsv[kQkUnroll];
#pragma unroll
      for (int u = 0; u < kQkUnroll; ++u) {
        const int r = min(rb + u * G::RPP + sub, n_rows - 1), t = t0 + r / H, h = r % H;
        graw[u] = ld_stream_16(g.row(t, h) + c * 8);
        if (NORM) {
          xraw[u] = ld_stream_16(in.row(t, h) + c * 8);
          rsv[u] = h < in.Hq ? rstd_q[(size_t)t * in.Hq + h] : rstd_k[(size_t)t * in.Hkv + (h - in.Hq)];
        }
      }
#pragma unroll
      for (int u = 0; u < kQkUnroll; ++u) {
        const int r_raw = rb + u * G::RPP + sub;
        const bool live = r_raw < n_rows;
        const int r = min(r_raw, n_rows - 1), tt = r / H, h = r % H;
        bool is_q;
        const size_t o = qk_out_index(t0 + tt, h, in.Hq, in.Hkv, is_q);
        float gv[8], cs[8], sn[8], s[8], ps[8], gn[8];
        unpack8(graw[u], gv);
        unpack8(s_cs[0][tt][c], cs);
        unpack8(s_cs[1][tt][c], sn);
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = gv[j] * sn[j];  // rounded by the pack: bf16(g sin), the partner's term
        unpack8(partner<L>(pack8(s)), ps);
#pragma unroll
        for (int j = 0; j < 8; ++j) gn[j] = bf16r(bf16r(gv[j] * cs[j]) + (first ? ps[j] : -ps[j]));
        if (NORM) {
          float x[8], wg[8], dot = 0.f;
          unpack8(xraw[u], x);
          const float rs = rsv[u];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float gj = live ? gn[j] : 0.f;
            if (is_q) dwq[j] = fmaf(gj * rs, x[j], dwq[j]);
            else dwk[j] = fmaf(gj * rs, x[j], dwk[j]);
            wg[j] = gn[j] * (is_q ? wq[j] : wk[j]);
            dot = fmaf(wg[j], x[j], dot);
          }
          const float cterm = row_sum<L>(dot) * rs * rs / (float)D;
#pragma unroll
          for (int j = 0; j < 8; ++j) gn[j] = (wg[j] - x[j] * cterm) * rs;
        }
        if (live) st_stream_16((is_q ? dx_q : dx_k) + o * D + c * 8, pack8(gn));
      }
    }
  }
  if (NORM && partial) {
    const int slot = warp * G::RPW + sub;
#pragma unroll
    for (int j = 0; j < 8; ++j) s_red[slot][c * 8 + j] = dwq[j], s_red[slot][D + c * 8 + j] = dwk[j];
    __syncthreads();
    for (int col = threadIdx.x; col < 2 * D; col += blockDim.x) {
      float acc = 0.f;
#pragma unroll 8
      for (int sl = 0; sl < G::RPP; ++sl) acc += s_red[sl][col];
      partial[(size_t)blockIdx.x * 2 * D + col] = acc;
    }
  }
}

static int qk_bwd_blocks(int64_t T) {  // persistent grid: the 2 CTAs per SM that fit, one per token group at least
  return (int)max((int64_t)1, min((int64_t)sm_count() * 2, (T + kQkTokens - 1) / kQkTokens));
}

static bool qk_aligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace xtb

using namespace xtb;

extern "C" int xtb_qk_norm_rope(const void* q_bf16, int64_t q_stride_t, int64_t q_stride_h, const void* k_bf16,
                                int64_t k_stride_t, int64_t k_stride_h, const void* cos_bf16, const void* sin_bf16,
                                const float* w_q_f32, const float* w_k_f32, float eps, int T, int Hq, int Hkv, int D,
                                void* out_q_bf16, void* out_k_bf16, float* rstd_q, float* rstd_k, xtb_stream_t stream) {
  XTB_CHECK_ARG(q_bf16 && k_bf16 && cos_bf16 && sin_bf16 && out_q_bf16 && out_k_bf16, "xtb_qk_norm_rope: null pointer");
  XTB_CHECK_ARG(D == 64 || D == 128 || D == 256, "xtb_qk_norm_rope: head dim D=%d must be 64, 128 or 256", D);
  XTB_CHECK_ARG(T >= 0 && Hq > 0 && Hkv > 0, "xtb_qk_norm_rope: T=%d Hq=%d Hkv=%d", T, Hq, Hkv);
  XTB_CHECK_ARG((w_q_f32 == nullptr) == (w_k_f32 == nullptr), "xtb_qk_norm_rope: pass both norm weights or neither");
  XTB_CHECK_ARG(!w_q_f32 || (rstd_q && rstd_k), "xtb_qk_norm_rope: the norm needs rstd_q and rstd_k");
  XTB_CHECK_ARG(qk_aligned(q_bf16) && qk_aligned(k_bf16) && qk_aligned(cos_bf16) && qk_aligned(sin_bf16) &&
                    qk_aligned(out_q_bf16) && qk_aligned(out_k_bf16) && q_stride_t % 8 == 0 && q_stride_h % 8 == 0 &&
                    k_stride_t % 8 == 0 && k_stride_h % 8 == 0,
                "xtb_qk_norm_rope: pointers must be 16-byte aligned and strides multiples of 8 elements");
  if (T == 0) return XTB_OK;
  XTB_ENSURE_CTX(q_bf16);
  cudaStream_t st = as_stream(stream);
  const QkOperands in{static_cast<const __nv_bfloat16*>(q_bf16), static_cast<const __nv_bfloat16*>(k_bf16), q_stride_t,
                      q_stride_h, k_stride_t, k_stride_h, Hq, Hkv};
  const dim3 grid((unsigned)((T + kQkTokens - 1) / kQkTokens));
  const bool norm = w_q_f32 != nullptr;
  auto* kernel = D == 64    ? (norm ? qk_norm_rope_kernel<64, true> : qk_norm_rope_kernel<64, false>)
                 : D == 128 ? (norm ? qk_norm_rope_kernel<128, true> : qk_norm_rope_kernel<128, false>)
                            : (norm ? qk_norm_rope_kernel<256, true> : qk_norm_rope_kernel<256, false>);
  XTB_LAUNCH(kernel, grid, dim3(256), 0, st, true, in, static_cast<const __nv_bfloat16*>(cos_bf16),
             static_cast<const __nv_bfloat16*>(sin_bf16), w_q_f32, w_k_f32, static_cast<__nv_bfloat16*>(out_q_bf16),
             static_cast<__nv_bfloat16*>(out_k_bf16), rstd_q, rstd_k, T, eps);
  return XTB_OK;
}

extern "C" size_t xtb_qk_norm_rope_bwd_workspace_bytes(int T, int D) {
  return (size_t)qk_bwd_blocks(T) * 2 * D * sizeof(float);
}

extern "C" int xtb_qk_norm_rope_bwd(const void* g_q_bf16, int64_t g_q_stride_t, int64_t g_q_stride_h,
                                    const void* g_k_bf16, int64_t g_k_stride_t, int64_t g_k_stride_h, const void* q_bf16,
                                    int64_t q_stride_t, int64_t q_stride_h, const void* k_bf16, int64_t k_stride_t,
                                    int64_t k_stride_h, const void* cos_bf16, const void* sin_bf16, const float* w_q_f32,
                                    const float* w_k_f32, const float* rstd_q, const float* rstd_k, int T, int Hq,
                                    int Hkv, int D, void* dx_q_bf16, void* dx_k_bf16, float* dw, void* workspace,
                                    xtb_stream_t stream) {
  XTB_CHECK_ARG(g_q_bf16 && g_k_bf16 && cos_bf16 && sin_bf16 && dx_q_bf16 && dx_k_bf16, "xtb_qk_norm_rope_bwd: null pointer");
  XTB_CHECK_ARG(D == 64 || D == 128 || D == 256, "xtb_qk_norm_rope_bwd: head dim D=%d must be 64, 128 or 256", D);
  XTB_CHECK_ARG(T >= 0 && Hq > 0 && Hkv > 0, "xtb_qk_norm_rope_bwd: T=%d Hq=%d Hkv=%d", T, Hq, Hkv);
  XTB_CHECK_ARG((w_q_f32 == nullptr) == (w_k_f32 == nullptr), "xtb_qk_norm_rope_bwd: pass both norm weights or neither");
  XTB_CHECK_ARG(!w_q_f32 || (q_bf16 && k_bf16 && rstd_q && rstd_k), "xtb_qk_norm_rope_bwd: the norm needs q, k and rstd");
  XTB_CHECK_ARG(!dw || w_q_f32, "xtb_qk_norm_rope_bwd: dw needs the norm weights");
  XTB_CHECK_ARG(!dw || workspace, "xtb_qk_norm_rope_bwd: workspace required for the weight gradient");
  XTB_CHECK_ARG(qk_aligned(g_q_bf16) && qk_aligned(g_k_bf16) && qk_aligned(cos_bf16) && qk_aligned(sin_bf16) &&
                    qk_aligned(dx_q_bf16) && qk_aligned(dx_k_bf16) && qk_aligned(q_bf16) && qk_aligned(k_bf16) &&
                    g_q_stride_t % 8 == 0 && g_q_stride_h % 8 == 0 && g_k_stride_t % 8 == 0 && g_k_stride_h % 8 == 0 &&
                    q_stride_t % 8 == 0 && q_stride_h % 8 == 0 && k_stride_t % 8 == 0 && k_stride_h % 8 == 0,
                "xtb_qk_norm_rope_bwd: pointers must be 16-byte aligned and strides multiples of 8 elements");
  XTB_ENSURE_CTX(g_q_bf16);
  cudaStream_t st = as_stream(stream);
  const QkOperands gg{static_cast<const __nv_bfloat16*>(g_q_bf16), static_cast<const __nv_bfloat16*>(g_k_bf16),
                      g_q_stride_t, g_q_stride_h, g_k_stride_t, g_k_stride_h, Hq, Hkv};
  const QkOperands in{static_cast<const __nv_bfloat16*>(q_bf16), static_cast<const __nv_bfloat16*>(k_bf16), q_stride_t,
                      q_stride_h, k_stride_t, k_stride_h, Hq, Hkv};
  const int blocks = T ? qk_bwd_blocks(T) : 0;  // T = 0: no launch; the reduce over zero partial rows writes dw = 0
  float* partial = dw ? static_cast<float*>(workspace) : nullptr;
  const bool norm = w_q_f32 != nullptr;
  if (T > 0) {
    auto* kernel = D == 64    ? (norm ? qk_norm_rope_bwd_kernel<64, true> : qk_norm_rope_bwd_kernel<64, false>)
                   : D == 128 ? (norm ? qk_norm_rope_bwd_kernel<128, true> : qk_norm_rope_bwd_kernel<128, false>)
                              : (norm ? qk_norm_rope_bwd_kernel<256, true> : qk_norm_rope_bwd_kernel<256, false>);
    XTB_LAUNCH(kernel, dim3(blocks), dim3(256), 0, st, true, gg, in, static_cast<const __nv_bfloat16*>(cos_bf16),
               static_cast<const __nv_bfloat16*>(sin_bf16), w_q_f32, w_k_f32, rstd_q, rstd_k,
               static_cast<__nv_bfloat16*>(dx_q_bf16), static_cast<__nv_bfloat16*>(dx_k_bf16), partial, T);
  }
  if (dw) {
    XTB_LAUNCH(reduce_partial_rows_kernel<32>, dim3((2 * D + 31) / 32), dim3(1024), 0, st, true, (const float*)partial,
               dw, blocks, (int64_t)2 * D);
  }
  return XTB_OK;
}
