// fp8 (e4m3) tile-wise quantisation kernels for the fp8 expert path (SURVEY.md §8a row a15, config 5).
// Bit-exact on an H100 against reference-made golden vectors and the oracle (tests/test_gpu_fp8.py; oracle/moe_oracle.py:
// per_tile_quant, per_block_fp8_scales, cast_to_per_block_fp8), and against the reference's own functions on CUDA tensors
// (tests/test_gpu_fp8_edges.py): every bf16 value in [-448, 448] through the cast, all-zero and sub-1e-12 blocks, fp32 and
// bf16 weights, and NaN / inf inputs, where the scale follows torch's amax (a NaN makes its whole tile or block NaN, an
// inf gives an inf scale and inf / inf = NaN).  Nothing on the bf16 default path calls them;
// plugin.install_fp8_cast() rebinds the reference's fp8 FSDP all-gather cast and scale precompute to them.
//
//   xtb_fp8_per_tile_quant   activations [M,K] bf16 -> e4m3 [M,K] + fp32 scale per 1x128 tile
//                            (float8/triton_kernels/per_tile_quant.py:61-100 / torch ref :145-155)
//   xtb_fp8_block_scales     weights [nw,dout,din] fp32/bf16 -> fp32 scale per 128x128 block
//                            (float8/fsdp_utils.py:75-116, dout >= 128 branch)
//   xtb_fp8_block_cast       weights [dout,din] + scales -> e4m3 [dout,din]   (float8/fsdp_utils.py:195-223)
// scale = clamp(amax, 1e-12) / 448 evaluated in double like the reference (fsdp_utils.py:106-110), value / scale in
// fp32, saturating round-to-nearest-even conversion (float8_utils.py:16-32; NaN stays NaN, +-inf and finite overflow
// become +-448).
#include <cuda_fp8.h>

#include "common.cuh"

namespace xtb {

// max that keeps NaN, as torch's amax does (fmaxf drops a NaN operand, which would leave the scale finite)
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }
__device__ __forceinline__ float warp_nan_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float fp8_scale_from_amax(float amax) {
  const double a = amax < 1e-12 ? 1e-12 : (double)amax;
  return (float)(a / 448.0);
}

// satfinite: finite overflow and +-inf saturate to +-448 (the reference's clamp), NaN converts to NaN
__device__ __forceinline__ uint8_t to_e4m3_sat(float v) {
  return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
}

// one warp per 1x128 tile: lane holds 4 consecutive elements
__global__ void __launch_bounds__(256) fp8_per_tile_quant_kernel(const __nv_bfloat16* __restrict__ x,
                                                                 uint8_t* __restrict__ q, float* __restrict__ scales,
                                                                 long long n_tiles) {
  const int lane = threadIdx.x & 31;
  const long long tile = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (tile >= n_tiles) return;
  const uint2 raw = *reinterpret_cast<const uint2*>(x + tile * 128 + lane * 4);
  float f[4];
  unpack_bf16x2(raw.x, f[0], f[1]);
  unpack_bf16x2(raw.y, f[2], f[3]);
  float amax = nan_max(nan_max(fabsf(f[0]), fabsf(f[1])), nan_max(fabsf(f[2]), fabsf(f[3])));
  amax = warp_nan_max(amax);
  const float s = fp8_scale_from_amax(amax);
  if (lane == 0) scales[tile] = s;
  uint32_t out = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) out |= (uint32_t)to_e4m3_sat(__fdiv_rn(f[j], s)) << (8 * j);
  *reinterpret_cast<uint32_t*>(q + tile * 128 + lane * 4) = out;
}

// one 256-thread block per 128x128 block: amax -> scale (pass 1), optional cast (pass 2)
template <typename T, bool CAST>
__global__ void __launch_bounds__(256) fp8_block_kernel(const T* __restrict__ w, int dout, int din,
                                                        float* __restrict__ scales_out,
                                                        const float* __restrict__ scales_in, uint8_t* __restrict__ q) {
  __shared__ float s_red[8];
  const int bj = blockIdx.x, bi = blockIdx.y;
  const long long mat = blockIdx.z;
  const T* base = w + mat * (long long)dout * din + (long long)bi * 128 * din + bj * 128;
  const int nbj = din / 128, nbi = dout / 128;
  float s;
  if (!CAST) {
    float amax = 0.f;
    for (int i = threadIdx.x; i < 128 * 128; i += 256) {
      const int r = i >> 7, c = i & 127;
      float v;
      if constexpr (sizeof(T) == 2) v = __bfloat162float(base[(long long)r * din + c]);
      else v = (float)base[(long long)r * din + c];
      amax = nan_max(amax, fabsf(v));
    }
    amax = warp_nan_max(amax);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = amax;
    __syncthreads();
    if (threadIdx.x == 0) {
      float m = s_red[0];
      for (int i = 1; i < 8; ++i) m = nan_max(m, s_red[i]);
      scales_out[(mat * nbi + bi) * nbj + bj] = fp8_scale_from_amax(m);
    }
    return;
  } else {
    s = scales_in[(mat * nbi + bi) * nbj + bj];
    uint8_t* qb = q + mat * (long long)dout * din + (long long)bi * 128 * din + bj * 128;
    for (int i = threadIdx.x; i < 128 * 128; i += 256) {
      const int r = i >> 7, c = i & 127;
      float v;
      if constexpr (sizeof(T) == 2) v = __bfloat162float(base[(long long)r * din + c]);
      else v = (float)base[(long long)r * din + c];
      qb[(long long)r * din + c] = to_e4m3_sat(__fdiv_rn(v, s));
    }
  }
}

}  // namespace xtb

using namespace xtb;

extern "C" int xtb_fp8_per_tile_quant(const void* x_bf16, void* q_e4m3, float* scales, int64_t M, int64_t K,
                                      xtb_stream_t stream) {
  XTB_CHECK_ARG(x_bf16 && q_e4m3 && scales, "xtb_fp8_per_tile_quant: null pointer");
  XTB_CHECK_ARG(M >= 0 && K > 0 && K % 128 == 0, "xtb_fp8_per_tile_quant: K=%lld must be a multiple of 128", (long long)K);
  // 8-byte loads of x, 4-byte stores of q
  XTB_CHECK_ARG(reinterpret_cast<uintptr_t>(x_bf16) % 8 == 0 && reinterpret_cast<uintptr_t>(q_e4m3) % 4 == 0 &&
                    reinterpret_cast<uintptr_t>(scales) % 4 == 0,
                "xtb_fp8_per_tile_quant: x must be 8-byte aligned, q and scales 4-byte aligned");
  XTB_ENSURE_CTX(x_bf16);
  const long long n_tiles = M * (K / 128);
  if (n_tiles == 0) return XTB_OK;
  fp8_per_tile_quant_kernel<<<(unsigned)((n_tiles + 7) / 8), 256, 0, as_stream(stream)>>>(
      static_cast<const __nv_bfloat16*>(x_bf16), static_cast<uint8_t*>(q_e4m3), scales, n_tiles);
  XTB_LAUNCH_OK();
  return XTB_OK;
}

extern "C" int xtb_fp8_block_scales(const void* w, int w_is_f32, int64_t nw, int dout, int din, float* scales,
                                    xtb_stream_t stream) {
  XTB_CHECK_ARG(w && scales, "xtb_fp8_block_scales: null pointer");
  XTB_CHECK_ARG(nw >= 0 && dout > 0 && din > 0 && dout % 128 == 0 && din % 128 == 0,
                "xtb_fp8_block_scales: dout=%d, din=%d must be multiples of 128", dout, din);
  XTB_CHECK_ARG(nw <= 65535, "xtb_fp8_block_scales: nw=%lld exceeds the grid's z limit 65535", (long long)nw);
  XTB_ENSURE_CTX(w);
  if (nw == 0) return XTB_OK;
  dim3 grid(din / 128, dout / 128, (unsigned)nw);
  if (w_is_f32) fp8_block_kernel<float, false><<<grid, 256, 0, as_stream(stream)>>>(static_cast<const float*>(w), dout, din, scales, nullptr, nullptr);
  else fp8_block_kernel<__nv_bfloat16, false><<<grid, 256, 0, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(w), dout, din, scales, nullptr, nullptr);
  XTB_LAUNCH_OK();
  return XTB_OK;
}

extern "C" int xtb_fp8_block_cast(const void* w, int w_is_f32, int64_t nw, int dout, int din, const float* scales,
                                  void* q_e4m3, xtb_stream_t stream) {
  XTB_CHECK_ARG(w && scales && q_e4m3, "xtb_fp8_block_cast: null pointer");
  XTB_CHECK_ARG(nw >= 0 && dout > 0 && din > 0 && dout % 128 == 0 && din % 128 == 0,
                "xtb_fp8_block_cast: dout=%d, din=%d must be multiples of 128", dout, din);
  XTB_CHECK_ARG(nw <= 65535, "xtb_fp8_block_cast: nw=%lld exceeds the grid's z limit 65535", (long long)nw);
  XTB_ENSURE_CTX(w);
  if (nw == 0) return XTB_OK;
  dim3 grid(din / 128, dout / 128, (unsigned)nw);
  if (w_is_f32) fp8_block_kernel<float, true><<<grid, 256, 0, as_stream(stream)>>>(static_cast<const float*>(w), dout, din, nullptr, scales, static_cast<uint8_t*>(q_e4m3));
  else fp8_block_kernel<__nv_bfloat16, true><<<grid, 256, 0, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(w), dout, din, nullptr, scales, static_cast<uint8_t*>(q_e4m3));
  XTB_LAUNCH_OK();
  return XTB_OK;
}
