// Expert-parallel token exchange over NVLink peer memory with the split sizes kept ON THE DEVICE (SURVEY.md §8a row a10,
// §8e row 3).  The reference (xtuner/v1/module/dispatcher/torch_all2all.py:279-674) exchanges the per-expert counts with
// an all-to-all (:91-95), reads them back on the host to size a variable-split NCCL all-to-all (:102-114), and then
// re-sorts the received rows by local expert (repeat_interleave + permute, :485-495).  Here every rank leaves its rows —
// already sorted by GLOBAL expert id by the dispatch kernel — in a symmetric staging buffer behind a small header holding
// its per-expert counts; after ONE barrier each rank pulls exactly the row ranges of its local experts from every peer and
// writes them straight into expert-major order (the second permute of the reference disappears into the addressing).
// The way back is the mirrored pull.  No host read, no NCCL; both directions are one kernel each, and the same two
// kernels serve the backward pass (gradients travel the opposite way through the same addressing).
//
// Layout of a staging buffer (symmetric memory, same size on every rank):
//   [0, hdr)         int32 cnt[E]       rows this rank holds per GLOBAL expert (only read in the forward dispatch)
//   [hdr, ...)       rows               source-major: this rank's permuted tokens (sorted by global expert, M rows)
//                                       expert-major: this rank's local-expert rows (grouped by local expert, then source)
// cnt_all[s][e] (int32, world x E, local copy on every rank) is produced by the forward dispatch pull and drives every
// later kernel of the layer.
#include "common.cuh"

namespace xtb {

constexpr int kEpMaxExperts = 1024;
constexpr int kEpMaxWorld = 16;

__device__ __forceinline__ uint4 ep_ld_peer(const void* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}

// one warp copies one row of row_vec 16-byte vectors (batches of 8 loads in flight per lane)
__device__ __forceinline__ void ep_copy_row(const uint4* __restrict__ src, uint4* __restrict__ dst, int row_vec, int lane) {
  int v = lane;
  for (; v + 7 * 32 < row_vec; v += 8 * 32) {
    uint4 b[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) b[u] = ep_ld_peer(src + v + u * 32);
#pragma unroll
    for (int u = 0; u < 8; ++u) st_stream_16(dst + v + u * 32, b[u]);
  }
  for (; v < row_vec; v += 32) st_stream_16(dst + v, ep_ld_peer(src + v));
}

struct EpArgs {
  int me, world, E, E_loc;
  int row_vec;          // row bytes / 16
  long long hdr_vec;    // header bytes / 16
  int cap_rows;         // capacity (rows) of the expert-major buffer
  int m_rows;           // rows of the source-major buffer of THIS rank (T * K)
};

// ---- addressing tables (same code on the device — one thread per source / owner — and, for the CPU tests, on the host) ----
// to-experts: segment (j, s) = rows of local expert j that came from rank s; destination rows are ordered by (j, s)
__host__ __device__ inline void ep_src0_for_source(const int* cnt, const EpArgs& a, int s, int* src0) {
  int run = 0;
  for (int e = 0; e < a.me * a.E_loc; ++e) run += cnt[s * a.E + e];
  for (int j = 0; j < a.E_loc; ++j) {
    src0[j * a.world + s] = run;  // first row of expert me*E_loc + j inside rank s's source-major buffer
    run += cnt[s * a.E + a.me * a.E_loc + j];
  }
}
__host__ __device__ inline void ep_dst0_all(const int* cnt, const EpArgs& a, int* dst0) {
  const int nseg = a.E_loc * a.world;
  int run = 0;
  for (int seg = 0; seg < nseg; ++seg) {
    dst0[seg] = run;
    const int j = seg / a.world, s = seg - j * a.world;
    run += cnt[s * a.E + a.me * a.E_loc + j];
  }
  dst0[nseg] = run;
}
// to-sources: my rows of global expert e start at mine0[e] in my permuted order and at rem0[e] inside the owner's buffer
__host__ __device__ inline void ep_mine0_all(const int* cnt, const EpArgs& a, int* mine0) {
  int run = 0;
  for (int e = 0; e < a.E; ++e) {
    mine0[e] = run;
    run += cnt[a.me * a.E + e];
  }
  mine0[a.E] = run;
}
__host__ __device__ inline void ep_rem0_for_owner(const int* cnt, const EpArgs& a, int d, int* rem0) {
  int run = 0;
  for (int j = 0; j < a.E_loc; ++j) {
    const int e = d * a.E_loc + j;
    int before = 0, all = 0;
    for (int s = 0; s < a.world; ++s) {
      const int c = cnt[s * a.E + e];
      if (s < a.me) before += c;
      all += c;
    }
    rem0[e] = run + before;  // after every row of experts j' < j and the rows of expert e from ranks s' < me
    run += all;
  }
}
// largest index i in [0, n) with start[i] <= row (start is non-decreasing; empty ranges are skipped)
__host__ __device__ inline int ep_find(const int* start, int n, int row) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (start[mid] <= row) lo = mid; else hi = mid;
  }
  return lo;
}

// shared tables: s_cnt[s*E + e]; built once per CTA
__device__ __forceinline__ void ep_load_counts(int* s_cnt, const int32_t* cnt_all, const uint4* const* peer, const EpArgs& a) {
  const int n = a.world * a.E;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int s = i / a.E, e = i - s * a.E;
    s_cnt[i] = cnt_all ? cnt_all[i] : reinterpret_cast<const int32_t*>(peer[s])[e];
  }
  __syncthreads();
}

// ---- source-major (every rank's permuted rows) -> expert-major on the expert's owner ---------------------------------
// segment (j, s): rows of local expert j that came from rank s.  dst rows are ordered by (j, s); within a segment the
// source order is kept (= ascending flat token index on the source, as in the reference's stable sorts).
__global__ void __launch_bounds__(256) ep_pull_to_experts_kernel(const uint4* const* __restrict__ peer,
                                                                 const int32_t* __restrict__ cnt_all_in,
                                                                 int32_t* __restrict__ cnt_all_out, uint4* __restrict__ out,
                                                                 int64_t* __restrict__ tpe_local, int32_t* __restrict__ status,
                                                                 EpArgs a) {
  extern __shared__ int s_mem[];
  int* s_cnt = s_mem;                           // [world*E]
  int* s_src0 = s_cnt + a.world * a.E;          // [E_loc*world]  first source row of segment (j, s) in rank s's buffer
  int* s_dst0 = s_src0 + a.E_loc * a.world + 1; // [E_loc*world + 1]  first destination row of segment
  ep_load_counts(s_cnt, cnt_all_in, peer, a);
  const int nseg = a.E_loc * a.world;
  // source offsets: exclusive prefix of cnt[s][.] up to expert me*E_loc + j   (one thread per source rank)
  if (threadIdx.x < a.world) ep_src0_for_source(s_cnt, a, threadIdx.x, s_src0);
  if (threadIdx.x == 32) ep_dst0_all(s_cnt, a, s_dst0);
  __syncthreads();
  int total = s_dst0[nseg];
  if (blockIdx.x == 0) {
    if (cnt_all_out)
      for (int i = threadIdx.x; i < a.world * a.E; i += blockDim.x) cnt_all_out[i] = s_cnt[i];
    if (tpe_local)
      for (int j = threadIdx.x; j < a.E_loc; j += blockDim.x) {
        int n = 0;
        for (int s = 0; s < a.world; ++s) n += s_cnt[s * a.E + a.me * a.E_loc + j];
        tpe_local[j] = n;
      }
    if (threadIdx.x == 0 && status) {
      status[0] = total;                       // rows received
      if (total > a.cap_rows) status[1] = 1;   // capacity overflow (rows beyond the capacity are NOT transferred)
    }
  }
  if (total > a.cap_rows) total = a.cap_rows;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  for (int row = blockIdx.x * (blockDim.x >> 5) + warp; row < total; row += n_warps) {
    const int lo = ep_find(s_dst0, nseg, row);
    const int s = lo % a.world;
    const long long src_row = s_src0[lo] + (row - s_dst0[lo]);
    ep_copy_row(peer[s] + a.hdr_vec + src_row * a.row_vec, out + (long long)row * a.row_vec, a.row_vec, lane);
  }
}

// ---- expert-major (on the owners) -> source-major (back on the rank the tokens came from) ----------------------------
__global__ void __launch_bounds__(256) ep_pull_to_sources_kernel(const uint4* const* __restrict__ peer,
                                                                 const int32_t* __restrict__ cnt_all, uint4* __restrict__ out,
                                                                 EpArgs a) {
  extern __shared__ int s_mem[];
  int* s_cnt = s_mem;                       // [world*E]
  int* s_mine0 = s_cnt + a.world * a.E;     // [E+1]  first of MY rows of global expert e (my permuted order)
  int* s_rem0 = s_mine0 + a.E + 1;          // [E]    where my rows of expert e start inside the owner's expert-major buffer
  ep_load_counts(s_cnt, cnt_all, peer, a);
  if (threadIdx.x == 0) ep_mine0_all(s_cnt, a, s_mine0);
  if (threadIdx.x >= 32 && threadIdx.x < 32 + a.world) ep_rem0_for_owner(s_cnt, a, threadIdx.x - 32, s_rem0);
  __syncthreads();
  const int total = min(s_mine0[a.E], a.m_rows);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  for (int row = blockIdx.x * (blockDim.x >> 5) + warp; row < total; row += n_warps) {
    const int lo = ep_find(s_mine0, a.E, row);
    const int d = lo / a.E_loc;
    const long long src_row = s_rem0[lo] + (row - s_mine0[lo]);
    if (src_row < a.cap_rows)
      ep_copy_row(peer[d] + a.hdr_vec + src_row * a.row_vec, out + (long long)row * a.row_vec, a.row_vec, lane);
  }
}

// writes this rank's per-expert counts (int64 tokens_per_expert of the dispatch kernel) as the int32 header of a staging buffer
__global__ void ep_write_header_kernel(const int64_t* __restrict__ tpe, int32_t* __restrict__ hdr, int E) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x) hdr[e] = (int32_t)tpe[e];
}

static size_t ep_smem_bytes(int world, int E, int E_loc) {
  return sizeof(int) * ((size_t)world * E + 2 * ((size_t)E_loc * world + 1) + 2 * ((size_t)E + 1) + 8);
}

static int ep_check(const char* name, const void* peers, int rank, int world, int E, int64_t row_bytes, int64_t hdr_bytes) {
  XTB_CHECK_ARG(peers, "%s: null pointer", name);
  XTB_CHECK_ARG(world >= 1 && world <= kEpMaxWorld && rank >= 0 && rank < world, "%s: bad rank/world (%d/%d)", name, rank, world);
  XTB_CHECK_ARG(E > 0 && E <= kEpMaxExperts && E % world == 0, "%s: E=%d must be in 1..%d and divisible by the group size", name, E,
                kEpMaxExperts);
  XTB_CHECK_ARG(row_bytes > 0 && row_bytes % 16 == 0 && hdr_bytes >= (int64_t)E * 4 && hdr_bytes % 16 == 0,
                "%s: row_bytes=%lld / hdr_bytes=%lld must be multiples of 16 (header >= 4*E)", name, (long long)row_bytes,
                (long long)hdr_bytes);
  return XTB_OK;
}

}  // namespace xtb

using namespace xtb;

// Pure host code (no CUDA call; CPU-testable): the row addressing the two pull kernels use, from the same functions.
//   to_experts[r] = {source rank, row inside that rank's source-major buffer}   for r < rows received (2 ints per row)
//   to_sources[p] = {owner rank, row inside the owner's expert-major buffer}    for p < this rank's rows (2 ints per row)
extern "C" int xtb_ep_plan(const int32_t* cnt_all, int rank, int world, int E, int32_t* to_experts, int64_t max_rows_e,
                           int32_t* to_sources, int64_t max_rows_s, int64_t* n_rows_e, int64_t* n_rows_s) {
  XTB_CHECK_ARG(cnt_all && to_experts && to_sources && n_rows_e && n_rows_s, "xtb_ep_plan: null pointer");
  XTB_CHECK_ARG(world >= 1 && world <= kEpMaxWorld && rank >= 0 && rank < world && E > 0 && E <= kEpMaxExperts && E % world == 0,
                "xtb_ep_plan: bad rank/world/E");
  EpArgs a{};
  a.me = rank; a.world = world; a.E = E; a.E_loc = E / world;
  const int nseg = a.E_loc * world;
  int* src0 = new int[nseg + 1];
  int* dst0 = new int[nseg + 1];
  int* mine0 = new int[E + 1];
  int* rem0 = new int[E];
  for (int s = 0; s < world; ++s) ep_src0_for_source(cnt_all, a, s, src0);
  ep_dst0_all(cnt_all, a, dst0);
  ep_mine0_all(cnt_all, a, mine0);
  for (int d = 0; d < world; ++d) ep_rem0_for_owner(cnt_all, a, d, rem0);
  *n_rows_e = dst0[nseg];
  *n_rows_s = mine0[E];
  int rc = XTB_OK;
  if (dst0[nseg] > max_rows_e || mine0[E] > max_rows_s) {
    rc = fail(XTB_ERR_INVALID, "xtb_ep_plan: output too small (%d / %d rows)", dst0[nseg], mine0[E]);
  } else {
    for (int row = 0; row < dst0[nseg]; ++row) {
      const int seg = ep_find(dst0, nseg, row);
      to_experts[2 * row] = seg % world;
      to_experts[2 * row + 1] = src0[seg] + (row - dst0[seg]);
    }
    for (int row = 0; row < mine0[E]; ++row) {
      const int e = ep_find(mine0, E, row);
      to_sources[2 * row] = e / a.E_loc;
      to_sources[2 * row + 1] = rem0[e] + (row - mine0[e]);
    }
  }
  delete[] src0; delete[] dst0; delete[] mine0; delete[] rem0;
  return rc;
}

extern "C" int xtb_ep_write_header(const int64_t* tokens_per_expert, void* header, int E, xtb_stream_t stream) {
  XTB_CHECK_ARG(tokens_per_expert && header, "xtb_ep_write_header: null pointer");
  XTB_CHECK_ARG(E > 0, "xtb_ep_write_header: bad E=%d", E);
  XTB_ENSURE_CTX(header);
  XTB_LAUNCH(ep_write_header_kernel, dim3(1), dim3(256), 0, as_stream(stream), false, tokens_per_expert,
             static_cast<int32_t*>(header), E);
  return XTB_OK;
}

extern "C" int xtb_ep_pull_to_experts(void* const* peer_ptrs_dev, const int32_t* cnt_all_in, int32_t* cnt_all_out, void* out,
                                      int64_t* tokens_per_expert_local, int32_t* status, int rank, int world, int E,
                                      int64_t row_bytes, int64_t hdr_bytes, int64_t cap_rows, xtb_stream_t stream) {
  XTB_CHECK_ARG(peer_ptrs_dev && out, "xtb_ep_pull_to_experts: null pointer");
  int rc = ep_check("xtb_ep_pull_to_experts", peer_ptrs_dev, rank, world, E, row_bytes, hdr_bytes);
  if (rc) return rc;
  XTB_CHECK_ARG(out && cap_rows >= 0 && cap_rows < (1ll << 31), "xtb_ep_pull_to_experts: bad output / capacity");
  XTB_CHECK_ARG(cnt_all_in || cnt_all_out, "xtb_ep_pull_to_experts: either cnt_all_in (reuse) or cnt_all_out (first use) is needed");
  XTB_ENSURE_CTX(out);
  EpArgs a;
  a.me = rank; a.world = world; a.E = E; a.E_loc = E / world;
  a.row_vec = (int)(row_bytes / 16); a.hdr_vec = hdr_bytes / 16; a.cap_rows = (int)cap_rows; a.m_rows = 0;
  const size_t smem = ep_smem_bytes(world, E, a.E_loc);
  XTB_CHECK_ARG(smem <= 96 * 1024, "xtb_ep_pull_to_experts: count tables need %zu bytes of shared memory", smem);
  XTB_LAUNCH(ep_pull_to_experts_kernel, dim3(sm_count() * 2), dim3(256), smem, as_stream(stream), false,
             reinterpret_cast<const uint4* const*>(peer_ptrs_dev), cnt_all_in, cnt_all_out, static_cast<uint4*>(out),
             tokens_per_expert_local, status, a);
  return XTB_OK;
}

extern "C" int xtb_ep_pull_to_sources(void* const* peer_ptrs_dev, const int32_t* cnt_all, void* out, int rank, int world, int E,
                                      int64_t row_bytes, int64_t hdr_bytes, int64_t cap_rows, int64_t m_rows,
                                      xtb_stream_t stream) {
  XTB_CHECK_ARG(peer_ptrs_dev && cnt_all && out, "xtb_ep_pull_to_sources: null pointer");
  int rc = ep_check("xtb_ep_pull_to_sources", peer_ptrs_dev, rank, world, E, row_bytes, hdr_bytes);
  if (rc) return rc;
  XTB_CHECK_ARG(cnt_all && out && m_rows >= 0 && m_rows < (1ll << 31) && cap_rows >= 0 && cap_rows < (1ll << 31),
                "xtb_ep_pull_to_sources: bad arguments");
  XTB_ENSURE_CTX(out);
  if (m_rows == 0) return XTB_OK;
  EpArgs a;
  a.me = rank; a.world = world; a.E = E; a.E_loc = E / world;
  a.row_vec = (int)(row_bytes / 16); a.hdr_vec = hdr_bytes / 16; a.cap_rows = (int)cap_rows; a.m_rows = (int)m_rows;
  const size_t smem = ep_smem_bytes(world, E, a.E_loc);
  XTB_CHECK_ARG(smem <= 96 * 1024, "xtb_ep_pull_to_sources: count tables need %zu bytes of shared memory", smem);
  XTB_LAUNCH(ep_pull_to_sources_kernel, dim3(sm_count() * 2), dim3(256), smem, as_stream(stream), false,
             reinterpret_cast<const uint4* const*>(peer_ptrs_dev), cnt_all, static_cast<uint4*>(out), a);
  return XTB_OK;
}
