// bf16 GEMM for sm_90a on the Hopper warpgroup tensor cores (wgmma), optionally fused with a tensor-parallel
// collective over NVLink peer memory.
//
//   D[M,N] (+)= op(A)[M,K] · op(B)[K,N]           fp32 accumulation in registers
//
// One persistent CTA per SM, 384 threads: a TMA producer warpgroup and two consumer warpgroups (see gemm_bf16_kernel).
//
// Operand majors are template parameters so forward (A K-major, B K-major), dgrad (B MN-major) and wgrad
// (A and B MN-major) all run without transposition copies — only the TMA boxes and wgmma descriptors differ.
//
// Fused collective modes (no NCCL call on these paths — reference call sites layers_utils.py:56,
// layers.py:1035-1038, mappings.py:125-157, 347-352):
//   MODE 1  all-gather → GEMM : `comm_sms` CTAs push this rank's A shard into every peer's symmetric
//           buffer (st.global over NVLink, 16 B vectors) and publish per-(source,row-block) flags with
//           st.release.sys; GEMM CTAs walk row-chunks in arrival order and their TMA producer acquires
//           the flag (ld.acquire.sys + fence.proxy.async) before loading tiles of that chunk.
//   MODE 2  GEMM → reduce-scatter : the epilogue stores each partial tile straight into the owner rank's
//           staging slot (peer st.global), then bumps the owner's per-(source,row-block) counter with
//           red.release.sys; after its last tile every CTA turns into a reducer that acquires the 8
//           counters of a row-block, sums the partials in fp32 and writes the bf16 result.
//   Payload regions are double-buffered by call parity and flags are monotonic, so consecutive calls need
//   no barrier (DESIGN.md, "symmetric memory protocol").
//
// NVLS modes (NVSwitch multicast / in-switch reduction over a VMM symmetric region; without a multicast mapping,
// `mc_base == nullptr`, the same kernels use unicast peer stores / loads with the identical flag protocol):
//   MODE 5  all-gather → GEMM : `comm_sms` CTAs stream this rank's shard to the multicast address with `multimem.st`
//           (the switch replicates it into every rank's buffer) and release per-(source, 128-row block, quarter) epoch
//           flags on every peer; GEMM CTAs start on the own chunk (read in place) and then walk the remote chunks in the
//           order they were pushed, the TMA producer acquiring the four quarter flags of a block before loading it.
//   MODE 6  GEMM → reduce-scatter : every rank walks the row blocks in the same global order and stores its partial
//           tiles (bf16, or fp32 for the fp32 wire format) into its own buffer; the CTA that completes a 128-row block
//           releases one flag at the block's owner.  The owner pulls the sum of all ranks' partials with
//           `multimem.ld_reduce` (fp32 accumulation in the switch); 16-row reduction items are claimed dynamically by the
//           comm CTAs while the GEMM runs, and by the GEMM CTAs after their tiles when `gemm_join` is set.
#include <cuda.h>

#include "common.cuh"
#include "kernels.h"
#include "sm90_ptx.cuh"

namespace nxd {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 256;
constexpr int BLOCK_K = 64;           // 64 bf16 = 128 bytes = one swizzle row
constexpr int WG_K = 16;              // K of one bf16 wgmma (32 for e4m3: the same 32 bytes)
constexpr int kStages = 4;
constexpr int kABytes = BLOCK_M * BLOCK_K * 2;   // 16 KB
constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;   // 32 KB
constexpr int kStageBytes = kABytes + kBBytes;   // 48 KB
constexpr int kThreads = 384;                    // producer warpgroup + 2 consumer warpgroups
constexpr int kEpiBoxBytes = 64 * 128;           // TMA epilogue box: 64 rows x 128 bytes (64 bf16 / 32 fp32 columns)
constexpr int kEpiBytes = 2 * 2 * kEpiBoxBytes;  // two boxes per consumer warpgroup: 32 KB
constexpr int kSmemBytes = kStages * kStageBytes + kEpiBytes + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int kMaxRowBlocks = 64;   // flag index = source_rank * kMaxRowBlocks + row_block (shape independent)

struct CommDev {
  int rank, world;
  const int64_t* peer_bufs;
  const int64_t* peer_flags;
  long buf_offset;
  int flag_offset;
  uint32_t epoch;
  int comm_sms;
  int rows_per_rank;      // M / world
  uint32_t rs_targets[kMaxRowBlocks];   // MODE 2: cumulative n-tile count expected per row-block counter
  const void* a_local;    // MODE 1: this rank's [rows_per_rank, K] shard
  void* rs_out;           // MODE 2: reduced [rows_per_rank, N] output
  // grouped (MoE blockwise) modes.  MODE 3: every `grp_block_rows`-row block of A belongs to one expert whose weight
  // matrix is `grp_b_rows` rows further down the stacked 2-D B tensor.  MODE 4 (wgrad): one output matrix per expert,
  // reduced over that expert's row blocks [seg_first_block[e], seg_first_block[e+1]).
  const float* scale_a;   // FP8: per-row (token) scales [M]
  const float* scale_b;   // FP8: per-column (output channel) scales [N]
  const int* block_expert;
  const int* seg_first_block;
  int grp_block_rows, grp_b_rows, num_groups;
  long out_group_stride;
  // NVLS modes 5 / 6 (peer_bufs = every rank's region base, flag_offset_bytes = flags inside the region)
  uint8_t* mc_base;
  uint8_t* local_base;
  long flag_offset_bytes;
  uint32_t* tile_done;     // MODE 6: per-128-row-block completed n-tile counters (re-armed by the completing CTA)
  uint32_t* claim;         // MODE 6: reducer claim counter, monotonic across calls
  uint32_t claim_base;
  int gemm_join;
};

constexpr int kNvlsMaxRowBlocks = 256;   // 128-row blocks per rank in the NVLS flag layout
constexpr int kAgParts = 4;              // MODE 5 flag granularity: quarter of a 128-row block
constexpr int kRsRowsPerItem = 16;       // MODE 6 reduction item: 16 full rows

NXD_DEVICE uint32_t atom_add_acqrel_gpu(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
NXD_DEVICE void multimem_st_v4(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
               ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
NXD_DEVICE uint4 multimem_ld_reduce_bf16x2(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
NXD_DEVICE uint4 multimem_ld_reduce_f32(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
NXD_DEVICE uint4 ld_relaxed_sys_v4(const void* p) {      // peer payload published through a flag: never the nc path
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

// MODE 4 tile → (expert, m_blk, n_blk, first k-block, number of k-blocks)
struct GroupTile { int e, m_blk, n_blk, kb0, nkb; };
NXD_DEVICE GroupTile group_tile(int tile, int tiles_m, int tiles_n, const CommDev& c) {
  GroupTile g;
  const int per = tiles_m * tiles_n;
  g.e = tile / per;
  const int in = tile - g.e * per;
  g.m_blk = in % tiles_m;
  g.n_blk = in / tiles_m;
  const int b0 = c.seg_first_block[g.e], b1 = c.seg_first_block[g.e + 1];
  const int per_blk = c.grp_block_rows / 64;
  g.kb0 = b0 * per_blk;
  g.nkb = (b1 - b0) * per_blk;
  return g;
}

// tile index → (m_blk, n_blk).  `chunk_order` visits row-chunks (one per rank) in communication order.
template <int MODE>
NXD_DEVICE void tile_coords(int tile, int tiles_m, int tiles_n, const CommDev& c, int& m_blk, int& n_blk) {
  if constexpr (MODE == 5) {
    // own chunk first (no wait), then the remote chunks block-major in the order their pushes were issued
    const int mbr = c.rows_per_rank / BLOCK_M;
    const int seq = tile / tiles_n;
    n_blk = tile - seq * tiles_n;
    if (seq < mbr) { m_blk = c.rank * mbr + seq; return; }
    const int s2 = seq - mbr;
    const int mb = s2 / (c.world - 1), s = s2 - mb * (c.world - 1);
    m_blk = ((c.rank + 1 + s) % c.world) * mbr + mb;
  } else if constexpr (MODE == 6) {
    // the same order on every rank: block b of every owner completes everywhere at about the same time
    const int mbr = c.rows_per_rank / BLOCK_M;
    const int seq = tile / tiles_n;
    n_blk = tile - seq * tiles_n;
    const int mb = seq / c.world, chunk = seq - mb * c.world;
    m_blk = chunk * mbr + mb;
  } else if constexpr (MODE == 0 || MODE == 3) {
    constexpr int GROUP = 8;  // rasterise 8 M-blocks at a time so B tiles are re-used from L2
    const int per_group = GROUP * tiles_n;
    const int g = tile / per_group;
    const int first_m = g * GROUP;
    const int gsz = min(GROUP, tiles_m - first_m);
    const int in = tile - g * per_group;
    m_blk = first_m + in % gsz;
    n_blk = in / gsz;
  } else {
    const int mb_per_rank = c.rows_per_rank / BLOCK_M;
    const int per_chunk = mb_per_rank * tiles_n;
    const int step = tile / per_chunk;           // 0 .. world-1
    const int in = tile - step * per_chunk;
    int chunk;
    if constexpr (MODE == 1) chunk = (c.rank - step + c.world) % c.world;        // own, then rank-1, rank-2, …
    else chunk = (c.rank + 1 + step) % c.world;                                  // rank+1, …, own last
    m_blk = chunk * mb_per_rank + in % mb_per_rank;
    n_blk = in / mb_per_rank;
  }
}

// FP8: operands are e4m3 bytes (both K-major), one k-block is 128 elements (= the same 128-byte swizzle row), the wgmma is
// m64n256k32.e4m3 and the epilogue applies the outer product of per-row / per-column scales.
//
// Epilogue store of one consumer thread's accumulator fragment (wgmma m64n256 layout: register 4j + {0,1} holds row
// lane/4, columns 8j + 2(lane%4) + {0,1}; register 4j + {2,3} the same columns eight rows further down).
template <int MODE, typename OutT, bool FP8>
NXD_DEVICE void store_tile(const float (&acc)[128], OutT* orow0, OutT* orow1, int row0, int n0, int M, int N, int accumulate,
                           const CommDev& comm) {
  const int lane = threadIdx.x & 31;
  const bool ok0 = row0 < M, ok1 = row0 + 8 < M;
  float sa0 = 1.f, sa1 = 1.f;
  if constexpr (FP8) { sa0 = comm.scale_a[ok0 ? row0 : 0]; sa1 = comm.scale_a[ok1 ? row0 + 8 : 0]; }
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = n0 + 8 * j + 2 * (lane & 3);
    if (col >= N) continue;                          // N is even: col < N → col + 1 < N
    float v0 = acc[4 * j], v1 = acc[4 * j + 1], v2 = acc[4 * j + 2], v3 = acc[4 * j + 3];
    if constexpr (FP8) {
      const float sb0 = comm.scale_b[col], sb1 = comm.scale_b[col + 1];
      v0 *= sa0 * sb0; v1 *= sa0 * sb1; v2 *= sa1 * sb0; v3 *= sa1 * sb1;
    }
    if constexpr (sizeof(OutT) == 2) {
      __nv_bfloat162* p0 = (__nv_bfloat162*)(orow0 + col);
      __nv_bfloat162* p1 = (__nv_bfloat162*)(orow1 + col);
      if (accumulate && MODE != 2) {
        if (ok0) { const float2 o = __bfloat1622float2(*p0); v0 += o.x; v1 += o.y; }
        if (ok1) { const float2 o = __bfloat1622float2(*p1); v2 += o.x; v3 += o.y; }
      }
      if (ok0) *p0 = __floats2bfloat162_rn(v0, v1);
      if (ok1) *p1 = __floats2bfloat162_rn(v2, v3);
    } else {
      float2* p0 = (float2*)(orow0 + col);
      float2* p1 = (float2*)(orow1 + col);
      if (accumulate) {
        if (ok0) { const float2 o = *p0; v0 += o.x; v1 += o.y; }
        if (ok1) { const float2 o = *p1; v2 += o.x; v3 += o.y; }
      }
      if (ok0) *p0 = make_float2(v0, v1);
      if (ok1) *p1 = make_float2(v2, v3);
    }
  }
}

// TMA epilogue of one consumer warpgroup's 64 x 256 slice (rows row_base.., columns n0..): it leaves in boxes of 64 rows x
// 128 bytes, each written into one of the warpgroup's two 128B-swizzled staging buffers and sent by one thread as a bulk
// tensor store, or, to accumulate into fp32, a bulk tensor reduce-add performed at L2.  The tensor map clips rows >= M and
// columns >= N.  Per element the arithmetic is the register epilogue's: the fp32 accumulator (times the fp8 scales), rounded
// once to bf16 for a bf16 out, or added once in fp32 to the old value (which, unlike the register path's flush-to-zero
// FADD, keeps subnormal operands and sums: DESIGN.md §2).
//
// Ordering: every thread fences its shared-memory writes for the async proxy; before the warpgroup barrier the leader waits
// until its previous box has been read out of shared memory, so after the barrier the other buffer is free to rewrite.
template <typename OutT, bool FP8>
NXD_DEVICE void store_tile_tma(const float (&acc)[128], const CUtensorMap* tma_out, uint32_t stage, int row_base, int n0,
                               int M, int N, bool reduce_add, const CommDev& comm, uint32_t bar_id, bool leader) {
  constexpr int kCols = 128 / sizeof(OutT);        // columns of a box
  constexpr int kJ = kCols / 8;                    // accumulator column groups (8 columns each) of a box
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const int r = wq * 16 + (lane >> 2);             // box rows r and r + 8; both have r % 8 = lane / 4 → same swizzle
  const int sw = lane >> 2;
  float sa0 = 1.f, sa1 = 1.f;
  if constexpr (FP8) {
    const int row0 = row_base + r;
    sa0 = comm.scale_a[row0 < M ? row0 : 0]; sa1 = comm.scale_a[row0 + 8 < M ? row0 + 8 : 0];
  }
#pragma unroll
  for (int box = 0; box < BLOCK_N / kCols; ++box) {
    const uint32_t buf = stage + (box & 1) * kEpiBoxBytes;
#pragma unroll
    for (int jj = 0; jj < kJ; ++jj) {
      const int j = box * kJ + jj;
      float v0 = acc[4 * j], v1 = acc[4 * j + 1], v2 = acc[4 * j + 2], v3 = acc[4 * j + 3];
      if constexpr (FP8) {
        const int col = n0 + 8 * j + 2 * (lane & 3);
        const float sb0 = col < N ? comm.scale_b[col] : 0.f, sb1 = col < N ? comm.scale_b[col + 1] : 0.f;
        v0 *= sa0 * sb0; v1 *= sa0 * sb1; v2 *= sa1 * sb0; v3 *= sa1 * sb1;
      }
      // 16-byte chunk c of row r sits at chunk c ^ (r % 8) (SWIZZLE_128B)
      if constexpr (sizeof(OutT) == 2) {
        const int off = ((jj ^ sw) << 4) + 4 * (lane & 3);
        const __nv_bfloat162 h0 = __floats2bfloat162_rn(v0, v1), h1 = __floats2bfloat162_rn(v2, v3);
        st_shared_b32(buf + r * 128 + off, *(const uint32_t*)&h0);
        st_shared_b32(buf + (r + 8) * 128 + off, *(const uint32_t*)&h1);
      } else {
        const int off = (((2 * jj + ((lane & 3) >> 1)) ^ sw) << 4) + 8 * (lane & 1);
        st_shared_v2f32(buf + r * 128 + off, v0, v1);
        st_shared_v2f32(buf + (r + 8) * 128 + off, v2, v3);
      }
    }
    fence_proxy_async_smem();
    if (leader) bulk_wait_group_read<0>();
    named_barrier_sync(bar_id, 128);
    if (leader) {
      if (reduce_add) tma_reduce_add_2d(tma_out, buf, n0 + box * kCols, row_base);
      else tma_store_2d(tma_out, buf, n0 + box * kCols, row_base);
      bulk_commit_group();
    }
  }
}

// Structure (one persistent CTA per SM, 384 threads):
//   warpgroup 0     TMA producer : one thread fills a 4-stage ring of 128B-swizzled [128 x 64] A / [256 x 64] B tiles
//   warpgroups 1-2  consumers    : consumer c owns rows 64c..64c+63 of the 128 x 256 tile, issues wgmma m64n256k16 from
//                                  shared memory into a register accumulator (one wgmma group in flight, which releases
//                                  the previous stage), then stores the tile: through shared memory by TMA when
//                                  `tma_epi` is set (store_tile_tma, MODE 0 / 3), else straight from registers.
template <bool A_KMAJOR, bool B_KMAJOR, int MODE, typename OutT, bool FP8 = false>
__global__ void __launch_bounds__(kThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                 const __grid_constant__ CUtensorMap tma_a_local, const __grid_constant__ CUtensorMap tma_out,
                 OutT* __restrict__ out, int M, int N, int K, int accumulate, int tma_epi, CommDev comm) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B needs 1 KB alignment
  uint8_t* epi_stage = smem + kStages * kStageBytes;                               // [2 warpgroups][2 boxes] of 8 KB
  uint64_t* bars = (uint64_t*)(epi_stage + kEpiBytes);
  // [0,kStages) full, [kStages,2kStages) empty
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + kStages);
  const uint32_t smem_base = smem_u32(smem);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + BLOCK_M - 1) / BLOCK_M, tiles_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = (MODE == 4 ? comm.num_groups : 1) * tiles_m * tiles_n;
  constexpr int KB_ELEMS = FP8 ? 2 * BLOCK_K : BLOCK_K;
  const int num_kb_all = (K + KB_ELEMS - 1) / KB_ELEMS;

  // ---- one-time setup ------------------------------------------------------------
  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tma_a);
    prefetch_tmap(&tma_b);
    for (int i = 0; i < kStages; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 2); }
    fence_barrier_init();
  }
  __syncthreads();

  // ---- role split ------------------------------------------------------------------
  int gemm_cta = blockIdx.x, gemm_ctas = gridDim.x;
  bool is_comm_cta = false;
  if constexpr (MODE == 1 || MODE == 5 || MODE == 6) {
    is_comm_cta = (int)blockIdx.x < comm.comm_sms;
    gemm_cta = blockIdx.x - comm.comm_sms;
    gemm_ctas = gridDim.x - comm.comm_sms;
  }

  if constexpr (MODE == 1) {
    if (is_comm_cta) {
      // ===== all-gather pusher: (destination, row-block) items, destinations in rotated order =====
      const int mb_per_rank = comm.rows_per_rank / BLOCK_M;
      const int items = comm.world * mb_per_rank;
      const size_t row_bytes = (size_t)K * 2;
      const size_t blk_bytes = (size_t)BLOCK_M * row_bytes;
      for (int it = blockIdx.x; it < items; it += comm.comm_sms) {
        const int step = it / mb_per_rank, mb = it % mb_per_rank;
        const int dst = (comm.rank + step) % comm.world;          // step 0 = local copy
        const uint8_t* src = (const uint8_t*)comm.a_local + (size_t)mb * blk_bytes;
        uint8_t* dbase = (uint8_t*)comm.peer_bufs[dst] + comm.buf_offset +
                         ((size_t)comm.rank * comm.rows_per_rank + (size_t)mb * BLOCK_M) * row_bytes;
        const size_t nvec = blk_bytes / 16;
        const uint4* s4 = (const uint4*)src;
        uint4* d4 = (uint4*)dbase;
        size_t i = threadIdx.x;
        // 4 independent 16-byte loads in flight per thread
        for (; i + 3 * kThreads < nvec; i += 4 * kThreads) {
          const uint4 v0 = __ldg(s4 + i), v1 = __ldg(s4 + i + kThreads), v2 = __ldg(s4 + i + 2 * kThreads),
                      v3 = __ldg(s4 + i + 3 * kThreads);
          d4[i] = v0; d4[i + kThreads] = v1; d4[i + 2 * kThreads] = v2; d4[i + 3 * kThreads] = v3;
        }
        for (; i < nvec; i += kThreads) d4[i] = __ldg(s4 + i);
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
          uint32_t* f = (uint32_t*)comm.peer_flags[dst] + comm.flag_offset + comm.rank * kMaxRowBlocks + mb;
          st_release_sys(f, comm.epoch);
        }
      }
    }
  }

  if constexpr (MODE == 5) {
    if (is_comm_cta) {
      // ===== NVLS all-gather pusher: (128-row block, quarter) items of this rank's shard =====
      constexpr int U = 8;
      constexpr int rows_part = BLOCK_M / kAgParts;
      const int items = (comm.rows_per_rank / BLOCK_M) * kAgParts;
      const size_t nvec = (size_t)rows_part * K / 8;          // 16-byte vectors per item
      for (int it = blockIdx.x; it < items; it += comm.comm_sms) {
        const int mb = it / kAgParts, part = it - mb * kAgParts;
        const size_t row0 = (size_t)mb * BLOCK_M + part * rows_part;
        const uint4* src = (const uint4*)((const uint8_t*)comm.a_local + row0 * K * 2);
        const size_t dst_off = (size_t)comm.buf_offset + ((size_t)comm.rank * comm.rows_per_rank + row0) * K * 2;
        for (size_t base = threadIdx.x; base < nvec; base += (size_t)U * kThreads) {
          uint4 v[U];
#pragma unroll
          for (int u = 0; u < U; ++u) { const size_t i = base + (size_t)u * kThreads; if (i < nvec) v[u] = __ldg(src + i); }
          if (comm.mc_base != nullptr) {
            uint4* dst = (uint4*)(comm.mc_base + dst_off);
#pragma unroll
            for (int u = 0; u < U; ++u) { const size_t i = base + (size_t)u * kThreads; if (i < nvec) multimem_st_v4(dst + i, v[u]); }
          } else {
            for (int p = 0; p < comm.world; ++p) {
              uint4* dst = (uint4*)((uint8_t*)comm.peer_bufs[p] + dst_off);
#pragma unroll
              for (int u = 0; u < U; ++u) { const size_t i = base + (size_t)u * kThreads; if (i < nvec) dst[i] = v[u]; }
            }
          }
        }
        __threadfence_system();
        __syncthreads();
        if ((int)threadIdx.x < comm.world && (int)threadIdx.x != comm.rank) {
          uint32_t* f = (uint32_t*)((uint8_t*)comm.peer_bufs[threadIdx.x] + comm.flag_offset_bytes) +
                        ((size_t)comm.rank * kNvlsMaxRowBlocks + mb) * kAgParts + part;
          st_release_sys(f, comm.epoch);
        }
      }
    }
  }

  if (!is_comm_cta) {
    if (warp < 4) {
      // ===== TMA producer =====
      if (warp == 0 && lane == 0) {
        int stage = 0; uint32_t phase = 0;
        for (int tile = gemm_cta; tile < num_tiles; tile += gemm_ctas) {
          int m_blk, n_blk, kb0 = 0, num_kb = num_kb_all, b_off = 0;
          if constexpr (MODE == 4) {
            const GroupTile g = group_tile(tile, tiles_m, tiles_n, comm);
            m_blk = g.m_blk; n_blk = g.n_blk; kb0 = g.kb0; num_kb = g.nkb;
          } else {
            tile_coords<MODE>(tile, tiles_m, tiles_n, comm, m_blk, n_blk);
          }
          if constexpr (MODE == 3) b_off = comm.block_expert[(m_blk * BLOCK_M) / comm.grp_block_rows] * comm.grp_b_rows;
          if constexpr (MODE == 1) {
            const int mb_per_rank = comm.rows_per_rank / BLOCK_M;
            const uint32_t* f = (const uint32_t*)comm.peer_flags[comm.rank] + comm.flag_offset +
                                (m_blk / mb_per_rank) * kMaxRowBlocks + (m_blk % mb_per_rank);
            wait_flag_ge(f, comm.epoch);
            fence_proxy_async_global();   // peer generic-proxy writes → visible to our TMA reads
          }
          const int m0 = m_blk * BLOCK_M, n0 = n_blk * BLOCK_N;
          const CUtensorMap* map_a = &tma_a;
          int a_row = m0;
          if constexpr (MODE == 5) {
            const int mbr = comm.rows_per_rank / BLOCK_M, src_rank = m_blk / mbr;
            if (src_rank == comm.rank) {                      // own shard, read in place
              map_a = &tma_a_local;
              a_row = m0 - src_rank * comm.rows_per_rank;
            } else {
              const uint32_t* f = (const uint32_t*)(comm.local_base + comm.flag_offset_bytes) +
                                  ((size_t)src_rank * kNvlsMaxRowBlocks + (m_blk - src_rank * mbr)) * kAgParts;
              for (int p = 0; p < kAgParts; ++p) wait_flag_ge(f + p, comm.epoch);
              fence_proxy_async_global();
            }
          }
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(bar_empty + 8 * stage, phase ^ 1);
            const uint32_t full = bar_full + 8 * stage;
            mbar_expect_tx(full, kStageBytes);
            const uint32_t sa = smem_base + stage * kStageBytes, sb = sa + kABytes;
            const int k0 = (kb0 + kb) * KB_ELEMS;
            if constexpr (A_KMAJOR) {
              tma_load_2d(sa, map_a, full, k0, a_row);                        // box {64 k, 128 m}
            } else {
#pragma unroll
              for (int j = 0; j < BLOCK_M / 64; ++j) tma_load_2d(sa + j * 8192, &tma_a, full, m0 + j * 64, k0);  // box {64 m, 64 k}
            }
            if constexpr (B_KMAJOR) {
              tma_load_2d(sb, &tma_b, full, k0, b_off + n0);                  // box {64 k, 256 n}
            } else {
#pragma unroll
              for (int j = 0; j < BLOCK_N / 64; ++j) tma_load_2d(sb + j * 8192, &tma_b, full, n0 + j * 64, b_off + k0);  // box {64 n, 64 k}
            }
            if (++stage == kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
      __syncwarp();
    } else {
      // ===== consumers: wgmma + epilogue =====
      const int cw = (threadIdx.x - 128) >> 7;            // consumer warpgroup 0 / 1 → rows 64*cw ..
      const int wq = warp & 3;                            // warp inside the warpgroup → 16-row slice
      int stage = 0; uint32_t phase = 0;
      float acc[128];
      for (int tile = gemm_cta; tile < num_tiles; tile += gemm_ctas) {
        int m_blk, n_blk, num_kb = num_kb_all;
        OutT* out_base = out;
        if constexpr (MODE == 4) {
          const GroupTile g = group_tile(tile, tiles_m, tiles_n, comm);
          m_blk = g.m_blk; n_blk = g.n_blk; num_kb = g.nkb;   // expert without tokens: zero accumulator is stored
          out_base = out + (long)g.e * comm.out_group_stride;
        } else {
          tile_coords<MODE>(tile, tiles_m, tiles_n, comm, m_blk, n_blk);
        }
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
        int prev_stage = -1;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bar_full + 8 * stage, phase);
          const uint32_t sa = smem_base + stage * kStageBytes + cw * 8192, sb = smem_base + stage * kStageBytes + kABytes;
          fence_acc(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BLOCK_K / WG_K; ++k) {
            // K-major: advance 32 B inside the 128 B swizzle row; MN-major: 16 k-rows × 128 B = 2 KB
            const uint64_t da = A_KMAJOR ? make_smem_desc(sa + k * 32, 16, 1024) : make_smem_desc(sa + k * 2048, 8192, 1024);
            const uint64_t db = B_KMAJOR ? make_smem_desc(sb + k * 32, 16, 1024) : make_smem_desc(sb + k * 2048, 8192, 1024);
            if constexpr (FP8) wgmma_m64n256k32_e4m3(acc, da, db, 1u);
            else wgmma_m64n256k16_bf16<A_KMAJOR ? 0 : 1, B_KMAJOR ? 0 : 1>(acc, da, db, 1u);
          }
          wgmma_commit();
          fence_acc(acc);
          wgmma_wait<1>();                                  // the previous k-block's MMAs have retired
          if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_empty + 8 * prev_stage);
          prev_stage = stage;
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_empty + 8 * prev_stage);

        const int n0 = n_blk * BLOCK_N;
        if constexpr (MODE == 0 || MODE == 3) {
          if (tma_epi) {
            // named barrier 2 + cw: 0 is __syncthreads, 1 the MODE 2 / 6 publish barrier
            store_tile_tma<OutT, FP8>(acc, &tma_out, smem_u32(epi_stage) + cw * 2 * kEpiBoxBytes, m_blk * BLOCK_M + cw * 64,
                                      n0, M, N, accumulate != 0, comm, 2 + cw, (threadIdx.x & 127) == 0);
            continue;
          }
        }
        const int row0 = m_blk * BLOCK_M + cw * 64 + wq * 16 + (lane >> 2);
        OutT *orow0, *orow1;
        if constexpr (MODE == 2) {
          // partial tile goes to the owner's staging slot [src = my rank][row in chunk][N]
          const int owner = (m_blk * BLOCK_M) / comm.rows_per_rank;
          const int lrow = row0 - owner * comm.rows_per_rank;
          OutT* base = (OutT*)((uint8_t*)comm.peer_bufs[owner] + comm.buf_offset) + (size_t)comm.rank * comm.rows_per_rank * N;
          orow0 = base + (size_t)lrow * N;
          orow1 = base + (size_t)(lrow + 8) * N;
        } else if constexpr (MODE == 6) {
          OutT* base = (OutT*)(comm.local_base + comm.buf_offset);     // this rank's partial of every row
          orow0 = base + (size_t)row0 * N;
          orow1 = base + (size_t)(row0 + 8) * N;
        } else {
          orow0 = out_base + (size_t)row0 * N;
          orow1 = out_base + (size_t)(row0 + 8) * N;
        }
        store_tile<MODE, OutT, FP8>(acc, orow0, orow1, row0, n0, M, N, accumulate, comm);
        if constexpr (MODE == 2) {
          // publish: all 256 consumer threads' peer stores, then one counter bump on the owner
          __threadfence_system();
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (threadIdx.x == 128) {
            const int owner = (m_blk * BLOCK_M) / comm.rows_per_rank;
            const int mb_in = m_blk - owner * (comm.rows_per_rank / BLOCK_M);
            uint32_t* f = (uint32_t*)comm.peer_flags[owner] + comm.flag_offset + comm.rank * kMaxRowBlocks + mb_in;
            red_add_release_sys(f, 1u);
          }
        }
        if constexpr (MODE == 6) {
          // the CTA completing a 128-row block (all its n-tiles, any CTA) releases the block's flag at its owner
          __threadfence_system();
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (threadIdx.x == 128 && atom_add_acqrel_gpu(comm.tile_done + m_blk, 1u) == (uint32_t)(tiles_n - 1)) {
            comm.tile_done[m_blk] = 0;                              // re-armed for the next call
            const int mbr = comm.rows_per_rank / BLOCK_M, owner = m_blk / mbr;
            uint32_t* f = (uint32_t*)((uint8_t*)comm.peer_bufs[owner] + comm.flag_offset_bytes) +
                          (size_t)comm.rank * kNvlsMaxRowBlocks + (m_blk - owner * mbr);
            st_release_sys(f, comm.epoch);
          }
        }
      }
      // the last boxes' global writes are complete before the kernel ends (the next kernel may read `out` on another stream)
      if ((MODE == 0 || MODE == 3) && tma_epi && (threadIdx.x & 127) == 0) bulk_wait_group<0>();
    }
  }

  if constexpr (MODE == 2) {
    // ===== reducer phase: (row-block, 256-column slab) items of my chunk =====
    __syncthreads();
    const int mb_per_rank = comm.rows_per_rank / BLOCK_M;
    const int slabs = (N + 255) / 256;
    const int items = mb_per_rank * slabs;
    const uint32_t* myflags = (const uint32_t*)comm.peer_flags[comm.rank] + comm.flag_offset;
    const __nv_bfloat16* stage_base = (const __nv_bfloat16*)((const uint8_t*)comm.peer_bufs[comm.rank] + comm.buf_offset);
    __nv_bfloat16* rout = (__nv_bfloat16*)comm.rs_out;
    for (int it = blockIdx.x; it < items; it += gridDim.x) {
      const int mb = it / slabs, slab = it % slabs;
      if (threadIdx.x < comm.world) {
        // counter reaches epoch (cumulative number of n-tiles this source has ever sent for this row-block)
        wait_flag_ge(myflags + threadIdx.x * kMaxRowBlocks + mb, comm.rs_targets[mb]);
      }
      __syncthreads();
      const int c0 = slab * 256;
      const int cols = min(256, N - c0);
      const int vec_per_row = cols / 8;
      for (int idx = threadIdx.x; idx < BLOCK_M * vec_per_row; idx += kThreads) {
        const int r = idx / vec_per_row, v = idx % vec_per_row;
        const size_t off = ((size_t)(mb * BLOCK_M + r)) * N + c0 + v * 8;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int s = 0; s < comm.world; ++s) {
          const uint4 raw = *(const uint4*)(stage_base + (size_t)s * comm.rows_per_rank * N + off);
          const __nv_bfloat162* h = (const __nv_bfloat162*)&raw;
#pragma unroll
          for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); acc[2 * j] += f.x; acc[2 * j + 1] += f.y; }
        }
        uint4 o; __nv_bfloat162* oh = (__nv_bfloat162*)&o;
#pragma unroll
        for (int j = 0; j < 4; ++j) oh[j] = __floats2bfloat162_rn(acc[2 * j], acc[2 * j + 1]);
        *(uint4*)(rout + off) = o;
      }
      __syncthreads();
    }
  }

  if constexpr (MODE == 6) {
    // ===== NVLS reducer: dynamically claimed 16-row items of my chunk =====
    __shared__ int s_item;
    if (is_comm_cta || comm.gemm_join) {
      constexpr bool W32 = sizeof(OutT) == 4;
      const int items = comm.rows_per_rank / kRsRowsPerItem;
      const uint32_t* myflags = (const uint32_t*)(comm.local_base + comm.flag_offset_bytes);
      __nv_bfloat16* rout = (__nv_bfloat16*)comm.rs_out;
      for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) s_item = (int)(atomicAdd(comm.claim, 1u) - comm.claim_base);
        __syncthreads();
        const int item = s_item;
        if (item >= items) break;
        const int mb = item / (BLOCK_M / kRsRowsPerItem), row0 = item * kRsRowsPerItem;
        if ((int)threadIdx.x < comm.world) wait_flag_ge(myflags + (size_t)threadIdx.x * kNvlsMaxRowBlocks + mb, comm.epoch);
        __syncthreads();
        const size_t src_off = (size_t)comm.buf_offset + ((size_t)comm.rank * comm.rows_per_rank + row0) * N * sizeof(OutT);
        const size_t nvec = (size_t)kRsRowsPerItem * N / 8;          // 8 output elements per step
        for (size_t i = threadIdx.x; i < nvec; i += kThreads) {
          float acc[8];
          if (comm.mc_base != nullptr) {
            const uint8_t* src = comm.mc_base + src_off;
            if constexpr (W32) {
              const uint4 lo = multimem_ld_reduce_f32(src + i * 32), hi = multimem_ld_reduce_f32(src + i * 32 + 16);
              acc[0] = __uint_as_float(lo.x); acc[1] = __uint_as_float(lo.y); acc[2] = __uint_as_float(lo.z); acc[3] = __uint_as_float(lo.w);
              acc[4] = __uint_as_float(hi.x); acc[5] = __uint_as_float(hi.y); acc[6] = __uint_as_float(hi.z); acc[7] = __uint_as_float(hi.w);
            } else {
              const uint4 v = multimem_ld_reduce_bf16x2(src + i * 16);
              const __nv_bfloat162* h = (const __nv_bfloat162*)&v;
#pragma unroll
              for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); acc[2 * j] = f.x; acc[2 * j + 1] = f.y; }
            }
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = 0.f;
            for (int p = 0; p < comm.world; ++p) {
              const uint8_t* src = (const uint8_t*)comm.peer_bufs[p] + src_off;
              if constexpr (W32) {
                const uint4 lo = ld_relaxed_sys_v4(src + i * 32), hi = ld_relaxed_sys_v4(src + i * 32 + 16);
                acc[0] += __uint_as_float(lo.x); acc[1] += __uint_as_float(lo.y); acc[2] += __uint_as_float(lo.z); acc[3] += __uint_as_float(lo.w);
                acc[4] += __uint_as_float(hi.x); acc[5] += __uint_as_float(hi.y); acc[6] += __uint_as_float(hi.z); acc[7] += __uint_as_float(hi.w);
              } else {
                const uint4 v = ld_relaxed_sys_v4(src + i * 16);
                const __nv_bfloat162* h = (const __nv_bfloat162*)&v;
#pragma unroll
                for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); acc[2 * j] += f.x; acc[2 * j + 1] += f.y; }
              }
            }
          }
          uint4 o; __nv_bfloat162* oh = (__nv_bfloat162*)&o;
#pragma unroll
          for (int j = 0; j < 4; ++j) oh[j] = __floats2bfloat162_rn(acc[2 * j], acc[2 * j + 1]);
          *(uint4*)(rout + (size_t)row0 * N + i * 8) = o;
        }
      }
    }
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    NXD_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    if (!p || q != cudaDriverEntryPointSuccess) nxd_throw("cuTensorMapEncodeTiled not available", __FILE__, __LINE__);
    fn = (PFN_encodeTiled)p;
  }
  return fn;
}

// cuTensorMapEncodeTiled is a DRIVER API call: it needs a current context on the calling thread.  Autograd worker threads may
// reach us before any runtime call made the primary context current there (PyTorch's device guard skips cudaSetDevice when the
// device index already matches, and the caching allocator can serve at::empty without touching the runtime) → error 201.
static void ensure_driver_context() {
  thread_local bool done = false;
  if (!done) {
    cudaFree(nullptr);      // forces the runtime to initialise / bind the primary context on this thread
    done = true;
  }
}

// 2-D bf16 row-major tensor [rows, cols] (cols contiguous); box = {box_cols, box_rows}; 128B swizzle.
static CUtensorMap make_tmap(const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_cols, uint32_t box_rows) {
  ensure_driver_context();
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) nxd_throw("cuTensorMapEncodeTiled failed: " + std::to_string((int)r), __FILE__, __LINE__);
  return m;
}

// e4m3 row-major [rows, cols] bytes; box = {128 k-bytes, box_rows}
static CUtensorMap make_tmap_u8(const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  ensure_driver_context();
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols};
  cuuint32_t box[2] = {128, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) nxd_throw("cuTensorMapEncodeTiled (u8) failed: " + std::to_string((int)r), __FILE__, __LINE__);
  return m;
}

static int sm_count() {
  static int n = 0;
  if (!n) { int dev; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); }
  return n;
}

CUtensorMap make_tmap_2d(const void* ptr, CUtensorMapDataType dt, uint64_t rows, uint64_t cols, uint64_t row_bytes,
                         uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle) {
  ensure_driver_context();
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(&m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) nxd_throw("cuTensorMapEncodeTiled failed: " + std::to_string((int)r), __FILE__, __LINE__);
  return m;
}

int device_sm_count() { return sm_count(); }

// The TMA epilogue (MODE 0 / 3) writes `out` [M, N] through a tensor map, which needs a 16-byte aligned base and row pitch.
// A bf16 accumulate stays on the register epilogue: a bf16 reduce-add would round the product to bf16 before the add.
// Returns false (register epilogue) when the map does not fit.
template <typename OutT>
static bool out_tmap(const void* out, int M, int N, bool accumulate, CUtensorMap* map) {
  constexpr bool bf16 = sizeof(OutT) == 2;
  if ((uintptr_t)out % 16 || ((size_t)N * sizeof(OutT)) % 16 || (accumulate && bf16)) return false;
  *map = make_tmap_2d(out, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, M, N,
                      (uint64_t)N * sizeof(OutT), kEpiBoxBytes / 64 / sizeof(OutT), 64, CU_TENSOR_MAP_SWIZZLE_128B);
  return true;
}

template <bool AK, bool BK, int MODE, typename OutT, bool FP8 = false>
static void launch(const CUtensorMap& ta, const CUtensorMap& tb, void* out, int M, int N, int K, bool accumulate,
                   const CommDev& c, int grid, cudaStream_t st, const CUtensorMap* ta_local = nullptr) {
  auto kern = gemm_bf16_kernel<AK, BK, MODE, OutT, FP8>;
  static bool configured = false;
  if (!configured) {
    NXD_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    configured = true;
  }
  CUtensorMap to = ta;
  const bool tma_epi = (MODE == 0 || MODE == 3) && out_tmap<OutT>(out, M, N, accumulate, &to);
  kern<<<grid, kThreads, kSmemBytes, st>>>(ta, tb, ta_local ? *ta_local : ta, to, (OutT*)out, M, N, K, accumulate ? 1 : 0,
                                           tma_epi ? 1 : 0, c);
  NXD_CUDA_CHECK(cudaGetLastError());
}

void gemm_bf16(const void* a, const void* b, void* out, int M, int N, int K, bool trans_a, bool trans_b, int out_dt,
               bool accumulate, const GemmComm& comm, const void* a_local_shard, cudaStream_t st) {
  // trans_a=false: a is [M,K] (K-major).  trans_a=true: a is [K,M] (MN-major).
  // trans_b=true : b is [N,K] (K-major).  trans_b=false: b is [K,N] (MN-major).
  const bool AK = !trans_a, BK = trans_b;
  const CUtensorMap ta = AK ? make_tmap(a, M, K, BLOCK_K, BLOCK_M) : make_tmap(a, K, M, 64, BLOCK_K);
  const CUtensorMap tb = BK ? make_tmap(b, N, K, BLOCK_K, BLOCK_N) : make_tmap(b, K, N, 64, BLOCK_K);
  CommDev c{};
  c.rank = comm.rank; c.world = comm.world; c.peer_bufs = comm.peer_bufs; c.peer_flags = comm.peer_flags;
  c.buf_offset = comm.buf_offset; c.flag_offset = comm.flag_offset; c.epoch = comm.epoch; c.comm_sms = comm.comm_sms;
  c.rows_per_rank = comm.world > 0 ? M / comm.world : M;
  c.a_local = a_local_shard; c.rs_out = out;
  for (int i = 0; i < kMaxRowBlocks; ++i) c.rs_targets[i] = comm.rs_targets ? comm.rs_targets[i] : 0u;
  if (comm.mode != 0 && c.rows_per_rank / BLOCK_M > kMaxRowBlocks) nxd_throw("too many row blocks per rank", __FILE__, __LINE__);
  const int tiles = ((M + BLOCK_M - 1) / BLOCK_M) * ((N + BLOCK_N - 1) / BLOCK_N);
  const int sms = sm_count();
  if (comm.mode != 0) {
    if (c.rows_per_rank % BLOCK_M || M % comm.world) nxd_throw("fused TP GEMM needs rows/rank % 128 == 0", __FILE__, __LINE__);
    if (comm.mode == 2 && (N % 8)) nxd_throw("GEMM→RS needs N % 8 == 0", __FILE__, __LINE__);
    if (comm.mode == 1) {
      if (N % 8 || K % 8) nxd_throw("AG→GEMM needs N and K multiples of 8", __FILE__, __LINE__);
      // no pusher: the GEMM CTAs wait for the shards forever; no GEMM CTA: nothing is computed
      if (comm.comm_sms < 1 || comm.comm_sms >= sms) nxd_throw("AG→GEMM: comm_sms must leave GEMM CTAs", __FILE__, __LINE__);
    }
  }
#define NXD_LAUNCH(AKv, BKv)                                                                                          \
  do {                                                                                                                \
    if (comm.mode == 1) {                                                                                             \
      if (out_dt == kBF16) launch<AKv, BKv, 1, __nv_bfloat16>(ta, tb, out, M, N, K, accumulate, c, sms, st);          \
      else launch<AKv, BKv, 1, float>(ta, tb, out, M, N, K, accumulate, c, sms, st);                                  \
    } else if (comm.mode == 2) {                                                                                      \
      launch<AKv, BKv, 2, __nv_bfloat16>(ta, tb, out, M, N, K, false, c, sms, st);                                    \
    } else {                                                                                                          \
      const int grid = tiles < sms ? tiles : sms;                                                                     \
      if (out_dt == kBF16) launch<AKv, BKv, 0, __nv_bfloat16>(ta, tb, out, M, N, K, accumulate, c, grid, st);         \
      else launch<AKv, BKv, 0, float>(ta, tb, out, M, N, K, accumulate, c, grid, st);                                 \
    }                                                                                                                 \
  } while (0)
  if (AK && BK) NXD_LAUNCH(true, true);
  else if (AK && !BK) NXD_LAUNCH(true, false);
  else if (!AK && !BK) NXD_LAUNCH(false, false);
  else NXD_LAUNCH(false, true);
#undef NXD_LAUNCH
}

// ---- grouped (MoE blockwise) GEMMs ---------------------------------------------------------------------------------
// out[M,N] = A[M,K] · W[e(block)]: rows of A are grouped in `block_rows`-row blocks, block i uses expert block_expert[i].
// trans_b: W is [E, N, K] (K-major) else [E, K, N] (MN-major).
void grouped_gemm_bf16(const void* a, const void* b, void* out, int M, int N, int K, int E, bool trans_b,
                       const int* block_expert, int block_rows, int out_dt, cudaStream_t st) {
  if (block_rows % BLOCK_M) nxd_throw("grouped GEMM: block size must be a multiple of 128", __FILE__, __LINE__);
  if (!trans_b && (K % BLOCK_K)) nxd_throw("grouped GEMM: K % 64 != 0 with [E,K,N] weights", __FILE__, __LINE__);
  const CUtensorMap ta = make_tmap(a, M, K, BLOCK_K, BLOCK_M);
  const CUtensorMap tb = trans_b ? make_tmap(b, (uint64_t)E * N, K, BLOCK_K, BLOCK_N) : make_tmap(b, (uint64_t)E * K, N, 64, BLOCK_K);
  CommDev c{};
  c.block_expert = block_expert; c.grp_block_rows = block_rows; c.grp_b_rows = trans_b ? N : K; c.num_groups = E;
  const int tiles = ((M + BLOCK_M - 1) / BLOCK_M) * ((N + BLOCK_N - 1) / BLOCK_N);
  const int grid = tiles < sm_count() ? tiles : sm_count();
  if (trans_b) {
    if (out_dt == kBF16) launch<true, true, 3, __nv_bfloat16>(ta, tb, out, M, N, K, false, c, grid, st);
    else launch<true, true, 3, float>(ta, tb, out, M, N, K, false, c, grid, st);
  } else {
    if (out_dt == kBF16) launch<true, false, 3, __nv_bfloat16>(ta, tb, out, M, N, K, false, c, grid, st);
    else launch<true, false, 3, float>(ta, tb, out, M, N, K, false, c, grid, st);
  }
}

// out[e] [Mo, No] (+)= A[rows of e, Mo]ᵀ · B[rows of e, No]; expert e owns row blocks [seg_first_block[e], seg_first_block[e+1]).
void grouped_wgrad_bf16(const void* a, const void* b, void* out, int rows_total, int Mo, int No, int E,
                        const int* seg_first_block, int block_rows, int out_dt, bool accumulate, cudaStream_t st) {
  if (block_rows % BLOCK_K) nxd_throw("grouped wgrad: block size must be a multiple of 64", __FILE__, __LINE__);
  const CUtensorMap ta = make_tmap(a, rows_total, Mo, 64, BLOCK_K);
  const CUtensorMap tb = make_tmap(b, rows_total, No, 64, BLOCK_K);
  CommDev c{};
  c.seg_first_block = seg_first_block; c.grp_block_rows = block_rows; c.num_groups = E; c.out_group_stride = (long)Mo * No;
  const int tiles = E * ((Mo + BLOCK_M - 1) / BLOCK_M) * ((No + BLOCK_N - 1) / BLOCK_N);
  const int grid = tiles < sm_count() ? tiles : sm_count();
  if (out_dt == kBF16) launch<false, false, 4, __nv_bfloat16>(ta, tb, out, Mo, No, rows_total, accumulate, c, grid, st);
  else launch<false, false, 4, float>(ta, tb, out, Mo, No, rows_total, accumulate, c, grid, st);
}

// out[M,N] = (a_e4m3[M,K] · b_e4m3[N,K]ᵀ) ∘ scale_a[M] ⊗ scale_b[N]: bf16 (quantised linears), or fp32 (the fp8 weight
// gradient), which `accumulate` adds into (TMA reduce-add at L2 when out's tensor map fits, else the register epilogue)
void gemm_fp8(const void* a, const void* b, void* out, int M, int N, int K, const float* scale_a, const float* scale_b,
              int out_dt, bool accumulate, cudaStream_t st) {
  if (K % 16) nxd_throw("fp8 GEMM needs K % 16 == 0", __FILE__, __LINE__);
  if (out_dt != kBF16 && out_dt != kF32) nxd_throw("fp8 GEMM writes bf16 or fp32", __FILE__, __LINE__);
  if (accumulate && out_dt != kF32) nxd_throw("fp8 GEMM accumulates into fp32 only", __FILE__, __LINE__);
  const CUtensorMap ta = make_tmap_u8(a, M, K, BLOCK_M);
  const CUtensorMap tb = make_tmap_u8(b, N, K, BLOCK_N);
  CommDev c{};
  c.scale_a = scale_a; c.scale_b = scale_b;
  const int tiles = ((M + BLOCK_M - 1) / BLOCK_M) * ((N + BLOCK_N - 1) / BLOCK_N);
  const int grid = tiles < sm_count() ? tiles : sm_count();
  if (out_dt == kBF16) launch<true, true, 0, __nv_bfloat16, true>(ta, tb, out, M, N, K, false, c, grid, st);
  else launch<true, true, 0, float, true>(ta, tb, out, M, N, K, accumulate, c, grid, st);
}

bool gemm_self_check_supported() { return true; }

// ---- NVLS fused tensor-parallel GEMMs (MODE 5 / 6).  mode 1: a_local = shard [M/world, K] → out [M, N]; the gathered A
// lands at buf_offset of every rank's region.  mode 2: a [M, K] → rs_out [M/world, N]; the partials live at buf_offset.
// Returns the number of reducer claims consumed (mode 2), 0 for mode 1.
int gemm_bf16_nvls(int mode, const void* a, const void* b, void* out, void* rs_out, const void* a_local, int M, int N, int K,
                   bool trans_b, int rank, int world, const int64_t* peer_bases, int64_t mc_base, int64_t local_base,
                   long buf_offset, long flag_offset, uint32_t epoch, int comm_ctas, uint32_t* tile_done, uint32_t* claim,
                   uint32_t claim_base, bool wire_fp32, bool gemm_join, cudaStream_t st) {
  CommDev c{};
  c.rank = rank; c.world = world; c.peer_bufs = peer_bases; c.mc_base = (uint8_t*)mc_base; c.local_base = (uint8_t*)local_base;
  c.buf_offset = buf_offset; c.flag_offset_bytes = flag_offset; c.epoch = epoch; c.comm_sms = comm_ctas;
  c.rows_per_rank = M / world; c.a_local = a_local; c.rs_out = rs_out; c.tile_done = tile_done; c.claim = claim;
  c.claim_base = claim_base; c.gemm_join = gemm_join ? 1 : 0;
  if (M % world || c.rows_per_rank % BLOCK_M || c.rows_per_rank / BLOCK_M > kNvlsMaxRowBlocks)
    nxd_throw("NVLS TP GEMM: rows per rank must be a multiple of 128 and at most 32768", __FILE__, __LINE__);
  if (N % 8 || K % 8) nxd_throw("NVLS TP GEMM: N and K must be multiples of 8", __FILE__, __LINE__);
  const int grid = sm_count();
  if (comm_ctas < 1 || comm_ctas >= grid) nxd_throw("NVLS TP GEMM: comm_ctas must leave GEMM CTAs", __FILE__, __LINE__);
  const CUtensorMap tb = trans_b ? make_tmap(b, N, K, BLOCK_K, BLOCK_N) : make_tmap(b, K, N, 64, BLOCK_K);
  if (mode == 1) {
    const CUtensorMap ta = make_tmap((const uint8_t*)local_base + buf_offset, M, K, BLOCK_K, BLOCK_M);
    const CUtensorMap tal = make_tmap(a_local, c.rows_per_rank, K, BLOCK_K, BLOCK_M);
    if (trans_b) launch<true, true, 5, __nv_bfloat16>(ta, tb, out, M, N, K, false, c, grid, st, &tal);
    else launch<true, false, 5, __nv_bfloat16>(ta, tb, out, M, N, K, false, c, grid, st, &tal);
    return 0;
  }
  const CUtensorMap ta = make_tmap(a, M, K, BLOCK_K, BLOCK_M);
  if (trans_b) {
    if (wire_fp32) launch<true, true, 6, float>(ta, tb, nullptr, M, N, K, false, c, grid, st);
    else launch<true, true, 6, __nv_bfloat16>(ta, tb, nullptr, M, N, K, false, c, grid, st);
  } else {
    if (wire_fp32) launch<true, false, 6, float>(ta, tb, nullptr, M, N, K, false, c, grid, st);
    else launch<true, false, 6, __nv_bfloat16>(ta, tb, nullptr, M, N, K, false, c, grid, st);
  }
  return (c.rows_per_rank / kRsRowsPerItem) + (gemm_join ? grid : comm_ctas);
}

}  // namespace nxd
