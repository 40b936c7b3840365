// chain_kernel.cuh -- fused linear voice chains: one kernel launch = n_blocks Bank::operator()
// calls (reference MLDSPFunctional.h:328-337) for every voice.
//
// Work decomposition (DESIGN.md "K1/K2"):
//   * one LANE per voice: all oscillator / filter state and coefficients live in registers
//     for the whole launch (loaded once, stored once, SoA, coalesced 4 B/lane);
//   * one WARP per 32 consecutive voices (a "group"); the grid is persistent and work units
//     (a quarter of the launch's blocks for one group) come from an atomic queue; warps are
//     otherwise fully independent (no __syncthreads):
//     each warp owns a private ring of `stages` 8 KB shared-memory blocks and its own
//     mbarriers, and walks time sequentially (the recurrences cannot be split in time);
//   * the unit of transfer is one 64-sample block of 32 voices = 32 FULL 256-byte rows of one
//     plane of the reference layout [plane][V][64] f32 (8 KB), moved by ONE TMA instruction
//     through a 4-D tensor map {32 samples, V voices, 2 halves, planes} with strides
//     {256 B, 128 B, V*256 B} and box {32, 32, 2, 1}: it lands in shared memory as two 4 KB
//     half tiles [half][voice][32 samples], each SWIZZLE_128B.  (Full rows rather than half
//     rows through a 3-D map: fewer, larger TMA transfers; tools/ubench/tma_copy.cu compares
//     the two as a pure copy.)  With the 128-byte swizzle lane r finds
//     16-byte chunk j of its own row at  r*128 + ((j ^ (r & 7)) << 4): the eight lanes of
//     every quarter-warp hit eight different 16-byte bank groups, so the per-lane LDS.128 /
//     STS.128 row walk is bank-conflict free;
//   * results are written IN PLACE into the block and leave through one TMA store
//     (UTMASTG.4D); ragged V is clipped by the tensor map (zero fill on load, clip on store);
//   * optional mix bus: after a tile is computed, lane n sums column n over the 32 voice
//     rows into partial[plane][group][64].  This column walk is NOT conflict-free under the
//     row swizzle: it is where the kernel's shared-memory bank conflicts are;
//     a second tiny kernel adds the per-group partials in group order (deterministic).
#pragma once
#include "ops.cuh"
#include "tma.cuh"

namespace mlb
{
constexpr int kTileSamples = 32;
constexpr int kTileVoices = 32;
constexpr int kTileBytes = kTileSamples * kTileVoices * 4;  // 4096: one 128B-swizzled half tile
constexpr int kBlockBytes = 2 * kTileBytes;                 // 8192: 32 voices x one 64-sample block
constexpr int kChainMaxWarps = 14;                          // 14 x 2 stages x 8 KB = 224 KB per SM
constexpr int kMaxChainState = 8;
constexpr int kMaxChainCoef = 16;
constexpr int kMaxChainRows = 6;                            // coefficient rows of a *_V filter (HiShelf: 6)

__host__ __device__ constexpr int op_ns(int op)
{
  switch (op)
  {
#define MLB_X_NS(NAME, id, nin, nst, nco) \
  case id: return nst;
    MLB_OP_TABLE(MLB_X_NS)
#undef MLB_X_NS
  }
  return 0;
}
__host__ __device__ constexpr int op_nc(int op)
{
  switch (op)
  {
#define MLB_X_NC(NAME, id, nin, nst, nco) \
  case id: return nco;
    MLB_OP_TABLE(MLB_X_NC)
#undef MLB_X_NC
  }
  return 0;
}

__host__ __device__ constexpr int op_nin(int op)
{
  switch (op)
  {
#define MLB_X_NI(NAME, id, nin, nst, nco) \
  case id: return nin;
    MLB_OP_TABLE(MLB_X_NI)
#undef MLB_X_NI
  }
  return 0;
}
// the op table again, for dispatching the stateless elementwise ops
#define MLB_OP_TABLE_STATELESS(X) MLB_OP_TABLE(X)

enum ChainSrc
{
  SRC_INPUT = 0,  // generator/filter input = external signal plane (Contract R)
  SRC_PARAM = 1,  // = per-voice scalar broadcast, DSPVector(float) (Contract S)
  SRC_NONE = 2    // generator takes no input (NoiseGen)
};

struct ChainArgs
{
  uint32_t* state;     // [n_state_words][V]
  const float* coef;   // [n_coef_words][V]
  float* mix_partial;  // [T*n_out_planes][n_groups][64] or nullptr
  int V, T;                     // voices of this launch (a slice of the bank), blocks
  int v_stride;                 // voices of the whole bank = row length of the state/coef SoA
  int n_in_planes, in_plane;    // tile z = t*n_in_planes + in_plane
  int n_out_planes, out_plane;  // tile z = t*n_out_planes + out_plane
  int n_groups;                 // ceil(V/32) groups of this launch
  int groups_stride;            // groups of the whole bank = row length of the mix partials
  int write_out;                // store per-voice output planes
  int stages;
  unsigned* sched;              // unit counter; the warp that finishes the launch's last unit re-zeroes it
  unsigned* progress;           // [g] chunks finished by group g of this launch (monotonic)
  unsigned* done;               // units finished in this launch (re-zeroed with sched)
  unsigned* base_word;          // device-resident progress base: value of progress[g] "at launch"; the last
                                // warp advances it by n_chunks.  Nothing launch-specific is baked into the
                                // kernel arguments, so a captured CUDA graph of a process call can be replayed.
  int chunk_blocks, n_chunks;   // blocks per work unit, units per group
  int st_idx[kMaxChainState];  // SoA word index of each register state slot
  int co_idx[kMaxChainCoef];
  int cv_plane[kMaxChainRows];  // input plane of each coefficient ROW of a LOPASS_V-class filter
  unsigned long long* prof;     // team kernel, debugging only (MLB_TEAM_PROF=1): cycle counters of CTA 0
  int n_sms;                    // team kernel: SM count (role rotation between the CTAs that share an SM)
};

// GEN: generator op id or -1 (the chain filters the source directly)
// F1, F2: filter op ids or -1;  GAIN: multiply by a PARAM at the end
template <int GEN, int SRC, int F1, int F2, bool GAIN, bool EX>
struct Chain
{
  static constexpr int NS_GEN = GEN >= 0 ? op_ns(GEN) : 0;
  static constexpr int NS_F1 = F1 >= 0 ? op_ns(F1) : 0;
  static constexpr int NS_F2 = F2 >= 0 ? op_ns(F2) : 0;
  static constexpr int NS = NS_GEN + NS_F1 + NS_F2;
  static constexpr int NC_SRC = (SRC == SRC_PARAM) ? 1 : 0;
  static constexpr int NC_F1 = F1 >= 0 ? op_nc(F1) : 0;
  static constexpr int NC_F2 = F2 >= 0 ? op_nc(F2) : 0;
  static constexpr int NC = NC_SRC + NC_F1 + NC_F2 + (GAIN ? 1 : 0);
  static constexpr bool HAS_IN = (SRC == SRC_INPUT);
  // F1 may be a filter whose coefficients are per-sample ROWS (LOPASS_V ...): NV extra input planes
  static constexpr bool F1_V = (F1 == MLB_OP_LOPASS_V || F1 == MLB_OP_LOSHELF_V || F1 == MLB_OP_HISHELF_V);
  static constexpr int NV = F1_V ? op_nin(F1) - 1 : 0;
  static constexpr int NP = (HAS_IN ? 1 : 0) + NV;  // planes a stage of the ring holds (TMA loads per block)
  static constexpr int NPB = NP > 0 ? NP : 1;       // 8-KB blocks per stage (the output is written over plane 0)
  static_assert(NS <= kMaxChainState && NC <= kMaxChainCoef && NV <= kMaxChainRows, "chain too large");

  static MLB_DEV float tick(float in, uint32_t (&st)[NS > 0 ? NS : 1],
                            const float (&co)[NC > 0 ? NC : 1], const float* cv)
  {
    float x = (SRC == SRC_INPUT) ? in : ((SRC == SRC_PARAM) ? co[0] : 0.0f);
    float y = x;
    if (GEN >= 0) y = gen_tick<EX>(GEN, x, 0.0f, &st[0]);
    if (F1_V)
      y = vfilter_tick<EX>(F1, y, &st[NS_GEN], cv);
    else if (F1 >= 0)
      y = filter_tick<EX>(F1, y, &st[NS_GEN], &co[NC_SRC]);
    if (F2 >= 0) y = filter_tick<EX>(F2, y, &st[NS_GEN + NS_F1], &co[NC_SRC + NC_F1]);
    if (GAIN) y = A<EX>::mul(y, co[NC - 1]);  // operator*(DSPVector, DSPVector(float)), O:345-348
    return y;
  }
  // the same chain cut after the generator, for the two-warp team kernel (chain_team_kernel)
  static constexpr bool SPLIT = (GEN >= 0) && (F1 >= 0) && !F1_V;
  static MLB_DEV float tick_gen(float in, uint32_t (&st)[NS > 0 ? NS : 1], const float (&co)[NC > 0 ? NC : 1])
  {
    const float x = (SRC == SRC_INPUT) ? in : ((SRC == SRC_PARAM) ? co[0] : 0.0f);
    return gen_tick<EX>(GEN, x, 0.0f, &st[0]);
  }
  static MLB_DEV float tick_flt(float y, uint32_t (&st)[NS > 0 ? NS : 1], const float (&co)[NC > 0 ? NC : 1])
  {
    if (F1 >= 0) y = filter_tick<EX>(F1, y, &st[NS_GEN], &co[NC_SRC]);
    if (F2 >= 0) y = filter_tick<EX>(F2, y, &st[NS_GEN + NS_F1], &co[NC_SRC + NC_F1]);
    if (GAIN) y = A<EX>::mul(y, co[NC - 1]);
    return y;
  }
};

// Work distribution: the launch is cut into units (chunk c, group g) = `chunk_blocks`
// consecutive blocks of one 32-voice group, numbered chunk-major u = c * n_groups + g and
// handed out by an atomic counter, so any number of resident warps stays balanced.  A voice's
// time axis is sequential, so unit (c, g) may start only after (c-1, g) stored its state:
// progress[g] counts finished chunks; chunk-major order means that predecessor was handed
// out a whole round earlier and is practically always done.  A warp always holds its current
// unit and the next one, so its TMA load stream runs S-1 blocks ahead across unit boundaries.
struct UnitCursor
{
  int unit;  // unit id, >= total when exhausted
  int g, t0, nblk;
};

template <class P>
__global__ void __launch_bounds__(kChainMaxWarps * 32)
    chain_kernel(const __grid_constant__ CUtensorMap in_map,
                 const __grid_constant__ CUtensorMap out_map, const ChainArgs a)
{
  extern __shared__ __align__(1024) uint8_t smem_raw[];  // SWIZZLE_128B atom = 1024 B
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int W = blockDim.x >> 5;
  const int S = a.stages;
  const int total_units = a.n_chunks * a.n_groups;
  // read before this warp can finish a unit, i.e. before the launch's last unit can have been counted
  const unsigned progress_base = (a.n_chunks > 1) ? __ldcg(a.base_word) : 0u;

  const uint32_t base = smem_u32(smem_raw);
  if (base & 1023u) __trap();  // the swizzle formula below assumes 1024-byte aligned tiles
  constexpr uint32_t kStageBytes = (uint32_t)P::NPB * kBlockBytes;
  const uint32_t blocks = base + (uint32_t)(warp * S) * kStageBytes;
  const uint32_t bars = base + (uint32_t)(W * S) * kStageBytes + (uint32_t)(warp * S) * 8u;

  // Every warp draws unit indices until it gets one >= total_units: exactly ONE failing draw per warp, so the
  // counter ends at total_units + (warps of the grid), and the warp that draws that last value is the last one
  // ever to touch the counter in this launch: it puts it back to zero for the next launch (no memset).
  const unsigned last_draw = (unsigned)total_units + gridDim.x * (unsigned)W - 1u;
  auto grab = [&]() -> int
  {
    int u = 0;
    if (lane == 0)
    {
      const unsigned d = atomicAdd(a.sched, 1u);
      if (d == last_draw) atomicExch(a.sched, 0u);
      u = (int)min(d, (unsigned)total_units);
    }
    return __shfl_sync(0xffffffffu, u, 0);
  };
  auto decode = [&](int u) -> UnitCursor
  {
    UnitCursor c;
    c.unit = u;
    const int ch = u / a.n_groups;
    c.g = u - ch * a.n_groups;
    c.t0 = ch * a.chunk_blocks;
    const int rest = a.T - c.t0;
    c.nblk = (u < total_units) ? (rest < a.chunk_blocks ? rest : a.chunk_blocks) : 0;
    return c;
  };

  UnitCursor cur = decode(grab());
  if (cur.unit >= total_units) return;  // warp-uniform; warps never synchronise with each other
  // The next unit is reserved only when the load stream is about to need it (S-1 blocks before
  // the end of `cur`): reserving earlier would put more units in flight than there are groups
  // and make warps wait on predecessors that are still being computed.
  UnitCursor nxt = cur;
  nxt.nblk = 0;
  bool have_nxt = false;

  if (lane == 0)
  {
    if (P::NP > 0)
    {
      prefetch_tensormap(&in_map);
      for (int s = 0; s < S; ++s) mbar_init(bars + 8u * s, 1);
      fence_mbar_init();
    }
    if (a.write_out) prefetch_tensormap(&out_map);
  }
  __syncwarp();

  // ---- TMA load stream (lane 0): one op = one 64-sample block of 32 voices = 32 full
  // 256-byte rows (8 KB), landing as two 128B-swizzled 4 KB half tiles ----
  int ld_in_nxt = 0;  // 0: the load cursor is inside `cur`, 1: inside `nxt`
  int ld_blk = 0;     // next block of that unit to request
  int ld_stage = 0;   // stage the next load goes to
  auto issue_next_load = [&]() -> bool
  {
    const UnitCursor& u = ld_in_nxt ? nxt : cur;
    if (ld_blk >= u.nblk) return false;  // stream exhausted (or next unit not known yet)
    const uint32_t bar = bars + 8u * ld_stage;
    mbar_arrive_expect_tx(bar, (uint32_t)P::NP * kBlockBytes);
    const uint32_t dst = blocks + (uint32_t)ld_stage * kStageBytes;
    const int z0 = (u.t0 + ld_blk) * a.n_in_planes;
    // The input rows are read once, yet they stream faster with an evict-last hint than with evict-first or
    // evict-normal: 0.776 / 0.800 / 0.788 ms for config A on an H100 SXM at 700 W (DESIGN.md 7).  The hint only
    // changes which lines L2 gives up first; why that helps the write-backs of the output rows is not measured.
    if (P::HAS_IN) tma_load_4d(dst, &in_map, bar, 0, u.g * kTileVoices, 0, z0 + a.in_plane, kEvictLast);
#pragma unroll
    for (int p = 0; p < P::NV; ++p)
      tma_load_4d(dst + (uint32_t)((P::HAS_IN ? 1 : 0) + p) * kBlockBytes, &in_map, bar, 0, u.g * kTileVoices, 0,
                  z0 + a.cv_plane[p], kEvictFirst);
    if (++ld_stage == S) ld_stage = 0;
    if (++ld_blk == u.nblk && !ld_in_nxt)
    {
      ld_in_nxt = 1;
      ld_blk = 0;
    }
    return true;
  };
  int ahead = 0;  // (lane 0) loads issued minus blocks whose computation has started
  if (P::NP > 0 && lane == 0)
    while (ahead < S - 1 && issue_next_load()) ++ahead;

  const uint32_t row_off = (uint32_t)lane * 128u;
  const uint32_t sw = (uint32_t)(lane & 7) << 4;
  uint32_t mix_off[8];
#pragma unroll
  for (int j = 0; j < 8; ++j)
    mix_off[j] = ((((uint32_t)lane >> 2) ^ (uint32_t)j) << 4) + (((uint32_t)lane & 3u) << 2);
  const size_t mix_block_stride = (size_t)a.n_out_planes * a.groups_stride * MLB_BLOCK;

  uint32_t st[P::NS > 0 ? P::NS : 1];
  float co[P::NC > 0 ? P::NC : 1];
  int s = 0;            // stage of the block being computed
  uint32_t parity = 0;  // parity of the current use of stage s
  int stores = 0;       // bulk stores issued by this warp so far

  while (cur.unit < total_units)
  {
    // ---- unit start: wait for this group's previous chunk, then state HBM -> registers ----
    const int v0 = cur.g * kTileVoices;
    const int v = v0 + lane;
    const bool live = v < a.V;
    const bool full_group = (v0 + kTileVoices <= a.V);
    if (cur.t0 > 0)
    {
      const unsigned want = progress_base + (unsigned)(cur.t0 / a.chunk_blocks);
      const volatile unsigned* pr = a.progress + cur.g;
      while ((int)(*pr - want) < 0) __nanosleep(64);
      __threadfence();  // acquire: the predecessor's state stores are visible
    }
#pragma unroll
    for (int i = 0; i < P::NS; ++i)
      st[i] = live ? __ldcg(a.state + (size_t)a.st_idx[i] * a.v_stride + v) : 0u;
#pragma unroll
    for (int i = 0; i < P::NC; ++i) co[i] = live ? a.coef[(size_t)a.co_idx[i] * a.v_stride + v] : 0.0f;
    // partial[t*n_out + plane][group][h*32 + lane]
    float* mix_row = a.mix_partial ? a.mix_partial + (size_t)cur.t0 * mix_block_stride +
                                         ((size_t)a.out_plane * a.groups_stride + cur.g) * MLB_BLOCK + lane
                                   : nullptr;

    for (int b = 0; b < cur.nblk; ++b)
    {
      if (!have_nxt && b >= cur.nblk - (S - 1))
      {
        nxt = decode(grab());
        have_nxt = true;
      }
      const uint32_t blk = blocks + (uint32_t)s * kStageBytes;
      if (P::NP > 0)
      {
        --ahead;
        mbar_wait(bars + 8u * s, parity);
      }
      else
      {
        // output-only ring (2 stages): the store that last read this stage is done
        if (lane == 0) bulk_wait_read<1>();
        __syncwarp();
      }

#pragma unroll 1
      for (int h = 0; h < 2; ++h)
      {
        const uint32_t tile = blk + (uint32_t)h * kTileBytes;
        // all eight LDS.128 first so their latency overlaps the arithmetic
        float4 xin[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
          xin[j] = P::HAS_IN ? lds128(tile + row_off + (((uint32_t)j << 4) ^ sw))
                             : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 8; ++j)
        {
          float4 y;
          if (P::NV > 0)
          {
            // this quad of every coefficient row (same swizzled position in the following 8-KB planes)
            float4 cq[P::NV > 0 ? P::NV : 1];
#pragma unroll
            for (int p = 0; p < P::NV; ++p)
              cq[p] = lds128(tile + (uint32_t)((P::HAS_IN ? 1 : 0) + p) * kBlockBytes + row_off +
                             (((uint32_t)j << 4) ^ sw));
            float cv[P::NV > 0 ? P::NV : 1];
#pragma unroll
            for (int p = 0; p < P::NV; ++p) cv[p] = cq[p].x;
            y.x = P::tick(xin[j].x, st, co, cv);
#pragma unroll
            for (int p = 0; p < P::NV; ++p) cv[p] = cq[p].y;
            y.y = P::tick(xin[j].y, st, co, cv);
#pragma unroll
            for (int p = 0; p < P::NV; ++p) cv[p] = cq[p].z;
            y.z = P::tick(xin[j].z, st, co, cv);
#pragma unroll
            for (int p = 0; p < P::NV; ++p) cv[p] = cq[p].w;
            y.w = P::tick(xin[j].w, st, co, cv);
          }
          else
          {
            y.x = P::tick(xin[j].x, st, co, nullptr);
            y.y = P::tick(xin[j].y, st, co, nullptr);
            y.z = P::tick(xin[j].z, st, co, nullptr);
            y.w = P::tick(xin[j].w, st, co, nullptr);
          }
          sts128(tile + row_off + (((uint32_t)j << 4) ^ sw), y);
          if (P::NP > 0 && j == 3 && h == 0 && lane == 0)
          {
            // Refill point, a quarter block after the previous block's store was issued: that
            // store has drained its shared-memory reads by now, so the wait does not stall.
            if (a.write_out && stores > 0) bulk_wait_read<0>();
            while (ahead < S - 1 && issue_next_load()) ++ahead;
          }
        }

        if (a.mix_partial != nullptr)
        {
          // lane n sums sample column n over the 32 voice rows, rows in voice order, from +0.
          // Element (r, n) sits at r*128 + (((n>>2) ^ (r&7)) << 4) + (n&3)*4: mix_off[r&7]
          // holds the lane-dependent part, the rest folds into LDS immediates.
          __syncwarp();
          float acc = 0.0f;
          if (full_group)
          {
#pragma unroll
            for (int r = 0; r < 32; ++r)
              acc = __fadd_rn(acc, lds32(tile + mix_off[r & 7] + (uint32_t)r * 128u));
          }
          else
          {
            // ragged last group: rows beyond V hold garbage computed from zero-filled input
            for (int r = 0; r < 32; ++r)
              if (v0 + r < a.V)
                acc = __fadd_rn(acc, lds32(tile + mix_off[r & 7] + (uint32_t)r * 128u));
          }
          mix_row[h * kTileSamples] = acc;
        }
      }
      if (a.mix_partial != nullptr) mix_row += mix_block_stride;

      // make this lane's generic-proxy writes visible to the TMA unit, then hand the block over
      fence_proxy_async();
      __syncwarp();
      if (lane == 0 && a.write_out)
      {
        tma_store_4d(&out_map, blk, 0, v0, 0, (cur.t0 + b) * a.n_out_planes + a.out_plane);
        bulk_commit();
      }
      ++stores;
      if (++s == S)
      {
        s = 0;
        parity ^= 1u;
      }
    }

    // ---- unit done: state back to HBM, publish progress, move to the next unit ----
#pragma unroll
    for (int i = 0; i < P::NS; ++i)
      if (live) __stcg(a.state + (size_t)a.st_idx[i] * a.v_stride + v, st[i]);
    if (a.n_chunks > 1)
    {
      __threadfence();  // release: state stores before the progress flag
      __syncwarp();
      if (lane == 0)
        atomicExch(a.progress + cur.g, progress_base + (unsigned)(cur.t0 / a.chunk_blocks) + 1u);
    }
    // the launch's last unit: advance the device-resident progress base for the next launch on this stream
    if (lane == 0 && atomicAdd(a.done, 1u) + 1u == (unsigned)total_units)
    {
      atomicExch(a.done, 0u);
      if (a.n_chunks > 1) atomicAdd(a.base_word, (unsigned)a.n_chunks);
    }
    if (!have_nxt) nxt = decode(grab());
    cur = nxt;
    nxt.nblk = 0;
    have_nxt = false;
    // The load cursor was inside the old `nxt`, which is now `cur` (it always is when there are
    // loads: every block of a unit is requested before it is computed).  If it already
    // requested all of it (units shorter than the ring), move on and top the ring up again.
    if (ld_in_nxt)
      ld_in_nxt = 0;
    else
      ld_blk = 0;
    if (!ld_in_nxt && ld_blk >= cur.nblk)
    {
      ld_in_nxt = 1;
      ld_blk = 0;
    }
    if (P::NP > 0 && lane == 0 && ahead < S - 1)
    {
      if (a.write_out) bulk_wait_read<0>();  // all stages but the ones in flight are free again
      while (ahead < S - 1 && issue_next_load()) ++ahead;
    }
  }

  // shared memory must outlive the last bulk stores
  if (lane == 0) bulk_wait_read<0>();
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// chain_team_kernel: the same fused chains for SMALL banks (fewer voice groups than ~4 per SM).
//
// With so few groups the persistent kernel above runs one lone warp per scheduler, and a lone warp
// is latency-bound: every one of the ~39 instructions of a voice-sample waits for its operands.  A voice's
// time axis cannot be split, but the CHAIN can: the generator (phase accumulate + waveshape: a long
// but time-parallel computation, the only recurrence is one integer add) and the filter (a short
// 16-cycle recurrence) are different pipeline stages.  Here every 32-voice group is run by a TEAM
// of three warps in one 96-thread CTA (the third, M, takes everything that is not arithmetic of the chain off F):
//   warp G: waits for the TMA load of block t (mbarrier `full`), overwrites the frequency tile with the
//           generator's output in place, arrives on the stage's `gen` NAMED barrier (bar.arrive, 64 threads);
//   warp F: bar.sync on `gen`, runs filter(s) + gain in place, fences for the async proxy, arrives on `flt`;
//   warp M: bar.sync on `flt`, hands the block to the TMA store, sums the mix-bus columns (reads only), and
//           arrives on the stage's `free` barrier once the store has drained its shared-memory reads; G syncs
//           on `free` before it refills the stage.
// (Named barriers -- ids 1..S gen, S+1..2S flt, 2S+1..3S free, S = 5 -- make every lane a participant of the
// hand-off at the price of one warp-level instruction; compute-sanitizer racecheck follows them.)
// All walk a ring of S 8-KB stages; G's lane 0 keeps S-3 loads in flight.  Per sample each warp now
// has roughly half the dependent instructions, and the halves overlap: ~2x per group.
template <class P>
__global__ void __launch_bounds__(128) chain_team_kernel(const __grid_constant__ CUtensorMap in_map,
                                                        const __grid_constant__ CUtensorMap out_map,
                                                        const ChainArgs a)
{
  static_assert(P::SPLIT, "team kernel needs a generator and a filter");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31;
  // Which scheduler a warp lands on, and with whom it shares it, decides the pace of the busiest role (F).
  // Four-warp CTAs rotate the roles by CTA index (the fourth warp exits at once); three-warp CTAs keep fixed roles and
  // rotate by themselves, since the SM hands out warp slots round robin.  The host launches 128 threads (rotation) up
  // to two teams per SM and 96 threads (fixed roles) above; tools/probe_team.py times the variants.
  const bool four = blockDim.x == 128;
  const int rot = four ? (int)((blockIdx.x + blockIdx.x / (unsigned)a.n_sms) & 3u) : 0;
  const int warp = four ? (int)(((threadIdx.x >> 5) - rot) & 3) : (int)(threadIdx.x >> 5);  // role: 0 = G, 1 = F, 2 = M
  const int S = a.stages;
  const int LA = S - 3;               // loads in flight ahead of the generator
  const uint32_t base = smem_u32(smem_raw);
  if (base & 1023u) __trap();
  const uint32_t bar_full = base + (uint32_t)S * kBlockBytes;
  // named barrier ids of stage s (3 S <= 15): G -> F, F -> M, M -> G
  const int id_gen = 1, id_flt = 1 + S, id_free = 1 + 2 * S;
  if (threadIdx.x == 0)
  {
    for (int s = 0; s < S; ++s) mbar_init(bar_full + 8u * s, 1);
    fence_mbar_init();
    if (P::HAS_IN) prefetch_tensormap(&in_map);
    if (a.write_out) prefetch_tensormap(&out_map);
  }
  __syncthreads();
  if (warp == 3) return;

  const int g = blockIdx.x;
  const int v0 = g * kTileVoices;
  const int v = v0 + lane;
  const bool live = v < a.V;
  const bool full_group = (v0 + kTileVoices <= a.V);
  const uint32_t row_off = (uint32_t)lane * 128u;
  const uint32_t sw = (uint32_t)(lane & 7) << 4;
  const int T = a.T;

  if (warp == 2)
  {
    // ---------------- M: mix-bus column sums + TMA store + stage recycling ----------------
    uint32_t mix_off[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      mix_off[j] = ((((uint32_t)lane >> 2) ^ (uint32_t)j) << 4) + (((uint32_t)lane & 3u) << 2);
    const size_t mix_block_stride = (size_t)a.n_out_planes * a.groups_stride * MLB_BLOCK;
    float* mix_row = a.mix_partial
                         ? a.mix_partial + ((size_t)a.out_plane * a.groups_stride + g) * MLB_BLOCK + lane
                         : nullptr;
    for (int b = 0; b < T; ++b)
    {
      const int s = b % S;
      const uint32_t blk = base + (uint32_t)s * kBlockBytes;
      named_bar_sync(id_flt + s, 64);  // F's rows of the block are written (and fenced for the async proxy)
      if (lane == 0 && a.write_out)
      {
        tma_store_4d(&out_map, blk, 0, v0, 0, b * a.n_out_planes + a.out_plane);
        bulk_commit();
      }
      if (a.mix_partial != nullptr)
      {
        // lane n sums sample column n over the 32 voice rows, rows in voice order, from +0 (reads only:
        // concurrent with the store's reads)
#pragma unroll 1
        for (int h = 0; h < 2; ++h)
        {
          const uint32_t tile = blk + (uint32_t)h * kTileBytes;
          float acc = 0.0f;
          if (full_group)
          {
#pragma unroll
            for (int r = 0; r < 32; ++r) acc = __fadd_rn(acc, lds32(tile + mix_off[r & 7] + (uint32_t)r * 128u));
          }
          else
          {
            for (int r = 0; r < 32; ++r)
              if (v0 + r < a.V) acc = __fadd_rn(acc, lds32(tile + mix_off[r & 7] + (uint32_t)r * 128u));
          }
          mix_row[h * kTileSamples] = acc;
        }
        mix_row += mix_block_stride;
      }
      if (lane == 0 && a.write_out) bulk_wait_read<0>();  // the store has drained its shared-memory reads
      __syncwarp();
      named_bar_arrive(id_free + s, 64);  // G may refill the stage
    }
    return;
  }

  uint32_t st[P::NS > 0 ? P::NS : 1];
  float co[P::NC > 0 ? P::NC : 1];
#pragma unroll
  for (int i = 0; i < P::NS; ++i) st[i] = live ? __ldcg(a.state + (size_t)a.st_idx[i] * a.v_stride + v) : 0u;
#pragma unroll
  for (int i = 0; i < P::NC; ++i) co[i] = live ? a.coef[(size_t)a.co_idx[i] * a.v_stride + v] : 0.0f;

  if (warp == 0)
  {
    // ---------------- G: TMA loads + generator ----------------
    auto issue_load = [&](int blk_t)  // lane 0, after the warp has synced on the stage's `free` barrier
    {
      const int s = blk_t % S;
      mbar_arrive_expect_tx(bar_full + 8u * s, kBlockBytes);
      tma_load_4d(base + (uint32_t)s * kBlockBytes, &in_map, bar_full + 8u * s, 0, v0, 0,
                  blk_t * a.n_in_planes + a.in_plane, kEvictFirst);
    };
    if (P::HAS_IN && lane == 0)
      for (int t = 0; t < LA && t < T; ++t) issue_load(t);
    long long g_wait = 0, g_comp = 0;
    for (int b = 0; b < T; ++b)
    {
      const int s = b % S, use = b / S;
      const uint32_t blk = base + (uint32_t)s * kBlockBytes;
      const long long c0 = a.prof ? clock64() : 0;
      if (P::HAS_IN)
      {
        if (b + LA < T)
        {
          if ((b + LA) / S > 0) named_bar_sync(id_free + (b + LA) % S, 64);  // the store of the previous use drained
          if (lane == 0) issue_load(b + LA);
        }
        mbar_wait(bar_full + 8u * s, (uint32_t)use & 1u);
      }
      else if (use > 0)
        named_bar_sync(id_free + s, 64);
      const long long c1 = a.prof ? clock64() : 0;
#pragma unroll 1
      for (int h = 0; h < 2; ++h)
      {
        const uint32_t tile = blk + (uint32_t)h * kTileBytes;
        float4 xin[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
          xin[j] = P::HAS_IN ? lds128(tile + row_off + (((uint32_t)j << 4) ^ sw)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 8; ++j)
        {
          xin[j].x = P::tick_gen(xin[j].x, st, co);
          xin[j].y = P::tick_gen(xin[j].y, st, co);
          xin[j].z = P::tick_gen(xin[j].z, st, co);
          xin[j].w = P::tick_gen(xin[j].w, st, co);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) sts128(tile + row_off + (((uint32_t)j << 4) ^ sw), xin[j]);
      }
      named_bar_arrive(id_gen + s, 64);  // the block's rows are written
      if (a.prof) g_wait += c1 - c0, g_comp += clock64() - c1;
    }
    if (a.prof && blockIdx.x == 0 && lane == 0) a.prof[0] = (unsigned long long)g_wait, a.prof[1] = (unsigned long long)g_comp;
#pragma unroll
    for (int i = 0; i < P::NS_GEN; ++i)
      if (live) __stcg(a.state + (size_t)a.st_idx[i] * a.v_stride + v, st[i]);
  }
  else
  {
    // ---------------- F: filter(s) + gain, nothing else ----------------
    long long f_wait = 0, f_comp = 0;
    for (int b = 0; b < T; ++b)
    {
      const int s = b % S;
      const uint32_t blk = base + (uint32_t)s * kBlockBytes;
      const long long c0 = a.prof ? clock64() : 0;
      named_bar_sync(id_gen + s, 64);
      const long long c1 = a.prof ? clock64() : 0;
#pragma unroll 1
      for (int h = 0; h < 2; ++h)
      {
        const uint32_t tile = blk + (uint32_t)h * kTileBytes;
        float4 xin[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) xin[j] = lds128(tile + row_off + (((uint32_t)j << 4) ^ sw));
#pragma unroll
        for (int j = 0; j < 8; ++j)
        {
          xin[j].x = P::tick_flt(xin[j].x, st, co);
          xin[j].y = P::tick_flt(xin[j].y, st, co);
          xin[j].z = P::tick_flt(xin[j].z, st, co);
          xin[j].w = P::tick_flt(xin[j].w, st, co);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) sts128(tile + row_off + (((uint32_t)j << 4) ^ sw), xin[j]);
      }
      fence_proxy_async();               // this lane's rows are visible to the TMA unit ...
      named_bar_arrive(id_flt + s, 64);  // ... before M hands the block to it
      if (a.prof) f_wait += c1 - c0, f_comp += clock64() - c1;
    }
    if (a.prof && blockIdx.x == 0 && lane == 0)
      a.prof[2] = (unsigned long long)f_wait, a.prof[3] = (unsigned long long)f_comp, a.prof[4] = 0ull;
#pragma unroll
    for (int i = P::NS_GEN; i < P::NS; ++i)
      if (live) __stcg(a.state + (size_t)a.st_idx[i] * a.v_stride + v, st[i]);
  }
}

// second stage of the mix bus.  Deterministic two-level sum (DESIGN.md "mix bus"):
//   chunk[c][n] = sum over the (up to) 64 group partials of chunk c, in group order, from +0
//   mix[p][n]   = sum over chunks c = 0..C-1, in order, from +0
// One CTA per plane, 64 x 16 threads: thread (n, w) owns chunks w, w+16, ...
constexpr int kMixChunkGroups = 64;  // 64 groups x 32 voices = 2048 voices per chunk

// Multi-GPU mix bus (DESIGN.md 6): the sum over voices continues over the GPUs of one box INSIDE this
// kernel, through peer memory over NVLink -- a one-shot all-reduce executed by the CTA that just finished
// plane p's local tree.  Every rank owns an exchange buffer xchg[2 parities][world][n_floats] and flags
// flag[2][world][n_planes]; peer r's buffer is mapped here as peers[r] (cudaIpc).  Protocol for plane p of
// call number `seq` (parity = seq & 1):
//   1. write my 64 local sums into slot [parity][my_rank] of EVERY rank's buffer (remote stores, 256 B rows);
//   2. __threadfence_system, then store-release flag[parity][my_rank][p] = seq on every rank;
//   3. wait until my own flag[parity][r][p] == seq for every r (acquire loads at system scope);
//   4. mix[p][n] = sum over r = 0..world-1, left to right from +0, of my slot [parity][r] -- the same order on
//      every rank, so all ranks hold bit-identical results (and the CPU checker reproduces it: shards in rank
//      order).
// A parity is reused two calls later; a peer can only get there after it has seen this rank's flags of the
// call in between, which this rank writes only after it finished reading: double buffering suffices.
// No rank ever waits for a peer to FINISH, only for its writes, and every rank launches the same sequence
// of kernels, so there is no circular wait.
constexpr int kMaxBusRanks = 16;
struct MixBusArgs
{
  float* xchg[kMaxBusRanks];     // [r]: rank r's exchange buffer (xchg[my_rank] is local memory)
  unsigned* flags[kMaxBusRanks];  // [r]: rank r's flag words
  int rank, world;
  unsigned seq;
  int n_floats;   // floats per slot (>= n_planes * 64 of this call)
  int n_planes_cap;  // planes per flag row
  // async mode: this kernel only leaves the local sums in `stage` (local memory, nothing on the caller's
  // stream touches a peer); mixbus_exchange_kernel on the bus's own stream runs steps 1-4 while the next
  // call's chain kernel already computes, then acknowledges on every rank; a post waits for the acks of the
  // call two before it (the previous user of this parity), which have normally long arrived.
  int async;
  float* stage;                  // this call's staging row block [n_floats] (one of four, local)
  unsigned* acks[kMaxBusRanks];  // [r]: rank r's ack words [2][world][n_planes_cap]
};

MLB_DEV unsigned ld_acquire_sys_u32(const unsigned* p)
{
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
MLB_DEV void st_release_sys_u32(unsigned* p, unsigned v)
{
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__global__ void __launch_bounds__(1024) mix_reduce_kernel(const float* __restrict__ partial,
                                                          float* __restrict__ chunk_scratch,
                                                          float* __restrict__ mix, int n_groups,
                                                          const MixBusArgs bus)
{
  const int p = blockIdx.x, n = threadIdx.x, w = threadIdx.y;
  const int n_chunks = (n_groups + kMixChunkGroups - 1) / kMixChunkGroups;
  const float* src = partial + (size_t)p * n_groups * MLB_BLOCK + n;
  float* scratch = chunk_scratch + (size_t)p * n_chunks * MLB_BLOCK + n;
  for (int c = w; c < n_chunks; c += blockDim.y)
  {
    const int g0 = c * kMixChunkGroups;
    const int g1 = min(g0 + kMixChunkGroups, n_groups);
    float acc = 0.0f;
    int g = g0;
    for (; g + 8 <= g1; g += 8)
    {
      float x[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] = src[(size_t)(g + i) * MLB_BLOCK];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc = __fadd_rn(acc, x[i]);
    }
    for (; g < g1; ++g) acc = __fadd_rn(acc, src[(size_t)g * MLB_BLOCK]);
    scratch[(size_t)c * MLB_BLOCK] = acc;
  }
  __syncthreads();  // also orders the global scratch writes within the CTA
  if (w != 0) return;
  float acc = 0.0f;
  for (int c = 0; c < n_chunks; ++c) acc = __fadd_rn(acc, scratch[(size_t)c * MLB_BLOCK]);
  if (bus.world <= 1)
  {
    mix[(size_t)p * MLB_BLOCK + n] = acc;
    return;
  }
  // ---- the sum continues over the GPUs of the box (threads (n, 0): two warps of this CTA) ----
  if (bus.async)
  {
    bus.stage[(size_t)p * MLB_BLOCK + n] = acc;
    return;
  }
  const unsigned parity = bus.seq & 1u;
  const size_t slot = ((size_t)parity * bus.world + bus.rank) * bus.n_floats + (size_t)p * MLB_BLOCK + n;
  for (int r = 0; r < bus.world; ++r) bus.xchg[r][slot] = acc;  // 1. my sums into everyone's buffer
  __threadfence_system();
  asm volatile("bar.sync 1, 64;" ::: "memory");  // both warps' stores are fenced before the flags go out
  if (n < bus.world)
  {
    const size_t f = ((size_t)parity * bus.world + bus.rank) * bus.n_planes_cap + p;
    st_release_sys_u32(bus.flags[n] + f, bus.seq);  // 2. one flag per destination rank
    // 3. wait for rank n's flag in MY memory
    const unsigned* mine = bus.flags[bus.rank] + ((size_t)parity * bus.world + n) * bus.n_planes_cap + p;
    while (ld_acquire_sys_u32(mine) != bus.seq) __nanosleep(40);
  }
  asm volatile("bar.sync 1, 64;" ::: "memory");
  __threadfence_system();
  const float* loc = bus.xchg[bus.rank] + (size_t)parity * bus.world * bus.n_floats + (size_t)p * MLB_BLOCK + n;
  float sum = 0.0f;
  for (int r = 0; r < bus.world; ++r) sum = __fadd_rn(sum, __ldcv(loc + (size_t)r * bus.n_floats));  // 4.
  mix[(size_t)p * MLB_BLOCK + n] = sum;
}

// the whole exchange (steps 1-4) for the async mode, on the bus's own stream: 256-thread CTAs, each 64-thread
// quarter owns one plane (few CTAs: this kernel runs beside the next call's chain kernel)
constexpr int kExchangePlanesPerCta = 4;
__global__ void __launch_bounds__(64 * kExchangePlanesPerCta) mixbus_exchange_kernel(float* __restrict__ mix,
                                                                                     const MixBusArgs bus, int n_planes)
{
  const int n = threadIdx.x & 63;
  const int p = blockIdx.x * kExchangePlanesPerCta + (threadIdx.x >> 6);
  const bool active = p < n_planes;
  const unsigned parity = bus.seq & 1u;
  // (polls its own memory with plain volatile loads at a relaxed pace and fences once after the flag showed up)
  if (active && bus.seq > 2u && n < bus.world)
  {
    // every rank has finished reading this parity's slots of call seq - 2
    const volatile unsigned* ack = bus.acks[bus.rank] + ((size_t)parity * bus.world + n) * bus.n_planes_cap + p;
    while ((int)(*ack - (bus.seq - 2u)) < 0) __nanosleep(100);
    __threadfence_system();
  }
  __syncthreads();
  const size_t slot = ((size_t)parity * bus.world + bus.rank) * bus.n_floats + (size_t)p * MLB_BLOCK + n;
  if (active)
  {
    const float acc = bus.stage[(size_t)p * MLB_BLOCK + n];
    for (int r = 0; r < bus.world; ++r) bus.xchg[r][slot] = acc;  // 1.
  }
  __threadfence_system();
  __syncthreads();
  if (active && n < bus.world)
  {
    st_release_sys_u32(bus.flags[n] + ((size_t)parity * bus.world + bus.rank) * bus.n_planes_cap + p, bus.seq);  // 2.
    const volatile unsigned* mine = bus.flags[bus.rank] + ((size_t)parity * bus.world + n) * bus.n_planes_cap + p;
    while (*mine != bus.seq) __nanosleep(100);  // 3.
    __threadfence_system();
  }
  __syncthreads();
  __threadfence_system();
  if (active)
  {
    const float* loc = bus.xchg[bus.rank] + (size_t)parity * bus.world * bus.n_floats + (size_t)p * MLB_BLOCK + n;
    float sum = 0.0f;
    for (int r = 0; r < bus.world; ++r) sum = __fadd_rn(sum, __ldcv(loc + (size_t)r * bus.n_floats));  // 4.
    mix[(size_t)p * MLB_BLOCK + n] = sum;
  }
  __syncthreads();  // every thread has read its column of every slot
  if (active && n < bus.world)
    st_release_sys_u32(bus.acks[n] + ((size_t)parity * bus.world + bus.rank) * bus.n_planes_cap + p, bus.seq);
}

}  // namespace mlb
