// cmix_b200/csrc/mixer_bulk.cuh
//
// The bulk mixer kernel: the three-layer gated mixer + SSE of one stream for a whole sub-chunk of bits
// (reference src/mixer/mixer.cpp:38-72, src/predictor.cpp:361-469, src/mixer/sse.cpp:243-328),
// one thread-block cluster of 2 CTAs per stream, warp-specialised. The arithmetic is mixer.cuh's,
// which documents the parity rules; this file is only about scheduling.
//
// Per coded bit the mixer touches 26*(2078+i) + 20*(29+i) + 49 = 55 172 fp32 weights twice (dot, then SGD).
// The cluster stays resident over the whole sub-chunk. CTA r keeps the currently selected weight rows of layer-0
// mixers [13r, 13r+13) in shared memory (13 x 8.4 KB): a row is read from HBM only when its selector context changes
// (16 of the 26 selectors change once per byte, not per bit) and written back only when it is evicted, so
// steady-state HBM traffic is well under the algorithmic 450 KB/bit. The parallelism is across the 13 serial chains
// of a CTA (13 lanes of one warp, conflict-free row pitch in shared memory) and across the other warps, which stage
// inputs, move rows and apply the SGD update.
//
// Per bit, a CTA's critical loop is
//     13 serial dot-product chains  ->  forward substitution through the extra inputs
//     ->  SGD coefficient  ->  (movers) SGD step  ->  next bit's chains,
// and the last arrow is pipelined: the 2104-float rows are cut into 8 chunks, the mover warps
// apply bit t-1's step chunk by chunk and publish chunk_seq[c], and the chain warp starts bit t's
// chain on chunk 0 as soon as that chunk carries the step - the update runs just ahead of the chain.
//
// Warp roles (roles are pinned to schedulers: the arbiter prefers high warp ids):
// * C warp (15): lanes 0..12 = the CTA's 13 layer-0 mixers. Chain out of shared memory with
//   LDS.128 ping-pong buffers and __fmul_rn products feeding one FADD chain per lane; then the
//   triangular extra-input substitution; then u = decay*lr*(sigma(p)-bit) with decay*lr
//   pre-computed by the movers (mixer.cpp:58-60).
// * mover warps (11): while bit t's chains run they plan bit t+1 - stage the 2078 inputs (triple
//   buffered, stretch LUT in shared memory), resolve every mixer's weight row, move rows whose
//   selector changed with the TMA (cp.async.bulk + mbarrier; bit-level selectors own a spare
//   buffer so the load never waits for the eviction), pre-compute the step-dependent learning
//   rate - then apply bit t's SGD step chunk by chunk.
// * T warp (14, CTA 0): layers 1 and 2, SSE and p_out, trailing by up to 4 bits behind a ring of
//   {value, sequence} slots; rows resident per lane, SSE candidate buckets prefetched a bit ahead.
// * CTA 0 publishes each clamped output the moment it exists (8-byte value+sequence "LL" slots
//   through distributed shared memory), so CTA 1's extra-input prefix overlaps CTA 0's loop and no
//   cluster barrier or cluster fence is ever executed inside the bit loop.
#pragma once
#include "jitter.cuh"
#include "mixer.cuh"

namespace cmixb200 {

enum { MIX_NBUF = 20, MIX_RING = 4, MIX_M_WARPS = 11, MIX_M_THREADS = MIX_M_WARPS * 32, MIX_CM = MIX_M_THREADS + 32,
       MIX_C_WARP = 15, MIX_T_WARP = 14,
       BAR_READY0 = 1, BAR_COEFF0 = 3, BAR_MOVERS = 5,     // named barriers; READY and COEFF alternate with the bit's parity
       ROW_PITCH_S = 2108,     // shared-memory row pitch: 527 float4 (odd) -> LDS.128 conflict-free across lanes
       K_SAME = 0, K_SWAP = 1, K_LATE_SWITCH = 3, T_ELEMS = 819 };

__device__ __forceinline__ void named_sync(int id, int count, int site) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); jit_point(site); }
__device__ __forceinline__ void named_arrive(int id, int count, int site) { jit_point(site); asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void spin_until_ge(volatile u32* p, u32 v, int site) {
  while (*p < v) { }
  jit_point(site);
}

// "LL" message slots (as in NCCL's low-latency protocol): a float and its sequence number are written
// with one 8-byte store, so the consumer needs no fence - it polls the slot until the sequence matches.
// (A cluster-scope fence costs an L1 invalidate + a drain of the warp's outstanding global stores.)
__device__ __forceinline__ void ll_store(uint2* slot, float v, u32 seq) {
  *reinterpret_cast<volatile unsigned long long*>(slot) = ((unsigned long long)seq << 32) | (unsigned long long)__float_as_uint(v);
}
__device__ __forceinline__ float ll_wait(const uint2* slot, u32 seq, int site) {
  unsigned long long m;
  do { m = *reinterpret_cast<const volatile unsigned long long*>(slot); } while ((u32)(m >> 32) != seq);
  jit_point(site);
  return __uint_as_float((u32)m);
}

// ---- TMA (bulk async copy) helpers: one instruction moves a whole 8.4 KB weight row ----
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity, int site) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "W: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra W;\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
  jit_point(site);
}
__device__ __forceinline__ void tma_load_row(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_row(void* gmem_dst, const void* smem_src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}

// Selectors that change every bit: their mixers get a spare row buffer.
__device__ __forceinline__ bool selector_is_bit_level(int sel) {
  return sel == S_AUX || sel == S_LONGBIT || (sel >= S_BC0 && sel <= S_BC_RB1);
}

// A row move of the movers: write buffer `buf` back to row evict_slot and/or fill it from row load_slot.
struct RowJob { int buf; int mixer; u32 load_slot; u32 evict_slot; int do_evict; int do_load; };

struct MixBulkShared {
  alignas(16) float rows[MIX_NBUF][ROW_PITCH_S];
  alignas(16) float x[3][N_INPUTS + 2];
  // plan of bit t (parity t&1): movers -> chain warp
  int plan_buf[2][16]; float plan_dl[2][16]; u32 plan_shrink[2][16];
  // results of bit t (parity t&1): chain warp -> movers
  float upd[2][16]; float cext[2][32];
  // mover bookkeeping
  int buf_cur[16], buf_alt[16]; u32 tag[MIX_NBUF]; u32 dirty[MIX_NBUF]; u64 steps[MIX_NBUF]; u64 max_steps[16];
  u32 want[16]; u32 kind[16]; int mupd[16]; int n_late;
  RowJob jobs[32]; int n_jobs;
  u32 sel[2][SEL_PITCH];
  alignas(8) unsigned long long row_bar; u32 row_bar_phase;
  // messages
  alignas(8) uint2 ring_in[MIX_RING][16];
  alignas(8) uint2 ring_t[MIX_RING][32];
  volatile u32 peer_progress, t_consumed;
  volatile u32 chunk_seq[8];                 // chunk c carries every SGD step of bits < chunk_seq[c]
  // T warp
  float in1[L1_IN + 3], in2[L2_IN + 3];
  alignas(16) float l1row[N_L1 + 1][ROW_PITCH_L1];     // row 20 = the layer-2 mixer
  float l1extra[N_L1 + 4]; float tu[N_L1 + 4]; u32 tshr[N_L1 + 4];
  unsigned short emap[T_ELEMS + 5];
  float lut12[4100];
};

// Per-phase cycle accounting into ChunkArgs::prof (debug; tools/gpu_prof.py reads slots 8-30). BAR.SYNC does not
// block at issue, so a clock read placed right after a barrier would capture the issue time; a dependent
// shared-memory load + MOV in front of the clock read makes the sample wait for the barrier's release.
#define MIX_PROF(cond, slot) do { if (cond) { \
    unsigned dummy_ = *reinterpret_cast<volatile unsigned*>(&sh.n_jobs), sink_; \
    asm volatile("mov.u32 %0, %1;" : "=r"(sink_) : "r"(dummy_)); \
    const long long now_ = clock64(); pacc[(slot) & 7] += (unsigned long long)(now_ - tprev) + (sink_ & 0u); tprev = now_; } } while (0)
#define MIX_PROF_DUMP(cond, base, n) do { if (cond) { for (int q_ = 0; q_ < (n); ++q_) a.prof[(base) + q_] += pacc[((base) + q_) & 7]; } } while (0)

// movers: apply the SGD step of one bit, chunk c only, to the rows listed in sh.mupd (-1 = none).
// Work item = (row, half chunk of 32 float4): one warp instruction stream per item, no index division.
__device__ __forceinline__ void movers_update_chunk(MixBulkShared& sh, int m0, int mwarp, int lane, int par_prev, const float* xprev, int c) {
  const float4* xp4 = reinterpret_cast<const float4*>(xprev);
#pragma unroll 1
  for (int item = mwarp; item < 2 * MIX_PER_CTA; item += MIX_M_WARPS) {
    const int i = item >> 1, half = item & 1;
    const int b = sh.mupd[i];
    if (b < 0) continue;
    const float u = sh.upd[par_prev][i];
    const bool shr = sh.plan_shrink[par_prev][i] != 0;
    float4* row4 = reinterpret_cast<float4*>(sh.rows[b]);
    {
      const int k4 = c * MIX_CHUNK4 + half * 32 + lane;
      const float4 xv = xp4[k4];
      sgd_step4(row4[k4], u, xv, shr);
    }
    if (c == MIX_CHUNKS - 1 && half == 1) {
      // leftovers of the row: float4 512..518, scalars 2076/2077 and this mixer's extra-input weights
      if (lane < 7) {
        const int k4 = 512 + lane;
        const float4 xv = xp4[k4];
        sgd_step4(row4[k4], u, xv, shr);
      } else {
        const int n = N_INPUTS + m0 + i;
        float* row = sh.rows[b];
#pragma unroll 1
        for (int k = 2076 + (lane - 7); k < n; k += 25) {   // lanes 7..31 sweep elements 2076 .. n-1
          const float xin = k < N_INPUTS ? xprev[k] : sh.cext[par_prev][k - N_INPUTS];
          sgd_step(row[k], u, xin, shr);
        }
      }
    }
  }
}
// all chunks; after chunk c is complete the chain warp of bit `seq` may read it
__device__ __forceinline__ void movers_update(MixBulkShared& sh, int m0, int mtid, int par_prev, const float* xprev, u32 seq) {
#pragma unroll 1
  for (int c = 0; c < MIX_CHUNKS; ++c) {
    movers_update_chunk(sh, m0, mtid >> 5, mtid & 31, par_prev, xprev, c);
    named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
    if (mtid == 0) sh.chunk_seq[c] = seq;
  }
}

// movers: run sh.jobs through the TMA - evictions first (bulk stores, waited for until their reads of shared
// memory are done), then every load on one mbarrier; threads 32.. move the rows' step counters alongside.
__device__ __forceinline__ void run_row_jobs(MixBulkShared& sh, StreamState* st, int m0, int mtid) {
  const int nj = sh.n_jobs;
  if (nj == 0) return;
  if (mtid == 0) {
    const unsigned bytes = ROW_PITCH_L0 * 4;
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    bool any_evict = false, any_load = false;
#pragma unroll 1
    for (int j = 0; j < nj; ++j) { any_evict |= sh.jobs[j].do_evict != 0; any_load |= sh.jobs[j].do_load != 0; }
    if (any_evict) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#pragma unroll 1
      for (int j = 0; j < nj; ++j) {
        const RowJob jb = sh.jobs[j];
        if (jb.do_evict) tma_store_row(st->mixer[m0 + jb.mixer].rows + (size_t)jb.evict_slot * ROW_PITCH_L0, sh.rows[jb.buf], bytes);
      }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
    if (any_load) {
      unsigned total = 0;
#pragma unroll 1
      for (int j = 0; j < nj; ++j) if (sh.jobs[j].do_load) total += bytes;
      mbar_expect_tx(&sh.row_bar, total);
#pragma unroll 1
      for (int j = 0; j < nj; ++j) {
        const RowJob jb = sh.jobs[j];
        if (jb.do_load) tma_load_row(sh.rows[jb.buf], st->mixer[m0 + jb.mixer].rows + (size_t)jb.load_slot * ROW_PITCH_L0, bytes, &sh.row_bar);
      }
    }
  }
  if (mtid >= 32 && mtid < 32 + nj) {
    const RowJob jb = sh.jobs[mtid - 32];
    MixerState& m = st->mixer[m0 + jb.mixer];
    if (jb.do_evict) m.row_steps[jb.evict_slot] = sh.steps[jb.buf];
    if (jb.do_load) { sh.steps[jb.buf] = m.row_steps[jb.load_slot]; sh.tag[jb.buf] = jb.load_slot; sh.dirty[jb.buf] = 0; }
  }
  if (mtid == 0) {
    bool any_load = false;
#pragma unroll 1
    for (int j = 0; j < nj; ++j) any_load |= sh.jobs[j].do_load != 0;
    if (any_load) { mbar_wait(&sh.row_bar, sh.row_bar_phase & 1, JIT_HERE); sh.row_bar_phase++; }
  }
  named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
}

// movers: the learning-rate factor of bit t for local mixer i, on the step counters kept in shared memory
__device__ __forceinline__ void plan_rate(MixBulkShared& sh, int par, int i, float decay, float lr) {
  const int b = sh.plan_buf[par][i];
  const u64 rs = sh.steps[b], ms = sh.max_steps[i];
  sh.plan_dl[par][i] = mixer_rate(decay, lr, rs, ms);
  mixer_step(rs, ms, sh.steps[b], sh.max_steps[i], sh.plan_shrink[par][i]);
  sh.dirty[b] = 1;
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(MIX_THREADS, 1)
mix_kernel_v3(const ChunkArgs* __restrict__ args_all, Tables T) { jit_entry(JK_MIX);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const ChunkArgs a = args_all[blockIdx.x / 2];
  StreamState* st = a.st;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MixBulkShared& sh = *reinterpret_cast<MixBulkShared*>(smem_raw);
  MixBulkShared* sh0 = cluster.map_shared_rank(&sh, 0);
  MixBulkShared* sh1 = cluster.map_shared_rank(&sh, 1);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = rank * MIX_PER_CTA;
  const u64 n_bits = (u64)a.n_bytes * 8;

  if (tid == 0) {
    int next = MIX_PER_CTA;
    for (int i = 0; i < MIX_PER_CTA; ++i) {
      sh.buf_cur[i] = i;
      sh.buf_alt[i] = -1;
      if (selector_is_bit_level(st->mixer[m0 + i].sel) && next < MIX_NBUF) sh.buf_alt[i] = next++;
      sh.max_steps[i] = st->mixer[m0 + i].max_steps;
      sh.mupd[i] = -1;
    }
    for (int b = 0; b < MIX_NBUF; ++b) { sh.tag[b] = 0xffffffffu; sh.dirty[b] = 0; sh.steps[b] = 0; }
    for (int r = 0; r < MIX_RING; ++r) for (int k = 0; k < 32; ++k) { sh.ring_t[r][k] = make_uint2(0, 0); if (k < 16) sh.ring_in[r][k] = make_uint2(0, 0); }
    sh.peer_progress = 0; sh.t_consumed = 0; sh.n_jobs = 0; sh.row_bar_phase = 0; sh.n_late = 0;
    for (int c = 0; c < 8; ++c) sh.chunk_seq[c] = 0;
    mbar_init(&sh.row_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    int e = 0;
    for (int i = 0; i <= N_L1; ++i) { const int n = i < N_L1 ? L1_IN + i : L2_IN; for (int c = 0; c < n; ++c) sh.emap[e++] = (unsigned short)((i << 8) | c); }
  }
  for (int k = tid; k < 4097; k += MIX_THREADS) sh.lut12[k] = T.lut12[k];
  JIT_SYNCTHREADS();
  jit_cluster_sync(cluster, JIT_HERE);

  if (warp == MIX_C_WARP) {
    // =============================== C warp ===============================
    const bool pc_on = a.prof != nullptr && lane == 0; const int pb = rank == 0 ? 8 : 14;
    unsigned long long pacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long tprev = clock64();
    float u_prev = 0.0f;
    for (u64 t = 0; t < n_bits; ++t) {
      const int par = (int)(t & 1), r = (int)(t & (MIX_RING - 1));
      const int bit = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
      named_sync(BAR_READY0 + par, MIX_CM, JIT_HERE);
      MIX_PROF(pc_on, pb + 0);
      const float* x = sh.x[t % 3];
      float* row = sh.rows[lane < MIX_PER_CTA ? sh.plan_buf[par][lane] : 0];
      const float dl = lane < MIX_PER_CTA ? sh.plan_dl[par][lane] : 0.0f;
      float main = 0.0f;
      {
        const float4* x4 = reinterpret_cast<const float4*>(x);
        const float4* w4 = reinterpret_cast<const float4*>(row);
#pragma unroll 1
        for (int c = 0; c < MIX_CHUNKS; ++c) {
          while (sh.chunk_seq[c] < (u32)t) { }            // the movers have applied bit t-1's step to this chunk
          jit_point(JIT_HERE);
          if (lane < MIX_PER_CTA) main = chain_chunk(x4, w4, c * MIX_CHUNK4, chain_chunk_end(c), main);
        }
        if (lane < MIX_PER_CTA) main = chain_tail(x, row, main);
      }
      __syncwarp();
      MIX_PROF(pc_on, pb + 1);
      // ---- forward substitution through the extra inputs ----
      // (substitute() in mixer.cuh is the same recurrence on one warp; here the 26 mixers are split over the two CTAs,
      // CTA 1 first folds in CTA 0's 13 outputs, and each output is published to the peer and the T warp as it appears)
      float e = 0.0f, pfin = 0.0f, cmine = 0.0f;
      int kbase = 0;
      if (rank == 1) {
#pragma unroll 1
        for (int k = 0; k < MIX_PER_CTA; ++k) {
          const float ck = ll_wait(&sh.ring_in[r][k], (u32)(t + 1), JIT_HERE);
          if (lane == k) sh.cext[par][k] = ck;
          if (lane < MIX_PER_CTA) e = XM_FADD(e, XM_FMUL(ck, row[N_INPUTS + k]));
        }
        if (lane == 0) sh0->peer_progress = (u32)(t + 1);
        kbase = MIX_PER_CTA;
      } else {
        if (lane == 0 && t >= MIX_RING) { spin_until_ge(&sh.peer_progress, (u32)(t + 1 - MIX_RING), JIT_HERE); spin_until_ge(&sh.t_consumed, (u32)(t + 1 - MIX_RING), JIT_HERE); }
        __syncwarp();
      }
      if (rank == 1 && lane == 0 && t >= MIX_RING) spin_until_ge(&sh.t_consumed, (u32)(t + 1 - MIX_RING), JIT_HERE);
      __syncwarp();
      MIX_PROF(pc_on, pb + 2);
      float wnext = lane < MIX_PER_CTA ? row[N_INPUTS + kbase] : 0.0f;
#pragma unroll 1
      for (int k = 0; k < MIX_PER_CTA; ++k) {
        if (lane == k) pfin = XM_FADD(main, e);
        const float pk = __shfl_sync(0xffffffffu, pfin, k);
        const float ck = clamp_stretched(T, pk);
        const float wk = wnext;
        if (lane < MIX_PER_CTA && k + 1 < MIX_PER_CTA) wnext = row[N_INPUTS + kbase + k + 1];
        if (lane == k) {
          cmine = ck;
          if (rank == 0) { ll_store(&sh1->ring_in[r][k], ck, (u32)(t + 1)); ll_store(&sh.ring_t[r][k], ck, (u32)(t + 1)); }
          else ll_store(&sh0->ring_t[r][MIX_PER_CTA + k], ck, (u32)(t + 1));
        }
        if (lane > k && lane < MIX_PER_CTA) e = XM_FADD(e, XM_FMUL(ck, wk));
      }
      MIX_PROF(pc_on, pb + 3);
      // ---- coefficient: the movers pre-computed decay*lr; only the logistic is left (mixer.cpp:60) ----
      if (lane < MIX_PER_CTA) {
        u_prev = sgd_coeff(dl, pfin, bit);
        sh.upd[par][lane] = u_prev;
        sh.cext[par][m0 + lane] = cmine;
      } else if (rank == 0 && lane < MIX_PER_CTA + 3) {
        const int idx = lane == MIX_PER_CTA ? 433 : (lane == MIX_PER_CTA + 1 ? 2024 : 2077);
        ll_store(&sh.ring_t[r][N_L0 + (lane - MIX_PER_CTA)], clamp_stretched(T, x[idx]), (u32)(t + 1));
      }
      __syncwarp();
      MIX_PROF(pc_on, pb + 4);
      named_arrive(BAR_COEFF0 + par, MIX_CM, JIT_HERE);
      MIX_PROF(pc_on, pb + 5);
    }
    MIX_PROF_DUMP(pc_on, pb, 6);
  } else if (warp < MIX_T_WARP && (warp & 3) != 3) {
    // =============================== M warps ===============================
    const int mtid = (warp - (warp >> 2)) * 32 + lane;
    const bool pm_on = a.prof != nullptr && mtid == 0 && rank == 0;
    unsigned long long pacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long tprev = clock64();
    const float my_lr = mtid < MIX_PER_CTA ? st->mixer[m0 + mtid].lr : 0.0f;
    for (u64 t = 0; t <= n_bits; ++t) {
      const int par = (int)(t & 1), parp = par ^ 1;
      bool coeff_synced = (t == 0);
      if (t < n_bits) {
        // ---- plan bit t ----
        if (mtid < SEL_PITCH) sh.sel[par][mtid] = mtid < N_MIXERS ? a.sel[t * SEL_PITCH + mtid] : 0;
        if (mtid >= 64 && mtid < 64 + MIX_PER_CTA && !(rank == 0 && mtid - 64 == 12))
          sh.want[mtid - 64] = resolve_slot(st->mixer[m0 + mtid - 64], a.sel[t * SEL_PITCH + m0 + mtid - 64]);
        stage_inputs<MIX_M_THREADS>(sh.x[t % 3], sh.lut12, a.ext ? a.ext + t * N_EXT : nullptr, a.small_x + t * SMALL_X_PITCH, a.lstm_x[2 * t], mtid);
        named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
        MIX_PROF(pm_on, 20);
        if (mtid == 0) {
          if (rank == 0) { const u32 ax = aux_context(sh.x[t % 3]); sh.sel[par][12] = ax; sh.want[12] = resolve_slot(st->mixer[12], ax); }
          int nj = 0, nlate = 0;
#pragma unroll 1
          for (int i = 0; i < MIX_PER_CTA; ++i) {
            const u32 s = sh.want[i];
            const int cur = sh.buf_cur[i], alt = sh.buf_alt[i];
            sh.mupd[i] = -1;
            if (sh.tag[cur] == s) {
              sh.kind[i] = K_SAME;
              sh.plan_buf[par][i] = cur;
              if (t > 0) sh.mupd[i] = cur;          // applied chunk by chunk just ahead of the chain
            } else if (alt >= 0) {
              sh.kind[i] = K_SWAP;
              sh.plan_buf[par][i] = alt;
              if (t > 0) sh.mupd[i] = cur;          // its pending step is applied by the movers, off the critical path
              if (sh.tag[alt] != s) {
                RowJob jb; jb.buf = alt; jb.mixer = i; jb.load_slot = s; jb.evict_slot = sh.tag[alt];
                jb.do_evict = (sh.tag[alt] != 0xffffffffu && sh.dirty[alt]) ? 1 : 0; jb.do_load = 1;
                sh.jobs[nj++] = jb;
              }
              sh.buf_cur[i] = alt; sh.buf_alt[i] = cur;
            } else {
              sh.kind[i] = K_LATE_SWITCH;
              ++nlate;
              sh.plan_buf[par][i] = cur;
            }
          }
          sh.n_jobs = nj; sh.n_late = nlate;
        }
        named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
        MIX_PROF(pm_on, 21);
        run_row_jobs(sh, st, m0, mtid);
        const float decay = a.decay[t];
        if (mtid < MIX_PER_CTA && sh.kind[mtid] != K_LATE_SWITCH) plan_rate(sh, par, mtid, decay, my_lr);
        named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
        MIX_PROF(pm_on, 22);
        if (sh.n_late) {
          // rows that must carry bit t-1's step BEFORE bit t's chain: shrink due, or single-buffered switch
          if (t > 0) { named_sync(BAR_COEFF0 + parp, MIX_CM, JIT_HERE); coeff_synced = true; }
          if (mtid < MIX_PER_CTA) {
            if (t > 0 && sh.kind[mtid] == K_LATE_SWITCH && sh.tag[sh.buf_cur[mtid]] != 0xffffffffu) sh.mupd[mtid] = sh.buf_cur[mtid];
          }
          named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
          if (t > 0) movers_update(sh, m0, mtid, parp, sh.x[(t + 2) % 3], (u32)t);
          named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
          if (mtid == 0) {
            int nj = 0;
#pragma unroll 1
            for (int i = 0; i < MIX_PER_CTA; ++i) {
              if (sh.kind[i] == K_LATE_SWITCH) {
                const int cur = sh.buf_cur[i];
                RowJob jb; jb.buf = cur; jb.mixer = i; jb.load_slot = sh.want[i]; jb.evict_slot = sh.tag[cur];
                jb.do_evict = (sh.tag[cur] != 0xffffffffu && sh.dirty[cur]) ? 1 : 0; jb.do_load = 1;
                sh.jobs[nj++] = jb;
              }
              sh.mupd[i] = -1;                     // every pending step was applied just above
            }
            sh.n_jobs = nj;
          }
          named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
          run_row_jobs(sh, st, m0, mtid);
          if (mtid < MIX_PER_CTA && sh.kind[mtid] == K_LATE_SWITCH) plan_rate(sh, par, mtid, decay, my_lr);
          named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
        }
        MIX_PROF(pm_on, 23);
        named_arrive(BAR_READY0 + par, MIX_CM, JIT_HERE);
      }
      // ---- bit t-1's step for the rows that were switched away (or, at the end, for all rows) ----
      if (t > 0) {
        if (!coeff_synced) named_sync(BAR_COEFF0 + parp, MIX_CM, JIT_HERE);
        MIX_PROF(pm_on, 24);
        if (t == n_bits) { if (mtid < MIX_PER_CTA) sh.mupd[mtid] = sh.buf_cur[mtid]; named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE); }
        movers_update(sh, m0, mtid, parp, sh.x[(t + 2) % 3], (u32)t);
        MIX_PROF(pm_on, 25);
      }
    }
    MIX_PROF_DUMP(pm_on, 20, 6);
    // ---- epilogue: write every dirty resident row back ----
    if (mtid == 0) {
      int nj = 0;
#pragma unroll 1
      for (int i = 0; i < MIX_PER_CTA; ++i) {
#pragma unroll 1
        for (int w = 0; w < 2; ++w) {
          const int b = w == 0 ? sh.buf_cur[i] : sh.buf_alt[i];
          if (b < 0 || sh.tag[b] == 0xffffffffu || !sh.dirty[b]) continue;
          RowJob jb; jb.buf = b; jb.mixer = i; jb.load_slot = 0; jb.evict_slot = sh.tag[b]; jb.do_evict = 1; jb.do_load = 0;
          sh.jobs[nj++] = jb;
        }
        st->mixer[m0 + i].max_steps = sh.max_steps[i];
      }
      sh.n_jobs = nj;
    }
    named_sync(BAR_MOVERS, MIX_M_THREADS, JIT_HERE);
    run_row_jobs(sh, st, m0, mtid);
    if (mtid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  } else if (rank == 0 && warp == MIX_T_WARP) {
    // =============================== T warp ===============================
    SseState& sse = st->sse;
    u32 sj = sse.j, spc = sse.pc, sffl = sse.ffl;
    const u16* __restrict__ tst = sse.st; const u16* __restrict__ tsq = sse.sq;
    const int mi = lane < N_L1 + 1 ? lane : 0;
    MixerState& mym = st->mixer[N_L0 + mi];
    float* const myrows = mym.rows; u64* const mysteps = mym.row_steps; u32* const mytable = mym.slot_table;
    const float mylr = mym.lr;
    u64 my_max = mym.max_steps; u32 my_assigned = mym.n_assigned; const u32 my_nrows = mym.n_rows;
    const bool pt_on = a.prof != nullptr && lane == 0;
    unsigned long long pacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long tprev = clock64();
    u32 myslot = 0xffffffffu; u64 my_rs = 0;
    u32 ctx_next = lane < N_L1 + 1 ? a.sel[N_L0 + lane] : 0;
    u32 sl_next = lane < N_L1 + 1 ? mytable[ctx_next] : 0;
    for (u64 t = 0; t < n_bits; ++t) {
      const int r = (int)(t & (MIX_RING - 1));
      const int bit = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
      // ---- candidate SSE buckets for every possible quantisation of p (sse.cpp:250-270) ----
      uint4 cand = make_uint4(0, 0, 0, 0); size_t cand_idx = 0;
      if (lane < 3) {
        cand_idx = sse_i6(lane, sj, spc, sffl);
        cand = *reinterpret_cast<const uint4*>(sse.s6 + cand_idx * 8);
      } else if (lane < 6) {
        cand_idx = sse_i7(lane - 3, sj, spc, sffl);
        cand = *reinterpret_cast<const uint4*>(sse.s7 + cand_idx * 8);
      } else if (lane < 9) {
        cand_idx = sse_ix2(lane - 6, sj, spc, sffl);
        cand.x = (u32)sse.x2[cand_idx];
      } else if (lane < 13) {
        cand_idx = sse_ix1(lane - 9, sj, spc, sffl);
        cand.x = (u32)sse.x1[cand_idx];
      }
      const float decay = a.decay[t];
      const float ov = a.lstm_x[2 * t + 1];
      // ---- rows of layers 1/2 (resident per lane; table look-up issued one bit ahead) ----
      if (lane < N_L1 + 1) {
        const u32 ctx = ctx_next;
        u32 sl = sl_next;
        if (sl == 0) sl = mytable[ctx];               // may have been assigned since the look-ahead read
        sl = assign_row(mytable, ctx, sl, my_assigned, my_nrows);
        if (t + 1 < n_bits) { ctx_next = a.sel[(t + 1) * SEL_PITCH + N_L0 + lane]; sl_next = mytable[ctx_next]; }
        const u32 want = sl - 1;
        if (want != myslot) {
          float4* srow = reinterpret_cast<float4*>(sh.l1row[lane]);
          if (myslot != 0xffffffffu) {
            float4* g = reinterpret_cast<float4*>(myrows + (size_t)myslot * ROW_PITCH_L1);
#pragma unroll
            for (int q = 0; q < ROW_PITCH_L1 / 4; ++q) g[q] = srow[q];
            mysteps[myslot] = my_rs;
          }
          const float4* g = reinterpret_cast<const float4*>(myrows + (size_t)want * ROW_PITCH_L1);
          float4 tmp[ROW_PITCH_L1 / 4];
#pragma unroll
          for (int q = 0; q < ROW_PITCH_L1 / 4; ++q) tmp[q] = g[q];
          my_rs = mysteps[want];
#pragma unroll
          for (int q = 0; q < ROW_PITCH_L1 / 4; ++q) srow[q] = tmp[q];
          myslot = want;
        }
      }
      __syncwarp();
      MIX_PROF(pt_on, 26);
      {
        float c = 0.0f;
        if (lane < N_L0 + N_AUX) c = ll_wait(&sh.ring_t[r][lane], (u32)(t + 1), JIT_HERE);
        if (lane < N_L0) { sh.in1[lane] = c; sh.in2[lane] = c; }
        else if (lane < N_L0 + N_AUX) { sh.in1[lane] = c; sh.in2[N_L1 + lane] = c; }
      }
      __syncwarp();
      MIX_PROF(pt_on, 27);
      if (lane == 0) { sh.t_consumed = (u32)(t + 1); sh1->t_consumed = (u32)(t + 1); }
      float pfin = layer1_forward(sh.l1row[lane], sh.in1, sh.l1extra, sh.in2, T, lane);
      __syncwarp();
      MIX_PROF(pt_on, 28);
      float s2 = 0.0f;
      if (lane == N_L1) {
        s2 = layer2_forward(sh.l1row[N_L1], sh.in2);
        pfin = s2;
      }
      s2 = __shfl_sync(0xffffffffu, s2, N_L1);
      // ---- SSE (sse.cpp:243-289) on the prefetched buckets ----
      int q3, q4;
      const int discrete = sse_quantise(xm_logistic(s2), q3, q4);
      const uint4 b6 = make_uint4(__shfl_sync(0xffffffffu, cand.x, q3), __shfl_sync(0xffffffffu, cand.y, q3),
                                  __shfl_sync(0xffffffffu, cand.z, q3), __shfl_sync(0xffffffffu, cand.w, q3));
      const uint4 b7 = make_uint4(__shfl_sync(0xffffffffu, cand.x, 3 + q3), __shfl_sync(0xffffffffu, cand.y, 3 + q3),
                                  __shfl_sync(0xffffffffu, cand.z, 3 + q3), __shfl_sync(0xffffffffu, cand.w, 3 + q3));
      int wx2 = (int)__shfl_sync(0xffffffffu, cand.x, 6 + q3);
      int wx1 = (int)__shfl_sync(0xffffffffu, cand.x, 9 + q4);
      const size_t i6 = __shfl_sync(0xffffffffu, (unsigned long long)cand_idx, q3);
      const size_t i7 = __shfl_sync(0xffffffffu, (unsigned long long)cand_idx, 3 + q3);
      const size_t ix2 = __shfl_sync(0xffffffffu, (unsigned long long)cand_idx, 6 + q3);
      const size_t ix1 = __shfl_sync(0xffffffffu, (unsigned long long)cand_idx, 9 + q4);
      if (lane == 0) {
        SseCarry sc;
        u16 k6[8] = {(u16)b6.x, (u16)(b6.x >> 16), (u16)b6.y, (u16)(b6.y >> 16), (u16)b6.z, (u16)(b6.z >> 16), (u16)b6.w, (u16)(b6.w >> 16)};
        u16 k7[8] = {(u16)b7.x, (u16)(b7.x >> 16), (u16)b7.y, (u16)(b7.y >> 16), (u16)b7.z, (u16)(b7.z >> 16), (u16)b7.w, (u16)(b7.w >> 16)};
        const float p = sse_estimate(sc, tst, tsq, discrete, k6, k7, wx1, wx2);
        a.p_out[t] = ov >= 0.0f ? ov : p;
        sse_learn(sc, bit, k6, k7, &wx1, &wx2);
        u16* g6 = sse.s6 + i6 * 8; g6[sc.q6] = k6[sc.q6]; g6[sc.q6 + 1] = k6[sc.q6 + 1];
        u16* g7 = sse.s7 + i7 * 8; g7[sc.q7] = k7[sc.q7]; g7[sc.q7 + 1] = k7[sc.q7 + 1];
        sse.x1[ix1] = wx1; sse.x2[ix2] = wx2;
      }
      MIX_PROF(pt_on, 29);
      sse_advance(sj, spc, sffl, bit);
      // ---- SGD of layers 1/2 (mixer.cpp:56-72): coefficients per lane, then a flat (row, column) sweep ----
      if (lane < N_L1 + 1) {
        u32 shr;
        sh.tu[lane] = sgd_coeff(mixer_rate(decay, mylr, my_rs, my_max), pfin, bit);
        mixer_step(my_rs, my_max, my_rs, my_max, shr);
        sh.tshr[lane] = shr;
      }
      __syncwarp();
#pragma unroll 2
      for (int el = lane; el < T_ELEMS; el += 32) {
        const int i = sh.emap[el] >> 8, c = sh.emap[el] & 255;
        const float xin = i < N_L1 ? (c < L1_IN ? sh.in1[c] : sh.l1extra[c - L1_IN]) : sh.in2[c];
        sgd_step(sh.l1row[i][c], sh.tu[i], xin, sh.tshr[i]);
      }
      __syncwarp();
      MIX_PROF(pt_on, 30);
    }
    MIX_PROF_DUMP(pt_on, 26, 5);
    if (lane < N_L1 + 1) {
      if (myslot != 0xffffffffu) {
        const float* srow = sh.l1row[lane];
        float* g = myrows + (size_t)myslot * ROW_PITCH_L1;
        for (int q = 0; q < ROW_PITCH_L1; ++q) g[q] = srow[q];
        mysteps[myslot] = my_rs;
      }
      mym.max_steps = my_max; mym.n_assigned = my_assigned;
    }
    if (lane == 0) { sse.j = sj; sse.pc = spc; sse.ffl = sffl; st->bits_done += n_bits; }
  }
  JIT_SYNCTHREADS();
  jit_cluster_sync(cluster, JIT_HERE);
}

}  // namespace cmixb200
