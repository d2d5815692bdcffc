// cmix_b200/csrc/mixer_v3.cuh
//
// Kernel "mix" v3: the three-layer gated mixer + SSE of one stream for a whole sub-chunk of bits
// (reference src/mixer/mixer.cpp:38-72, src/predictor.cpp:361-469, src/mixer/sse.cpp:243-328),
// one thread-block cluster of 2 CTAs per stream, warp-specialised. Same arithmetic as mixer.cuh,
// which documents the parity rules; this file is only about scheduling.
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
#include "mixer_prims.cuh"

namespace cmixb200 {

enum { V3_NBUF = 20, V3_RING = 4, V3_M_WARPS = 11, V3_M_THREADS = V3_M_WARPS * 32, V3_CM = V3_M_THREADS + 32,
       B3_READY0 = 1, B3_COEFF0 = 3, B3_MOVERS = 5,
       K_SAME = 0, K_SWAP = 1, K_LATE_SAME = 2, K_LATE_SWITCH = 3, T_ELEMS = 819 };

struct MixShared3 {
  alignas(16) float rows[V3_NBUF][ROW_PITCH_S];
  alignas(16) float x[3][N_INPUTS + 2];
  // plan of bit t (parity t&1): movers -> chain warp
  int plan_buf[2][16]; float plan_dl[2][16]; u32 plan_shrink[2][16];
  // results of bit t (parity t&1): chain warp -> movers
  float upd[2][16]; float cext[2][32];
  // mover bookkeeping
  int buf_cur[16], buf_alt[16]; u32 tag[V3_NBUF]; u32 dirty[V3_NBUF]; u64 steps[V3_NBUF]; u64 max_steps[16];
  u32 want[16]; u32 kind[16]; int mupd[16]; int n_late;
  RowJob jobs[32]; int n_jobs;
  u32 sel[2][SEL_PITCH];
  alignas(8) unsigned long long row_bar; u32 row_bar_phase;
  // messages
  alignas(8) uint2 ring_in[V3_RING][16];
  alignas(8) uint2 ring_t[V3_RING][32];
  volatile u32 peer_progress, t_consumed;
  volatile u32 chunk_seq[8];                 // chunk c carries every SGD step of bits < chunk_seq[c]
  // T warp
  float in1[L1_IN + 3], in2[L2_IN + 3];
  alignas(16) float l1row[N_L1 + 1][ROW_PITCH_L1];     // row 20 = the layer-2 mixer
  float l1extra[N_L1 + 4]; float tu[N_L1 + 4]; u32 tshr[N_L1 + 4];
  unsigned short emap[T_ELEMS + 5];
  float lut12[4100];
};

enum { V3_CHUNKS = 8, V3_CHUNK4 = 64 };          // 8 chunks of 64 float4; the last also takes float4 512..518 and the scalar tail

// One chunk (64 float4) of the serial dot product; the SGD step is applied by the movers chunk by
// chunk just ahead of this warp. Ping-pong register buffers keep 8 LDS.128 in flight under the FADD chain.
__device__ __forceinline__ float chain_chunk(const float4* __restrict__ x4, const float4* __restrict__ w4, int k0, int k1, float p) {
  float4 xa[4], wa[4], xb[4], wb[4];
#define CC_LOAD(X, W, k) { _Pragma("unroll") for (int q = 0; q < 4; ++q) { X[q] = x4[(k) + q]; W[q] = w4[(k) + q]; } }
#define CC_EAT(X, W) { _Pragma("unroll") for (int q = 0; q < 4; ++q) { \
    float p0_, p1_, p2_, p3_; \
    xm_fmul2(X[q].x, X[q].y, W[q].x, W[q].y, p0_, p1_); xm_fmul2(X[q].z, X[q].w, W[q].z, W[q].w, p2_, p3_); \
    p = XM_FADD(p, p0_); p = XM_FADD(p, p1_); p = XM_FADD(p, p2_); p = XM_FADD(p, p3_); } }
  CC_LOAD(xa, wa, k0);
#pragma unroll 1
  for (int k = k0; k < k0 + 56; k += 8) {          // blocks 0..13 consumed, block 14 left in A
    CC_LOAD(xb, wb, k + 4);
    CC_EAT(xa, wa);
    CC_LOAD(xa, wa, k + 8);
    CC_EAT(xb, wb);
  }
  CC_LOAD(xb, wb, k0 + 60);
  CC_EAT(xa, wa);
  CC_EAT(xb, wb);
#undef CC_LOAD
#undef CC_EAT
#pragma unroll 1
  for (int k = k0 + 64; k < k1; ++k) {              // only the last chunk: float4 512..518
    const float4 a = x4[k], b = w4[k];
    p = XM_FADD(p, XM_FMUL(a.x, b.x)); p = XM_FADD(p, XM_FMUL(a.y, b.y));
    p = XM_FADD(p, XM_FMUL(a.z, b.z)); p = XM_FADD(p, XM_FMUL(a.w, b.w));
  }
  return p;
}

// movers: apply the SGD step of one bit, chunk c only, to the rows listed in sh.mupd (-1 = none).
// Work item = (row, half chunk of 32 float4): one warp instruction stream per item, no index division.
__device__ __forceinline__ void movers_update_chunk(MixShared3& sh, int m0, int mwarp, int lane, int par_prev, const float* xprev, int c) {
  const float4* xp4 = reinterpret_cast<const float4*>(xprev);
#pragma unroll 1
  for (int item = mwarp; item < 2 * MIX_PER_CTA; item += V3_M_WARPS) {
    const int i = item >> 1, half = item & 1;
    const int b = sh.mupd[i];
    if (b < 0) continue;
    const float u = sh.upd[par_prev][i];
    const bool shr = sh.plan_shrink[par_prev][i] != 0;
    float4* row4 = reinterpret_cast<float4*>(sh.rows[b]);
    {
      const int k4 = c * V3_CHUNK4 + half * 32 + lane;
      const float4 xv = xp4[k4];
      float4 w = row4[k4];
      w.x = XM_FSUB(w.x, XM_FMUL(u, xv.x)); w.y = XM_FSUB(w.y, XM_FMUL(u, xv.y));
      w.z = XM_FSUB(w.z, XM_FMUL(u, xv.z)); w.w = XM_FSUB(w.w, XM_FMUL(u, xv.w));
      if (shr) { w.x = XM_FMUL(w.x, 1.0f - 3.0e-6f); w.y = XM_FMUL(w.y, 1.0f - 3.0e-6f); w.z = XM_FMUL(w.z, 1.0f - 3.0e-6f); w.w = XM_FMUL(w.w, 1.0f - 3.0e-6f); }
      row4[k4] = w;
    }
    if (c == V3_CHUNKS - 1 && half == 1) {
      // leftovers of the row: float4 512..518, scalars 2076/2077 and this mixer's extra-input weights
      if (lane < 7) {
        const int k4 = 512 + lane;
        const float4 xv = xp4[k4];
        float4 w = row4[k4];
        w.x = XM_FSUB(w.x, XM_FMUL(u, xv.x)); w.y = XM_FSUB(w.y, XM_FMUL(u, xv.y));
        w.z = XM_FSUB(w.z, XM_FMUL(u, xv.z)); w.w = XM_FSUB(w.w, XM_FMUL(u, xv.w));
        if (shr) { w.x = XM_FMUL(w.x, 1.0f - 3.0e-6f); w.y = XM_FMUL(w.y, 1.0f - 3.0e-6f); w.z = XM_FMUL(w.z, 1.0f - 3.0e-6f); w.w = XM_FMUL(w.w, 1.0f - 3.0e-6f); }
        row4[k4] = w;
      } else {
        const int n = N_INPUTS + m0 + i;
        float* row = sh.rows[b];
#pragma unroll 1
        for (int k = 2076 + (lane - 7); k < n; k += 25) {   // lanes 7..31 sweep elements 2076 .. n-1
          const float xin = k < N_INPUTS ? xprev[k] : sh.cext[par_prev][k - N_INPUTS];
          float w = XM_FSUB(row[k], XM_FMUL(u, xin));
          if (shr) w = XM_FMUL(w, 1.0f - 3.0e-6f);
          row[k] = w;
        }
      }
    }
  }
}
// all chunks; after chunk c is complete the chain warp of bit `seq` may read it
__device__ __forceinline__ void movers_update(MixShared3& sh, int m0, int mtid, int par_prev, const float* xprev, u32 seq) {
#pragma unroll 1
  for (int c = 0; c < V3_CHUNKS; ++c) {
    movers_update_chunk(sh, m0, mtid >> 5, mtid & 31, par_prev, xprev, c);
    named_sync(B3_MOVERS, V3_M_THREADS);
    if (mtid == 0) sh.chunk_seq[c] = seq;
  }
}

// movers: run sh.jobs through the TMA (same protocol as mixer_prims.cuh::run_row_jobs)
__device__ __forceinline__ void run_row_jobs3(MixShared3& sh, StreamState* st, int m0, int mtid) {
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
    if (any_load) { mbar_wait(&sh.row_bar, sh.row_bar_phase & 1); sh.row_bar_phase++; }
  }
  named_sync(B3_MOVERS, V3_M_THREADS);
}

// movers: the step-dependent learning-rate factor of bit t for local mixer i (mixer.cpp:58-66),
// and the bookkeeping of ContextData::steps / Mixer::max_steps_.
__device__ __forceinline__ void plan_rate(MixShared3& sh, int par, int i, float decay, float lr) {
  const int b = sh.plan_buf[par][i];
  const u64 rs = sh.steps[b], ms = sh.max_steps[i];
  float d = decay;
  d = (float)((double)d * (1.5 - ((1.0 * (double)rs) / (double)ms)));
  sh.plan_dl[par][i] = XM_FMUL(d, lr);
  const u64 ns = rs + 1;
  sh.steps[b] = ns;
  if (ns > ms) sh.max_steps[i] = ns;
  sh.plan_shrink[par][i] = ((ns & 1023) == 0) ? 1u : 0u;
  sh.dirty[b] = 1;
}

#define V3_PROF(cond, slot) do { if (cond) { \
    unsigned dummy_ = *reinterpret_cast<volatile unsigned*>(&sh.n_jobs), sink_; \
    asm volatile("mov.u32 %0, %1;" : "=r"(sink_) : "r"(dummy_)); \
    const long long now_ = clock64(); pacc[(slot) & 7] += (unsigned long long)(now_ - tprev) + (sink_ & 0u); tprev = now_; } } while (0)

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(MIX_THREADS, 1)
mix_kernel_v3(const ChunkArgs* __restrict__ args_all, Tables T) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const ChunkArgs a = args_all[blockIdx.x / 2];
  StreamState* st = a.st;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MixShared3& sh = *reinterpret_cast<MixShared3*>(smem_raw);
  MixShared3* sh0 = cluster.map_shared_rank(&sh, 0);
  MixShared3* sh1 = cluster.map_shared_rank(&sh, 1);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = rank * MIX_PER_CTA;
  const u64 n_bits = (u64)a.n_bytes * 8;

  if (tid == 0) {
    int next = MIX_PER_CTA;
    for (int i = 0; i < MIX_PER_CTA; ++i) {
      sh.buf_cur[i] = i;
      sh.buf_alt[i] = -1;
      if (selector_is_bit_level(st->mixer[m0 + i].sel) && next < V3_NBUF) sh.buf_alt[i] = next++;
      sh.max_steps[i] = st->mixer[m0 + i].max_steps;
      sh.mupd[i] = -1;
    }
    for (int b = 0; b < V3_NBUF; ++b) { sh.tag[b] = 0xffffffffu; sh.dirty[b] = 0; sh.steps[b] = 0; }
    for (int r = 0; r < V3_RING; ++r) for (int k = 0; k < 32; ++k) { sh.ring_t[r][k] = make_uint2(0, 0); if (k < 16) sh.ring_in[r][k] = make_uint2(0, 0); }
    sh.peer_progress = 0; sh.t_consumed = 0; sh.n_jobs = 0; sh.row_bar_phase = 0; sh.n_late = 0;
    for (int c = 0; c < 8; ++c) sh.chunk_seq[c] = 0;
    mbar_init(&sh.row_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    int e = 0;
    for (int i = 0; i <= N_L1; ++i) { const int n = i < N_L1 ? L1_IN + i : L2_IN; for (int c = 0; c < n; ++c) sh.emap[e++] = (unsigned short)((i << 8) | c); }
  }
  for (int k = tid; k < 4097; k += MIX_THREADS) sh.lut12[k] = T.lut12[k];
  __syncthreads();
  cluster.sync();

  if (warp == V2_C_WARP) {
    // =============================== C warp ===============================
    const bool pc_on = a.prof != nullptr && lane == 0; const int pb = rank == 0 ? 8 : 14;
    unsigned long long pacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long tprev = clock64();
    float u_prev = 0.0f;
    for (u64 t = 0; t < n_bits; ++t) {
      const int par = (int)(t & 1), r = (int)(t & (V3_RING - 1));
      const int bit = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
      named_sync(B3_READY0 + par, V3_CM);
      V3_PROF(pc_on, pb + 0);
      const float* x = sh.x[t % 3];
      float* row = sh.rows[lane < MIX_PER_CTA ? sh.plan_buf[par][lane] : 0];
      const float dl = lane < MIX_PER_CTA ? sh.plan_dl[par][lane] : 0.0f;
      float main = 0.0f;
      {
        const float4* x4 = reinterpret_cast<const float4*>(x);
        const float4* w4 = reinterpret_cast<const float4*>(row);
#pragma unroll 1
        for (int c = 0; c < V3_CHUNKS; ++c) {
          while (sh.chunk_seq[c] < (u32)t) { }            // the movers have applied bit t-1's step to this chunk
          if (lane < MIX_PER_CTA) main = chain_chunk(x4, w4, c * V3_CHUNK4, c == V3_CHUNKS - 1 ? 519 : (c + 1) * V3_CHUNK4, main);
        }
        if (lane < MIX_PER_CTA) {
          main = XM_FADD(main, XM_FMUL(x[2076], row[2076]));
          main = XM_FADD(main, XM_FMUL(x[2077], row[2077]));
        }
      }
      __syncwarp();
      V3_PROF(pc_on, pb + 1);
      // ---- forward substitution through the extra inputs ----
      float e = 0.0f, pfin = 0.0f, cmine = 0.0f;
      int kbase = 0;
      if (rank == 1) {
#pragma unroll 1
        for (int k = 0; k < MIX_PER_CTA; ++k) {
          const float ck = ll_wait(&sh.ring_in[r][k], (u32)(t + 1));
          if (lane == k) sh.cext[par][k] = ck;
          if (lane < MIX_PER_CTA) e = XM_FADD(e, XM_FMUL(ck, row[N_INPUTS + k]));
        }
        if (lane == 0) sh0->peer_progress = (u32)(t + 1);
        kbase = MIX_PER_CTA;
      } else {
        if (lane == 0 && t >= V3_RING) { spin_until_ge(&sh.peer_progress, (u32)(t + 1 - V3_RING)); spin_until_ge(&sh.t_consumed, (u32)(t + 1 - V3_RING)); }
        __syncwarp();
      }
      if (rank == 1 && lane == 0 && t >= V3_RING) spin_until_ge(&sh.t_consumed, (u32)(t + 1 - V3_RING));
      __syncwarp();
      V3_PROF(pc_on, pb + 2);
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
      V3_PROF(pc_on, pb + 3);
      // ---- coefficient: the movers pre-computed decay*lr; only the logistic is left (mixer.cpp:60) ----
      if (lane < MIX_PER_CTA) {
        u_prev = XM_FMUL(dl, XM_FSUB(xm_logistic(pfin), (float)bit));
        sh.upd[par][lane] = u_prev;
        sh.cext[par][m0 + lane] = cmine;
      } else if (rank == 0 && lane < MIX_PER_CTA + 3) {
        const int idx = lane == MIX_PER_CTA ? 433 : (lane == MIX_PER_CTA + 1 ? 2024 : 2077);
        ll_store(&sh.ring_t[r][N_L0 + (lane - MIX_PER_CTA)], clamp_stretched(T, x[idx]), (u32)(t + 1));
      }
      __syncwarp();
      V3_PROF(pc_on, pb + 4);
      named_arrive(B3_COEFF0 + par, V3_CM);
      V3_PROF(pc_on, pb + 5);
    }
    V2_PROF_DUMP(pc_on, pb, 6);
  } else if (warp < V2_T_WARP && (warp & 3) != 3) {
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
        stage_inputs_v2<V3_M_THREADS>(sh.x[t % 3], sh.lut12, a.ext ? a.ext + t * N_EXT : nullptr, a.small_x + t * SMALL_X_PITCH, a.lstm_x[2 * t], mtid);
        named_sync(B3_MOVERS, V3_M_THREADS);
        V3_PROF(pm_on, 20);
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
        named_sync(B3_MOVERS, V3_M_THREADS);
        V3_PROF(pm_on, 21);
        run_row_jobs3(sh, st, m0, mtid);
        const float decay = a.decay[t];
        if (mtid < MIX_PER_CTA && sh.kind[mtid] != K_LATE_SWITCH) plan_rate(sh, par, mtid, decay, my_lr);
        named_sync(B3_MOVERS, V3_M_THREADS);
        V3_PROF(pm_on, 22);
        if (sh.n_late) {
          // rows that must carry bit t-1's step BEFORE bit t's chain: shrink due, or single-buffered switch
          if (t > 0) { named_sync(B3_COEFF0 + parp, V3_CM); coeff_synced = true; }
          if (mtid < MIX_PER_CTA) {
            if (t > 0 && sh.kind[mtid] == K_LATE_SWITCH && sh.tag[sh.buf_cur[mtid]] != 0xffffffffu) sh.mupd[mtid] = sh.buf_cur[mtid];
          }
          named_sync(B3_MOVERS, V3_M_THREADS);
          if (t > 0) movers_update(sh, m0, mtid, parp, sh.x[(t + 2) % 3], (u32)t);
          named_sync(B3_MOVERS, V3_M_THREADS);
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
          named_sync(B3_MOVERS, V3_M_THREADS);
          run_row_jobs3(sh, st, m0, mtid);
          if (mtid < MIX_PER_CTA && sh.kind[mtid] == K_LATE_SWITCH) plan_rate(sh, par, mtid, decay, my_lr);
          named_sync(B3_MOVERS, V3_M_THREADS);
        }
        V3_PROF(pm_on, 23);
        named_arrive(B3_READY0 + par, V3_CM);
      }
      // ---- bit t-1's step for the rows that were switched away (or, at the end, for all rows) ----
      if (t > 0) {
        if (!coeff_synced) named_sync(B3_COEFF0 + parp, V3_CM);
        V3_PROF(pm_on, 24);
        if (t == n_bits) { if (mtid < MIX_PER_CTA) sh.mupd[mtid] = sh.buf_cur[mtid]; named_sync(B3_MOVERS, V3_M_THREADS); }
        movers_update(sh, m0, mtid, parp, sh.x[(t + 2) % 3], (u32)t);
        V3_PROF(pm_on, 25);
      }
    }
    V2_PROF_DUMP(pm_on, 20, 6);
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
    named_sync(B3_MOVERS, V3_M_THREADS);
    run_row_jobs3(sh, st, m0, mtid);
    if (mtid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  } else if (rank == 0 && warp == V2_T_WARP) {
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
      const int r = (int)(t & (V3_RING - 1));
      const int bit = (a.bytes[t >> 3] >> (7 - (t & 7))) & 1;
      // ---- candidate SSE buckets for every possible quantisation of p (sse.cpp:250-270) ----
      uint4 cand = make_uint4(0, 0, 0, 0); size_t cand_idx = 0;
      if (lane < 3) {
        cand_idx = (((((size_t)lane << 7) + (sffl & 127)) << 8) + (spc & 255)) * 256 + sj;
        cand = *reinterpret_cast<const uint4*>(sse.s6 + cand_idx * 8);
      } else if (lane < 6) {
        cand_idx = (((((size_t)(lane - 3) << 5) + (sffl & 31)) << 8) + (spc & 255)) * 255 + (sj < 2 ? 0 : sj - 1);
        cand = *reinterpret_cast<const uint4*>(sse.s7 + cand_idx * 8);
      } else if (lane < 9) {
        cand_idx = (((((size_t)(lane - 6) << 1) + (sffl & 1)) << 8) + (spc & 255)) * 256 + sj;
        cand.x = (u32)sse.x2[cand_idx];
      } else if (lane < 13) {
        cand_idx = (((((size_t)(lane - 9) << 8) + (sffl & 255)) << 3) + ((spc >> 5) & 7)) * 79 + sse_mask1((int)sj);
        cand.x = (u32)sse.x1[cand_idx];
      }
      const float decay = a.decay[t];
      const float ov = a.lstm_x[2 * t + 1];
      // ---- rows of layers 1/2 (resident per lane; table look-up issued one bit ahead) ----
      if (lane < N_L1 + 1) {
        const u32 ctx = ctx_next;
        u32 sl = sl_next;
        if (sl == 0) sl = mytable[ctx];               // may have been assigned since the look-ahead read
        if (sl == 0) {
          const u32 cap = my_nrows - 1;
          if (my_assigned < cap && my_assigned < (u32)SLOT_LIMIT) { sl = ++my_assigned; mytable[ctx] = sl; }
          else sl = my_nrows;
        }
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
      V3_PROF(pt_on, 26);
      {
        float c = 0.0f;
        if (lane < N_L0 + N_AUX) c = ll_wait(&sh.ring_t[r][lane], (u32)(t + 1));
        if (lane < N_L0) { sh.in1[lane] = c; sh.in2[lane] = c; }
        else if (lane < N_L0 + N_AUX) { sh.in1[lane] = c; sh.in2[N_L1 + lane] = c; }
      }
      __syncwarp();
      V3_PROF(pt_on, 27);
      if (lane == 0) { sh.t_consumed = (u32)(t + 1); sh1->t_consumed = (u32)(t + 1); }
      // ---- layer 1 ----
      float main = 0.0f;
      if (lane < N_L1) {
        const float* w = sh.l1row[lane];
#pragma unroll 4
        for (int k = 0; k < L1_IN; ++k) main = XM_FADD(main, XM_FMUL(sh.in1[k], w[k]));
      }
      float e = 0.0f, pfin = 0.0f;
      float wnext = lane < N_L1 ? sh.l1row[lane][L1_IN] : 0.0f;
#pragma unroll 1
      for (int k = 0; k < N_L1; ++k) {
        if (lane == k) pfin = XM_FADD(main, e);
        const float pk = __shfl_sync(0xffffffffu, pfin, k);
        const float ck = clamp_stretched(T, pk);
        const float wk = wnext;
        if (lane < N_L1 && k + 1 < N_L1) wnext = sh.l1row[lane][L1_IN + k + 1];
        if (lane == k) { sh.l1extra[k] = ck; sh.in2[N_L0 + k] = ck; }
        if (lane > k && lane < N_L1) e = XM_FADD(e, XM_FMUL(ck, wk));
      }
      __syncwarp();
      V3_PROF(pt_on, 28);
      // ---- layer 2 ----
      float s2 = 0.0f;
      if (lane == N_L1) {
        const float* w = sh.l1row[N_L1];
#pragma unroll 7
        for (int k = 0; k < L2_IN; ++k) s2 = XM_FADD(s2, XM_FMUL(sh.in2[k], w[k]));
        s2 = XM_FADD(s2, 0.0f);
        pfin = s2;
      }
      s2 = __shfl_sync(0xffffffffu, s2, N_L1);
      // ---- SSE (sse.cpp:243-289) on the prefetched buckets ----
      const float pin = xm_logistic(s2);
      const int discrete = (int)XM_FADD(1.0f, XM_FMUL(XM_FSUB(1.0f, pin), 32766.0f));
      const u32 prq = (u32)discrete >> 11;
      const int q3 = (prq > 0) + (prq > 14), q4 = (prq > 0) + (prq > 7) + (prq > 14);
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
        u16 k6[8] = {(u16)b6.x, (u16)(b6.x >> 16), (u16)b6.y, (u16)(b6.y >> 16), (u16)b6.z, (u16)(b6.z >> 16), (u16)b6.w, (u16)(b6.w >> 16)};
        u16 k7[8] = {(u16)b7.x, (u16)(b7.x >> 16), (u16)b7.y, (u16)(b7.y >> 16), (u16)b7.z, (u16)(b7.z >> 16), (u16)b7.w, (u16)(b7.w >> 16)};
        const int stp = __ldg(&tst[discrete]);
        int sw6, qq6, P6, sw7, qq7, P7;
        const int p1 = sse_pred(k6, __ldg(&tsq[sse_extrap(stp, 10240)]), &sw6, &qq6, &P6);
        const int s0 = sse_extrap(stp, 7935);
        const int s1 = sse_extrap(__ldg(&tst[p1]), 9592);
        int sm = sse_mixup(wx1, s0, s1);
        sm = sse_extrap(sm, 8092);
        const int mix1_p = __ldg(&tsq[sm]);
        const int p2 = sse_pred(k7, __ldg(&tsq[sse_extrap(stp, 8200)]), &sw7, &qq7, &P7);
        const int s4 = sse_extrap(__ldg(&tst[p2]), 7677);
        int s5 = sse_mixup(wx2, sm, s4);
        s5 = sse_extrap(s5, 8202);
        const int mix2_p = __ldg(&tsq[s5]);
        const float p = (float)(1.0 - ((double)(mix2_p - 1) / 32766.0));
        a.p_out[t] = ov >= 0.0f ? ov : p;
        sse_bucket_update(k6, bit, 106, sw6, qq6, P6);
        sse_mix_update(&wx1, bit, s0, s1, 6202, mix1_p);
        sse_bucket_update(k7, bit, 127, sw7, qq7, P7);
        sse_mix_update(&wx2, bit, sm, s4, 8320, mix2_p);
        u16* g6 = sse.s6 + i6 * 8; g6[qq6] = k6[qq6]; g6[qq6 + 1] = k6[qq6 + 1];
        u16* g7 = sse.s7 + i7 * 8; g7[qq7] = k7[qq7]; g7[qq7 + 1] = k7[qq7 + 1];
        sse.x1[ix1] = wx1; sse.x2[ix2] = wx2;
      }
      V3_PROF(pt_on, 29);
      sj += sj + bit;
      if (sj >= 256) { sffl = (u8)(sffl * 2 + (spc >= 0x40)); spc = (u8)sj; sj = 1; }
      // ---- SGD of layers 1/2 (mixer.cpp:56-72): coefficients per lane, then a flat (row, column) sweep ----
      if (lane < N_L1 + 1) {
        float d = decay;
        d = (float)((double)d * (1.5 - ((1.0 * (double)my_rs) / (double)my_max)));
        sh.tu[lane] = XM_FMUL(XM_FMUL(d, mylr), XM_FSUB(xm_logistic(pfin), (float)bit));
        my_rs += 1;
        if (my_rs > my_max) my_max = my_rs;
        sh.tshr[lane] = (my_rs & 1023) == 0 ? 1u : 0u;
      }
      __syncwarp();
#pragma unroll 2
      for (int el = lane; el < T_ELEMS; el += 32) {
        const int i = sh.emap[el] >> 8, c = sh.emap[el] & 255;
        const float xin = i < N_L1 ? (c < L1_IN ? sh.in1[c] : sh.l1extra[c - L1_IN]) : sh.in2[c];
        float w = XM_FSUB(sh.l1row[i][c], XM_FMUL(sh.tu[i], xin));
        if (sh.tshr[i]) w = XM_FMUL(w, 1.0f - 3.0e-6f);
        sh.l1row[i][c] = w;
      }
      __syncwarp();
      V3_PROF(pt_on, 30);
    }
    V2_PROF_DUMP(pt_on, 26, 5);
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
  __syncthreads();
  cluster.sync();
}

}  // namespace cmixb200
