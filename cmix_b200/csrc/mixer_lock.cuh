// cmix_b200/csrc/mixer_lock.cuh
//
// Lock-step mixer kernels: Predict() / Perceive(bit) one bit at a time, the decoder's order (reference
// coder/decoder.cpp:20-39), on the arithmetic of mixer.cuh. Nothing can stay resident between the two calls, so
// the work is spread over SMs instead: one CTA per layer-0 mixer for the 26 serial chains and for the 26 row
// updates, one CTA for layers 1-2 + SSE. Rows stay in HBM; what Perceive needs is parked in StreamState.
#pragma once
#include "mixer.cuh"

namespace cmixb200 {

// mix_predict_rows_kernel<<<26, 256>>>: CTA i stages the 2078 inputs, resolves mixer i's row
// (mixer 12's selector is the auxiliary context of the staged inputs, predictor.cpp:388-393),
// copies the row into shared memory and runs its chain on one thread (Mixer::Mix, mixer.cpp:41-43).
struct LockRowShared {
  alignas(16) float x[N_INPUTS + 2];
  alignas(16) float row[ROW_PITCH_L0];
  u32 slot;
};

__global__ void __launch_bounds__(256, 1)
mix_predict_rows_kernel(StreamState* st, Tables T, const u16* ext /* device, N_EXT codes or null */) { jit_entry(JK_MIX_ROWS);
  __shared__ LockRowShared sh;
  const int tid = threadIdx.x, i = blockIdx.x;
  stage_inputs<256>(sh.x, T.lut12, ext, st->small_x, st->lstm_x, tid);
  JIT_SYNCTHREADS();
  if (tid == 0) {
    const u32 sel = i == 12 ? aux_context(sh.x) : st->sel[i];
    const u32 s = resolve_slot(st->mixer[i], sel);
    st->slot[i] = s;
    sh.slot = s;
  }
  JIT_SYNCTHREADS();
  {
    const float4* g = reinterpret_cast<const float4*>(st->mixer[i].rows + (size_t)sh.slot * ROW_PITCH_L0);
    float4* d = reinterpret_cast<float4*>(sh.row);
    for (int k = tid; k < ROW_PITCH_L0 / 4; k += 256) d[k] = g[k];
  }
  if (i == 0) for (int k = tid; k < N_INPUTS; k += 256) st->x[k] = sh.x[k];
  JIT_SYNCTHREADS();
  if (tid == 0) {
    const float4* x4 = reinterpret_cast<const float4*>(sh.x);
    const float4* w4 = reinterpret_cast<const float4*>(sh.row);
    float p = 0.0f;
    for (int c = 0; c < MIX_CHUNKS; ++c) p = chain_chunk(x4, w4, c * MIX_CHUNK4, chain_chunk_end(c), p);
    st->mains[i] = chain_tail(sh.x, sh.row, p);
  }
}

// mix_predict_final_kernel<<<1, 512>>>: extra-input substitution, layers 1-2, SSE (mixer.cpp:45-53,
// predictor.cpp:394-418, sse.cpp:243-289) from the 26 main sums, on one warp.
struct LockFinalShared {
  float mains[N_L0];              // main dot products of the 26 layer-0 mixers
  float we[N_L0][N_L0 + 2];       // their extra-input weights
  float aux[N_AUX];               // inputs 433, 2024 and 2077
  float in1[L1_IN + 3], in2[L2_IN + 3];
  float l1row[N_L1 + 1][ROW_PITCH_L1];     // row 20 = the layer-2 mixer
  float l1extra[N_L1 + 4];
  float mixp[N_MIXERS + 1];
  u32 slot1[N_L1 + 4];
};

__global__ void __launch_bounds__(MIX_THREADS, 1)
mix_predict_final_kernel(StreamState* st, Tables T) { jit_entry(JK_MIX_FINAL);
  __shared__ LockFinalShared sh;
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid < N_L0) sh.mains[tid] = st->mains[tid];
  if (tid >= 32 && tid < 32 + N_AUX) sh.aux[tid - 32] = st->x[tid == 32 ? 433 : (tid == 33 ? 2024 : 2077)];
  if (tid >= N_L0 && tid < N_MIXERS) { const u32 s = resolve_slot(st->mixer[tid], st->sel[tid]); st->slot[tid] = s; sh.slot1[tid - N_L0] = s; }
  JIT_SYNCTHREADS();
  for (int k = tid; k < (N_L1 + 1) * ROW_PITCH_L1; k += MIX_THREADS) {
    const int i = k / ROW_PITCH_L1, c = k - i * ROW_PITCH_L1;
    sh.l1row[i][c] = st->mixer[N_L0 + i].rows[(size_t)sh.slot1[i] * ROW_PITCH_L1 + c];
  }
  for (int k = tid; k < N_L0 * N_L0; k += MIX_THREADS) {
    const int i = k / N_L0, c = k - i * N_L0;
    sh.we[i][c] = st->mixer[i].rows[(size_t)st->slot[i] * ROW_PITCH_L0 + N_INPUTS + c];
  }
  JIT_SYNCTHREADS();
  if (tid < 32) {
    // layer 0's clamped outputs are the first inputs of layers 1 and 2, followed by the 3 auxiliary inputs
    const float p0 = substitute<N_L0>(lane < N_L0 ? sh.mains[lane] : 0.0f, sh.we[lane], T, sh.in1, sh.in2, lane);
    if (lane < N_L0) sh.mixp[lane] = p0;
    if (lane < N_AUX) {
      const float c = clamp_stretched(T, sh.aux[lane]);
      sh.in1[N_L0 + lane] = c;
      sh.in2[N_L0 + N_L1 + lane] = c;
    }
    __syncwarp();
    const float p1 = layer1_forward(sh.l1row[lane], sh.in1, sh.l1extra, sh.in2, T, lane);
    if (lane < N_L1) sh.mixp[N_L0 + lane] = p1;
    __syncwarp();
    if (lane == 0) {
      const float s = layer2_forward(sh.l1row[N_L1], sh.in2);
      sh.mixp[N_L0 + N_L1] = s;
      SseState& S = st->sse;
      int q3, q4;
      const int discrete = sse_quantise(xm_logistic(s), q3, q4);
      const size_t i6 = sse_i6(q3, S.j, S.pc, S.ffl), i7 = sse_i7(q3, S.j, S.pc, S.ffl);
      const size_t ix2 = sse_ix2(q3, S.j, S.pc, S.ffl), ix1 = sse_ix1(q4, S.j, S.pc, S.ffl);
      SseCarry c;
      const float p = sse_estimate(c, S.st, S.sq, discrete, S.s6 + i6 * 8, S.s7 + i7 * 8, S.x1[ix1], S.x2[ix2]);
      S.i6 = (u32)i6; S.i7 = (u32)i7; S.ix1 = (u32)ix1; S.ix2 = (u32)ix2;
      S.c = c;
      st->last_p = st->lstm_override >= 0.0f ? st->lstm_override : p;
    }
  }
  JIT_SYNCTHREADS();
  if (tid < N_L0) st->extras0[tid] = sh.in1[tid];
  if (tid < N_L1) st->extras1[tid] = sh.l1extra[tid];
  if (tid < L2_IN) st->in2[tid] = sh.in2[tid];
  if (tid < N_MIXERS) st->mix_p[tid] = sh.mixp[tid];
}

// mix_perceive_kernel<<<26 + 2, 512>>>: Mixer::Perceive (mixer.cpp:56-72) for every mixer and
// SSE::Perceive (sse.cpp:291-305). CTA i < 26 owns layer-0 mixer i's row; CTA 26 the 21 small rows of
// layers 1-2, the SSE update and the step counter; CTA 27 the LSTM read-out's bit update
// (ByteModel::Perceive, byte-model.cpp:17-30).
__global__ void __launch_bounds__(MIX_THREADS, 1)
mix_perceive_kernel(StreamState* st, int bit, float decay_base, const u32* dbit = nullptr) { jit_entry(JK_MIX_PERCEIVE);
  if (dbit) {                            // decode loop: the bit and the step's decay factor come from the device
    const DecodeState* ds = reinterpret_cast<const DecodeState*>(dbit);
    bit = (int)ds->bit;
    if (ds->decay) decay_base = ds->decay[ds->t - 1];
  }
  __shared__ float upd[N_L1 + 2];
  __shared__ u32 shrink[N_L1 + 2];
  const int tid = threadIdx.x, blk = blockIdx.x;
  if (blk < N_L0) {
    const int i = blk;
    MixerState& m = st->mixer[i];
    if (tid == 0) {
      u64& steps = m.row_steps[st->slot[i]];
      const u64 rs = steps, ms = m.max_steps;
      upd[0] = sgd_coeff(mixer_rate(decay_base, m.lr, rs, ms), st->mix_p[i], bit);
      mixer_step(rs, ms, steps, m.max_steps, shrink[0]);
    }
    JIT_SYNCTHREADS();
    float* row = m.rows + (size_t)st->slot[i] * ROW_PITCH_L0;
    const int n = N_INPUTS + i;
    const float u = upd[0];
    const u32 shr = shrink[0];
    for (int k = tid; k < n; k += MIX_THREADS) sgd_step(row[k], u, k < N_INPUTS ? st->x[k] : st->extras0[k - N_INPUTS], shr);
    return;
  }
  if (blk == N_L0 + 1) {
    if (tid == 0) bm_perceive(st->lstm.bm, bit);
    return;
  }
  if (tid < N_L1 + 1) {
    MixerState& m = st->mixer[N_L0 + tid];
    u64& steps = m.row_steps[st->slot[N_L0 + tid]];
    const u64 rs = steps, ms = m.max_steps;
    upd[tid] = sgd_coeff(mixer_rate(decay_base, m.lr, rs, ms), st->mix_p[N_L0 + tid], bit);
    mixer_step(rs, ms, steps, m.max_steps, shrink[tid]);
  }
  if (tid == 64) {
    SseState& S = st->sse;
    const SseCarry c = S.c;
    sse_learn(c, bit, S.s6 + (size_t)S.i6 * 8, S.s7 + (size_t)S.i7 * 8, &S.x1[S.ix1], &S.x2[S.ix2]);
    sse_advance(S.j, S.pc, S.ffl, bit);
  }
  JIT_SYNCTHREADS();
  for (int k = tid; k < (N_L1 + 1) * ROW_PITCH_L1; k += MIX_THREADS) {
    const int i = k / ROW_PITCH_L1, c = k - i * ROW_PITCH_L1;
    const int mi = N_L0 + i;
    const int n = i < N_L1 ? L1_IN + i : L2_IN;
    if (c < n) {
      float xin;
      if (i < N_L1) {
        if (c < N_L0) xin = st->extras0[c];                       // layer-1 input c = clamp(layer-0 output c)
        else if (c < L1_IN) xin = st->in2[N_L0 + N_L1 + (c - N_L0)];   // the 3 auxiliary inputs
        else xin = st->extras1[c - L1_IN];
      } else xin = st->in2[c];
      sgd_step(st->mixer[mi].rows[(size_t)st->slot[mi] * ROW_PITCH_L1 + c], upd[i], xin, shrink[i]);
    }
  }
  if (tid == 0) st->bits_done += 1;
}

}  // namespace cmixb200
