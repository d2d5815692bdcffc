// cmix_b200/csrc/state.h — device-resident state of one predictor stream.
//
// One "stream" = one reference Predictor instance (reference src/predictor.h:17-53):
// everything Predict()/Perceive() mutate lives in HBM in the structs below, laid
// out flat (no pointers-to-pointers) so that kernels address it with coalesced,
// vectorised accesses. See DESIGN.md §3 for sizes.
#ifndef CMIXB200_STATE_H
#define CMIXB200_STATE_H

#include <stdint.h>

#include "ppmd_model.h"

namespace cmixb200 {
namespace fx { struct State; }     // resident FXCM model (fxcm_model.h)

typedef uint64_t u64;
typedef uint32_t u32;
typedef uint16_t u16;
typedef uint8_t u8;

// ---- network topology (reference predictor.cpp:194-356, SURVEY Appendix A) ----
enum {
  N_INPUTS = 2078,         // layer-0 inputs
  N_EXT = 2022,            // FXCM 431 + PAQ8 1591 replayed 12-bit codes
  N_SMALL = 54,            // small cmix models (Direct/DirectHash/Indirect/Match/Bracket)
  N_L0 = 26, N_L1 = 20, N_AUX = 3, N_MIXERS = 47,
  L1_IN = N_L0 + N_AUX,            // 29
  L2_IN = N_L0 + N_L1 + N_AUX,     // 49
  ROW_PITCH_L0 = 2104,     // 2078 inputs + up to 25 extras, padded to a multiple of 4 floats
  ROW_PITCH_L1 = 52,       // 29 + up to 19 extras, padded
  ROW_PITCH_L2 = 52,
  SLOT_LIMIT = 10000,      // mixer.cpp:17
  SMALL_X_PITCH = 56,      // 54 small-model inputs + PPMD bit input + pad
  SEL_PITCH = 48,
  LSTM_CELLS = 200, LSTM_HORIZON = 100, LSTM_HID = 401,
};

// Selector ids: which shared context variable picks a mixer's weight row.
enum Sel : int { S_ZERO, S_LONGBIT, S_RB0, S_RB1, S_RB2, S_RB3, S_LINEBREAK, S_LONGEST, S_WRT, S_AUX,
                 S_IV0, S_IV1, S_IV2, S_IV3, S_IV4, S_IV6, S_IVH,
                 S_BC0, S_BC1, S_BC2, S_BC3, S_BC_ALNUM, S_BC_W2, S_BC_W3, S_BC_RB1, S_COMB0, S_COMB1,
                 S_COUNT };

// ---- gated mixer (reference mixer/mixer.{h,cpp}) ----
struct MixerState {
  u32* slot_table;      // [table_size]: 0 = context never seen, else row index + 1
  float* rows;          // [n_rows][pitch] weights then extra weights, zero-initialised
  u64* row_steps;       // [n_rows] ContextData::steps
  u32 table_size;       // number of distinct selector values
  u32 n_rows;           // min(table_size, SLOT_LIMIT) + 1 (last = overflow row, mixer.cpp:18-25)
  u32 n_assigned;       // context_map_.size() without the overflow entry
  u32 pitch;
  u64 max_steps;        // Mixer::max_steps_
  float lr;
  int n_in, n_extra, sel;
};

// ---- final SSE stage (reference mixer/sse.cpp) ----
// What SSE's estimate leaves for its update (M_T::su6/su7/mix*, sse.cpp:243-305): interpolation and mixing terms.
struct SseCarry {
  int sw6, q6, P6, sw7, q7, P7;
  int s0, s1, sm, s4, mix1_p, mix2_p;
};
struct SseState {
  u16* s6; u16* s7;     // [vol][7] interpolation buckets (padded to 8 u16 per bucket set)
  int* x1; int* x2;     // 1-weight integer mixers
  u16* st; u16* sq;     // stretch / squash tables (32768 each, host-built with libm)
  u32 j, pc, ffl;
  // carried from Predict to Perceive: the bucket sets and weights the estimate used, and its terms
  u32 i6, i7, ix1, ix2;
  SseCarry c;
};

// ---- small models + shared contexts (reference context-manager.cpp, contexts/, models/) ----
struct DirectTable { float* pred; u8* count; u64* checksum; u64 rows; u64 index; int limit; float delta, divisor; int hashed; };
struct IndirectState { u64 map_index, map_offset; float divisor; int run; float pred[256]; };
struct MatchState { u64 history_pos, cur_match; u32* map; u64 map_size; int limit; float delta, divisor;
                    u8 cur_byte, bit_pos, match_length, pad; float pred[256]; int count[256]; };
struct ByteModelState { int top, mid, bot, ex; float probs[256]; };
struct IHashState { u64* hashes; u64 ctx1, ctx, size; u32 size1, h1, h2, pad; };

struct alignas(16) SmallState {
  // ContextManager scalars (context-manager.h:23-27)
  u32 bit_context, wrt_state;
  u64 long_bit_context, history_pos, line_break, longest_match, wrt_context;
  u64 words[8], recent_bytes[8];
  u8* history;          // 100 000 000
  u8* shared_map;       // 2 048 000 000
  // byte-level contexts
  u64 bracket_ctx; u32 br_depth, br_cap; u8* br_char; u32* br_dist;
  u64 sparse[18], chash[13], interval[8], ivh_ctx, bitctx[8], combined[2];
  u32 ivh_interval, pad0;
  IHashState ihash[11];
  // models in models_ order (predictor.cpp:28-35), FXCM/PAQ8 excluded
  ByteModelState bracket_bm; u32 bk_depth; u32 bk_active[16]; u32 bk_distance[16]; u32* bk_first; u32* bk_second;
  DirectTable direct_bracket, dhash_word, direct_o[3], dhash_o3;
  IndirectState indirect[31];   // 0 bracket, 1..18 word, 19 run, 20..30 double
  MatchState match[16];         // 0..5 word, 6..15 order
  ByteModelState ppmd_bm;
  u8 vocab[256];
  u32 error;                    // sticky error flags (stack overflow etc.)
};
static_assert(sizeof(SmallState) % 16 == 0, "SmallState is copied to shared memory in 16-byte units");

// ---- LSTM byte mixer (reference mixer/lstm.cpp, lstm-layer.cpp, byte-mixer.cpp) ----
struct GateState {
  float* w;        // [8][row][25] cell-block-major (lstm_widx): the 25 cells owned by one CTA of the
                   //              LSTM cluster are contiguous for every column
  float* m; float* v;           // Adam moments, same layout
  float* state; float* norm;    // [H][C]
  float* err;                   // [H][C] post-normalisation gate error of every BPTT step
  float ivar[LSTM_HORIZON];
  float gamma[LSTM_CELLS], gamma_m[LSTM_CELLS], gamma_v[LSTM_CELLS];
  float beta[LSTM_CELLS], beta_m[LSTM_CELLS], beta_v[LSTM_CELLS];
  int row;                      // 2V+201 (layer 0) / 2V+401 (layer 1)
};
struct LayerState {
  GateState gate[3];            // forget, input node, output gate
  float state[LSTM_CELLS], state_error[LSTM_CELLS], stored_error[LSTM_CELLS];
  float* tanh_state; float* input_gate_state; float* last_state;   // [H][C]
  float* input;                 // [H][in_size]
  int in_size, epoch;
  u64 update_steps;
};
struct LstmState {
  LayerState layer[2];
  float* out_w;                 // [H][V][401]
  float* output;                // [H][V]
  float hidden[LSTM_HID + 3], hidden_error[LSTM_CELLS];
  u32 input_history[LSTM_HORIZON];
  int V, epoch;
  int byte_map[256];            // byte -> vocab index
  u8 vocab[256];
  ByteModelState bm;            // ByteMixer's ByteModel base (probs over 256 bytes)
  const float* adam;            // [3001][4] alpha, bc1, bc2 per update_steps (host-built with libm)
};

// ---- one stream ----
struct StreamState {
  MixerState mixer[N_MIXERS];
  SseState sse;
  SmallState small;
  LstmState lstm;
  u64 bits_done;                // Mixer::steps_ (same for all 47 mixers)
  // lock-step scratch carried from Predict to Perceive
  float x[N_INPUTS + 2];
  float extras0[N_L0 + 2], extras1[N_L1], in2[L2_IN + 3];
  float mix_p[N_MIXERS + 1];
  float mains[N_L0 + 2];        // layer-0 main dot products (lock-step: row kernel -> final kernel)
  u32 slot[N_MIXERS + 1];
  u32 sel[SEL_PITCH];
  float small_x[SMALL_X_PITCH];
  PpmdModel* ppmd;              // resident PPMD model (ppmd_model.h); its arenas are separate allocations
  float lstm_x, lstm_override;  // override: -1 none, else 0 or 1 (predictor.cpp:383)
  u32 lstm_fx;                  // lock-step: lstmpr | lstmex << 16 of the next bit (predictor.cpp:462-465)
  float last_p;
};

// Shared read-only tables.
struct Tables {
  const float* logit;           // [100001] sigmoid.cpp:5-10
  const float* lut12;           // [4097] stretch of k/4095 (k<=4095) and of 0.5 (index 4096)
  float stretch_min, stretch_max;
};

// Per-launch arguments of the bulk kernels, one entry per stream.
// Arithmetic coder state of one stream (coder.cuh), persistent across bulk calls.
struct CoderState {
  u32 x1, x2;                   // Encoder::x1_, x2_ (encoder.cpp:3-4)
  u32 overflow, pad;
  u64 n_out, cap;               // archive bytes produced / capacity of out
  u8* out;
};

// Decoder::Decode on the device (coder.cuh decode_step_kernel): the arithmetic decoder's registers, the archive and what the
// lock-step kernels of a decode loop read instead of host arguments (bit / full, in this order: they are passed as one pointer).
struct DecodeState {
  u32 bit, full;                // the bit just decoded; the byte it completed (valid on the 8th bit of a byte)
  u32 x1, x2, x, ctx;           // Decoder::x1_, x2_, x_ (decoder.cpp:3-8); bits of the current byte with a leading 1
  u64 pos, n_arch, t;           // next archive byte, archive length, bits decoded
  const u8* arch; u8* out;
  const float* decay;           // [bit of this call] the mixers' learning-rate factor 0.9 / pow(1e-7 * steps + 0.8, 0.8), host-built (glibc pow)
};

struct ChunkArgs {
  StreamState* st;
  const u8* bytes;              // [n_bytes] the coded stream
  const u16* ext;               // [n_bytes*8][N_EXT] or null (all 0.5)
  const float* ppmd;            // [n_bytes][256] PPMD distribution after each byte: replayed, or == ppmd_gen; null = flat
  float* ppmd_gen;              // when non-null the resident PPMD model (ppmd.cuh) writes the distributions here
  const float* decay;           // [n_bytes*8] 0.9/pow(1e-7*steps+0.8, 0.8) (mixer.cpp:58), host-built
  float* small_x;               // [n_bytes*8][SMALL_X_PITCH] scratch: small-model inputs (+ PPMD)
  u32* sel;                     // [n_bytes*8][SEL_PITCH]   scratch: mixer selector values
  float* lstm_x;                // [n_bytes*8][2]           scratch: LSTM bit input + override
  float* p_out;                 // [n_bytes*8] result
  u32 n_bytes;
  u32 pretrain;                 // 1: Pretrain() semantics (models + contexts only)
  // resident FXCM / PAQ8 (fxcm.cuh, paq8.cuh): they write their 12-bit codes into ext_gen ([n_bytes*8][N_EXT]); `ext` above is
  // then == ext_gen. ext_replay is the caller's codes (or null); no kernel reads it: the host stages the slots of a model
  // that is NOT resident into ext_gen before the mixer runs (RunPipelined).
  fx::State* fx;                // null = FXCM replayed
  void* paq8;                   // null = PAQ8 replayed
  u16* ext_gen;
  const u16* ext_replay;
  u32* lstm_fx;                 // [n_bytes*8] lstmpr | lstmex << 16 FXCM consumes while perceiving bit t (written by the LSTM kernel)
  CoderState* coder;            // optional device arithmetic coder fed with (p_out, bit); null = off
  unsigned long long* prof;     // optional [32] per-phase SM-cycle accumulators (null = off)
};

}  // namespace cmixb200
#endif
