// oracle/port/port.h — TEST INFRASTRUCTURE (CPU restatement of the hot path).
//
// Plain scalar C++ restatement of the reference's Predictor::Predict/Perceive
// path (reference src/predictor.cpp:361-487) for the rows of SURVEY.md §8(a)
// that the CUDA engine runs on the device: a1-a12 and a16-a18. The three big
// third-party model families (PAQ8 a13, FXCM a14, PPMD a15) are NOT restated:
// their per-bit outputs are *replayed* from a dump produced by the real
// reference (oracle/_ref/oracle_dump, built from the reference checkout by
// oracle/Makefile).
//
// Pinning: tests/test_oracle_port.py checks this port bit-for-bit against the
// per-bit Predict() floats, the 2078 stretched inputs, the 47 mixer outputs and
// the LSTM byte distributions dumped from the unmodified reference (golden
// fixtures under tests/golden/, generator script committed).
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may
// load this library. The product (cmix_b200/) never links or calls it.
#ifndef ORACLE_PORT_H
#define ORACLE_PORT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  OP_N_FXCM = 431,
  OP_N_PAQ8 = 1591,
  OP_N_EXT = 431 + 1591,   // replayed 12-bit codes per bit (0xFFFF = 0.5)
  OP_N_INPUTS = 2078,
  OP_N_MIXERS = 47,
};

typedef struct op_predictor op_predictor;

// vocab[i] != 0 iff byte i occurs in the coded stream (runner.cpp:196-202).
op_predictor* op_create(const uint8_t vocab[256]);
void op_destroy(op_predictor*);

// One Predict() (predictor.cpp:361). `ext` = the 2022 FXCM+PAQ8 codes the
// reference's models hold for THIS bit.
float op_predict(op_predictor*, const uint16_t* ext);
// One Perceive(bit) (predictor.cpp:421). When this bit completes a byte,
// `ppmd_after_byte` must hold the 256-entry PPMD distribution produced by
// PPMD::ByteUpdate for that byte (ppmd.cpp:1328); otherwise it is ignored.
void op_perceive(op_predictor*, int bit, const float* ppmd_after_byte);
// One Pretrain(bit) (predictor.cpp:471): models + contexts only.
void op_pretrain(op_predictor*, int bit);

// Introspection for component-level parity tests.
void op_get_inputs(const op_predictor*, float out[OP_N_INPUTS]);
void op_get_mixer_outputs(const op_predictor*, float out[OP_N_MIXERS]);
void op_get_mixer_contexts(const op_predictor*, uint32_t out[OP_N_MIXERS]);
void op_get_lstm_probs(const op_predictor*, float out[256]);

// Whole-stream helper: replays n_bytes of `stream` and writes one float per bit.
void op_run(op_predictor*, const uint8_t* stream, size_t n_bytes,
            const uint16_t* ext /*[n_bytes*8][OP_N_EXT]*/,
            const float* ppmd /*[n_bytes][256]*/, float* p_out /*[n_bytes*8]*/);

// Arithmetic coder restatement (coder/encoder.cpp:10-39, coder/decoder.cpp:16-39).
typedef struct op_encoder op_encoder;
op_encoder* op_enc_create(void);
void op_enc_encode(op_encoder*, float p, int bit);
// Flushes and copies the coded bytes out; returns their count (needs cap >= count).
size_t op_enc_finish(op_encoder*, uint8_t* out, size_t cap);
void op_enc_destroy(op_encoder*);
typedef struct op_decoder op_decoder;
op_decoder* op_dec_create(const uint8_t* data, size_t n);
int op_dec_decode(op_decoder*, float p);
void op_dec_destroy(op_decoder*);

// libm probes used by tests to pin the device transcendental restatements.
float op_libm_expf(float x);
float op_libm_tanhf(float x);
float op_logistic(float x);

#ifdef __cplusplus
}
#endif
#endif
