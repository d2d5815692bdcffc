/* include/cmixb200.h — C-ABI of the H100-native cmix predictor.
 *
 * Drop-in boundary: the reference's `class Predictor` (reference
 * src/predictor.h:17-53), the only interface the reference's arithmetic coder
 * (src/coder/encoder.cpp:15,23, src/coder/decoder.cpp:21,31), its runner
 * (src/runner.cpp:205,246) and its pretrainer (src/preprocess/preprocessor.cpp:52,66)
 * use. cmix_b200/shim/predictor.{h,cpp} re-declares that class with the same
 * signature on top of these entry points (see INTEGRATION.md).
 *
 * Plain pointers and sizes only; no C++ or torch types. All functions return
 * CMIXB200_OK (0) or an error code; cmixb200_last_error() describes the failure.
 * There is no CPU fallback behind any of them: without a usable sm_90 device
 * they fail with CMIXB200_ERR_CUDA.
 */
#ifndef CMIXB200_H
#define CMIXB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { CMIXB200_OK = 0, CMIXB200_ERR_CUDA = 1, CMIXB200_ERR_ARG = 2,
       CMIXB200_ERR_CAPACITY = 3 /* a model arena is full (PPMD: raise CMIXB200_PPMD_MB); the stream is unusable */,
       CMIXB200_ERR_UNSUPPORTED = 4 /* the resident PAQ8 met an image / 16-bit PCM WAV audio / JPEG block it does not model; the stream is unusable */ };

enum {
  CMIXB200_N_EXT = 2022,  /* replayed FXCM (431) + PAQ8 (1591) outputs per bit, as 12-bit codes k
                             meaning k/4095 (paq8.cpp:497-500, fxcmv1.cpp:97-101); 0xFFFF = 0.5 */
};

typedef struct cmixb200_predictor cmixb200_predictor;

/* Predictor::Predictor(const std::vector<bool>& vocab) (predictor.cpp:24-37) plus the
 * `char* dictionary_path` side channel of runner.cpp:17 (may be NULL). `device` = CUDA ordinal. */
int cmixb200_create(const uint8_t vocab[256], const char* dictionary_path, int device,
                    cmixb200_predictor** out);
void cmixb200_destroy(cmixb200_predictor*);

/* Same, choosing which of the big model groups are REPLAYED instead of device resident: a replayed group costs no HBM
 * and takes its codes from cmixb200_feed_external_bit / the `ext` argument of the bulk calls; a bulk call without `ext`
 * gives its inputs p = 0.5. CMIXB200_REPLAY_PAQ8 is how image, 16-bit PCM WAV audio and JPEG data are coded (the resident
 * PAQ8 returns CMIXB200_ERR_UNSUPPORTED there; it codes 8-bit PCM WAV audio itself). Predictors of one batch must replay the same groups, and decode_bytes needs
 * every group resident. cmixb200_create == replay_mask 0 == everything that is resident is used. */
enum { CMIXB200_REPLAY_FXCM = 1, CMIXB200_REPLAY_PAQ8 = 2 };
int cmixb200_create_ex(const uint8_t vocab[256], const char* dictionary_path, int device, unsigned replay_mask,
                       cmixb200_predictor** out);

/* float Predictor::Predict() (predictor.cpp:361). Returns -1 on failure. */
float cmixb200_predict(cmixb200_predictor*);
/* void Predictor::Perceive(int bit) (predictor.cpp:421). */
int cmixb200_perceive(cmixb200_predictor*, int bit);
/* void Predictor::Pretrain(int bit) (predictor.cpp:471). */
int cmixb200_pretrain(cmixb200_predictor*, int bit);

/* Model groups that are not yet device resident (SURVEY §8 rows a13-a15: PAQ8, FXCM, PPMD) enter
 * as replayed streams. Lock-step: feed the codes for the NEXT Predict(), and the 256-entry PPMD
 * byte distribution (ppmd.cpp:1328-1338) for the byte the next Perceive() calls complete.
 * Without them those inputs carry p = 0.5 / a flat distribution. */
int cmixb200_feed_external_bit(cmixb200_predictor*, const uint16_t codes[CMIXB200_N_EXT]);
int cmixb200_feed_external_byte(cmixb200_predictor*, const float ppmd[256]);

/* Bulk compress-direction path: the n_bytes*8 Predict()/Perceive() pairs of runner.cpp:101-119
 * (Compress) in one call; p_out receives the value Predict() returned before each bit.
 * HOST buffers (copies are part of the call). ext: [n_bytes*8][2022] or NULL; ppmd: [n_bytes][256] or NULL. */
int cmixb200_code_bytes(cmixb200_predictor*, const uint8_t* bytes, size_t n_bytes, const uint16_t* ext,
                        const float* ppmd, float* p_out);
/* Same with every buffer already in device memory. */
int cmixb200_code_bytes_device(cmixb200_predictor*, const uint8_t* d_bytes, size_t n_bytes,
                               const uint16_t* d_ext, const float* d_ppmd, float* d_p_out);
/* n_streams independent predictors (independent files) advanced together in one launch set. */
int cmixb200_code_batch_device(cmixb200_predictor** preds, int n_streams, const uint8_t* const* d_bytes,
                               size_t n_bytes, const uint16_t* const* d_ext, const float* const* d_ppmd,
                               float* const* d_p_out);
/* The batch entry point with HOST buffers: inputs are staged to the device in 1024-byte sub-steps on a
 * copy stream, double buffered, so the transfer of sub-step k+1 overlaps the kernels of sub-step k; the
 * probabilities return to p_out[s] the same way. All predictors must live on one device. */
int cmixb200_code_batch(cmixb200_predictor** preds, int n_streams, const uint8_t* const* bytes, size_t n_bytes,
                        const uint16_t* const* ext, const float* const* ppmd, float* const* p_out);
/* Device arithmetic coder for the compress direction: replaces Encoder::Encode / Encoder::Flush
 * (src/coder/encoder.cpp:14-39). Between begin and finish every bulk call (code_bytes*, code_batch*)
 * also feeds its (probability, bit) pairs through the coder on the device; finish flushes and copies
 * the archive bytes (without runner.cpp's header) to the HOST buffer `out`. capacity_bytes bounds the
 * archive; overflow is reported by finish, never written past. */
int cmixb200_coder_begin(cmixb200_predictor*, size_t capacity_bytes);
int cmixb200_coder_finish(cmixb200_predictor*, uint8_t* out, size_t cap, size_t* n_out);

/* Decompress direction on the device (SURVEY.md §8f rank 1): replaces the loop of Decompress() (reference src/runner.cpp:121-137,
 * i.e. Decoder::Decoder + n_bytes*8 calls of Decoder::Decode, src/coder/decoder.cpp:3-39). `archive` is the arithmetic-coded body
 * (what follows the header runner.cpp:62-86 reads), `out` receives n_bytes decoded bytes. Per bit the library queues the predict
 * kernels, one decoder step and the perceive kernels; the bit never visits the host. Needs every model group resident and a stream
 * standing on a byte boundary. */
int cmixb200_decode_bytes(cmixb200_predictor*, const uint8_t* archive, size_t n_archive, uint8_t* out, size_t n_bytes);
/* preprocessor::Pretrain's loop (preprocessor.cpp:37-69) over a byte buffer (HOST). */
int cmixb200_pretrain_bytes(cmixb200_predictor*, const uint8_t* bytes, size_t n_bytes);

const char* cmixb200_last_error(void);
/* kernels launched by this predictor so far (bench.py's gpu_launches). */
unsigned long long cmixb200_kernel_launches(const cmixb200_predictor*);
/* CUDA-event timing of every bulk kernel on the stream it is launched on (bench.py's roofline):
 * enable, run bulk calls, then read the accumulated milliseconds and launch count of one kernel:
 * which = 0 mixer, 1 small models, 2 LSTM, 3 PPMD, 4 FXCM, 5 PAQ8 (each on its own CUDA stream). */
void cmixb200_time_mix_kernel(cmixb200_predictor*, int enable);
double cmixb200_kernel_ms(const cmixb200_predictor*, int which, unsigned long long* n_launches);
/* the cudaStream_t the mixer kernel runs on (for CUDA-event timing in bench.py). */
void* cmixb200_mix_stream(cmixb200_predictor*);

/* test hooks: copy intermediate arrays of the last bulk call to the host */
enum { CMIXB200_DBG_SMALL_X = 1, CMIXB200_DBG_SEL = 2, CMIXB200_DBG_LSTM_X = 3, CMIXB200_DBG_LSTM_PROBS = 4,
       CMIXB200_DBG_ERROR_FLAGS = 5,
       CMIXB200_DBG_PROFILE = 6 /* 64 u64 per-phase cycle counters; first fetch enables them */,
       CMIXB200_DBG_PPMD_PROBS = 7 /* 256 f32: the resident PPMD model's distribution after the last lock-step byte */,
       CMIXB200_DBG_PPMD_PROFILE = 9 /* 6 u64: cycles in symbol search, model update, suffix walk, ConvertSQ, emit; bytes */,
       CMIXB200_DBG_EXT_GEN = 10 /* [n_bytes*8][2022] u16: the codes the resident models wrote in the last bulk piece (<= 2048 bytes) */,
       CMIXB200_DBG_EXT_BIT = 11 /* [2022] u16: lock-step codes for the next Predict() */,
       CMIXB200_DBG_PPMD_USAGE = 12 /* 6 u32: contexts used / capacity, states used / capacity, text bytes used / capacity */,
       CMIXB200_DBG_PPMD_BULK = 8 /* [n_bytes][256] f32: the distributions the resident model produced in the last bulk call */ };
int cmixb200_debug_fetch(cmixb200_predictor*, int what, void* out, size_t bytes);

#ifdef __cplusplus
}
#endif
#endif
