// cmix_b200/shim/predictor.cpp — Predictor methods forwarding to the CUDA engine.
// Error convention of the reference: none (no return codes, no exceptions; allocation failure
// exits, e.g. fxcmv1.cpp:142). A CUDA failure therefore prints the C-ABI error and exits(1):
// a half-written archive is useless, and there is no CPU fallback to fall back to.
#include "predictor.h"

#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/cmixb200.h"

extern char* dictionary_path;   // defined in the reference's runner.cpp:17

static void die(const char* what) {
  fprintf(stderr, "cmix_b200: %s failed: %s\n", what, cmixb200_last_error());
  exit(1);
}

Predictor::Predictor(const std::vector<bool>& vocab) : impl_(0), pre_acc_(0), pre_nbits_(0) {
  uint8_t v[256];
  for (int i = 0; i < 256; ++i) v[i] = (i < (int)vocab.size() && vocab[i]) ? 1 : 0;
  const char* dev = getenv("CMIXB200_DEVICE");
  if (cmixb200_create(v, dictionary_path, dev ? atoi(dev) : 0, &impl_) != CMIXB200_OK) die("cmixb200_create");
}

Predictor::~Predictor() { cmixb200_destroy(impl_); }

void Predictor::FlushPretrain() {
  if (!pre_bytes_.empty()) {
    if (cmixb200_pretrain_bytes(impl_, pre_bytes_.data(), pre_bytes_.size()) != CMIXB200_OK) die("cmixb200_pretrain_bytes");
    pre_bytes_.clear();
  }
  // a trailing partial byte (never produced by the reference's callers) goes through the bit entry point
  for (unsigned k = pre_nbits_; k > 0; --k)
    if (cmixb200_pretrain(impl_, (pre_acc_ >> (k - 1)) & 1) != CMIXB200_OK) die("cmixb200_pretrain");
  pre_acc_ = pre_nbits_ = 0;
}

float Predictor::Predict() {
  if (!pre_bytes_.empty() || pre_nbits_) FlushPretrain();
  const float p = cmixb200_predict(impl_);
  if (p < 0) die("cmixb200_predict");
  return p;
}

void Predictor::Perceive(int bit) {
  if (cmixb200_perceive(impl_, bit) != CMIXB200_OK) die("cmixb200_perceive");
}

void Predictor::Pretrain(int bit) {
  pre_acc_ = (pre_acc_ << 1) | (bit ? 1u : 0u);
  if (++pre_nbits_ == 8) {
    pre_bytes_.push_back((unsigned char)pre_acc_);
    pre_acc_ = pre_nbits_ = 0;
    if (pre_bytes_.size() >= (64u << 10)) FlushPretrain();
  }
}
