// cmix_b200/csrc/census.cuh — per-bit census of the device's clash verdicts and of PAQ8's slot cache (TEST BUILD ONLY).
//
// The lane-per-context scheme of paq8.cuh and fxcm.cuh is exact only if the per-bit clash check finds every clash the
// rule defines, and PAQ8's slot cache (P8CmCache) only if no path leaves a stale copy valid. A device that flags too many
// clashes only loses time and one that flags too few, or reads a stale byte, may still code the fixtures correctly. Built
// with -DCMIXB200_CENSUS the kernels log, per coded bit and per stream, what tools/census.h computes on the host:
//   PAQ8, 3 u32 per bit   w0 = clashing 7-slot maps (bit k: p8_cm(S, k)) | clashing history maps << 16 | bpos << 20
//                         w1 = flagged draws (popcount of flag_mask) | copies of P8CmCache the probe checked << 16
//                         w2 = copies the probe filled because they were invalid
//   FXCM, 1 u32 per bit   the clashing maps among the 31
// and check every copy a staying bit reads (the slot's 7 bytes and the run record in p8_probe_cm and p8_cm_stay, the two
// StateMap words the probe loaded where cm_cell_inputs uses them) against HBM, counting checks and mismatches and keeping
// the first mismatch. The log lives in HBM, written by lane 0 of the model CTA and by atomics; a stream's log is found by
// its own model memory (the table of its first map: sparse.cm.t for PAQ8, map[0].t for FXCM), which the shared copy of its
// state block holds. Exported by engine.cu (cmixb200_census_*), not part of include/cmixb200.h. Without the flag every hook
// expands to nothing.
#pragma once

namespace cmixb200 {

enum { CENSUS_STREAMS = 8, CENSUS_P8_WORDS = 3 };
// One stream's counters (16 u32, read back as they are).
struct CensusHead {
  unsigned cap;                   // bits the per-bit arrays hold
  unsigned p8_bits, fx_bits;      // bits logged
  unsigned bit_checked, bit_filled;   // the current bit's probe (lane 0 of PAQ8's model CTA moves them into the record)
  unsigned slot_checks, sm_checks, mismatches;
  unsigned first_set, first_bit, first_map, first_ctx, first_byte, first_cached, first_hbm;
  unsigned overflow;              // bits past cap, not logged
};
static_assert(sizeof(CensusHead) == 16 * 4, "read back as 16 words");
struct CensusEntry { const void* p8_key; const void* fx_key; CensusHead* head; unsigned* p8; unsigned* fx; };

}  // namespace cmixb200

#ifdef CMIXB200_CENSUS
namespace cmixb200 {

static __device__ CensusEntry census_tab[CENSUS_STREAMS];

__device__ __forceinline__ const CensusEntry* census_find(const void* key, bool fx) {
  for (int k = 0; k < CENSUS_STREAMS; ++k) {
    const CensusEntry* e = &census_tab[k];
    if (e->head && (fx ? e->fx_key : e->p8_key) == key) return e;
  }
  return nullptr;
}
// a copy compared with HBM: byte 0-6 the slot, 7-8 the run record, 9-10 the StateMap words
__device__ __forceinline__ void census_check(const void* key, int map, int ctx, int byte, unsigned cached, unsigned hbm) {
  if (cached == hbm) return;
  const CensusEntry* e = census_find(key, false);
  if (!e) return;
  CensusHead* h = e->head;
  atomicAdd(&h->mismatches, 1u);
  if (atomicCAS(&h->first_set, 0u, 1u) == 0u) {
    h->first_bit = *(volatile unsigned*)&h->p8_bits; h->first_map = (unsigned)map; h->first_ctx = (unsigned)ctx;
    h->first_byte = (unsigned)byte; h->first_cached = cached; h->first_hbm = hbm;
  }
}
// p8_probe_cm / p8_cm_stay on a staying bit: lane tid's copy of context i of map k against HBM (before the lane's store)
template <class Cm> __device__ __forceinline__ void census_p8_copy(const void* key, const Cm& m, int k, int i, const unsigned char* slot,
                                                                  const unsigned char* run, bool probe, bool filled) {
  const CensusEntry* e = census_find(key, false);
  if (!e) return;
  atomicAdd(&e->head->slot_checks, 1u);
  if (probe) { atomicAdd(&e->head->bit_checked, 1u); if (filled) atomicAdd(&e->head->bit_filled, 1u); }
  for (int j = 0; j < 7; ++j) census_check(key, k, i, j, slot[j], m.t[m.cp0[i] + j]);
  census_check(key, k, i, 7, run[0], m.t[m.runp[i]]);
  census_check(key, k, i, 8, run[1], m.t[m.runp[i] + 1]);
}
// p8_cm_stay: the StateMap words the probe loaded, where cm_cell_inputs uses them (before its store of smt[so])
__device__ __forceinline__ void census_p8_sm(const void* key, int k, int i, const unsigned short* smt, int so, unsigned short sm_old, int s,
                                             unsigned short fresh) {
  const CensusEntry* e = census_find(key, false);
  if (!e) return;
  atomicAdd(&e->head->sm_checks, 1u);
  census_check(key, k, i, 9, sm_old, smt[so]);
  census_check(key, k, i, 10, fresh, smt[s]);
}
// lane 0 of PAQ8's model CTA after the epilogue: the bit's record
// (flag_mask: the ballots of the warps holding the first `lanes` lanes; the bits past them are not the map lanes')
__device__ __forceinline__ void census_p8_bit(const void* key, const int* clash, const int* clash2, const unsigned* flag_mask, int lanes, int bpos) {
  const CensusEntry* e = census_find(key, false);
  if (!e) return;
  CensusHead* h = e->head;
  unsigned w0 = (unsigned)bpos << 20, draws = 0;
  for (int k = 0; k < 16; ++k) w0 |= (clash[k] ? 1u : 0u) << k;
  for (int k = 0; k < 3; ++k) w0 |= (clash2[k] ? 1u : 0u) << (16 + k);
  for (int w = 0; 32 * w < lanes; ++w) draws += __popc(lanes - 32 * w >= 32 ? flag_mask[w] : flag_mask[w] & ((1u << (lanes - 32 * w)) - 1u));
  const unsigned checked = atomicExch(&h->bit_checked, 0u), filled = atomicExch(&h->bit_filled, 0u);
  const unsigned t = h->p8_bits;
  if (t < h->cap) {
    unsigned* r = e->p8 + (size_t)t * CENSUS_P8_WORDS;
    r[0] = w0; r[1] = draws | checked << 16; r[2] = filled;
  } else atomicAdd(&h->overflow, 1u);
  h->p8_bits = t + 1;
}
// lane 0 of FXCM's model CTA after phase C
__device__ __forceinline__ void census_fx_bit(const void* key, const int* clash) {
  const CensusEntry* e = census_find(key, true);
  if (!e) return;
  CensusHead* h = e->head;
  unsigned mask = 0;
  for (int k = 0; k < 31; ++k) mask |= (clash[k] ? 1u : 0u) << k;      // fx::N_MAPS
  const unsigned t = h->fx_bits;
  if (t < h->cap) e->fx[t] = mask;
  else atomicAdd(&h->overflow, 1u);
  h->fx_bits = t + 1;
}

// Host side, once per translation unit: CENSUS_MODULE(name) defines census_set_<name>, which installs the table.
#define CENSUS_MODULE(name) \
  cudaError_t census_set_##name(const CensusEntry* tab) { return cudaMemcpyToSymbol(census_tab, tab, sizeof(census_tab)); }
cudaError_t census_set_paq8(const CensusEntry*);
cudaError_t census_set_fxcm(const CensusEntry*);

}  // namespace cmixb200

#define CENSUS_P8_COPY(key, m, k, i, slot, run, probe, filled) ::cmixb200::census_p8_copy(key, m, k, i, slot, run, probe, filled)
#define CENSUS_P8_SM(key, k, i, smt, so, sm_old, s, fresh) ::cmixb200::census_p8_sm(key, k, i, smt, so, sm_old, s, fresh)
#define CENSUS_P8_BIT(key, clash, clash2, flag_mask, lanes, bpos) ::cmixb200::census_p8_bit(key, clash, clash2, flag_mask, lanes, bpos)
#define CENSUS_FX_BIT(key, clash) ::cmixb200::census_fx_bit(key, clash)
#else
#define CENSUS_P8_COPY(key, m, k, i, slot, run, probe, filled) do { } while (0)
#define CENSUS_P8_SM(key, k, i, smt, so, sm_old, s, fresh) do { } while (0)
#define CENSUS_P8_BIT(key, clash, clash2, flag_mask, lanes, bpos) do { } while (0)
#define CENSUS_FX_BIT(key, clash) do { } while (0)
#endif
