// tools/census.h — host census of the paths only the device kernels have (TEST INFRASTRUCTURE, not part of the product).
//
// paq8.cuh and fxcm.cuh run the contexts of a context map on separate lanes and fall back to one lane walking the map in order
// when two contexts touch the same 64-byte bucket in one bit; PAQ8's 7-slot maps also share one pseudo-random sequence, whose
// draws the device numbers across lanes (at most 24 per step of the generator, replayed from a snapshot beyond that). The
// host builds always run the in-order loops, so the CPU pinning of the models says nothing about how often those device paths
// run. Compiled into tools/paq8_check.cpp / tools/fxcm_check.cpp with -DCENSUS, this header applies the device's per-bit rule
// (cm_touched / cm2_touched / map_touched and p8_claim's bucket set, on a staying bit cm_slot_keys for the 7-slot maps, the
// >= 204 draw flag of p8_probe_cm) where the in-order loops start, and counts per coded bit:
//   clash7 / clash_hist / fx_clash   bits in which some PAQ8 7-slot map / PAQ8 history map / FXCM map clashed, and per map
//   clash7_stay                      bits with a 7-slot clash on a staying bit (bpos 1, 3, 4, 6, 7: the slot rule)
//   clash7_bpos / bucket7_bpos       7-slot clash bits per bpos under the device's rule / under the bucket rule on every bit
//   draw_bits, max_draws             bits with any draw of the shared sequence, the most draws in one bit
//   gt24, gt24_fast                  bits with more than 24 draws; of those, bits without a 7-slot clash (the replay path)
// Include it before paq8_host.h / fxcm_host.h; call end_bit() after every bit and reset() after pretraining.
#pragma once
#include <stdint.h>
#include <stdio.h>

#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

namespace census {

struct Counts {
  int draws = 0, bp = 0;                         // this bit
  bool clash7 = false, bucket7 = false, clash_hist = false, fx_clash = false;
  long bits = 0, draw_bits = 0, max_draws = 0, gt24 = 0, gt24_fast = 0, clash7_bits = 0, clash_hist_bits = 0, fx_clash_bits = 0;
  long clash7_stay = 0, clash7_bpos[8] = {}, bucket7_bpos[8] = {};
  std::map<const void*, long> p8_map;            // PAQ8 map -> bits with a clash in it
  std::map<int, long> fx_map;                    // FXCM map id -> bits with a clash in it
};
inline Counts& C() { static Counts c; return c; }
inline void reset() { C() = Counts(); }

// p8_claim / fx_claim: a context's own repeats are removed; a bucket another context of the map touched this bit is a clash
inline bool claim(std::set<uint32_t>& seen, const uint32_t* ids, int n) {
  bool clash = false;
  for (int a = 0; a < n; ++a) {
    bool dup = false;
    for (int b = 0; b < a; ++b) dup = dup || ids[b] == ids[a];
    if (!dup && !seen.insert(ids[a]).second) clash = true;
  }
  return clash;
}

inline bool staying(int bp) { return (0xDA >> bp) & 1; }     // cm_staying
// p8_probe_cm's verdict for a 7-slot map: its contexts' slot keys on a staying bit, their buckets on the others
template <class Map> bool p8_cm_clash(const Map& m, int c0, int bp) {
  std::set<uint32_t> seen;
  uint32_t ids[5];
  bool clash = false;
  for (int i = 0; i < m.cn; ++i)
    if (claim(seen, ids, staying(bp) ? cm_slot_keys(m, i, ids) : cm_touched(m, i, c0, bp, ids))) clash = true;
  return clash;
}
// p8_probe_cm: every context i < cn claims its keys and flags a draw when its aged state is >= 204
template <class Tab, class Map> void p8_cm(const Tab& T, const Map& m, int y, int c0, int bp) {
  std::set<uint32_t> seen;
  uint32_t ids[5];
  bool bucket = false;
  for (int i = 0; i < m.cn; ++i) {
    if (cm_next_state(T, m, i, y) >= 204) ++C().draws;
    if (claim(seen, ids, cm_touched(m, i, c0, bp, ids))) bucket = true;
  }
  C().bp = bp;
  C().bucket7 |= bucket;
  if (p8_cm_clash(m, c0, bp)) { C().clash7 = true; ++C().p8_map[&m]; }
}
#ifdef CENSUS_REVERSE
// Test of the slot rule's exactness: on a staying bit where it finds no clash in map m, evaluate the contexts in REVERSE
// order, each flagged context taking the draw of its in-order rank (what the device's lanes do in any order). Returns
// cm_mix's result, or -1 where cm_mix runs in order.
template <class Tab, class Map, class Out, class Rnd> int p8_cm_reverse(const Tab& T, Map& m, Out& o, Rnd& rnd, int y, int c0, int bp, int c1) {
  if (!staying(bp) || p8_cm_clash(m, c0, bp)) return -1;
  bool flag[64];
  uint32_t draw[64];
  for (int i = 0; i < m.cn; ++i) {
    flag[i] = cm_next_state(T, m, i, y) >= 204;
    if (flag[i]) draw[i] = rnd_next(rnd);
  }
  int result = 0;
  for (int i = m.cn - 1; i >= 0; --i) {
    int ns = cm_next_state(T, m, i, y);
    if (flag[i] && ns >= 204 && (uint32_t)(draw[i] << ((452 - ns) >> 3)) != 0) ns -= 4;   // cm_draw_hits
    Out oi = o;
    oi.n = o.n + 5 * i;
    result += cm_step(m, i, oi, ns, y, c0, bp, c1);
  }
  o.n += 5 * m.cn;
  if (bp == 7) m.cn = 0;
  return result;
}
#endif
// p8_probe_cm2 (after cm2_begin)
template <class Map> void p8_cm2(const Map& m, int bpos) {
  std::set<uint32_t> seen;
  uint32_t ids[5];
  bool clash = false;
  for (int i = 0; i < m.index; ++i) {
    const int n = cm2_touched(m, i, bpos, ids);
    if (n && claim(seen, ids, n)) clash = true;
  }
  if (clash) { C().clash_hist = true; ++C().p8_map[&m]; }
}
// fxcm.cuh phase C
template <class State> void fx_map(const State& S, int id) {
  std::set<uint32_t> seen;
  uint32_t ids[5];
  bool clash = false;
  for (int i = 0; i < S.map[id].cn; ++i) {
    const int n = map_touched(S, id, i, ids);
    if (n && claim(seen, ids, n)) clash = true;
  }
  if (clash) { C().fx_clash = true; ++C().fx_map[id]; }
}

inline void end_bit() {
  Counts& c = C();
  ++c.bits;
  c.draw_bits += c.draws > 0;
  if (c.draws > c.max_draws) c.max_draws = c.draws;
  c.gt24 += c.draws > 24;
  c.gt24_fast += c.draws > 24 && !c.clash7;
  c.clash7_bits += c.clash7;
  c.clash7_stay += c.clash7 && staying(c.bp);
  c.clash7_bpos[c.bp] += c.clash7;
  c.bucket7_bpos[c.bp] += c.bucket7;
  c.clash_hist_bits += c.clash_hist;
  c.fx_clash_bits += c.fx_clash;
  c.draws = 0;
  c.clash7 = c.bucket7 = c.clash_hist = c.fx_clash = false;
}

// One JSON line: "census {...}". `maps` names the PAQ8 maps (in the device's order); FXCM maps are named by id.
inline void print(FILE* f, const std::vector<std::pair<std::string, const void*>>& maps) {
  const Counts& c = C();
  fprintf(f, "census {\"bits\": %ld, \"draw_bits\": %ld, \"max_draws\": %ld, \"gt24\": %ld, \"gt24_fast\": %ld, \"clash7\": %ld, "
             "\"clash7_stay\": %ld, \"clash_hist\": %ld, \"fx_clash\": %ld, ", c.bits, c.draw_bits, c.max_draws, c.gt24, c.gt24_fast,
          c.clash7_bits, c.clash7_stay, c.clash_hist_bits, c.fx_clash_bits);
  const char* sep = "";
  for (const auto* v : {c.clash7_bpos, c.bucket7_bpos}) {
    fprintf(f, "\"%s\": [", v == c.clash7_bpos ? "clash7_bpos" : "bucket7_bpos");
    for (int b = 0; b < 8; ++b) fprintf(f, "%s%ld", b ? ", " : "", v[b]);
    fprintf(f, "], ");
  }
  fprintf(f, "\"maps\": {");
  for (const auto& nm : maps) {
    auto it = c.p8_map.find(nm.second);
    fprintf(f, "%s\"p8 %s\": %ld", sep, nm.first.c_str(), it == c.p8_map.end() ? 0L : it->second);
    sep = ", ";
  }
  for (const auto& kv : c.fx_map) { fprintf(f, "%s\"fxcm %d\": %ld", sep, kv.first, kv.second); sep = ", "; }
  fprintf(f, "}}\n");
}

}  // namespace census

#define P8_CENSUS_CM(T, m, y, c0, bp) census::p8_cm(T, m, y, c0, bp)
#define P8_CENSUS_CM2(m, bpos) census::p8_cm2(m, bpos)
#ifdef CENSUS_REVERSE
#define P8_CM_ORDER(T, m, o, rnd, y, c0, bp, c1) do { const int r_ = census::p8_cm_reverse(T, m, o, rnd, y, c0, bp, c1); if (r_ >= 0) return r_; } while (0)
#endif
#define FX_CENSUS_MAP(S, id) census::fx_map(S, id)
