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
//   grouped, groups, group_max       in the clashing 7-slot maps: the contexts that share a key with another (the ones
//                                    p8_number walks), their groups (contexts joined by shared keys, transitively) and the
//                                    largest group; group_maps2 counts the map-bits with two or more groups
// Include it before paq8_host.h / fxcm_host.h; call end_bit() after every bit and reset() after pretraining.
//
// Per-bit log (open_log; the census build of the device library writes the same words, paq8.cuh / fxcm.cuh CENSUS_*):
//   PAQ8, 3 u32 per bit   w0 = clashing 7-slot maps (bit k: map k of p8_cm's order) | clashing history maps << 16 | bpos << 20
//                         w1 = flagged draws | copies of P8CmCache the probe checks << 16 (the cn of every 7-slot map on a
//                              staying bit, 0 on a move bit)
//                         w2 = the 7-slot maps that clash under the bucket rule (cm_touched on every bit)
//   FXCM, 1 u32 per bit   the clashing maps among the 31
// The device's third PAQ8 word is not w2 but the copies its probe filled (the host has no cache).
//
// -DCENSUS_PERMUTE=<seed>: in every map the rule finds clash-free, the contexts are evaluated in a seeded pseudo-random
// order instead of in order, on every bit and in all three families (cm_mix: each flagged context takes the draw of its
// in-order rank, as the device's lanes do; cm2_mix_body; fxcm_model.h map_bit). If the rule is right, the codes stay the
// reference's. "permuted" in the JSON line counts the map-bits whose order changed. -DCENSUS_REVERSE: the reverse order, on
// the 7-slot maps' staying bits only.
// -DCENSUS_GROUPS_PERMUTE=<seed>: every clashing 7-slot map as the device runs it (p8_number, p8_apply_cm), its free contexts
// in a seeded pseudo-random order interleaved with the grouped ones (p8_cm_groups_order); "permuted" counts the map-bits whose
// order changed.
#pragma once
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

namespace census {

struct Counts {
  int draws = 0, bp = 0;                         // this bit
  bool clash7 = false, bucket7 = false, clash_hist = false, fx_clash = false;
  uint32_t mask7 = 0, mask_bucket = 0, mask_hist = 0, mask_fx = 0, checked = 0;
  long bits = 0, draw_bits = 0, max_draws = 0, gt24 = 0, gt24_fast = 0, clash7_bits = 0, clash_hist_bits = 0, fx_clash_bits = 0;
  long clash7_stay = 0, clash7_bpos[8] = {}, bucket7_bpos[8] = {}, permuted = 0;
  long grouped = 0, groups = 0, group_max = 0, group_maps2 = 0;
  std::map<const void*, long> p8_map;            // PAQ8 map -> bits with a clash in it
  std::map<int, long> fx_map;                    // FXCM map id -> bits with a clash in it
};
inline Counts& C() { static Counts c; return c; }
inline std::map<const void*, int>& order() { static std::map<const void*, int> o; return o; }   // PAQ8 map -> index (device order)
struct Log { FILE* f = nullptr; bool fx = false; };
inline Log& L() { static Log l; return l; }
inline void reset() { C() = Counts(); }

// The PAQ8 maps in the device's order: the sixteen 7-slot maps of p8_cm, then the three history maps of p8_cm2.
inline void set_maps(const std::vector<std::pair<std::string, const void*>>& maps) {
  for (size_t k = 0; k < maps.size(); ++k) order()[maps[k].second] = (int)k;
}
inline uint32_t map_flag(const void* m) {    // bit k: map k of set_maps' list
  auto it = order().find(m);
  return it == order().end() ? 0u : 1u << it->second;
}
// The per-bit log; path nullptr: none. fx: the FXCM layout.
inline void open_log(const char* path, bool fx) {
  if (path && *path) { L().f = fopen(path, "wb"); L().fx = fx; }
}

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
inline int root(const int* grp, int i) { while (grp[i] != i) i = grp[i]; return i; }
// The groups of a 7-slot map on this bit: contexts that share a key (p8_probe_cm's keys: slot keys on a staying bit, buckets
// on the others) are joined, transitively. grp[i] = the first context of i's group, size[i] = the size of i's group. Returns
// p8_probe_cm's verdict: whether any key is shared.
template <class Map> bool p8_cm_groups(const Map& m, int c0, int bp, int* grp, int* size) {
  std::map<uint32_t, int> first;            // key -> the first context that claimed it
  uint32_t ids[5];
  bool clash = false;
  for (int i = 0; i < m.cn; ++i) grp[i] = i;
  for (int i = 0; i < m.cn; ++i) {
    const int n = staying(bp) ? cm_slot_keys(m, i, ids) : cm_touched(m, i, c0, bp, ids);
    for (int a = 0; a < n; ++a) {
      const auto r = first.emplace(ids[a], i);
      if (r.second || r.first->second == i) continue;      // new, or the context's own repeat
      clash = true;
      const int x = root(grp, i), z = root(grp, r.first->second);
      grp[x > z ? x : z] = x > z ? z : x;
    }
  }
  for (int i = 0; i < m.cn; ++i) size[i] = 0;
  for (int i = 0; i < m.cn; ++i) ++size[grp[i] = root(grp, i)];
  for (int i = 0; i < m.cn; ++i) size[i] = size[grp[i]];
  return clash;
}
// p8_probe_cm's verdict for a 7-slot map
template <class Map> bool p8_cm_clash(const Map& m, int c0, int bp) {
  int grp[64], size[64];
  return p8_cm_groups(m, c0, bp, grp, size);
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
  if (bucket) C().mask_bucket |= map_flag(&m);
  if (staying(bp)) C().checked += m.cn;
  int grp[64], size[64];
  if (p8_cm_groups(m, c0, bp, grp, size)) {
    C().clash7 = true; C().mask7 |= map_flag(&m); ++C().p8_map[&m];
    int groups = 0;
    for (int i = 0; i < m.cn; ++i) {
      if (size[i] < 2) continue;
      ++C().grouped;
      if (grp[i] == i) ++groups;
      if (size[i] > C().group_max) C().group_max = size[i];
    }
    C().groups += groups;
    C().group_maps2 += groups >= 2;
  }
}

#if defined(CENSUS_PERMUTE) || defined(CENSUS_REVERSE)
// The order of n contexts: a seeded Fisher-Yates shuffle (one generator over the run), or the reverse order.
inline void order_of(int n, int* perm) {
  for (int i = 0; i < n; ++i) perm[i] = i;
#ifdef CENSUS_PERMUTE
  static uint64_t s = 0x9E3779B97F4A7C15ull ^ (uint64_t)(CENSUS_PERMUTE);
  for (int i = n - 1; i > 0; --i) {
    s ^= s << 13; s ^= s >> 7; s ^= s << 17;
    const int j = (int)(s % (uint64_t)(i + 1));
    const int t = perm[i]; perm[i] = perm[j]; perm[j] = t;
  }
#else
  for (int i = 0; i < n; ++i) perm[i] = n - 1 - i;
#endif
  for (int i = 0; i < n; ++i) if (perm[i] != i) { ++C().permuted; break; }
}
// cm_mix on a map the rule finds clash-free: the contexts in order_of's order, each flagged context taking the draw of its
// in-order rank (what the device's lanes do in any order) and storing the aged state pass 1 computed (p8_probe_cm).
// Returns cm_mix's result, or -1 where cm_mix runs in order.
template <class Tab, class Map, class Out, class Rnd> int p8_cm_order(const Tab& T, Map& m, Out& o, Rnd& rnd, int y, int c0, int bp, int c1) {
#ifdef CENSUS_REVERSE
  if (!staying(bp)) return -1;
#endif
  if (p8_cm_clash(m, c0, bp)) return -1;
  int ns[64], perm[64];
  uint32_t draw[64];
  for (int i = 0; i < m.cn; ++i) {
    ns[i] = cm_next_state(T, m, i, y);
    if (ns[i] >= 204) draw[i] = rnd_next(rnd);
  }
  order_of(m.cn, perm);
  int result = 0;
  for (int q = 0; q < m.cn; ++q) {
    const int i = perm[q];
    int s = ns[i];
    if (s >= 204 && (uint32_t)(draw[i] << ((452 - s) >> 3)) != 0) s -= 4;   // cm_draw_hits
    Out oi = o;
    oi.n = o.n + 5 * i;
    result += cm_step(m, i, oi, s, y, c0, bp, c1);
  }
  o.n += 5 * m.cn;
  if (bp == 7) m.cn = 0;
  return result;
}
#endif
#ifdef CENSUS_GROUPS_PERMUTE
// cm_mix on a map the rule finds clashing, as the device runs it: the grouped contexts (those that share a key with another,
// p8_number) in program order, each with the aged state and flag it finds when its turn comes; the free contexts (p8_apply_cm)
// with the state and flag pass 1 computed, in a seeded pseudo-random order interleaved with the grouped ones. Each flagged
// context takes the draw of its in-order rank among the final flags. That rank counts the flags of the grouped contexts before
// it, so a flagged free context goes after those; an unflagged one goes anywhere. Returns cm_mix's result, or -1 where
// cm_mix runs in order (a clash-free map).
template <class Tab, class Map, class Out, class Rnd> int p8_cm_groups_order(const Tab& T, Map& m, Out& o, Rnd& rnd, int y, int c0, int bp, int c1) {
  int grp[64], size[64];
  if (!p8_cm_groups(m, c0, bp, grp, size)) return -1;
  static uint64_t s = 0x9E3779B97F4A7C15ull ^ (uint64_t)(CENSUS_GROUPS_PERMUTE);
  const int cn = m.cn;
  int ns[64];
  bool flag[64];
  uint32_t draw[64];
  Rnd r = rnd;
  for (int j = 0; j < cn; ++j) draw[j] = rnd_next(r);          // the draw of each rank
  // grouped context q (program order among them) at time 2q + 1, a free one at a random even time: 0 is before the first
  // grouped context, 2G after the last; a flagged one not before 2 * (the grouped contexts before it)
  std::vector<std::pair<uint64_t, int>> order;
  int g = 0;
  for (int i = 0; i < cn; ++i) g += size[i] > 1;
  for (int i = 0, before = 0; i < cn; ++i) {
    ns[i] = cm_next_state(T, m, i, y);
    flag[i] = ns[i] >= 204;
    s ^= s << 13; s ^= s >> 7; s ^= s << 17;
    if (size[i] > 1) { order.push_back({(uint64_t)(2 * before + 1) << 32, i}); ++before; continue; }
    const int lo = flag[i] ? before : 0;
    const uint64_t gap = (uint64_t)lo + s % (uint64_t)(g - lo + 1);
    order.push_back({(2 * gap) << 32 | (s >> 40), i});
  }
  std::sort(order.begin(), order.end());
  for (int q = 0; q < cn; ++q) if (order[q].second != q) { ++C().permuted; break; }
  int result = 0;
  for (const auto& e : order) {
    const int i = e.second;
    int st = ns[i];
    if (size[i] > 1) { st = cm_next_state(T, m, i, y); flag[i] = st >= 204; }
    if (flag[i]) {
      int rank = 0;
      for (int j = 0; j < i; ++j) rank += flag[j];
      if ((uint32_t)(draw[rank] << ((452 - st) >> 3)) != 0) st -= 4;   // cm_draw_hits
    }
    Out oi = o;
    oi.n = o.n + 5 * i;
    result += cm_step(m, i, oi, st, y, c0, bp, c1);
  }
  for (int i = 0; i < cn; ++i) if (flag[i]) rnd_next(rnd);
  o.n += 5 * cn;
  if (bp == 7) m.cn = 0;
  return result;
}
#endif
#ifdef CENSUS_PERMUTE
// cm2_mix_body on a history map the rule finds clash-free: cm2_step per context (p8_apply_cm2's lanes) in order_of's order
template <class Map, class Out> int p8_cm2_order(Map& m, Out& o, int y, int bpos) {
  std::set<uint32_t> seen;
  uint32_t ids[5];
  for (int i = 0; i < m.index; ++i) {
    const int n = cm2_touched(m, i, bpos, ids);
    if (n && claim(seen, ids, n)) return -1;
  }
  int perm[64], result = 0;
  order_of(m.index, perm);
  for (int q = 0; q < m.index; ++q) {
    Out oi = o;
    oi.n = o.n + 7 * perm[q];
    result += cm2_step(m, perm[q], oi, y, bpos);
  }
  o.n += 7 * m.index;
  return result;
}
// map_bit on an FXCM map the rule finds clash-free: map_ctx_bit per context (fxcm.cuh phase D) in order_of's order.
// Returns false where map_bit runs in order.
template <class State, class Out> bool fx_map_order(State& S, int id, const Out& o) {
  std::set<uint32_t> seen;
  uint32_t ids[5];
  const int cn = S.map[id].cn;
  for (int i = 0; i < cn; ++i) {
    const int n = map_touched(S, id, i, ids);
    if (n && claim(seen, ids, n)) return false;
  }
  int perm[64];
  uint32_t result = 0;
  order_of(cn, perm);
  for (int q = 0; q < cn; ++q) result += map_ctx_bit(S, id, perm[q], o);
  map_finish(S, id, result);
  return true;
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
  if (clash) { C().clash_hist = true; C().mask_hist |= map_flag(&m) >> 16; ++C().p8_map[&m]; }
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
  if (clash) { C().fx_clash = true; C().mask_fx |= 1u << id; ++C().fx_map[id]; }
}

inline void end_bit() {
  Counts& c = C();
  if (L().f) {
    if (L().fx) fwrite(&c.mask_fx, 4, 1, L().f);
    else {
      const uint32_t w[3] = {c.mask7 | c.mask_hist << 16 | (uint32_t)c.bp << 20, (uint32_t)c.draws | c.checked << 16, c.mask_bucket};
      fwrite(w, 4, 3, L().f);
    }
  }
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
  c.mask7 = c.mask_bucket = c.mask_hist = c.mask_fx = c.checked = 0;
}

// One JSON line: "census {...}". `maps` names the PAQ8 maps (in the device's order); FXCM maps are named by id.
inline void print(FILE* f, const std::vector<std::pair<std::string, const void*>>& maps) {
  if (L().f) { fclose(L().f); L().f = nullptr; }
  const Counts& c = C();
  fprintf(f, "census {\"bits\": %ld, \"draw_bits\": %ld, \"max_draws\": %ld, \"gt24\": %ld, \"gt24_fast\": %ld, \"clash7\": %ld, "
             "\"clash7_stay\": %ld, \"clash_hist\": %ld, \"fx_clash\": %ld, \"permuted\": %ld, ", c.bits, c.draw_bits, c.max_draws,
          c.gt24, c.gt24_fast, c.clash7_bits, c.clash7_stay, c.clash_hist_bits, c.fx_clash_bits, c.permuted);
  fprintf(f, "\"grouped\": %ld, \"groups\": %ld, \"group_max\": %ld, \"group_maps2\": %ld, ", c.grouped, c.groups, c.group_max,
          c.group_maps2);
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
#if defined(CENSUS_PERMUTE) || defined(CENSUS_REVERSE)
#define P8_CM_ORDER(T, m, o, rnd, y, c0, bp, c1) do { const int r_ = census::p8_cm_order(T, m, o, rnd, y, c0, bp, c1); if (r_ >= 0) return r_; } while (0)
#elif defined(CENSUS_GROUPS_PERMUTE)
#define P8_CM_ORDER(T, m, o, rnd, y, c0, bp, c1) do { const int r_ = census::p8_cm_groups_order(T, m, o, rnd, y, c0, bp, c1); if (r_ >= 0) return r_; } while (0)
#endif
#ifdef CENSUS_PERMUTE
#define P8_CM2_ORDER(m, o, y, bpos) do { const int r_ = census::p8_cm2_order(m, o, y, bpos); if (r_ >= 0) return r_; } while (0)
#define FX_MAP_ORDER(S, id, o) do { if (census::fx_map_order(S, id, o)) return; } while (0)
#endif
#define FX_CENSUS_MAP(S, id) census::fx_map(S, id)
