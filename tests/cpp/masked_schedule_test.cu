// Host-side checks of the masked arg-min kernel's schedule (expanded_tc.cuh EPI_MINLOC_MASKED, masked_nn.cuh); no GPU
// needed.
//   classify          reads "m n G", G group ends and m rows of G 0/1 characters from stdin and prints the class of
//                     every (64-row slab, 128-column half) tile from masked_tile_class, one row of digits per slab
//                     (compared with a numpy restatement by tests/test_masked_nn.py)
//   replay            replays the producer and the two consumer warpgroups of expanded_tc_kernel<kResident,
//                     EPI_MINLOC_MASKED> over random class bytes, resident and streaming (the kernel's own
//                     tc_producer_walk and skip helpers; only the consumers' waits and hand-backs are restated), and
//                     checks the invariants of
//                     DESIGN.md section 2 K3m: the same stage sequence on both sides, every loaded stage released by
//                     both warpgroups exactly once, the y block of every loaded item waited for and handed back by
//                     both, and nothing for a skipped item.  (Counts and order per warpgroup: that every warp of a
//                     warpgroup waits for each stage and the warpgroup meets before a NONE half's hand-back is the
//                     per-warp side of the protocol, DESIGN.md K3m.)
#include <cstdio>
#include <cstring>
#include <map>
#include <random>
#include <string>
#include <vector>
#include "../../raft_b200/csrc/masked_nn.cuh"

using namespace b2d;

static int classify()
{
  long long m, n, G;
  if (std::scanf("%lld %lld %lld", &m, &n, &G) != 3) return 2;
  std::vector<int> gi(G);
  for (auto& v : gi) if (std::scanf("%d", &v) != 1) return 2;
  const long long W = (m + 31) / 32;
  std::vector<unsigned> bits(static_cast<size_t>(W * G + 1), 0u);
  std::vector<char> row(G + 2);
  for (long long i = 0; i < m; ++i) {
    if (G == 0) continue;
    if (std::scanf("%s", row.data()) != 1) return 2;
    for (long long g = 0; g < G; ++g)
      if (row[g] == '1') bits[(i / 32) * G + g] |= 1u << (i % 32);
  }
  for (long long s = 0; s < (m + 63) / 64; ++s) {
    for (long long h = 0; h < (n + 127) / 128; ++h) std::printf("%d", masked_tile_class(bits.data(), gi.data(), G, m, n, s, h));
    std::printf("\n");
  }
  return 0;
}

// one (tile, k-block) stage load of the producer, and what the consumers did with it
struct Stage {
  int n_blk, mt0, mt, h, kb;
  int waits[2] = {0, 0}, releases[2] = {0, 0};
};

template <bool kResident>
static int replay_case(int nkb, int tiles_m, int nblocks, int n_last_half, int chunk, int grid, std::mt19937& rng, double p_dead)
{
  int bad = 0;
  // class bytes: a tile is dead with probability p_dead, otherwise random classes per (slab, half); a y block's second
  // half exists only if the block is not the last one or n_last_half
  std::vector<uint8_t> cls(static_cast<size_t>(nblocks) * tiles_m);
  std::uniform_real_distribution<double> u(0, 1);
  for (int nb = 0; nb < nblocks; ++nb)
    for (int mt = 0; mt < tiles_m; ++mt) {
      unsigned b = 0;
      const int nh = (nb < nblocks - 1 || n_last_half) ? 2 : 1;
      if (u(rng) >= p_dead)
        for (int h = 0; h < nh; ++h)
          for (int s = 0; s < 2; ++s) b |= static_cast<unsigned>(rng() % 3) << (2 * (2 * h + s));
      cls[static_cast<size_t>(nb) * tiles_m + mt] = static_cast<uint8_t>(b);
    }
  // the schedule fields as launch_tc fills them (every y block selected); the last y block has one half unless n_last_half
  TcParams p{};
  p.n = static_cast<int64_t>(nblocks) * TC_BN - (n_last_half ? 0 : TC_HN);
  p.tiles_m = tiles_m; p.tiles_sel = nblocks; p.chunk = chunk; p.chunks_m = (tiles_m + chunk - 1) / chunk;
  p.n_items  = static_cast<int64_t>(nblocks) * p.chunks_m;
  p.mask_cls = cls.data();
  // liveness of the ring: the producer refills position P - stages as position P, so a warpgroup must have handed
  // P - stages back before it waits for P
  constexpr int stages = TcCarve<kResident, EPI_MINLOC_MASKED>::stages;
  for (int cta = 0; cta < grid; ++cta) {
    // ---- producer: the kernel's own load order, recorded ----
    std::vector<Stage> loads;
    std::vector<int> b_loads;   // it_local of every y block load
    int items_loaded = 0;
    tc_producer_walk<kResident, true>(
        p, nkb, cta, grid,
        [&](int kb, uint32_t it_local, const TcItem&) { if (kb == 0) b_loads.push_back(static_cast<int>(it_local)); },
        [&](uint32_t a_it, const TcItem& t, int mt, int h, int kb) {
          if (a_it != loads.size()) ++bad;   // a_it counts the loaded stages
          if (loads.empty() || loads.back().n_blk != t.n_blk || loads.back().mt0 != t.mt0) ++items_loaded;
          loads.push_back(Stage{t.n_blk, t.mt0, mt, h, kb});
        });
    // ---- consumer warpgroups: the masked paths of the consumer loop, with the kernel's own skip decisions ----
    std::vector<int> a_end(2);
    std::map<int, int> bwait_item[2], brel_item[2];   // it_local -> count
    for (int wg = 0; wg < 2; ++wg) {
      std::vector<char> released(loads.size() + 1, 0);
      auto wait_at = [&](uint32_t it) {
        if (it >= static_cast<uint32_t>(stages) && it - stages < released.size() && !released[it - stages]) ++bad;
      };
      auto release_at = [&](uint32_t it) { if (it < released.size()) released[it] = 1; };
      uint32_t a_it = 0, itl = 0;
      for (int64_t item = cta; item < p.n_items; item += grid, ++itl) {
        const TcItem t     = tc_item(p, item);
        const uint8_t* c   = p.mask_cls + static_cast<int64_t>(t.n_blk) * p.tiles_m;
        const int mt_last  = mask_mt_last(c, t.mt0, t.mt1);
        if (mt_last < 0) { --itl; continue; }
        bool b_first = true;
        for (int mt = t.mt0; mt < t.mt1; ++mt) {
          const unsigned tcls = mask_cls_at(c, mt);
          if (tcls == 0u) continue;
          for (int h = 0; h < t.nh; ++h) {
            const bool release = tc_half_releases(kResident, h, t.nh);
            auto stage_at = [&](uint32_t it) -> Stage* {
              if (it >= loads.size()) { ++bad; return nullptr; }
              Stage* st = &loads[it];
              if (st->n_blk != t.n_blk || st->mt != mt || (!kResident && st->h != h)) ++bad;   // the same stage sequence
              return st;
            };
            if (mask_class_of(tcls, h, wg) == MASK_NONE) {
              if (!mask_half_loaded(kResident, tcls, h)) continue;
              if (release) {
                for (int kb = 0; kb < nkb; ++kb) {   // wait, meet, hand back: one stage at a time
                  wait_at(a_it + kb);
                  release_at(a_it + kb);
                  if (Stage* st = stage_at(a_it + kb)) { st->waits[wg]++; st->releases[wg]++; if (st->kb != kb) ++bad; }
                }
                a_it += nkb;
                if (kResident && mt == mt_last) brel_item[wg][static_cast<int>(itl)]++;
              }
              continue;
            }
            for (int kb = 0; kb < nkb; ++kb) {   // live: wait for kb, then hand back kb - 1 (the last after the loop)
              if (kResident && b_first && kb == 0) bwait_item[wg][static_cast<int>(itl)]++;
              wait_at(a_it + kb);
              if (release && kb > 0) release_at(a_it + kb - 1);
              if (Stage* st = stage_at(a_it + kb)) { st->waits[wg]++; if (release) st->releases[wg]++; if (st->kb != kb) ++bad; }
            }
            if (release) release_at(a_it + nkb - 1);
            b_first = false;
            if (release) {
              a_it += nkb;
              if (kResident && mt == mt_last && h == t.nh - 1) brel_item[wg][static_cast<int>(itl)]++;
            }
          }
        }
      }
      a_end[wg] = static_cast<int>(a_it);
      if (static_cast<int>(itl) != items_loaded) ++bad;   // both sides count the same loaded items
    }
    // ---- invariants ----
    for (int wg = 0; wg < 2; ++wg)
      if (a_end[wg] != static_cast<int>(loads.size())) ++bad;   // a_it counts exactly the loaded stages
    for (const Stage& st : loads)
      for (int wg = 0; wg < 2; ++wg)
        if (st.releases[wg] != 1 || st.waits[wg] < 1) ++bad;   // waited for, and released once by each warpgroup
    if (kResident)
      for (int it : b_loads)
        for (int wg = 0; wg < 2; ++wg) {
          if (brel_item[wg][it] != 1) ++bad;                    // the y block handed back once per loaded item
          if (bwait_item[wg][it] > 1) ++bad;                    // and waited for at most once (not at all: no MMAs)
        }
    if (kResident)   // it_local counts only loaded items: the i-th y block load has parity count i
      for (size_t i = 0; i < b_loads.size(); ++i)
        if (b_loads[i] != static_cast<int>(i)) ++bad;
    if (kResident && static_cast<int>(b_loads.size()) != items_loaded) ++bad;
  }
  return bad;
}

static int replay()
{
  std::mt19937 rng(12345);
  int bad = 0, cases = 0;
  for (bool resident : {true, false})
    for (int nkb : resident ? std::vector<int>{1, 2, 3, 4} : std::vector<int>{5, 7, 10})
      for (double p_dead : {0.0, 0.5, 0.9, 1.0})
        for (int rep = 0; rep < 6; ++rep) {
          const int tiles_m = 1 + static_cast<int>(rng() % 40), nblocks = 1 + static_cast<int>(rng() % 9);
          const int chunk = 1 + static_cast<int>(rng() % 8), grid = 1 + static_cast<int>(rng() % 5);
          const int nlh = static_cast<int>(rng() % 2);
          const int b   = resident ? replay_case<true>(nkb, tiles_m, nblocks, nlh, chunk, grid, rng, p_dead)
                                   : replay_case<false>(nkb, tiles_m, nblocks, nlh, chunk, grid, rng, p_dead);
          if (b) std::printf("case resident=%d nkb=%d tiles_m=%d blocks=%d: %d violations\n", resident, nkb, tiles_m, nblocks, b);
          bad += b;
          ++cases;
        }
  std::printf(bad ? "FAIL %d (%d cases)\n" : "PASS (%d cases)\n", bad ? bad : cases, cases);
  return bad ? 1 : 0;
}

int main(int argc, char** argv)
{
  if (argc > 1 && std::strcmp(argv[1], "classify") == 0) return classify();
  return replay();
}
