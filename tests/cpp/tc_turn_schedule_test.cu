// Host-side replay of the resident schedule of expanded_tc_kernel (expanded_tc.cuh, kResident = true); no GPU needed.
// The two producer warps (the kernel's own tc_producer_walk, warp w feeding x ring w, warp 0 alone loading the y block),
// the two consumer warpgroups (their waits, hand-backs, ordered MMA turns and the per-item meeting at named barrier 1,
// restated from the consumer loop with the kernel's own skip helpers) run as a small state machine under random
// interleavings.  Checked:
//   - no state is ever stuck: some actor can always move until all are done (on the GPU a stuck state is a hang);
//   - every mbarrier wait that passes sees exactly the phase it is meant to see (not an older or a later load), and the
//     stage it reads holds the (y block, x tile, k-block) the consumer multiplies;
//   - the turns alternate: a warpgroup never has two turns pending (a second bar.arrive before the waiter's bar.sync
//     would complete the 256-thread barrier without it), and at the end every arrival has been matched;
//   - no mbarrier is left with a partial phase.
// Cases: unmasked (4 stages as EPI_STORE, 5 as the arg-min / top-k epilogues) and EPI_MINLOC_MASKED with random class
// bytes; nkb 1-4; one or two halves in the last y block; m % 128 in {1, 64, 65, 127} (slab 1 of the last tile wholly
// outside the matrix for 1 and 64, NONE in the masked class bytes); random chunk sizes and grids down to one item per CTA.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>
#include "../../raft_b200/csrc/masked_nn.cuh"

using namespace b2d;

namespace {

enum Kind { WAIT, ARRIVE, LOAD, TAKE, PASS, MEET_ARRIVE, MEET_WAIT };
// mbarrier ids: x ring r full / empty stage s, y block full / empty k-block kb
int afull_id(int r, int s) { return 16 * r + s; }
int aempty_id(int r, int s) { return 16 * r + 8 + s; }
int bfull_id(int kb) { return 32 + kb; }
int bempty_id(int kb) { return 40 + kb; }
constexpr int NBARS = 48;

struct Op {
  Kind kind;
  int bar        = 0;   // mbarrier id (WAIT / ARRIVE / LOAD)
  uint32_t par   = 0;   // WAIT: try_wait.parity operand
  int expect     = 0;   // WAIT: completed phases it must see when it passes
  long long tag  = -1;  // LOAD: what the slot now holds; WAIT on a full barrier: what the slot must hold
};

struct Mbar {
  int count = 1, pending = 0, completed = 0;
  long long content = -1;   // full barriers: the load the slot holds
};

struct Sim {
  std::vector<Op> ops[4];   // actors 0, 1: producer warps; 2, 3: consumer warpgroups
  size_t pc[4] = {0, 0, 0, 0};
  Mbar bars[NBARS];
  int turns[2] = {0, 0};    // pending passes to warpgroup w (arrivals on named barrier 4 + w, in warpgroups)
  int met[2]   = {0, 0};    // arrivals at named barrier 1
  int bad      = 0;

  // can actor a execute its next op?  (executes it if so)
  bool step(int a)
  {
    if (pc[a] >= ops[a].size()) return false;
    const Op& o = ops[a][pc[a]];
    const int w = a - 2;
    switch (o.kind) {
      case WAIT: {
        Mbar& b = bars[o.bar];
        if ((static_cast<uint32_t>(b.completed) & 1u) == o.par) return false;   // the phase of parity o.par is open
        if (b.completed != o.expect) ++bad;                                    // passed on an older / later phase
        if (o.tag >= 0 && b.content != o.tag) ++bad;                           // the slot holds another load
        break;
      }
      case LOAD:
        bars[o.bar].content = o.tag;
        [[fallthrough]];
      case ARRIVE: {
        Mbar& b = bars[o.bar];
        if (++b.pending == b.count) { b.pending = 0; ++b.completed; }
        break;
      }
      case TAKE:
        if (turns[w] == 0) return false;
        --turns[w];
        break;
      case PASS:
        if (++turns[1 - w] > 1) ++bad;
        break;
      case MEET_ARRIVE: ++met[w]; break;
      case MEET_WAIT:
        if (met[1 - w] < met[w]) return false;
        break;
    }
    ++pc[a];
    return true;
  }

  // random interleaving until done or stuck; returns false when stuck
  bool run(std::mt19937& rng)
  {
    for (;;) {
      int order[4] = {0, 1, 2, 3};
      std::shuffle(order, order + 4, rng);
      bool moved = false, done = true;
      for (int i = 0; i < 4 && !moved; ++i) {
        const int a = order[i];
        if (pc[a] < ops[a].size()) done = false;
        // a few ops in a row, so that one actor can run ahead of the others
        for (int burst = 1 + static_cast<int>(rng() % 4); burst > 0 && step(a); --burst) moved = true;
      }
      if (done) return true;
      if (!moved) {
        for (int a = 0; a < 4; ++a)
          if (pc[a] < ops[a].size()) return false;
        return true;
      }
    }
  }
};

Op wait_op(int bar, uint32_t par, int expect, long long tag = -1) { Op o{WAIT}; o.bar = bar; o.par = par; o.expect = expect; o.tag = tag; return o; }
Op arrive_op(int bar) { Op o{ARRIVE}; o.bar = bar; return o; }
Op load_op(int bar, long long tag) { Op o{LOAD}; o.bar = bar; o.tag = tag; return o; }
Op simple(Kind k) { return Op{k}; }

// what a stage holds: (y block, x tile, k-block)
long long stage_tag(int n_blk, int mt, int kb) { return (static_cast<long long>(n_blk) << 32) | (mt << 4) | kb; }

template <bool kMasked, int kStages>
int replay_case(const TcParams& p, int nkb, int grid, std::mt19937& rng)
{
  int bad = 0;
  for (int cta = 0; cta < grid; ++cta) {
    Sim sim;
    for (int kb = 0; kb < TC_MAX_RES_KB; ++kb) sim.bars[bempty_id(kb)].count = 2;   // both warpgroups hand the y block back
    // ---- producer warps: the kernel's own load order ----
    for (int w = 0; w < 2; ++w)
      tc_producer_walk<true, kMasked>(
          p, nkb, cta, grid,
          [&](int kb, uint32_t it_local, const TcItem&) {
            if (w != 0) return;
            sim.ops[w].push_back(wait_op(bempty_id(kb), (it_local & 1) ^ 1, static_cast<int>(it_local)));
            sim.ops[w].push_back(load_op(bfull_id(kb), it_local));
          },
          [&](uint32_t a_it, const TcItem& t, int mt, int, int kb) {
            const int s = static_cast<int>(a_it % kStages), ph = static_cast<int>((a_it / kStages) & 1);
            sim.ops[w].push_back(wait_op(aempty_id(w, s), ph ^ 1, static_cast<int>(a_it / kStages)));
            sim.ops[w].push_back(load_op(afull_id(w, s), stage_tag(t.n_blk, mt, kb)));
          });
    // ---- consumer warpgroups: the resident paths of the consumer loop ----
    for (int w = 0; w < 2; ++w) {
      std::vector<Op>& ops = sim.ops[2 + w];
      if (w == 1) ops.push_back(simple(PASS));   // warpgroup 0 takes the first turn
      uint32_t a_it = 0, itl = 0;
      auto afull_wait = [&](uint32_t it, const TcItem& t, int mt, int kb) {
        ops.push_back(wait_op(afull_id(w, static_cast<int>(it % kStages)), (it / kStages) & 1,
                              static_cast<int>(it / kStages) + 1, stage_tag(t.n_blk, mt, kb)));
      };
      for (int64_t item = cta; item < p.n_items; item += grid, ++itl) {
        const TcItem t  = tc_item(p, item);
        const uint8_t* c = kMasked ? p.mask_cls + static_cast<int64_t>(t.n_blk) * p.tiles_m : nullptr;
        int mt_last      = t.mt1 - 1;
        if (kMasked) {
          mt_last = mask_mt_last(c, t.mt0, t.mt1);
          if (mt_last < 0) {
            if (w == 0 && item + grid >= p.n_items) ops.push_back(simple(TAKE));   // warpgroup 1's last pass
            --itl;
            continue;
          }
        }
        bool b_first = true;
        for (int rep = 0; rep < 2; ++rep) { ops.push_back(simple(MEET_ARRIVE)); ops.push_back(simple(MEET_WAIT)); }
        for (int mt = t.mt0; mt < t.mt1; ++mt) {
          const unsigned tcls = kMasked ? mask_cls_at(c, mt) : 0u;
          if (kMasked && tcls == 0u) continue;
          for (int h = 0; h < t.nh; ++h) {
            const bool release = tc_half_releases(true, h, t.nh);
            if (kMasked && mask_class_of(tcls, h, w) == MASK_NONE) {
              ops.push_back(simple(TAKE));
              ops.push_back(simple(PASS));
              if (!mask_half_loaded(true, tcls, h)) continue;
              if (release) {
                for (int kb = 0; kb < nkb; ++kb) {
                  afull_wait(a_it + kb, t, mt, kb);
                  ops.push_back(arrive_op(aempty_id(w, static_cast<int>((a_it + kb) % kStages))));
                }
                if (mt == mt_last)
                  for (int kb = 0; kb < nkb; ++kb) ops.push_back(arrive_op(bempty_id(kb)));
                a_it += nkb;
              }
              continue;
            }
            ops.push_back(simple(TAKE));
            for (int kb = 0; kb < nkb; ++kb) {
              const uint32_t it = a_it + kb;
              if (kMasked ? b_first : (mt == t.mt0 && h == 0))
                ops.push_back(wait_op(bfull_id(kb), itl & 1, static_cast<int>(itl) + 1, itl));
              afull_wait(it, t, mt, kb);
            }
            ops.push_back(simple(PASS));   // every MMA issued; then the stages go back in order
            b_first = false;
            if (release) {
              for (int kb = 0; kb < nkb; ++kb) ops.push_back(arrive_op(aempty_id(w, static_cast<int>((a_it + kb) % kStages))));
              a_it += nkb;
              if (mt == mt_last && h == t.nh - 1)
                for (int kb = 0; kb < nkb; ++kb) ops.push_back(arrive_op(bempty_id(kb)));
            }
          }
        }
        if (w == 0 && item + grid >= p.n_items) ops.push_back(simple(TAKE));   // warpgroup 1's last pass
      }
    }
    // a few interleavings of the same CTA
    for (int seed = 0; seed < 3; ++seed) {
      Sim s = sim;
      if (!s.run(rng)) {
        std::printf("stuck: cta %d of %d, pcs %zu/%zu %zu/%zu %zu/%zu %zu/%zu\n", cta, grid, s.pc[0], s.ops[0].size(), s.pc[1],
                    s.ops[1].size(), s.pc[2], s.ops[2].size(), s.pc[3], s.ops[3].size());
        ++bad;
        break;
      }
      bad += s.bad;
      if (s.turns[0] != 0 || s.turns[1] != 0 || s.met[0] != s.met[1]) ++bad;   // every named-barrier arrival matched
      for (const Mbar& b : s.bars)
        if (b.pending != 0) ++bad;                                              // no partial phase left behind
    }
  }
  return bad;
}

int replay()
{
  std::mt19937 rng(20261015);
  int bad = 0, cases = 0;
  for (int variant = 0; variant < 3; ++variant)   // unmasked with 4 stages (EPI_STORE), 5 stages, masked (5 stages)
    for (int nkb = 1; nkb <= TC_MAX_RES_KB; ++nkb)
      for (int mrem : {1, 64, 65, 127})
        for (int rep = 0; rep < 8; ++rep) {
          const int tiles_m = 1 + static_cast<int>(rng() % 24), nblocks = 1 + static_cast<int>(rng() % 6);
          const int nlh     = static_cast<int>(rng() % 2);   // 0: the last y block has one half
          TcParams p{};
          p.m         = static_cast<int64_t>(tiles_m - 1) * TC_BM + mrem;
          p.n         = static_cast<int64_t>(nblocks) * TC_BN - (nlh ? 0 : TC_HN);
          p.tiles_m   = tiles_m;
          p.tiles_n   = nblocks;
          p.tiles_sel = nblocks;
          p.chunk     = rep == 0 ? 1 : 1 + static_cast<int>(rng() % 8);
          p.chunk     = p.chunk < tiles_m ? p.chunk : tiles_m;
          p.chunks_m  = (tiles_m + p.chunk - 1) / p.chunk;
          p.n_items   = static_cast<int64_t>(nblocks) * p.chunks_m;
          // rep 0: one item per CTA; otherwise a few CTAs
          // (the launch never has more CTAs than items)
          int grid = rep == 0 ? static_cast<int>(p.n_items) : 1 + static_cast<int>(rng() % 5);
          grid     = grid < p.n_items ? grid : static_cast<int>(p.n_items);
          // class bytes: dead tiles, random (slab, half) classes, runs of tiles with one slab NONE; slabs outside the
          // matrix and the missing half of the last y block are NONE
          std::vector<uint8_t> cls(static_cast<size_t>(nblocks) * tiles_m, 0);
          const double p_dead = (rep % 4) * 0.3;
          for (int nb = 0; nb < nblocks; ++nb) {
            const int nh       = (nb < nblocks - 1 || nlh) ? 2 : 1;
            const int one_none = static_cast<int>(rng() % 3);   // 2: random; 0 / 1: slab 0 / 1 NONE for the whole block
            for (int mt = 0; mt < tiles_m; ++mt) {
              unsigned b = 0;
              if (std::uniform_real_distribution<double>(0, 1)(rng) >= p_dead)
                for (int h = 0; h < nh; ++h)
                  for (int s = 0; s < 2; ++s) {
                    unsigned k = static_cast<unsigned>(rng() % 3);
                    if (s == one_none || static_cast<int64_t>(mt) * TC_BM + 64 * s >= p.m) k = MASK_NONE;
                    b |= k << (2 * (2 * h + s));
                  }
              cls[static_cast<size_t>(nb) * tiles_m + mt] = static_cast<uint8_t>(b);
            }
          }
          p.mask_cls = cls.data();
          int b = 0;
          if (variant == 0) b = replay_case<false, TcCarve<true, EPI_STORE>::stages>(p, nkb, grid, rng);
          if (variant == 1) b = replay_case<false, TcCarve<true, EPI_MINLOC>::stages>(p, nkb, grid, rng);
          if (variant == 2) b = replay_case<true, TcCarve<true, EPI_MINLOC_MASKED>::stages>(p, nkb, grid, rng);
          if (b)
            std::printf("case variant=%d nkb=%d m=%lld n=%lld chunk=%d grid=%d: %d violations\n", variant, nkb,
                        static_cast<long long>(p.m), static_cast<long long>(p.n), p.chunk, grid, b);
          bad += b;
          ++cases;
        }
  std::printf(bad ? "FAIL %d (%d cases)\n" : "PASS (%d cases)\n", bad ? bad : cases, cases);
  return bad ? 1 : 0;
}

}  // namespace

int main() { return replay(); }
