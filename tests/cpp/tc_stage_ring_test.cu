// Host-side replay of the output staging ring of expanded_tc_kernel (tc_stage_store in expanded_tc.cuh): how the consumer
// warpgroup's 4 warps, its lead thread and the TMA unit share the ring's two boxes; no GPU needed.  The actors, each a
// restatement of tc_stage_store's order of operations over a run of tiles (4 boxes each, written as 2 pairs, box 2 q + s
// of a tile in slot s):
//   lead thread (lane 0 of warp 0): wait_group.read 0; named barrier; write its part of both boxes; fence; named barrier;
//     issue both stores and commit them as one group;
//   the other 31 lanes of warp 0 and warps 1-3: named barrier; write; fence; named barrier;
//   the TMA unit: finishes reading any issued store, in any order.
// Run under random interleavings.  Checked:
//   - no state is ever stuck (on the GPU a stuck state is a hang);
//   - no box is rewritten before the store that reads it has finished reading it, and every store reads only what the
//     whole warpgroup wrote for its own box;
//   - at the end every store has been read.
// Cases: 1-8 tiles, a few hundred interleavings each.
#include <algorithm>
#include <cstdio>
#include <random>
#include <vector>
#include "../../raft_b200/csrc/tc_params.cuh"

using namespace b2d;

namespace {

enum Kind { BAR_ARRIVE, BAR_WAIT, WAIT_READ0, WRITE, ISSUE };
constexpr int kSlots  = TC_STG_BOXES;
constexpr int kActors = 5;   // 0 lead, 1 the rest of warp 0, 2-4 warps 1-3
static_assert(kSlots == 2, "tc_stage_store writes one box per slot and pair");

struct Op {
  Kind kind;
  int box = 0;   // WRITE / ISSUE: box g (slot g % 2); ISSUE issues boxes g and g + 1
};

struct Sim {
  std::vector<Op> ops[kActors];
  size_t pc[kActors] = {};
  int bars[kActors]  = {};          // named-barrier arrivals per actor
  int content[kSlots][kActors];     // box whose values actor a wrote into the slot (-1: none)
  std::vector<int> read;            // stores that have finished reading, by box
  std::vector<int> in_flight;       // issued stores still reading
  int bad = 0;

  Sim()
  {
    for (auto& c : content)
      for (int& a : c) a = -1;
  }

  bool step(int a)
  {
    if (pc[a] >= ops[a].size()) return false;
    const Op& o = ops[a][pc[a]];
    switch (o.kind) {
      case BAR_ARRIVE: ++bars[a]; break;
      case BAR_WAIT:
        for (int b = 0; b < kActors; ++b)
          if (bars[b] < bars[a]) return false;
        break;
      case WAIT_READ0:   // wait_group.read 0 (and wait_group 0 after the last tile)
        if (!in_flight.empty()) return false;
        break;
      case WRITE: {
        const int s = o.box % kSlots, prev = content[s][a];
        // the slot's previous box must have been read by its store before any of it is overwritten
        if (prev >= 0 && std::find(read.begin(), read.end(), prev) == read.end()) ++bad;
        content[s][a] = o.box;
        break;
      }
      case ISSUE:
        for (int g = o.box; g < o.box + kSlots; ++g) {
          for (int w = 0; w < kActors; ++w)
            if (content[g % kSlots][w] != g) ++bad;   // a part of the box is missing or from another box
          in_flight.push_back(g);
        }
        break;
    }
    ++pc[a];
    return true;
  }

  // the TMA unit finishes reading one issued store (any of them); checks what it reads
  bool tma_step(std::mt19937& rng)
  {
    if (in_flight.empty()) return false;
    const size_t i = rng() % in_flight.size();
    const int g = in_flight[i];
    for (int w = 0; w < kActors; ++w)
      if (content[g % kSlots][w] != g) ++bad;   // rewritten while its store was reading it
    read.push_back(g);
    in_flight.erase(in_flight.begin() + static_cast<long>(i));
    return true;
  }

  bool run(std::mt19937& rng)
  {
    for (;;) {
      bool done = in_flight.empty();
      for (int a = 0; a < kActors; ++a)
        if (pc[a] < ops[a].size()) done = false;
      if (done) return true;
      int order[kActors + 1];
      for (int i = 0; i <= kActors; ++i) order[i] = i;
      std::shuffle(order, order + kActors + 1, rng);
      bool moved = false;
      for (int i = 0; i <= kActors && !moved; ++i) {
        const int a = order[i];
        if (a == kActors) {
          moved = (rng() % 2) && tma_step(rng);
          continue;
        }
        // a few ops in a row, so that one actor can run ahead of the others
        for (int burst = 1 + static_cast<int>(rng() % 4); burst > 0 && step(a); --burst) moved = true;
      }
      if (!moved && !tma_step(rng)) return false;   // nothing can move: stuck
    }
  }
};

int replay_case(int tiles, std::mt19937& rng)
{
  Sim sim;
  for (int t = 0; t < tiles; ++t)
    for (int q = 0; q < 2; ++q) {   // tc_stage_store, pair q of tile t: boxes g, g + 1 in slots 0, 1
      const int g = 4 * t + 2 * q;
      sim.ops[0].push_back(Op{WAIT_READ0});
      for (int a = 0; a < kActors; ++a)
        for (Op o : {Op{BAR_ARRIVE}, Op{BAR_WAIT}, Op{WRITE, g}, Op{WRITE, g + 1}, Op{BAR_ARRIVE}, Op{BAR_WAIT}})
          sim.ops[a].push_back(o);
      sim.ops[0].push_back(Op{ISSUE, g});
    }
  sim.ops[0].push_back(Op{WAIT_READ0});   // the CTA's last tile: every store done
  int bad = 0;
  for (int seed = 0; seed < 200; ++seed) {
    Sim s = sim;
    if (!s.run(rng)) {
      std::printf("stuck: tiles %d, lead at %zu of %zu\n", tiles, s.pc[0], s.ops[0].size());
      return bad + 1;
    }
    bad += s.bad;
    if (static_cast<int>(s.read.size()) != 4 * tiles) ++bad;   // every store read exactly once
  }
  return bad;
}

}  // namespace

int main()
{
  std::mt19937 rng(20261017);
  int bad = 0, cases = 0;
  for (int tiles = 1; tiles <= 8; ++tiles, ++cases) {
    const int b = replay_case(tiles, rng);
    if (b) std::printf("case tiles=%d: %d violations\n", tiles, b);
    bad += b;
  }
  std::printf(bad ? "FAIL %d (%d cases)\n" : "PASS (%d cases)\n", bad ? bad : cases, cases);
  return bad ? 1 : 0;
}
