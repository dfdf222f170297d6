// raft::matrix::SelectAlgo -- the enumerators of cpp/include/raft/matrix/select_k_types.hpp, kept so that callers naming
// an algorithm compile unchanged.  raft_b200 has one selection path (b2d_select_k), which every value selects.
#pragma once
#include <cstdint>

namespace raft {
namespace matrix {

enum class SelectAlgo : std::uint8_t {
  kAuto                 = 0,
  kRadix8bits           = 1,
  kRadix11bits          = 2,
  kRadix11bitsExtraPass = 3,
  kWarpAuto             = 4,
  kWarpImmediate        = 5,
  kWarpFiltered         = 6,
  kWarpDistributed      = 7,
  kWarpDistributedShm   = 8,
};

}  // namespace matrix
}  // namespace raft
