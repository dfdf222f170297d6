// Host run of select_k's key transform (raft_b200/csrc/select_k.cuh: select_key, the one definition of the order).
// Reads 32-bit patterns (hex, one per line) from stdin and prints "<min key> <max key>" in hex for each; compiled and
// compared with oracle/select_k.py by tests/test_select_k.py.
#include <cstdio>
#include <cstring>

#include "../../raft_b200/csrc/select_k.cuh"

int main()
{
  unsigned b;
  while (std::scanf("%x", &b) == 1) {
    float v;
    std::memcpy(&v, &b, sizeof v);
    std::printf("%08x %08x\n", b2d::select_key(v, true), b2d::select_key(v, false));
  }
  return 0;
}
