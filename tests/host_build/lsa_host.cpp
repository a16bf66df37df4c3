// TEST-ONLY host build of the set-criterion matcher's solver: trackformer_b200/csrc/lsa_core.h, the routine
// csrc/lsa.cu's kernels run, solved by one "thread" on the layout lsa_kernel hands it, so the CPU suite can compare
// it with scipy.optimize.linear_sum_assignment.  Built by tests/test_lsa_cpu.py; never shipped, never loaded by the
// package.
#include <vector>

#include "../../trackformer_b200/csrc/lsa_core.h"

namespace lsa = tfb200_lsa;

// One problem of lsa_kernel: cost[q * T + i] for query q < Q and target i < T <= Q.  query[i] = the query assigned to
// target i.  Returns 0, or 2 when the problem is infeasible (the kernel's status code).
extern "C" int tfb200_lsa_host(const float* cost, int Q, int T, int* query) {
  std::vector<double> shortest(Q), v(Q), u(T);
  std::vector<int> path(Q), row4col(Q), visited(T);
  std::vector<uint8_t> in_sc(Q);
  const lsa::Cols C{shortest.data(), v.data(), path.data(), row4col.data(), in_sc.data()};
  const lsa::Rows R{u.data(), query, visited.data()};
  lsa::Thread::Scratch scratch;
  return lsa::solve<lsa::Thread>(T, Q, lsa::Strided{cost, 1, size_t(T)}, R, C, scratch) ? 0 : 2;
}
