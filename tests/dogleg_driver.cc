// Reads one dogleg model per line: type radius gg ggn gngn jaja jajb jbjb; prints rank, the step's kind, cg, cn, its
// norm and the subspace branch (-1 for the traditional step), for tests/test_oracle_dogleg.py.
#include <cstdio>

#include "../ceres_solver_b200/csrc/dogleg.h"

int main() {
  int type;
  double radius;
  b200dl::Model m;
  while (std::scanf("%d %lf %lf %lf %lf %lf %lf %lf", &type, &radius, &m.gg, &m.ggn, &m.gngn, &m.jaja, &m.jajb, &m.jbjb) == 8) {
    b200dl::cauchy_point(&m);
    int branch = -1;
    b200dl::Step s;
    m.rank = 2;
    if (type == b200dl::kSubspace) {
      b200dl::subspace_model(&m);
      if (m.rank == 0) {
        std::printf("0 -1 0 0 0 -1\n");
        continue;
      }
      s = b200dl::subspace_step(m, radius, &branch);
    } else {
      s = b200dl::traditional_step(m, radius);
    }
    std::printf("%d %d %.17g %.17g %.17g %d\n", m.rank, s.kind, s.cg, s.cn, s.norm, branch);
  }
  return 0;
}
