// landmark_probe.cpp — TEST INFRASTRUCTURE: ovb200::SlamLandmark (the rpng_sim runner's ov_type::Landmark, include/ovb200_vio.hpp)
// on the command lines read from stdin, one result line each (17 significant digits):
//   rt REP px py pz qx qy qz      set_from_xyz(p, false), set_from_xyz(q, true)  ->  get_xyz(false) get_xyz(true) value[size] fej[size]
//   upd REP px py pz d0 d1 d2     set_from_xyz(p) (value and FEJ), update(d)      ->  get_xyz(false) get_xyz(true)
// REP is an ovb_feat_rep number; d has size() entries used (1 for ANCHORED_INVERSE_DEPTH_SINGLE).
#include "../../include/ovb200_vio.hpp"

#include <cstdio>
#include <iostream>
#include <sstream>

using namespace ovb200;

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op;
    SlamLandmark lm;
    Vec3 p, q;
    in >> op >> lm.rep >> p[0] >> p[1] >> p[2] >> q[0] >> q[1] >> q[2];
    if (!in || (op != "rt" && op != "upd"))
      return 2;
    lm.set_from_xyz(p, false);
    lm.set_from_xyz(op == "rt" ? q : p, true);
    if (op == "upd")
      lm.update(q.data());
    const Vec3 x = lm.get_xyz(false), xf = lm.get_xyz(true);
    std::printf("%.17g %.17g %.17g %.17g %.17g %.17g", x[0], x[1], x[2], xf[0], xf[1], xf[2]);
    if (op == "rt")
      for (int k = 0; k < 2 * lm.size(); k++)
        std::printf(" %.17g", k < lm.size() ? lm.value[k] : lm.fej[k - lm.size()]);
    std::printf("\n");
  }
  return 0;
}
