// host_propagation_backend.hpp — TEST INFRASTRUCTURE: the CUDA engine backend with the IMU accumulation of
// Propagator::propagate_and_clone left on the host (CovBackend's reference path: host loop, then ovb_cov_propagate and
// ovb_cov_clone). tools/run_simulation.cpp built with -DOVB_SIM_HOST_PROPAGATION runs on it, so the closed loop can be
// compared byte for byte with the product runner, whose EngineCov makes the one ovb_cov_propagate_imu call.
#pragma once
#include "../../include/ovb200_vio.hpp"

namespace ovb200 {
class HostPropagationEngineCov : public EngineCov {
public:
  using EngineCov::EngineCov;
  void propagate_imu(int n, int steps, const std::vector<double> &F, const std::vector<double> &G, const std::vector<double> &qc, int new_off,
                     const std::vector<int> &old_off, const std::vector<int> &old_sz, int clone_off, int clone_size, const double *dnc_dt, int dt_off) override {
    CovBackend::propagate_imu(n, steps, F, G, qc, new_off, old_off, old_sz, clone_off, clone_size, dnc_dt, dt_off);
  }
};
} // namespace ovb200
