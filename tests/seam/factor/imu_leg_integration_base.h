// tests/seam (see utils/parameters.h): the public results of the IMU / leg preintegration the binding copies.
#pragma once
#include <vector>
#include <eigen3/Eigen/Dense>
#include "../utils/parameters.h"

class IMULegIntegrationBase {
  public:
    Eigen::Matrix<double, RESIDUAL_STATE_SIZE, RESIDUAL_STATE_SIZE> jacobian, covariance;
    double sum_dt;
    Eigen::Vector3d delta_p;
    Eigen::Quaterniond delta_q;
    Eigen::Vector3d delta_v;
    std::vector<Eigen::Vector3d> delta_epsilon;
    Eigen::Vector3d linearized_ba, linearized_bg;
    Vector_rho linearized_rho;
};
