// tests/seam (see utils/parameters.h): what the binding reads of the marginalization prior.
#pragma once
#include <vector>
#include <eigen3/Eigen/Dense>

class MarginalizationInfo {
  public:
    int m, n;
    std::vector<int> keep_block_size;
    std::vector<int> keep_block_idx;
    std::vector<double *> keep_block_data;
    Eigen::MatrixXd linearized_jacobians;
    Eigen::VectorXd linearized_residuals;
    bool valid;
};
