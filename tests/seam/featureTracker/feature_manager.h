// tests/seam (see utils/parameters.h): the feature bookkeeping the binding walks (FeatureManager::feature).
#pragma once
#include <list>
#include <vector>
#include <eigen3/Eigen/Dense>
#include "../utils/parameters.h"

class FeaturePerFrame {
  public:
    double cur_td;
    Eigen::Vector3d point, pointRight;
    Eigen::Vector2d velocity, velocityRight;
    bool is_stereo;
};

class FeaturePerId {
  public:
    int start_frame;
    std::vector<FeaturePerFrame> feature_per_frame;
    int used_num;
};

class FeatureManager {
  public:
    std::list<FeaturePerId> feature;
};
