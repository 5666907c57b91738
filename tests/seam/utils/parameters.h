// tests/seam: the part of the reference's interface that tools/integration_stub.cpp reads, declared from scratch so that the
// binding type-checks without the reference's sources.  tests/golden/seam_v1.json pins every declaration here to the reference's
// own headers (see tests/golden/make_seam_golden.py).  Constants and globals of utils/parameters.h the binding uses:
#pragma once
#include <vector>
#include <eigen3/Eigen/Dense>

const double FOCAL_LENGTH = 460.0;
const int WINDOW_SIZE = 10;
const int NUM_OF_F = 1000;
#define NUM_OF_LEG 4
#define RESIDUAL_STATE_SIZE 31
typedef Eigen::Matrix<double, 4, 1> Vector_rho;
enum SIZE_PARAMETERIZATION { SIZE_POSE = 7, SIZE_SPEEDBIAS = 9, SIZE_LEG_BIAS = 4, SIZE_FEATURE = 1 };
extern int ESTIMATE_EXTRINSIC;
extern int ESTIMATE_TD;
extern int NUM_ITERATIONS;
extern int OPTIMIZE_LEG_BIAS;
extern Eigen::Vector3d G;
