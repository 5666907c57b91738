// Prints, as one JSON object, the type of every member, constant and global of the reference's interface that
// tools/integration_stub.cpp reads, and the value of every constant.  Built against tests/seam or against the reference's own
// headers (with the shims of oracle/shim either way), the two outputs must be equal: tests/golden/seam_v1.json holds the
// reference's, tests/test_abi.py compares.
#include <cstdio>
#include <typeinfo>
#include <utility>
#include "utils/parameters.h"
#include "featureTracker/feature_manager.h"
#include "factor/imu_leg_integration_base.h"
#include "factor/marginalization_factor.h"

#define MEMBER(cls, m) std::printf("  \"%s::%s\": \"%s\",\n", #cls, #m, typeid(decltype(std::declval<cls &>().m)).name())
#define GLOBAL(g) std::printf("  \"%s\": \"%s\",\n", #g, typeid(decltype(g)).name())
#define CONSTANT(c) std::printf("  \"%s\": \"%s = %.17g\",\n", #c, typeid(decltype(c)).name(), (double)(c))

int main() {
    std::printf("{\n");
    MEMBER(FeatureManager, feature);
    MEMBER(FeaturePerId, start_frame); MEMBER(FeaturePerId, used_num); MEMBER(FeaturePerId, feature_per_frame);
    MEMBER(FeaturePerFrame, point); MEMBER(FeaturePerFrame, velocity); MEMBER(FeaturePerFrame, pointRight); MEMBER(FeaturePerFrame, velocityRight);
    MEMBER(FeaturePerFrame, cur_td); MEMBER(FeaturePerFrame, is_stereo);
    MEMBER(IMULegIntegrationBase, sum_dt); MEMBER(IMULegIntegrationBase, delta_p); MEMBER(IMULegIntegrationBase, delta_q); MEMBER(IMULegIntegrationBase, delta_v);
    MEMBER(IMULegIntegrationBase, delta_epsilon); MEMBER(IMULegIntegrationBase, linearized_ba); MEMBER(IMULegIntegrationBase, linearized_bg);
    MEMBER(IMULegIntegrationBase, linearized_rho); MEMBER(IMULegIntegrationBase, jacobian); MEMBER(IMULegIntegrationBase, covariance);
    MEMBER(MarginalizationInfo, valid); MEMBER(MarginalizationInfo, m); MEMBER(MarginalizationInfo, n); MEMBER(MarginalizationInfo, keep_block_size);
    MEMBER(MarginalizationInfo, keep_block_idx); MEMBER(MarginalizationInfo, keep_block_data); MEMBER(MarginalizationInfo, linearized_jacobians);
    MEMBER(MarginalizationInfo, linearized_residuals);
    GLOBAL(ESTIMATE_EXTRINSIC); GLOBAL(ESTIMATE_TD); GLOBAL(NUM_ITERATIONS); GLOBAL(OPTIMIZE_LEG_BIAS); GLOBAL(G);
    CONSTANT(FOCAL_LENGTH); CONSTANT(WINDOW_SIZE); CONSTANT(NUM_OF_F); CONSTANT(NUM_OF_LEG); CONSTANT(RESIDUAL_STATE_SIZE);
    CONSTANT(SIZE_POSE); CONSTANT(SIZE_SPEEDBIAS); CONSTANT(SIZE_LEG_BIAS); CONSTANT(SIZE_FEATURE);
    std::printf("  \"\": \"\"\n}\n");
    return 0;
}
