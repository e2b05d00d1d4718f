// TEST INFRASTRUCTURE ONLY. Drives the reference's own DeformationGraph (Core/Utils/DeformationGraph.cpp, compiled
// unmodified together with Core/Utils/CholeskyDecomp.cpp and the CHOLMOD stand-in of this directory) through the host
// logic of Deformation::constrain for a local loop closure (Core/Deformation.cpp:73-207 with no ferns, fernMatch = false,
// relaxGraph = false). Deformation.cpp itself is not compiled because it needs OpenGL; the part of it used here is
// restated below, line for line.
#include <stdint.h>
#include <string.h>

#include <map>
#include <unordered_map>
#include <vector>

#include <Eigen/Dense>
#include <sophus/se3.hpp>

// the harness reads the graph's private state (constraint weights, factorisation count) to report it
#define private public
#include "CholeskyDecomp.h"
#include "DeformationGraph.h"
#undef private

extern "C" int refdef_solve(const double* pos3, const int32_t* node_times, int n, const double* src3, const double* dst3,
                            const int32_t* src_times, const int32_t* dst_times, int n_cons, int pin, int last_deform_time,
                            double* rt12, float* nodes16, int32_t* cons_nodes4, double* cons_weights4, float* error_out,
                            float* mean_cons_err_out, int32_t* iterations_out) {
  // Deformation::sampleGraphModel -> initialiseGraph (Deformation.cpp:291-301)
  std::vector<Eigen::Vector3d> graphPosePoints;
  std::vector<uint64_t> graphPoseTimes;
  for (int i = 0; i < n; ++i) {
    graphPosePoints.push_back(Eigen::Vector3d(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]));
    graphPoseTimes.push_back((uint64_t)node_times[i]);
  }
  std::vector<Eigen::Vector3d> pointPool;
  DeformationGraph def(4, &pointPool);  // Deformation.cpp:23
  def.initialiseGraph(&graphPosePoints, &graphPoseTimes);

  // Deformation::addConstraint (Deformation.cpp:73-86)
  struct C {
    Eigen::Vector3d src, target;
    uint64_t srcTime;
  };
  std::vector<C> constraints;
  for (int i = 0; i < n_cons; ++i) {
    const Eigen::Vector3d s(src3[3 * i], src3[3 * i + 1], src3[3 * i + 2]);
    const Eigen::Vector3d t(dst3[3 * i], dst3[3 * i + 1], dst3[3 * i + 2]);
    constraints.push_back({s, t, (uint64_t)src_times[i]});
    if (pin) constraints.push_back({t, t, (uint64_t)dst_times[i]});
  }

  // Deformation::constrain (Deformation.cpp:96-207), local case
  std::vector<uint64_t> times;
  std::vector<Sophus::SE3d> T_wcs;
  def.setPosesSeq(&times, T_wcs);
  std::vector<uint64_t> vertexTimes;
  const int originalPointPool = pointPool.size();
  std::vector<int> srcPointPoolId(constraints.size());
  for (size_t i = 0; i < constraints.size(); i++) {
    pointPool.push_back(constraints[i].src);
    vertexTimes.push_back(constraints[i].srcTime);
    srcPointPoolId[i] = pointPool.size() - 1;
  }
  def.appendVertices(&vertexTimes, originalPointPool);
  def.clearConstraints();
  for (size_t i = 0; i < constraints.size(); i++) {
    Eigen::Vector3d targetPoint = constraints[i].target;
    def.addConstraint(srcPointPoolId[i], targetPoint);
  }
  float error = 0;
  float meanConsError = 0;
  def.optimiseGraphSparse(error, meanConsError, false, (uint64_t)last_deform_time);

  std::vector<GraphNode*>& graphNodes = def.getGraph();
  std::vector<uint64_t> graphTimes = def.getGraphTimes();
  for (size_t i = 0; i < graphNodes.size(); i++) {
    const Eigen::Vector3f position = graphNodes.at(i)->position.cast<float>();
    const Eigen::Matrix3f rotation = graphNodes.at(i)->rotation.cast<float>();
    const Eigen::Vector3f translation = graphNodes.at(i)->translation.cast<float>();
    memcpy(&nodes16[i * 16], position.data(), sizeof(float) * 3);
    memcpy(&nodes16[i * 16 + 3], rotation.data(), sizeof(float) * 9);
    memcpy(&nodes16[i * 16 + 12], translation.data(), sizeof(float) * 3);
    nodes16[i * 16 + 15] = (float)graphTimes.at(i);
    memcpy(&rt12[i * 12], graphNodes.at(i)->rotation.data(), sizeof(double) * 9);
    memcpy(&rt12[i * 12 + 9], graphNodes.at(i)->translation.data(), sizeof(double) * 3);
  }
  for (size_t l = 0; l < constraints.size(); ++l)
    for (int k = 0; k < 4; ++k) {
      cons_nodes4[4 * l + k] = def.vertexMap.at(l).at(k).node;
      cons_weights4[4 * l + k] = def.vertexMap.at(l).at(k).weight;
    }
  *error_out = error;
  *mean_cons_err_out = meanConsError;
  *iterations_out = def.cholesky->Common.n_factorize;
  return 0;
}
