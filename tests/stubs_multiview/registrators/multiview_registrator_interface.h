// Stand-in for the reference's registrators/multiview_registrator_interface.h (:33-66) with the pieces of
// pcl::PointCloud and Eigen::Matrix4f it uses, for compiling MultiviewRegistratorLumPclB200 outside the reference
// tree.  TEST INFRASTRUCTURE.
#ifndef REGISTRATORS_MULTIVIEW_REGISTRATOR_INTERFACE_H_
#define REGISTRATORS_MULTIVIEW_REGISTRATOR_INTERFACE_H_

#include <cstddef>
#include <memory>
#include <vector>

namespace Eigen {
struct Matrix4f {   // column-major, like Eigen's default
  float m[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  float& operator()(int r, int c) { return m[c * 4 + r]; }
  const float* data() const { return m; }
};
}  // namespace Eigen

namespace pcl {
template <typename PointT>
struct PointCloud {
  using Ptr = std::shared_ptr<PointCloud>;
  using ConstPtr = std::shared_ptr<const PointCloud>;
  std::vector<PointT> points;
  size_t size() const { return points.size(); }
  void clear() { points.clear(); }
  PointCloud& operator+=(const PointCloud& o) {
    points.insert(points.end(), o.points.begin(), o.points.end());
    return *this;
  }
};
}  // namespace pcl

namespace static_map {
namespace registrator {

enum MultiviewType { kLumPCL, kMultiviewTypeCount };

template <typename PointT>
class MultiviewInterface {
 public:
  using PointCloudType = pcl::PointCloud<PointT>;
  using PointCloudPtr = typename PointCloudType::Ptr;
  using PointCloudConstPtr = typename PointCloudType::ConstPtr;

  MultiviewInterface() = default;
  ~MultiviewInterface() = default;

  struct InnerFrame {
    PointCloudPtr cloud;
    Eigen::Matrix4f pose;
  };

  inline void AddNewCloud(const PointCloudPtr& cloud, const Eigen::Matrix4f& pose) {
    if (cloud) inner_frames_.push_back({cloud, pose});
  }

  size_t Size() { return inner_frames_.size(); }

  virtual void AlignAll(const PointCloudPtr& output) = 0;

 protected:
  MultiviewType type_;
  std::vector<InnerFrame> inner_frames_;
};

}  // namespace registrator
}  // namespace static_map

#endif  // REGISTRATORS_MULTIVIEW_REGISTRATOR_INTERFACE_H_
