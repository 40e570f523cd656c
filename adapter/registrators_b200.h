// registrators_b200.h — drop-in C++ matcher for the StaticMapping tree, backed by
// libsm_b200.so (C ABI: include/sm_b200.h).
//
// Compile this header INSIDE the reference tree (it needs the reference's own headers:
// registrators/interface.h, builder/data/cloud_types.h, Eigen, glog).  It is not compiled in
// the sm_b200 repository, where those dependencies do not exist; tests/test_adapter_syntax.py
// checks its syntax against minimal stand-in headers.
//
//   registrator::IcpFastB200 replaces registrator::IcpFast (registrators/icp_fast.h:37-62):
//   same base class, same overrides, same option names, same CHECK behaviour.
#ifndef ADAPTER_REGISTRATORS_B200_H_
#define ADAPTER_REGISTRATORS_B200_H_

#include <stdio.h>

#include <algorithm>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "registrators/interface.h"
#include "sm_b200.h"

namespace static_map {
namespace registrator {

// float option -> text without losing bits (std::to_string prints 6 fixed decimals)
inline std::string OptionText(float v) {
  char buf[32];
  snprintf(buf, sizeof(buf), "%.9g", static_cast<double>(v));
  return buf;
}

class IcpFastB200 : public Interface {
 public:
  USE_REGISTRATOR_CLOUDS;

  explicit IcpFastB200(int device = 0) : Interface() {
    this->type_ = kFastIcp;
    const int rc = sm_create(SM_TYPE_FAST_ICP, device, &handle_);
    CHECK_EQ(rc, 0) << "sm_create failed (" << rc << "): no CUDA device / no CPU fallback";
    // same registry as IcpFast::IcpFast (icp_fast.cc:411-418): InitWithXml writes through
    // these pointers, InitWithOptions forwards the values to the engine.
    REG_REGISTRATOR_INNER_OPTION("knn_normal_estimate", OptionItemDataType::kInt32,
                                 options_.knn_for_normal_estimate);
    REG_REGISTRATOR_INNER_OPTION("max_iteration", OptionItemDataType::kInt32,
                                 options_.max_iteration);
    REG_REGISTRATOR_INNER_OPTION("dist_outlier_ratio", OptionItemDataType::kFloat32,
                                 options_.dist_outlier_ratio);
  }
  ~IcpFastB200() override { sm_destroy(handle_); }

  PROHIBIT_COPY_AND_ASSIGN(IcpFastB200);

  void InitWithOptions() override {
    Check(sm_set_option(handle_, "max_iteration", std::to_string(options_.max_iteration).c_str()));
    Check(sm_set_option(handle_, "dist_outlier_ratio", OptionText(options_.dist_outlier_ratio).c_str()));
  }

  // icp_fast.cc:421-425
  void SetInputSource(InnerCloudPtr cloud) override {
    CHECK(cloud);
    CHECK(cloud->GetEigenCloud());
    const auto& pts = cloud->GetEigenCloud()->points;          // 3xN, column-major doubles
    Check(sm_set_input_source(handle_, pts.data(), pts.cols()));
  }

  // icp_fast.cc:427-431
  void SetInputTarget(InnerCloudPtr cloud) override {
    CHECK(cloud);
    CHECK(cloud->GetEigenCloud());
    CHECK(cloud->GetEigenCloud()->HasNormals());
    const auto& ec = *cloud->GetEigenCloud();
    Check(sm_set_input_target(handle_, ec.points.data(), ec.normals.data(), ec.points.cols()));
  }

  // icp_fast.cc:455-529
  bool Align(const Eigen::Matrix4d& guess, Eigen::Matrix4d& result) override {  // NOLINT
    PrepareBatch();
    const int rc = sm_align(handle_, guess.data(), result.data());  // both column-major
    Check(rc);
    this->final_score_ = sm_get_fitness_score(handle_);
    return rc == 1;
  }

  // The ICP error minimizer (sm_icp_error_minimizer): SM_ICP_POINT_TO_PLANE, what IcpFast::Align calls
  // (icp_fast.cc:506-510) and the default, or SM_ICP_POINT_TO_POINT, its ComputePointToPoint (:326-375).  Kept for
  // every later Align and AlignBatch.  A value outside 0..1 CHECK-fails.
  void SetErrorMinimizer(int minimizer) { Check(sm_set_icp_error_minimizer(handle_, minimizer)); }

  // hooks of AlignBatch (below)
  sm_handle* handle() const { return handle_; }
  // Enable/DisableInnerCompensation are not virtual (interface.h:89-91): the flag is read at every Align
  // (icp_fast.cc:487, :509)
  void PrepareBatch() { Check(sm_set_inner_compensation(handle_, InnerCompensation(this, 0) ? 1 : 0)); }
  void SetFinalScore(double score) { this->final_score_ = score; }

 private:
  void Check(int rc) const {
    CHECK_GE(rc, 0) << "sm_b200: " << sm_last_error(handle_);   // reference aborts via glog
  }
  // Interface::inner_compensation_ (interface.h:115).  An Interface without that member (a reduced stand-in of
  // the header) still compiles the adapter, with the flag off.
  template <typename Self>
  static auto InnerCompensation(const Self* self, int) -> decltype(static_cast<bool>(self->inner_compensation_)) {
    return self->inner_compensation_;
  }
  template <typename Self>
  static bool InnerCompensation(const Self*, long) { return false; }

  sm_handle* handle_ = nullptr;
  struct {
    int32_t knn_for_normal_estimate = 7;
    int32_t max_iteration = 100;
    float dist_outlier_ratio = 0.7;
  } options_;
};

// registrator::Ndt (registrators/ndt.h, ndt.cc:28-64) and registrator::NdtWithGicp
// (ndt_gicp.h, ndt_gicp.cc:28-112) keep the caller's float cloud (base-class SetInput*,
// interface.cc:38-60) and hand it over at Align: std::vector<InnerPointType>, 20-byte stride.
template <int kType>
class FloatCloudMatcherB200 : public Interface {
 public:
  USE_REGISTRATOR_CLOUDS;
  explicit FloatCloudMatcherB200(int device = 0) : Interface() {
    this->type_ = static_cast<Type>(kType);
    const int rc = sm_create(kType, device, &handle_);
    CHECK_EQ(rc, 0) << "sm_create failed (" << rc << ")";
  }
  ~FloatCloudMatcherB200() override { sm_destroy(handle_); }

  bool Align(const Eigen::Matrix4d& guess, Eigen::Matrix4d& result) override {  // NOLINT
    if (!this->source_cloud_ || !this->target_cloud_) {
      if (kType == SM_TYPE_NDT) return false;                 // ndt.cc:40-42
      CHECK(this->source_cloud_ && this->target_cloud_);      // NdtWithGicp dereferences them
    }
    PrepareBatch();
    const int rc = sm_align(handle_, guess.data(), result.data());
    CheckRc(rc);
    this->final_score_ = sm_get_fitness_score(handle_);
    return rc == 1;
  }

  // hooks of AlignBatch (below): the clouds kept by the base class go to the engine
  sm_handle* handle() const { return handle_; }
  void PrepareBatch() {
    CHECK(this->source_cloud_ && this->target_cloud_);
    const auto& s = this->source_cloud_->GetInnerCloud()->points;
    const auto& t = this->target_cloud_->GetInnerCloud()->points;
    CheckRc(sm_set_input_source_f32(handle_, &s[0].x, static_cast<int64_t>(s.size()),
                                    sizeof(data::InnerPointType)));
    CheckRc(sm_set_input_target_f32(handle_, &t[0].x, static_cast<int64_t>(t.size()),
                                    sizeof(data::InnerPointType)));
  }
  void SetFinalScore(double score) { this->final_score_ = score; }

 protected:
  void CheckRc(int rc) const { CHECK_GE(rc, 0) << "sm_b200: " << sm_last_error(handle_); }
  sm_handle* handle_ = nullptr;
};

class NdtB200 : public FloatCloudMatcherB200<SM_TYPE_NDT> {   // registers no option, like Ndt
 public:
  explicit NdtB200(int device = 0) : FloatCloudMatcherB200<SM_TYPE_NDT>(device) {}
  // pclomp setNeighborhoodSearchMethod (ndt_omp.h:184) with pclomp's NeighborSearchMethod values (sm_ndt_search_method);
  // the engine keeps it for every later Align and AlignBatch.  The reference's Ndt sets KDTREE (ndt.cc:33), the
  // default.  A value outside 0..3 CHECK-fails.
  void SetNeighborhoodSearchMethod(int method) { CheckRc(sm_set_ndt_search_method(handle_, method)); }
};

class NdtWithGicpB200 : public FloatCloudMatcherB200<SM_TYPE_NDT_WITH_GICP> {
 public:
  explicit NdtWithGicpB200(int device = 0) : FloatCloudMatcherB200<SM_TYPE_NDT_WITH_GICP>(device) {
    REG_REGISTRATOR_INNER_OPTION("use_ndt", OptionItemDataType::kBool, options_.use_ndt);            // ndt_gicp.cc:31-36
    REG_REGISTRATOR_INNER_OPTION("using_voxel_filter", OptionItemDataType::kBool, options_.using_voxel_filter);
    REG_REGISTRATOR_INNER_OPTION("voxel_resolution", OptionItemDataType::kFloat32, options_.voxel_resolution);
  }
  void InitWithOptions() override {
    CheckRc(sm_set_option(handle_, "use_ndt", options_.use_ndt ? "1" : "0"));
    CheckRc(sm_set_option(handle_, "using_voxel_filter", options_.using_voxel_filter ? "1" : "0"));
    CheckRc(sm_set_option(handle_, "voxel_resolution", OptionText(options_.voxel_resolution).c_str()));
  }

 private:
  struct { float voxel_resolution = 0.2; bool using_voxel_filter = true; bool use_ndt = true; } options_;
};

// Stand-in for registrator::IcpUsingPointMatcher (icp_pointmatcher.h, .cc:125-247): the default
// libpointmatcher chain (random reading filter 0.9, surface-normal reference filter knn 7, k-d
// tree eps 3.16, trimmed 0.7, point-to-plane, 150 iterations / differential checker) run by the
// IcpFast kernels; Align() is false below score 0.6 (.cc:145).  Registers no option.  It is what
// loop_detector.cc:304-308 would construct instead of `new IcpUsingPointMatcher`.
class IcpUsingPointMatcherB200 : public FloatCloudMatcherB200<SM_TYPE_ICP_PM> {
 public:
  explicit IcpUsingPointMatcherB200(int device = 0) : FloatCloudMatcherB200<SM_TYPE_ICP_PM>(device) {}
  // The error minimizer of the ICP chain (sm_icp_error_minimizer): the reference's loadDefaultConfig builds
  // PointToPointErrorMinimizer (icp_pointmatcher.cc:202-204) and then installs point-to-plane (:239), the default
  // here.  A value outside 0..1 CHECK-fails.
  void SetErrorMinimizer(int minimizer) { CheckRc(sm_set_icp_error_minimizer(handle_, minimizer)); }
  // The leaf of the surface-normal reference filter (sm_pm_surface_normals): SM_PM_NORMALS_LEAST_SQUARES, the
  // default, is CalculateNormals' plane fit (cloud_types.cc:73-103); SM_PM_NORMALS_EIGENVECTOR is libpointmatcher's
  // own float box mean and smallest-eigenvector normal.  Applies from the next Align; a value outside 0..1
  // CHECK-fails.
  void SetSurfaceNormals(int mode) { CheckRc(sm_set_pm_surface_normals(handle_, mode)); }
  // The reading filter's random stream (sm_pm_reading_sampler): SM_PM_SAMPLING_HASH, the default, is a counter hash;
  // SM_PM_SAMPLING_GLIBC_RAND is glibc's rand() after srand(sample_seed), drawn from this matcher's stream position,
  // which every Align in that mode advances by the reading cloud's size.  To reproduce a process that shares one
  // rand() stream between matchers, hand each matcher the position the process had reached before its Align.
  // A mode outside 0..1 or a negative position CHECK-fails.
  void SetReadingSampler(int mode) { CheckRc(sm_set_pm_reading_sampler(handle_, mode)); }
  int64_t GetRandPosition() const {
    int64_t position = 0;
    CheckRc(sm_get_pm_rand_position(handle_, &position));
    return position;
  }
  void SetRandPosition(int64_t position) { CheckRc(sm_set_pm_rand_position(handle_, position)); }
};

// MotionCompensation (builder/map_builder.cc:232-257) on the GPU: same signature as the static
// function it replaces, so the two call sites (:325-327, :344-347) stay as they are.
inline void MotionCompensationB200(const data::InnerCloudType& raw_cloud, const Eigen::Matrix4d& delta_transform,
                                   data::InnerCloudType* const output_cloud, int device = 0) {
  CHECK(output_cloud);
  output_cloud->stamp = raw_cloud.stamp;
  output_cloud->points.resize(raw_cloud.points.size());
  if (raw_cloud.points.empty()) return;
  const int rc = sm_motion_compensation(device, &raw_cloud.points[0].x, static_cast<int64_t>(raw_cloud.points.size()),
                                        sizeof(data::InnerPointType), delta_transform.data(),
                                        &output_cloud->points[0].x);
  CHECK_EQ(rc, 0) << "MotionCompensation: factor outside [0, 1] (common/math.h:201) or CUDA failure";
}

// Batched CloseLoop / SubmapPairMatch: the reference starts one task (TBB / thread pool) per candidate
// pair, each constructing a matcher and calling Align (back_end/loop_detector.cc:216-228,304-308;
// builder/map_builder.cc:655,706-708).  With the engine ONE thread aligns all the candidates: the
// matchers have their clouds set as usual, AlignBatch enqueues every Align before it waits for the
// first result.  ok[i] / results[i] are what matchers[i]->Align(guesses[i], results[i]) would give.
template <typename MatcherB200>
inline void AlignBatch(const std::vector<MatcherB200*>& matchers, const std::vector<Eigen::Matrix4d>& guesses,
                       std::vector<Eigen::Matrix4d>* results, std::vector<bool>* ok) {
  CHECK(results && ok);
  CHECK_EQ(matchers.size(), guesses.size());
  const size_t n = matchers.size();
  std::vector<sm_handle*> handles(n);
  std::vector<double> g(16 * n), r(16 * n);
  std::vector<int32_t> rc(n);
  for (size_t i = 0; i < n; ++i) {
    matchers[i]->PrepareBatch();
    handles[i] = matchers[i]->handle();
    std::copy(guesses[i].data(), guesses[i].data() + 16, g.begin() + 16 * i);   // column-major, like Eigen
  }
  sm_align_batch(handles.data(), static_cast<int32_t>(n), g.data(), r.data(), rc.data());
  results->resize(n); ok->resize(n);
  for (size_t i = 0; i < n; ++i) {
    CHECK_GE(rc[i], 0) << "sm_b200: " << sm_last_error(handles[i]);               // reference aborts via glog
    std::copy(r.begin() + 16 * i, r.begin() + 16 * (i + 1), (*results)[i].data());
    (*ok)[i] = rc[i] != 0;
    matchers[i]->SetFinalScore(sm_get_fitness_score(handles[i]));
  }
}

// pre_processers::filter::VoxelGrid::Filter (pre_processors/filter_voxel_grid.cc:37-78) on the GPU:
// the body of that member becomes
//   this->FilterPrepare(cloud); registrator::VoxelGridFilterB200(*this->inner_cloud_, voxel_size_, cloud.get());
// Output points come in ascending voxel order instead of unordered_map iteration order.
inline void VoxelGridFilterB200(const data::InnerCloudType& input, float voxel_size,
                                data::InnerCloudType* const output, int device = 0) {
  CHECK(output);
  output->points.resize(input.points.size());
  int64_t m = 0;
  if (!input.points.empty()) {
    const int rc = sm_voxel_grid_filter(device, &input.points[0].x, static_cast<int64_t>(input.points.size()),
                                        sizeof(data::InnerPointType), voxel_size, &output->points[0].x, &m);
    // non-finite points are dropped by the engine (the reference keeps running on such input too).
    // SM_ERR_BAD_ARGUMENT is left for a cloud spanning >= 2^21 voxels along an axis or an invalid voxel
    // size (the reference refuses that one in ConfigsValid()): report and pass the cloud through
    // unfiltered rather than abort the mapper; only CUDA failures are fatal.
    CHECK_NE(rc, SM_ERR_CUDA) << "sm_voxel_grid_filter: CUDA failure";
    CHECK_NE(rc, SM_ERR_NO_DEVICE) << "sm_voxel_grid_filter: no CUDA device (no CPU fallback)";
    if (rc != 0) {
      LOG(ERROR) << "sm_voxel_grid_filter refused the cloud (" << rc << "): passing it through unfiltered";
      output->points = input.points;
      return;
    }
  }
  output->points.resize(m);
}

// The Filter body of FilterChainB200, StatisticRemovalB200 and GroundRemovalB200: CHECK-fails with last_error(h) when run (sm_*_run) fails
template <typename Handle, typename Run, typename LastError>
inline void FilterRecordsB200(Handle* h, Run run, LastError last_error, const char* run_name,
                              const data::InnerCloudType& input, data::InnerCloudType* const output,
                              std::vector<int>* const inliers) {
  CHECK(output);
  const int64_t n = static_cast<int64_t>(input.points.size());
  output->points.resize(input.points.size());
  std::vector<int32_t> index(input.points.size());
  int64_t m = 0;
  if (n > 0) {
    const int rc = run(h, &input.points[0].x, n, sizeof(data::InnerPointType), &output->points[0].x, &m, index.data());
    CHECK_EQ(rc, 0) << run_name << " failed (" << rc << "): " << last_error(h);
  }
  output->points.resize(m);
  if (inliers) inliers->assign(index.begin(), index.begin() + m);
}

// pre_processers::filter::Factory on the GPU (pre_processors/filter_factory.cc:63-106): one chain per Factory.  The
// body of Factory::InitFromXmlNode becomes one Add per <filter> and one SetParam per <param>, and the body of
// Factory::Filter (the call in DataCollector::CloudPreProcessing, builder/data/data_collector.cc:137-141)
//   this->FilterPrepare(cloud); chain_.Filter(*this->inner_cloud_, cloud.get(), &this->inliers_);
// RandomSampler is a deterministic stand-in for the reference's mt19937 draw (include/sm_b200.h).
class FilterChainB200 {
 public:
  explicit FilterChainB200(int device = 0) { CHECK_EQ(sm_filter_chain_create(device, &chain_), 0); }
  ~FilterChainB200() { sm_filter_chain_destroy(chain_); }
  FilterChainB200(const FilterChainB200&) = delete;
  FilterChainB200& operator=(const FilterChainB200&) = delete;

  // index of the new filter, or -1 for a name the reference skips too ("not supported yet.")
  int Add(const std::string& filter_name) {
    const int index = sm_filter_chain_add(chain_, filter_name.c_str());
    if (index == SM_ERR_UNKNOWN_OPTION) return -1;
    CHECK_GE(index, 0) << sm_filter_chain_last_error(chain_);
    return index;
  }
  // type: the <param>'s type attribute, -1 when it has none (the reference CHECK-fails, filter_interface.cc:57)
  void SetParam(int filter, const std::string& name, int type, const std::string& text) {
    CHECK_EQ(sm_filter_chain_set_param(chain_, filter, name.c_str(), type, text.c_str()), 0)
        << sm_filter_chain_last_error(chain_);
  }
  bool ConfigsValid(int filter) { return sm_filter_chain_validate(chain_, filter) == 1; }
  // true: Add also accepts GroundRemoval, StatisticRemoval and VoxelGrid (the chain option all_filters); false
  // restores their refusal.  Filters already added stay.
  void SetAllFilters(bool on) { CHECK_EQ(sm_filter_chain_set_option(chain_, "all_filters", on ? "1" : "0"), 0); }

  // inliers: the indices in `input` of the output records, in emission order (include/sm_b200.h)
  void Filter(const data::InnerCloudType& input, data::InnerCloudType* const output,
              std::vector<int>* const inliers = nullptr) {
    FilterRecordsB200(chain_, sm_filter_chain_run, sm_filter_chain_last_error, "sm_filter_chain_run", input, output,
                      inliers);
  }

  // RangeImage::DepthCluster (pre_processors/filter_range_image.cc:143-173) of the chain's RangeImage `filter` over
  // `input`, that filter's own input cloud: appends {x, y, z, label} records (pcl::PointXYZL, or any cloud whose
  // value_type has those members and that has push_back) in ascending label, each cluster in the reference's order.
  // An empty input CHECK-fails as in the reference (CHECK(inner_cloud_ != nullptr)).
  template <typename LabeledCloud>
  void DepthCluster(int filter, const data::InnerCloudType& input, LabeledCloud* const cloud) {
    const int64_t n = static_cast<int64_t>(input.points.size());
    std::vector<float> xyz(3 * input.points.size());
    std::vector<uint32_t> label(input.points.size());
    std::vector<int32_t> index(input.points.size());
    int64_t m = 0;
    const int rc = sm_filter_chain_depth_cluster(chain_, filter, n ? &input.points[0].x : nullptr, n,
                                                 sizeof(data::InnerPointType), xyz.data(), label.data(), index.data(),
                                                 &m, nullptr);
    CHECK_EQ(rc, 0) << "sm_filter_chain_depth_cluster failed (" << rc << "): " << sm_filter_chain_last_error(chain_);
    if (!cloud) return;
    for (int64_t j = 0; j < m; ++j) {
      typename LabeledCloud::value_type point;
      point.x = xyz[3 * j]; point.y = xyz[3 * j + 1]; point.z = xyz[3 * j + 2];
      point.label = label[j];
      cloud->push_back(point);
    }
  }

 private:
  sm_filter_chain* chain_ = nullptr;
};

// pre_processers::filter::StatisticRemoval as PCL's StatisticalOutlierRemoval (setMeanK(point_num_meank),
// setStddevMulThresh(std_mul)), the call filter_statistic_removal.cc:44-59 leaves as a TODO, on the GPU: one per
// StatisticRemoval.  The body of its InitFromXmlNode becomes one SetParam per <param>, and that of Filter
//   this->FilterPrepare(cloud); filter_.Filter(*this->inner_cloud_, cloud.get(), &this->inliers_);
// The two sums behind the threshold are correctly rounded instead of PCL's serial double sums (include/sm_b200.h).
class StatisticRemovalB200 {
 public:
  explicit StatisticRemovalB200(int device = 0) { CHECK_EQ(sm_statistic_removal_create(device, &filter_), 0); }
  ~StatisticRemovalB200() { sm_statistic_removal_destroy(filter_); }
  StatisticRemovalB200(const StatisticRemovalB200&) = delete;
  StatisticRemovalB200& operator=(const StatisticRemovalB200&) = delete;

  // point_num_meank (type 0) or std_mul (type 1); type -1 when the <param> has none (the reference CHECK-fails,
  // filter_interface.cc:57)
  void SetParam(const std::string& name, int type, const std::string& text) {
    CHECK_EQ(sm_statistic_removal_set_param(filter_, name.c_str(), type, text.c_str()), 0)
        << sm_statistic_removal_last_error(filter_);
  }

  // CHECK-fails for 1..point_num_meank finite points (PCL reads past its k-list there) and for a point_num_meank
  // outside 1..63
  void Filter(const data::InnerCloudType& input, data::InnerCloudType* const output,
              std::vector<int>* const inliers = nullptr) {
    FilterRecordsB200(filter_, sm_statistic_removal_run, sm_statistic_removal_last_error, "sm_statistic_removal_run",
                      input, output, inliers);
  }

 private:
  sm_statistic_removal* filter_ = nullptr;
};

// pre_processers::filter::GroundRemoval (v1, pre_processors/filter_ground_removal.{h,cc}) on the GPU: one per
// GroundRemoval.  The body of its InitFromXmlNode becomes one SetParam per <param>, and that of Filter
//   this->FilterPrepare(cloud);
//   filter_.Filter(*this->inner_cloud_, cloud.get(), &this->inliers_, &this->outliers_);
// The output is in the reference's voxel (std::map) order; inliers and outliers are ascending, and the points of a
// voxel below min_point_num_in_voxel are in neither.
class GroundRemovalB200 {
 public:
  explicit GroundRemovalB200(int device = 0) { CHECK_EQ(sm_ground_removal_create(device, &filter_), 0); }
  ~GroundRemovalB200() { sm_ground_removal_destroy(filter_); }
  GroundRemovalB200(const GroundRemovalB200&) = delete;
  GroundRemovalB200& operator=(const GroundRemovalB200&) = delete;

  // min_point_num_in_voxel (type 0), leaf_size or height_threshold (type 1); type -1 when the <param> has none (the
  // reference CHECK-fails, filter_interface.cc:57)
  void SetParam(const std::string& name, int type, const std::string& text) {
    CHECK_EQ(sm_ground_removal_set_param(filter_, name.c_str(), type, text.c_str()), 0)
        << sm_ground_removal_last_error(filter_);
  }

  // CHECK-fails when the voxel indices of an axis span more than 2^21 - 1 voxels (include/sm_b200.h)
  void Filter(const data::InnerCloudType& input, data::InnerCloudType* const output,
              std::vector<int>* const inliers = nullptr, std::vector<int>* const outliers = nullptr) {
    FilterRecordsB200(filter_, sm_ground_removal_run, sm_ground_removal_last_error, "sm_ground_removal_run", input,
                      output, nullptr);
    int64_t n_in = 0, n_out = 0;
    if (!input.points.empty()) CHECK_EQ(sm_ground_removal_indices(filter_, nullptr, &n_in, nullptr, &n_out), 0);
    std::vector<int32_t> in(static_cast<size_t>(n_in)), out(static_cast<size_t>(n_out));
    if (n_in + n_out > 0)
      CHECK_EQ(sm_ground_removal_indices(filter_, in.data(), &n_in, out.data(), &n_out), 0)
          << "sm_ground_removal_indices failed";
    if (inliers) inliers->assign(in.begin(), in.end());
    if (outliers) outliers->assign(out.begin(), out.end());
  }

 private:
  sm_ground_removal* filter_ = nullptr;
};

// The submap sampler RandomSamplerWithPlaneDetect (pre_processors/random_sample_with_plane_detect.h) on the GPU: one
// per sampler, with the class's setters.  Filter keeps the plane points of PlaneDetector and samples the rest at the
// rate, in input order; Inliers() / Outliers() / PlaneIndices() are ascending.  FilterDevice takes a device cloud and
// leaves its output on the device, where sm_set_input_target_f32_device (stride 20) reads it; Submap::InsertFrame's
// next step, CalculateNormals, reads the host output of Filter.  CHECK-fails past 2^24 points or the voxel key's span
// (include/sm_b200.h).
class RandomSamplerWithPlaneDetectB200 {
 public:
  explicit RandomSamplerWithPlaneDetectB200(int device = 0) { CHECK_EQ(sm_plane_sampler_create(device, &sampler_), 0); }
  ~RandomSamplerWithPlaneDetectB200() { sm_plane_sampler_destroy(sampler_); }
  RandomSamplerWithPlaneDetectB200(const RandomSamplerWithPlaneDetectB200&) = delete;
  RandomSamplerWithPlaneDetectB200& operator=(const RandomSamplerWithPlaneDetectB200&) = delete;

  void SetSamplingRate(float rate) { Warn(sm_plane_sampler_set_sampling_rate(sampler_, rate)); }
  void SetLeafSize(float size) { Warn(sm_plane_sampler_set_leaf_size(sampler_, size)); }
  void SetMinPointNumInVoxel(size_t num) { Warn(sm_plane_sampler_set_min_point_num_in_voxel(sampler_, num)); }

  void Filter(const data::InnerCloudType& input, data::InnerCloudType* const output) {
    FilterRecordsB200(sampler_, sm_plane_sampler_run, sm_plane_sampler_last_error, "sm_plane_sampler_run", input,
                      output, nullptr);
  }
  // n records of `stride_bytes` in device memory -> dev_out (capacity n 5-float records); the number kept
  int64_t FilterDevice(const float* dev_points, int64_t n, int64_t stride_bytes, float* dev_out,
                       void* cuda_stream = nullptr) {
    int64_t m = 0;
    const int rc = sm_plane_sampler_run_device(sampler_, dev_points, n, stride_bytes, dev_out, &m, nullptr,
                                               cuda_stream);
    CHECK_EQ(rc, 0) << "sm_plane_sampler_run_device failed (" << rc << "): " << sm_plane_sampler_last_error(sampler_);
    return m;
  }

  std::vector<int> Inliers() const { return Lists(0); }
  std::vector<int> Outliers() const { return Lists(1); }
  std::vector<int> PlaneIndices() const { return Lists(2); }

 private:
  void Warn(int rc) {
    CHECK_EQ(rc, 0);
    const char* message = sm_plane_sampler_last_error(sampler_);
    if (message && message[0]) LOG(WARNING) << message;
  }
  std::vector<int> Lists(int which) const {
    int64_t n[3] = {0, 0, 0};
    CHECK_EQ(sm_plane_sampler_indices(sampler_, nullptr, &n[0], nullptr, &n[1]), 0);
    CHECK_EQ(sm_plane_sampler_plane_indices(sampler_, nullptr, &n[2]), 0);
    std::vector<int32_t> list(static_cast<size_t>(n[which]));
    if (!list.empty() && which == 2) {
      CHECK_EQ(sm_plane_sampler_plane_indices(sampler_, list.data(), &n[2]), 0);
    } else if (!list.empty()) {
      CHECK_EQ(sm_plane_sampler_indices(sampler_, which == 0 ? list.data() : nullptr, &n[0],
                                        which == 1 ? list.data() : nullptr, &n[1]), 0);
    }
    return std::vector<int>(list.begin(), list.end());
  }

  sm_plane_sampler* sampler_ = nullptr;
};

// descriptor::M2dp::setInputCloud + getFinalDescriptor on the GPU (descriptor/m2dp.cc:129-153): the body of
// setInputCloud becomes   return registrator::M2dpB200(*source, r_, max_distance_, t_, p_, q_, &descriptor_);
inline bool M2dpB200(const data::InnerCloudType& source, double r, double max_distance, int32_t t, int32_t p,
                     int32_t q, std::vector<float>* descriptor, int device = 0) {
  CHECK(descriptor);
  const int64_t len = sm_m2dp_descriptor_length(r, max_distance, t, p, q);
  if (len < 0) return false;                              // "r is too small" (m2dp.cc:64-67)
  if (source.points.empty()) return false;                // "source is empty" (:130-133)
  descriptor->assign(static_cast<size_t>(len), 0.f);
  const int rc = sm_m2dp(device, &source.points[0].x, static_cast<int64_t>(source.points.size()),
                         sizeof(data::InnerPointType), r, max_distance, t, p, q, descriptor->data(), len, nullptr);
  CHECK_GE(rc, 0) << "sm_m2dp failed (" << rc << ")";
  return rc == 1;
}

// EigenPointCloud::CalculateNormals on the GPU (cloud_types.cc:347-368); call sites
// map_builder.cc:286,389 and submap.cc:161.
inline void CalculateNormalsB200(data::EigenPointCloud* cloud, int device = 0) {
  CHECK(cloud);
  const int64_t n = cloud->points.cols();
  Eigen::MatrixXd pts(3, n), nrm(3, n);
  int64_t m = 0;
  const int rc = sm_calculate_normals(device, cloud->points.data(), n, pts.data(), nrm.data(), &m);
  CHECK_EQ(rc, 0) << "sm_calculate_normals failed";
  cloud->points = pts.leftCols(m);
  cloud->normals = nrm.leftCols(m);
}

// libnabo's Nabo::NearestNeighbourSearch<double> with KDTREE_LINEAR_HEAP, searched on the GPU: construct it where the
// reference calls NNS::create(cloud, 3, KDTREE_LINEAR_HEAP, 0, {bucketSize}) and call knn() as NNS::knn.  Like libnabo
// it keeps a reference to `cloud`, which must outlive it; the tree is built on the device at every knn() call.
// indices (int32, e.g. Eigen::MatrixXi) and dists2 (double) must be sized k x query.cols(), as libnabo requires; k
// 1..64.  Rows past the neighbours found are -1 / +inf (libnabo's InvalidIndex / InvalidValue).
class KnnB200 {
 public:
  enum SearchOptionFlags { ALLOW_SELF_MATCH = SM_KNN_ALLOW_SELF_MATCH, SORT_RESULTS = SM_KNN_SORT_RESULTS };

  explicit KnnB200(const Eigen::MatrixXd& cloud, unsigned bucket_size = 8, int device = 0)
      : cloud_(cloud), bucket_size_(static_cast<int>(bucket_size)), device_(device) {
    CHECK_EQ(cloud.rows(), 3);
  }

  template <class IndexMatrix, class DistMatrix>
  void knn(const Eigen::MatrixXd& query, IndexMatrix& indices, DistMatrix& dists2, int k = 1, double epsilon = 0.0,
           unsigned option_flags = 0, double max_radius = std::numeric_limits<double>::infinity()) const {
    CHECK_EQ(query.rows(), 3);
    CHECK_EQ(static_cast<long>(indices.rows()), static_cast<long>(k));
    CHECK_EQ(static_cast<long>(indices.cols()), static_cast<long>(query.cols()));
    CHECK_EQ(static_cast<long>(dists2.rows()), static_cast<long>(k));
    CHECK_EQ(static_cast<long>(dists2.cols()), static_cast<long>(query.cols()));
    static_assert(sizeof(*indices.data()) == sizeof(int32_t), "indices: 32-bit integers, as libnabo's IndexMatrix");
    const int rc = sm_knn(device_, cloud_.data(), static_cast<int64_t>(cloud_.cols()), query.data(),
                          static_cast<int64_t>(query.cols()), k, epsilon, max_radius, option_flags, bucket_size_,
                          reinterpret_cast<int32_t*>(indices.data()), dists2.data());
    CHECK_EQ(rc, 0) << "sm_knn failed (" << rc << ")";
  }

 private:
  const Eigen::MatrixXd& cloud_;
  int bucket_size_;
  int device_;
};

}  // namespace registrator
}  // namespace static_map

#endif  // ADAPTER_REGISTRATORS_B200_H_
