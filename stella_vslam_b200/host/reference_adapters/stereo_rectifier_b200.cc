// Drop-in replacement for src/stella_vslam/util/stereo_rectifier.cc (same header, same members): link this translation unit instead of
// the original one.  The constructors keep their checks, exceptions and YAML parsing (stereo_rectifier.cc:12-56); the two maps per eye
// are built once by b200_rectifier_create, which also keeps their fixed-point form on the device, and rectify() runs cv::remap
// (INTER_LINEAR, BORDER_CONSTANT 0) of both eyes there, bit-exact to OpenCV.  undist_map_{x,y}_{l,r}_ are filled from
// b200_rectifier_maps so that the object holds what the reference's holds.
//
// Deviations: rectify() accepts CV_8UC1 / CV_8UC3 / CV_8UC4 frames of the camera's size only and throws otherwise; distortion vectors
// of 12 or 14 coefficients (thin prism, tilt) throw.
#include "stella_vslam/camera/perspective.h"
#include "stella_vslam/util/stereo_rectifier.h"
#include "stella_vslam/util/yaml.h"

#include <spdlog/spdlog.h>
#include <opencv2/core/mat.hpp>

#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>

#include "b200vslam.h"

namespace stella_vslam {
namespace util {

namespace {
// stereo_rectifier.h has no spare member for the handle; keep it in a side table keyed by `this` (as orb_extractor_b200.cc does).
std::mutex g_mtx;
std::unordered_map<const stereo_rectifier*, b200_rectifier_t> g_handles;

b200_rectifier_t handle_of(const stereo_rectifier* self) {
    std::lock_guard<std::mutex> lock(g_mtx);
    auto it = g_handles.find(self);
    if (it == g_handles.end()) throw std::runtime_error("stereo_rectifier: no device rectifier for this object");
    return it->second;
}

void copy9(double* dst, const std::vector<double>& v, const char* key) {
    if (v.size() < 9) throw std::runtime_error(std::string("StereoRectifier.") + key + " needs 9 values");
    std::memcpy(dst, v.data(), 9 * sizeof(double));
}
}  // namespace

stereo_rectifier::stereo_rectifier(const std::shared_ptr<stella_vslam::config>& cfg, camera::base* camera)
    : stereo_rectifier(camera, stella_vslam::util::yaml_optional_ref(cfg->yaml_node_, "StereoRectifier")) {}

stereo_rectifier::stereo_rectifier(camera::base* camera, const YAML::Node& yaml_node)
    : model_type_(load_model_type(yaml_node)) {
    spdlog::debug("CONSTRUCT: util::stereo_rectifier (b200)");
    if (camera->setup_type_ != camera::setup_type_t::Stereo) {
        throw std::runtime_error("When stereo rectification is used, 'setup' must be set to 'stereo'");
    }
    if (camera->model_type_ != camera::model_type_t::Perspective) {
        throw std::runtime_error("When stereo rectification is used, 'model' must be set to 'perspective'");
    }
    const auto K_l = yaml_node["K_left"].as<std::vector<double>>();
    const auto K_r = yaml_node["K_right"].as<std::vector<double>>();
    const auto R_l = yaml_node["R_left"].as<std::vector<double>>();
    const auto R_r = yaml_node["R_right"].as<std::vector<double>>();
    const auto D_l_vec = yaml_node["D_left"].as<std::vector<double>>();
    const auto D_r_vec = yaml_node["D_right"].as<std::vector<double>>();
    if (model_type_ != camera::model_type_t::Perspective && model_type_ != camera::model_type_t::Fisheye) {
        throw std::runtime_error("Invalid model type for stereo rectification: " + camera->get_model_type_string());
    }
    b200_rectifier_params_t p;
    std::memset(&p, 0, sizeof(p));
    p.model = model_type_ == camera::model_type_t::Fisheye ? 1 : 0;
    p.cols = static_cast<int32_t>(camera->cols_);
    p.rows = static_cast<int32_t>(camera->rows_);
    // camera matrix after rectification: cv_cam_matrix_ is CV_32F, the maps are built from its float values
    const cv::Mat& K_rect = static_cast<camera::perspective*>(camera)->cv_cam_matrix_;
    for (int k = 0; k < 9; ++k) p.K_rect[k] = K_rect.at<float>(k / 3, k % 3);
    copy9(p.K[0], K_l, "K_left");
    copy9(p.K[1], K_r, "K_right");
    copy9(p.R[0], R_l, "R_left");
    copy9(p.R[1], R_r, "R_right");
    const std::vector<double>* D[2] = {&D_l_vec, &D_r_vec};
    for (int eye = 0; eye < 2; ++eye) {
        if (D[eye]->size() > 8) throw std::runtime_error("stereo_rectifier (b200): the thin-prism and tilt distortion models are not supported");
        std::memcpy(p.D[eye], D[eye]->data(), D[eye]->size() * sizeof(double));
        p.n_dist[eye] = static_cast<int32_t>(D[eye]->size());
    }
    p.device = 0;
    b200_rectifier_t h = nullptr;
    if (b200_rectifier_create(&p, &h) != B200_OK) throw std::runtime_error(b200_last_error());
    {
        std::lock_guard<std::mutex> lock(g_mtx);
        g_handles[this] = h;
    }
    undist_map_x_l_.create(p.rows, p.cols, CV_32F);
    undist_map_y_l_.create(p.rows, p.cols, CV_32F);
    undist_map_x_r_.create(p.rows, p.cols, CV_32F);
    undist_map_y_r_.create(p.rows, p.cols, CV_32F);
    if (b200_rectifier_maps(h, 0, undist_map_x_l_.ptr<float>(), undist_map_y_l_.ptr<float>()) != B200_OK
        || b200_rectifier_maps(h, 1, undist_map_x_r_.ptr<float>(), undist_map_y_r_.ptr<float>()) != B200_OK)
        throw std::runtime_error(b200_last_error());
}

stereo_rectifier::~stereo_rectifier() {
    spdlog::debug("DESTRUCT: util::stereo_rectifier (b200)");
    b200_rectifier_t h = nullptr;
    {
        std::lock_guard<std::mutex> lock(g_mtx);
        auto it = g_handles.find(this);
        if (it != g_handles.end()) {
            h = it->second;
            g_handles.erase(it);
        }
    }
    b200_rectifier_destroy(h);
}

void stereo_rectifier::rectify(const cv::Mat& in_img_l, const cv::Mat& in_img_r,
                               cv::Mat& out_img_l, cv::Mat& out_img_r) const {
    const int type = in_img_l.type();
    if ((type != CV_8UC1 && type != CV_8UC3 && type != CV_8UC4) || in_img_r.type() != type) {
        throw std::runtime_error("stereo_rectifier (b200): both frames must be CV_8UC1, CV_8UC3 or CV_8UC4 of the same type");
    }
    if (in_img_l.cols != undist_map_x_l_.cols || in_img_l.rows != undist_map_x_l_.rows || in_img_r.cols != in_img_l.cols
        || in_img_r.rows != in_img_l.rows) {
        throw std::runtime_error("stereo_rectifier (b200): frames must have the camera's size");
    }
    // cv::remap copies a source that is also the destination; do the same before the outputs are (re)allocated
    const cv::Mat src_l = in_img_l.data == out_img_l.data || in_img_l.data == out_img_r.data ? in_img_l.clone() : in_img_l;
    const cv::Mat src_r = in_img_r.data == out_img_l.data || in_img_r.data == out_img_r.data ? in_img_r.clone() : in_img_r;
    out_img_l.create(src_l.rows, src_l.cols, type);
    out_img_r.create(src_r.rows, src_r.cols, type);
    if (b200_stereo_rectify(handle_of(this), src_l.channels(), src_l.data, src_l.step, src_r.data, src_r.step, out_img_l.data, out_img_l.step,
                            out_img_r.data, out_img_r.step)
        != B200_OK)
        throw std::runtime_error(b200_last_error());
}

cv::Mat stereo_rectifier::parse_vector_as_mat(const cv::Size& shape, const std::vector<double>& vec) {
    cv::Mat mat(shape, CV_64F);
    std::memcpy(mat.data, vec.data(), shape.height * shape.width * sizeof(double));
    return mat;
}

camera::model_type_t stereo_rectifier::load_model_type(const YAML::Node& yaml_node) {
    const auto model_type_str = yaml_node["model"].as<std::string>("perspective");
    if (model_type_str == "perspective") {
        return camera::model_type_t::Perspective;
    }
    else if (model_type_str == "fisheye") {
        return camera::model_type_t::Fisheye;
    }
    else if (model_type_str == "equirectangular") {
        return camera::model_type_t::Equirectangular;
    }

    throw std::runtime_error("Invalid camera model: " + model_type_str);
}

}  // namespace util
}  // namespace stella_vslam
