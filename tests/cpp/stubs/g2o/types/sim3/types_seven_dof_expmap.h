// Declaration-only stand-in for g2o's types_seven_dof_expmap.h (module/type.h includes it): the g2o::Sim3 interface the
// graph-optimiser adapter uses, for type-checking against the reference headers.
#pragma once
#include <Eigen/Core>
#include <Eigen/Geometry>

namespace g2o {
using Vector3 = Eigen::Matrix<double, 3, 1>;
using Vector7 = Eigen::Matrix<double, 7, 1>;
using Matrix3 = Eigen::Matrix<double, 3, 3>;
using Quaternion = Eigen::Quaternion<double>;
struct Sim3 {
    Sim3();
    Sim3(const Quaternion& r, const Vector3& t, double s);
    Sim3(const Matrix3& R, const Vector3& t, double s);
    explicit Sim3(const Vector7& update);
    Vector3 map(const Vector3& xyz) const;
    Vector7 log() const;
    Sim3 inverse() const;
    Sim3 operator*(const Sim3& other) const;
    Sim3& operator*=(const Sim3& other);
    const Vector3& translation() const;
    Vector3& translation();
    const Quaternion& rotation() const;
    Quaternion& rotation();
    const double& scale() const;
    double& scale();
};
}  // namespace g2o
