// IPC::CollisionObject<dim> and IPC::HalfSpace<dim> members the half-space adapter overrides or reads, restated from the reference for a compile
// check (src/CollisionObject/CollisionObject.h:29-33 origin / velocitydt / friction, :127-170 constraint virtuals, :323-325 computeConstraintSet,
// :386-390 isIntersected, :403-423 friction virtuals; src/CollisionObject/HalfSpace.hpp: normal, D, the constructors).  Test scaffolding only.
#pragma once
#include "LinSysSolver.hpp"
#include "Mesh.hpp"
#include <Eigen/Eigen>
#include <vector>
namespace ccd {
enum class CCDMethod { FLOATING_POINT_ROOT_FINDER };
}
namespace IPC {
template <int dim>
class CollisionObject {
public:
    Eigen::Matrix<double, dim, 1> origin;
    Eigen::Matrix<double, dim, 1> velocitydt;
    double friction;
    virtual ~CollisionObject() {}
    virtual void leftMultiplyConstraintJacobianT(const Mesh<dim>& mesh, const std::vector<int>& activeSet, const Eigen::VectorXd& input,
        Eigen::VectorXd& output_incremental, double coef = 1.0) const = 0;
    virtual void augmentIPHessian(const Mesh<dim>& mesh, const std::vector<int>& activeSet, LinSysSolver<Eigen::VectorXi, Eigen::VectorXd>* mtr_incremental,
        double dHat, double coef = 1.0, bool projectDBC = true) const = 0;
    virtual void largestFeasibleStepSize(const Mesh<dim>& mesh, const Eigen::VectorXd& searchDir, double slackness, std::vector<int>& activeSet_next,
        double& stepSize) = 0;
    virtual void computeConstraintSet(const Mesh<dim>& mesh, double dHat, std::vector<int>& constraintSet) const;
    virtual bool isIntersected(const Mesh<dim>& mesh, const Eigen::MatrixXd& V0, const ccd::CCDMethod method = ccd::CCDMethod::FLOATING_POINT_ROOT_FINDER) const;
    virtual void computeFrictionEnergy(const Eigen::MatrixXd& V, const Eigen::MatrixXd& Vt, const std::vector<int>& activeSet, const Eigen::VectorXd& multipliers,
        double& Ef, double eps2, double coef) const;
    virtual void augmentFrictionGradient(const Eigen::MatrixXd& V, const Eigen::MatrixXd& Vt, const std::vector<int>& activeSet, const Eigen::VectorXd& multipliers,
        Eigen::VectorXd& grad_inc, double eps2, double coef) const;
    virtual void augmentFrictionHessian(const Mesh<dim>& mesh, const Eigen::MatrixXd& Vt, const std::vector<int>& activeSet, const Eigen::VectorXd& multipliers,
        LinSysSolver<Eigen::VectorXi, Eigen::VectorXd>* H_inc, double eps2, double coef, bool projectDBC = true) const;
};
template <int dim>
class HalfSpace : public CollisionObject<dim> {
public:
    HalfSpace(const Eigen::Matrix<double, dim, 1>& p_origin, const Eigen::Matrix<double, dim, 1>& p_normal, const Eigen::Matrix<double, dim, 1>& p_velocitydt,
        double p_friction);
    HalfSpace(double p_Y, double p_friction);
    Eigen::Matrix<double, dim, 1> normal;
    double D;
    void leftMultiplyConstraintJacobianT(const Mesh<dim>& mesh, const std::vector<int>& activeSet, const Eigen::VectorXd& input, Eigen::VectorXd& output_incremental,
        double coef = 1.0) const override;
    void augmentIPHessian(const Mesh<dim>& mesh, const std::vector<int>& activeSet, LinSysSolver<Eigen::VectorXi, Eigen::VectorXd>* mtr_incremental, double dHat,
        double coef = 1.0, bool projectDBC = true) const override;
    void largestFeasibleStepSize(const Mesh<dim>& mesh, const Eigen::VectorXd& searchDir, double slackness, std::vector<int>& activeSet_next,
        double& stepSize) override;
};
} // namespace IPC
