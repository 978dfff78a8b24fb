// Instantiates the half-space adapter against the restated reference interface (syntax/semantic check only: g++ -fsyntax-only).
#include "IpcGpuHalfSpace.hpp"
void touch_halfspace(IPC::IpcGpuScene& s, const IPC::Mesh<3>& m, IPC::LinSysSolver<Eigen::VectorXi, Eigen::VectorXd>* sol, const Eigen::VectorXd& p)
{
    Eigen::Matrix<double, 3, 1> o, n, v;
    IPC::GpuHalfSpace ground(s, o, n, v, 0.3);
    IPC::CollisionObject<3>& co = ground; // called through the reference's base class, as Optimizer.cpp does
    std::vector<int> as, next;
    Eigen::VectorXd g, lam;
    Eigen::MatrixXd Vt;
    double alpha = 1.0, Ef = 0.0;
    co.computeConstraintSet(m, 1e-6, as);
    co.augmentIPHessian(m, as, sol, 1e-6, 1e8, true);
    co.largestFeasibleStepSize(m, p, 0.9, next, alpha);
    (void)co.isIntersected(m, m.V);
    IPC::GpuHalfSpace::lag(1e-6, 1e8);
    co.computeFrictionEnergy(m.V, Vt, as, lam, Ef, 1e-9, 1.0);
    co.augmentFrictionGradient(m.V, Vt, as, lam, g, 1e-9, 1.0);
    co.augmentFrictionHessian(m, Vt, as, lam, sol, 1e-9, 1.0, true);
    IPC::GpuHalfSpace::upload();
}
