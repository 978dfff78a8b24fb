// IpcGpuHalfSpace.hpp -- reference-side binding of the analytic half-space planes (include/ipcgpu.h: ipcgpu_set_halfspaces, ipcgpu_halfspace_*).
//
// Compiled inside an ipc-sim/IPC checkout next to IpcGpuAdapters.hpp; not built in this repository (tests/test_oracle_halfspace.py
// compile-checks it against tests/stubs/CollisionObject.h).
//
// The reference keeps one HalfSpace<3> per plane in animConfig.collisionObjects and calls each one's virtuals in turn (activeSet[coI]); the
// device runs every plane in one pass.  GpuHalfSpace derives from HalfSpace<3> (construction, QP functions, move, rendering stay the
// reference's) and overrides the IP-path virtuals with the reference's signatures:
//   computeConstraintSet (CollisionObject.h:323)       ipcgpu_halfspace_constraint_set, once per state (plane 0), each plane takes its entries
//   augmentIPHessian (HalfSpace.cpp:169)               ipcgpu_halfspace_hessian, every plane's blocks in plane 0's call; the others add nothing
//   largestFeasibleStepSize (HalfSpace.cpp:242)        ipcgpu_halfspace_step in plane 0's call (a minimum: the order of the planes does not matter)
//   isIntersected (CollisionObject.h:386)              ipcgpu_halfspace_crossings in plane 0's call
//   computeFrictionEnergy / augmentFriction* (:272)    the device's lagged set (GpuHalfSpace::lag at Optimizer.cpp:1555, in place of the loop there)
// The energies the reference forms from evaluateConstraints (Optimizer.cpp:3254-3267) stay its own host code; a caller that moves the whole
// iteration onto the device uses the NULL-output calls instead (INTEGRATION.md section 8).  Planes that move (HalfSpace::move, AnimScripter)
// are re-uploaded with GpuHalfSpace::upload after the motion.
#pragma once
#include "IpcGpuAdapters.hpp"
#include "CollisionObject.h"

namespace IPC {

class GpuHalfSpace : public HalfSpace<3> {
public:
    inline static IpcGpuScene* gpu = nullptr;
    inline static std::vector<GpuHalfSpace*> planes;    // in animConfig.collisionObjects order
    inline static std::vector<std::vector<int>> active; // the last device set, split by plane
    int k = 0;                                          // this plane's index on the device

    GpuHalfSpace(IpcGpuScene& scene, const Eigen::Matrix<double, 3, 1>& p_origin, const Eigen::Matrix<double, 3, 1>& p_normal,
        const Eigen::Matrix<double, 3, 1>& p_velocitydt, double p_friction)
        : HalfSpace<3>(p_origin, p_normal, p_velocitydt, p_friction)
    {
        gpu = &scene;
        k = (int)planes.size();
        planes.push_back(this);
        upload();
    }
    ~GpuHalfSpace() override
    {
        planes.erase(std::find(planes.begin(), planes.end(), this));
        for (size_t i = 0; i < planes.size(); ++i) planes[i]->k = (int)i;
        upload();
    }

    // every plane's origin / normal / velocitydt / friction to the device (after construction and after every scripted motion)
    static void upload()
    {
        const int n = (int)planes.size();
        std::vector<double> o(3 * n), nr(3 * n), v(3 * n), f(n);
        for (int i = 0; i < n; ++i) {
            for (int c = 0; c < 3; ++c) {
                o[3 * i + c] = planes[i]->origin.data()[c];
                nr[3 * i + c] = planes[i]->normal.data()[c];
                v[3 * i + c] = planes[i]->velocitydt.data()[c];
            }
            f[i] = planes[i]->friction;
        }
        IpcGpuScene::check(gpu->ctx, ipcgpu_set_halfspaces(gpu->ctx, n, o.data(), nr.data(), v.data(), f.data()), "ipcgpu_set_halfspaces");
    }
    // Optimizer.cpp:1555-1572: lagged set and lambda of every plane with friction > 0, on the device
    static void lag(double dHat, double kappa)
    {
        IpcGpuScene::check(gpu->ctx, ipcgpu_halfspace_friction_lag(gpu->ctx, dHat, kappa, nullptr), "ipcgpu_halfspace_friction_lag");
    }

    void computeConstraintSet(const Mesh<3>& mesh, double dHat, std::vector<int>& constraintSet) const override
    {
        if (k == 0) {
            int n = 0;
            IpcGpuScene::check(gpu->ctx, ipcgpu_halfspace_constraint_set(gpu->ctx, dHat, &n), "ipcgpu_halfspace_constraint_set");
            std::vector<int> pv(2 * (size_t)n);
            IpcGpuScene::check(gpu->ctx, ipcgpu_get_halfspace_sets(gpu->ctx, &n, pv.data(), nullptr, nullptr, nullptr), "ipcgpu_get_halfspace_sets");
            active.assign(planes.size(), {});
            for (int c = 0; c < n; ++c) active[pv[2 * c]].push_back(pv[2 * c + 1]);
        }
        constraintSet = active[k];
    }
    void augmentIPHessian(const Mesh<3>& mesh, const std::vector<int>& activeSet, LinSysSolver<Eigen::VectorXi, Eigen::VectorXd>* mtr_incremental, double dHat,
        double coef = 1.0, bool projectDBC = true) const override
    {
        if (k != 0) return;
        IpcGpuScene::check(gpu->ctx, ipcgpu_halfspace_hessian(gpu->ctx, dHat, coef, projectDBC ? 1 : 0, mtr_incremental->get_a().data()),
            "ipcgpu_halfspace_hessian");
    }
    void largestFeasibleStepSize(const Mesh<3>& mesh, const Eigen::VectorXd& searchDir, double slackness, std::vector<int>& activeSet_next,
        double& stepSize) override
    {
        if (k != 0) return;
        IpcGpuScene::check(gpu->ctx, ipcgpu_halfspace_step(gpu->ctx, searchDir.data(), slackness, &stepSize), "ipcgpu_halfspace_step");
    }
    bool isIntersected(const Mesh<3>& mesh, const Eigen::MatrixXd& V0, const ccd::CCDMethod method = ccd::CCDMethod::FLOATING_POINT_ROOT_FINDER) const override
    {
        if (k != 0) return false;
        int n = 0;
        IpcGpuScene::check(gpu->ctx, ipcgpu_halfspace_crossings(gpu->ctx, &n), "ipcgpu_halfspace_crossings");
        return n > 0;
    }
    // the friction terms of every lagged plane entry in plane 0's call (coef is 1.0 for collision objects, Optimizer.cpp:3361)
    void computeFrictionEnergy(const Eigen::MatrixXd& V, const Eigen::MatrixXd& Vt, const std::vector<int>& activeSet, const Eigen::VectorXd& multipliers,
        double& Ef, double eps2, double coef) const override
    {
        Ef = 0.0;
        if (k == 0) IpcGpuScene::check(gpu->ctx, ipcgpu_halfspace_friction_energy(gpu->ctx, eps2, &Ef), "ipcgpu_halfspace_friction_energy");
    }
    void augmentFrictionGradient(const Eigen::MatrixXd& V, const Eigen::MatrixXd& Vt, const std::vector<int>& activeSet, const Eigen::VectorXd& multipliers,
        Eigen::VectorXd& grad_inc, double eps2, double coef) const override
    {
        if (k == 0) IpcGpuScene::check(gpu->ctx, ipcgpu_halfspace_friction_gradient(gpu->ctx, eps2, grad_inc.data()), "ipcgpu_halfspace_friction_gradient");
    }
    void augmentFrictionHessian(const Mesh<3>& mesh, const Eigen::MatrixXd& Vt, const std::vector<int>& activeSet, const Eigen::VectorXd& multipliers,
        LinSysSolver<Eigen::VectorXi, Eigen::VectorXd>* H_inc, double eps2, double coef, bool projectDBC = true) const override
    {
        if (k == 0)
            IpcGpuScene::check(gpu->ctx, ipcgpu_halfspace_friction_hessian(gpu->ctx, eps2, projectDBC ? 1 : 0, H_inc->get_a().data()),
                "ipcgpu_halfspace_friction_hessian");
    }
};

} // namespace IPC
