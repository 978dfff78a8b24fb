#!/bin/sh
# Builds oracle/_ref/libref_pairs.so from the REFERENCE's own scalar code (MATLAB-codegen bodies of the
# pair-distance gradients/Hessians, the EE cross-norm derivatives, the mollifier polynomial and the C2 barrier)
# compiled from the sources where they lie under /root/reference, and oracle/_ref/libref_cubic.so from its
# inversion-filter root finders (getSmallestPositiveRealQuadRoot / getSmallestPositiveRealCubicRoot, pure double and
# std::complex) and its absolute-coordinate coefficient lines (a, b, c, d of computeInjectiveStepSize_3d), the latter
# inside a shim that declares the scalars they read.  The line ranges below are the pure-`double`
# overloads (no Eigen inside); they are streamed through sed into a scratch file OUTSIDE the repo, compiled, and
# the scratch file is deleted -- no reference source is ever copied into this repository.  Only the .so lands in
# oracle/_ref/ (git-ignored, travels to the GPU box).  The rest of the reference (Eigen/TBB/libigl/CCD-Wrapper
# dependent) is unbuildable here: see DESIGN.md.
set -e
REF=/root/reference/src
HERE=$(cd "$(dirname "$0")" && pwd)
OUT="$HERE/_ref"
CXX=/usr/bin/g++; [ -x "$CXX" ] || CXX=g++
mkdir -p "$OUT"
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
M="$REF/CollisionObject/MeshCollisionUtils.hpp"
B="$REF/Utils/BarrierFunctions.hpp"
{
  echo '#include <cmath>'
  echo 'namespace refsrc {'
  sed -n '235,287p;300,620p;696,757p;772,1217p;1298,1377p;1392,2002p;2419,2477p;2494,2762p;2834,2849p' "$M"
  sed -n '56,83p' "$B"
  echo '}'
  cat <<'SHIM'
extern "C" {
#define V9 v[0],v[1],v[2],v[3],v[4],v[5],v[6],v[7],v[8]
#define V12 V9,v[9],v[10],v[11]
void ref_g_PE(const double* v, double* g) { refsrc::g_PE(V9, g); }
void ref_H_PE(const double* v, double* H) { refsrc::H_PE(V9, H); }
void ref_g_PT(const double* v, double* g) { refsrc::g_PT(V12, g); }
void ref_H_PT(const double* v, double* H) { refsrc::H_PT(V12, H); }
void ref_g_EE(const double* v, double* g) { refsrc::g_EE(V12, g); }
void ref_H_EE(const double* v, double* H) { refsrc::H_EE(V12, H); }
void ref_EEcross_g(const double* v, double* g) { refsrc::computeEECrossSqNormGradient(V12, g); }
void ref_EEcross_H(const double* v, double* H) { refsrc::computeEECrossSqNormHessian(V12, H); }
void ref_q(double x, double eps, double* q, double* qg, double* qH) { refsrc::compute_q(x, eps, *q); refsrc::compute_q_g(x, eps, *qg); refsrc::compute_q_H(x, eps, *qH); }
void ref_barrier(double d, double dHat, double* b, double* g, double* H) { refsrc::b_C2(d, dHat, *b); refsrc::g_bC2(d, dHat, *g); refsrc::H_bC2(d, dHat, *H); }
}
SHIM
} > "$TMP/ref_pairs.cpp"
$CXX -O2 -std=c++17 -fPIC -ffp-contract=off -shared -o "$OUT/libref_pairs.so" "$TMP/ref_pairs.cpp"
echo "built $OUT/libref_pairs.so"
G="$REF/Utils/get_feasible_steps.cpp"
{
  echo '#include <cmath>'
  echo '#include <complex>'
  echo 'namespace refsrc {'
  echo 'using namespace std;'
  sed -n '9,28p;75,108p' "$G"
  echo 'void coefs(const double* X, const double* P, double slackness, double* out) {'
  echo 'const double x1 = X[0], y1 = X[1], z1 = X[2], x2 = X[3], y2 = X[4], z2 = X[5], x3 = X[6], y3 = X[7], z3 = X[8], x4 = X[9], y4 = X[10], z4 = X[11];'
  echo 'const double p1 = P[0], q1 = P[1], r1 = P[2], p2 = P[3], q2 = P[4], r2 = P[5], p3 = P[6], q3 = P[7], r3 = P[8], p4 = P[9], q4 = P[10], r4 = P[11];'
  echo 'double a, b, c, d;'
  sed -n '158,161p' "$G"
  echo 'out[0] = a; out[1] = b; out[2] = c; out[3] = d;'
  echo '}'
  echo '}'
  cat <<'SHIM'
extern "C" {
double ref_quad_root(double a, double b, double c, double tol) { return refsrc::getSmallestPositiveRealQuadRoot(a, b, c, tol); }
double ref_cubic_root(double a, double b, double c, double d, double tol) { return refsrc::getSmallestPositiveRealCubicRoot(a, b, c, d, tol); }
void ref_inversion_coefs(const double* X, const double* P, double slackness, double* out) { refsrc::coefs(X, P, slackness, out); }
}
SHIM
} > "$TMP/ref_cubic.cpp"
$CXX -O2 -std=c++17 -fPIC -ffp-contract=off -shared -o "$OUT/libref_cubic.so" "$TMP/ref_cubic.cpp"
echo "built $OUT/libref_cubic.so"
