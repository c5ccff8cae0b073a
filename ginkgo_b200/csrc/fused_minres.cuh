// What the fused MINRES paths share (fused_minres.cu, fused_minres_mrhs.cu): safe_divide and the scalar
// recurrence minres::step_1, both as krylov_steps.cu states them.
#pragma once
#include "fused_common.cuh"

namespace b200 {
namespace fminres {

// include/ginkgo/core/base/math.hpp, as krylov_steps.cu states them
template <typename V>
__device__ __forceinline__ V safe_divide(V a, V b)
{
    return b == V(0) ? V(0) : a / b;
}
template <typename V>
__device__ __forceinline__ V dev_abs(V a)
{
    return a < V(0) ? -a : a;
}

// minres::step_1 (krylov_steps.cu, reference/solver/minres_kernels.cpp:64-110) on one column's scalars,
// by ONE thread, with beta = v.z~ just summed.  Slot s of the column is sc[s * k] (fused_minres.cu's
// numbering; one column: k = 1).
template <typename V>
__device__ __forceinline__ void step_1(V beta_sq, V* sc, int64_t k)
{
    const V bt = sqrt(beta_sq);
    sc[1 * k] = bt;
    const V tmp_d = sc[2 * k];
    const V tmp_a = sc[0];
    sc[3 * k] = sc[11 * k] * tmp_d;
    const V c_old = sc[10 * k], s_old = sc[12 * k], cp_old = sc[9 * k];
    const V g1 = cp_old * c_old;
    const V g2 = g1 * tmp_d;
    const V g3 = s_old * tmp_a;
    sc[2 * k] = g2 + g3;
    const V a1 = (-s_old) * cp_old;
    const V a2 = a1 * tmp_d;
    const V a3 = c_old * tmp_a;
    V al = a2 + a3;
    sc[9 * k] = c_old;
    sc[11 * k] = s_old;
    V c, sn;
    if (al == V(0)) {
        c = V(0);
        sn = V(1);
    } else {
        const V scale = dev_abs(al) + dev_abs(bt);
        const V ra = dev_abs(al / scale), rb = dev_abs(bt / scale);
        const V h1 = ra * ra;
        const V h2 = rb * rb;
        const V hyp = scale * sqrt(h1 + h2);
        c = al / hyp;
        sn = bt / hyp;
    }
    const V n1 = c * al;
    const V n2 = sn * bt;
    al = n1 + n2;
    sc[0] = al;
    sc[10 * k] = c;
    sc[12 * k] = sn;
    const V t1 = sn * sn;
    sc[6 * k] = t1 * sc[6 * k];
    const V e = sc[8 * k];
    sc[7 * k] = e;
    sc[8 * k] = (-sn) * e;
}

}  // namespace fminres
}  // namespace b200
