/*
 * TEST INFRASTRUCTURE ONLY.  What the sources of the host-memory mock (the .c files next to it) share:
 * the context, the recorded graph operations, the error buffer and the stopping rule of the fused paths.
 */
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "ginkgo_b200.h"

typedef struct mock_graph mock_graph;
struct b200_ctx {
    int device;
    int64_t launches;
    mock_graph* capture; /* non-NULL between b200_graph_begin_capture and end_capture */
    unsigned char snap[2][256]; /* b200_snapshot_*: the mock executes in order, so begin copies at once */
};

/* ---- graphs: the calls made between begin_capture and end_capture are recorded, not executed (as
 * under CUDA stream capture).  Each recorded call carries the function that runs it again;
 * b200_graph_launch calls those in order and counts one launch per call. ---- */
typedef struct mock_op mock_op;
typedef b200_status (*mock_replay)(b200_ctx* ctx, const mock_op* op);
struct mock_op {
    mock_replay replay;
    void* p[16];
    int64_t n[4];
    int32_t i[4];
    double d;
    void* keep; /* a heap block of arguments, freed with the graph */
};
/* a zeroed operation appended to the graph being captured */
mock_op* mock_new_op(b200_ctx* ctx, mock_replay replay);

void mock_set_error(const char* fmt, ...);

/* fused::criteria_status (ginkgo_b200/csrc/fused_common.cuh): Iteration (ctl[2], -1 = none) and a
 * residual norm (ctl[3], 0 = none) in the user's order (ctl[4]) with ids 1 and 2.  `converged` says
 * whether the residual criterion holds; `finalized` is OR-ed into a stop. */
#define STOPPED(s) ((s) & 0x3f)
static inline uint8_t mock_criteria_status(int32_t iter, const int32_t* ctl, int converged, uint8_t finalized)
{
    const int32_t max_iters = ctl[2], res_kind = ctl[3], iter_first = ctl[4];
    uint8_t status = 0, id = 1;
    for (int k = 0; k < 2 && status == 0; ++k) {
        const int is_it = (k == 0) == (iter_first != 0);
        if (is_it) {
            if (max_iters < 0) continue;
            if (iter >= max_iters) status = (uint8_t)((id & 0x3f) | finalized);
            ++id;
        } else {
            if (!res_kind) continue;
            if (converged) status = (uint8_t)(0x80 | (id & 0x3f) | finalized);
            ++id;
        }
    }
    return status;
}

/* fused::finish_scalars, the top-of-iteration check of the one-column CG and BiCGStab: rho and ||r||^2
 * shifted into sc, the iteration counted, the status (finalized) into ctl[0] */
#define MOCK_FINISH_SCALARS(V, VT, SQRT, FABS)                                                         \
    static inline void mock_finish_scalars_##V(VT rho_new, VT rr, VT* sc, int32_t* ctl)                \
    {                                                                                                  \
        sc[1] = sc[0];                                                                                 \
        sc[0] = rho_new;                                                                               \
        sc[3] = rr;                                                                                    \
        const int32_t iter = ctl[1] + 1;                                                               \
        ctl[1] = iter;                                                                                 \
        const VT tau = ctl[3] == 1 ? SQRT(rr) : SQRT(FABS(rho_new));                                   \
        ctl[0] = mock_criteria_status(iter, ctl, tau <= sc[5], 0x40);                                  \
    }
MOCK_FINISH_SCALARS(f64, double, sqrt, fabs)
MOCK_FINISH_SCALARS(f32, float, sqrtf, fabsf)

/* the oracle's Givens update of the Hessenberg column, which the fused GMRES paths call as the loop does */
void orc_common_gmres_hessenberg_qr_f64(int64_t, double*, int64_t, double*, int64_t, double*, double*, int64_t,
                                        double*, int64_t, int64_t, uint64_t*, const uint8_t*);
void orc_common_gmres_hessenberg_qr_f32(int64_t, float*, int64_t, float*, int64_t, float*, float*, int64_t,
                                        float*, int64_t, int64_t, uint64_t*, const uint8_t*);
