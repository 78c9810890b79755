// ba_solver.cu -- host Levenberg-Marquardt controller + C ABI of the BA path.
//
// Mirrors, statement by statement where it decides anything:
//   sba_motstr_levmar_x     lib/sba-1.5/sba_levmar.c:457-2081  (controller quirks: SURVEY.md A.3)
//   run_sfm                 lib/sfm-driver/sfm.c:592-1003       (packing :652-703, unpacking :876-929)
// All array work runs in the sm_90a kernels of ba_kernels.cu / ba_chol.cu, set up by ba_setup.cu; the host only reads
// back one small scalar block per LM phase.  No CPU fallback.
#include "common.h"
#include "ba_kernels.cuh"
#include "ba_chol_large.cuh"
#include "ba_loop.h"
#include "../../include/bsfm_b200_ba.h"
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

using namespace bsfm;
using namespace bsfm::ba;

#define SBA_ERROR_RC (-1)
static const double SBA_EPSILON_SQ = 1E-12 * 1E-12;      // sba_levmar.c:34-35
static const double SBA_ONE_THIRD = 0.3333333334;         // sba_levmar.c:37

// PDL launch of a BA kernel on stream `st`
#define BA_LAUNCH(kernel, grid, block, ...)                                                              \
    do {                                                                                                \
        BSFM_CUDA_TRY(launch_pdl(kernel, dim3(grid), dim3(block), st, __VA_ARGS__));                    \
        BSFM_KERNEL_CHECK();                                                                            \
    } while (0)

namespace {

struct Timing {
    float ms[6] = {0, 0, 0, 0, 0, 0};
    int iterations = 0;
    int launches = 0;
};
thread_local Timing g_timing;

struct PhaseTimer {
    // accumulates device time per phase with event pairs; cheap (events only) and optional
    cudaStream_t st;
    bool on;
    std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> spans;
    std::vector<cudaEvent_t> pool;
    PhaseTimer(cudaStream_t s, bool enable) : st(s), on(enable) {}
    ~PhaseTimer() { for (auto e : pool) cudaEventDestroy(e); }
    cudaEvent_t get() { cudaEvent_t e; cudaEventCreate(&e); pool.push_back(e); return e; }
    void begin(int phase) { if (!on) return; cudaEvent_t a = get(), b = get(); cudaEventRecord(a, st); spans.push_back({phase, {a, b}}); }
    void end() { if (!on) return; cudaEventRecord(spans.back().second.second, st); }
    void collect(float *ms) {
        if (!on) return;
        for (auto &s : spans) { float t = 0; cudaEventElapsedTime(&t, s.second.first, s.second.second); ms[s.first] += t; }
    }
};

// BSFM_BA_HOST_TIMING=1: wall-clock marks of the host path (stderr), to see where an end-to-end call spends its time
struct HostMarks {
    bool on = getenv("BSFM_BA_HOST_TIMING") != nullptr;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now(), last = t0;
    void mark(const char *what)
    {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[ba host] %-28s +%8.3f ms  (%8.3f ms)\n", what, std::chrono::duration<double, std::milli>(now - last).count(),
                std::chrono::duration<double, std::milli>(now - t0).count());
        last = now;
    }
};

// stream, events and the pinned scalar blocks are created once per thread and device and reused: driver
// calls that allocate (cudaMallocHost, cudaStreamCreate, ...) serialise on a global lock and cost more than
// an LM iteration of the 50-camera configuration
// Point constraints that are on the device already, in the layout of Problem::pt_constrained / pt_constraints / pt_weights
struct DevicePointConstraints { const char *constrained; const double *constraints, *weights; };

struct SolverCtx { int device = -1; cudaStream_t st = nullptr; cudaEvent_t ev_begin = nullptr, ev_end = nullptr; Scalars *h_sc = nullptr; double *h_mu = nullptr; };
int solver_ctx(SolverCtx **out)
{
    static thread_local SolverCtx ctx;
    int dev = 0;
    BSFM_CUDA_TRY(cudaGetDevice(&dev));
    if (ctx.device != dev) {
        if (ctx.st) { cudaStreamDestroy(ctx.st); cudaEventDestroy(ctx.ev_begin); cudaEventDestroy(ctx.ev_end); cudaFreeHost(ctx.h_sc); cudaFreeHost(ctx.h_mu); ctx = SolverCtx(); }
        BSFM_CUDA_TRY(cudaStreamCreateWithFlags(&ctx.st, cudaStreamNonBlocking));
        BSFM_CUDA_TRY(cudaEventCreate(&ctx.ev_begin));
        BSFM_CUDA_TRY(cudaEventCreate(&ctx.ev_end));
        BSFM_CUDA_TRY(cudaMallocHost(&ctx.h_sc, sizeof(Scalars)));
        BSFM_CUDA_TRY(cudaMallocHost(&ctx.h_mu, sizeof(double)));
        ctx.device = dev;
    }
    *out = &ctx;
    return BSFM_OK;
}

// One LM solve: its device state, and the stages levmar_impl runs in turn.
//   mot == 0 : sba_motstr_levmar_x (cameras + points), p = (a_1..a_m, b_1..b_n)
//   mot == 1 : sba_mot_levmar_x (sba_levmar.c:2090-2690; cameras only), p = (a_1..a_m), the points are read from
//              `fixed_pts` (n x 3; what sfm_project_point3_mot takes from its adata, sfm.c:553-560) and never change
struct Solve {
    const int mot, n, m, mcon, cnp, Sdim, jac_mode;
    const cudaStream_t st;
    const char *const fname;
    DeviceArena D;
    PhaseTimer PT;
    HostMarks HM;
    Problem P{};
    CholBand band;            // envelope plan of S in its factorisation order (apply_camera_order), or none
    int nvis = 0, nobs = 0, useg = 0, red_blocks_obs = 0, red_blocks_var = 0;
    double *d_p, *d_pdp, *d_e, *d_enew, *d_camR_a, *d_camR_b, *d_Lmat, *d_linv, *d_da, *d_mu;
    double *const h_mu;
    Scalars *const h_sc;
    decltype(&residual_kernel<false, false>) k_residual = nullptr;
    decltype(&jacobian_kernel<false, false>) k_jacobian = nullptr;
    // what the controller ends with (info[], sba_levmar.c:2028-2049)
    double mu = 0.0, eab_inf = 0.0, p_eL2 = 0.0, dp_L2 = DBL_MAX, init_p_eL2 = 0.0, max_diag = DBL_MIN;
    int stop = 0, nfev = 0, njev = 0, nlss = 0, itno = 0;
    bool almost_singular = false;

    Solve(int mot_, int n_, int m_, int mcon_, int cnp_, const bsfm_sfm_model_t *model, int jac_mode_, const SolverCtx &ctx)
        : mot(mot_), n(n_), m(m_), mcon(mcon_), cnp(cnp_), Sdim((m_ - mcon_) * cnp_), jac_mode(jac_mode_), st(ctx.st),
          fname(mot_ ? "sba_mot_levmar_x" : "sba_motstr_levmar_x"), D(ctx.st), PT(ctx.st, getenv("BSFM_BA_TIMING") != nullptr),
          h_mu(ctx.h_mu), h_sc(ctx.h_sc)
    {
        P.n = n; P.m = m; P.mcon = mcon;
        P.M.cnp = cnp; P.M.est_focal = model->est_focal_length ? 1 : 0; P.M.undistort = model->undistort ? 1 : 0;
        P.M.explicit_centers = model->explicit_camera_centers ? 1 : 0;
        P.M.focal_idx = P.M.est_focal ? 6 : -1;
        P.M.k_idx = P.M.undistort ? (P.M.est_focal ? 7 : 6) : -1;
        P.M.f_scale = model->f_scale; P.M.k_scale = model->k_scale;
        P.nvars = m * cnp + n * 3;
        P.nlm = mot ? m * cnp : P.nvars;
        P.Sdim = Sdim;
    }
    int visibility(const VisSource &vis, const double *x);
    int upload(const bsfm_sfm_model_t *model, const bsfm_camera_params_t *init_params, bool fisheye, const double *p, const double *fixed_pts,
               int use_constraints, const bsfm_camera_constraints_t *constraints,
               int use_point_constraints, const bsfm_point_constraints_t *point_constraints, const DevicePointConstraints *dev_pc);
    int controller(int itmax, int verbose, const double opts[6], bool any_constraints, double *Vout);
    int export_blocks(double *Vout, double *Sout, double *Uout, double *Wout);

    int read_scalars()
    {
        BSFM_CUDA_TRY(cudaMemcpyAsync(h_sc, P.sc, sizeof(Scalars), cudaMemcpyDeviceToHost, st));
        BSFM_CUDA_TRY(cudaStreamSynchronize(st));
        return BSFM_OK;
    }
    int launch_residual(const double *pp, double *camR, double *eout, const double *eprev, double eps5v)
    {
        const int with_pert = (jac_mode == BSFM_BA_JAC_FD) ? 1 : 0;
        P.camR = camR;
        BA_LAUNCH(cam_prep_kernel, (m + 127) / 128, 128, P, pp, with_pert);
        BA_LAUNCH(k_residual, red_blocks_obs, 256, P, pp, eout, eprev, eps5v);
        return BSFM_OK;
    }
    // Jacobian at p, U_j / ea_j and, with structure, V_i / eb_i (sba_levmar.c:919-1082)
    int normal_equations()
    {
        P.camR = d_camR_a;
        k_jacobian<<<(nvis + 127) / 128, 128, 0, st>>>(P, d_p, jac_mode); ++njev;
        BSFM_KERNEL_CHECK();
        u_partial_kernel<<<m * useg, 128, 0, st>>>(P, d_e, useg);
        BA_LAUNCH(u_final_kernel, m, 96, P, d_p, useg);
        if (!mot) BA_LAUNCH(v_kernel, (n + 127) / 128, 128, P, d_p, d_e);
        return BSFM_OK;
    }
    // S and E of the Schur complement at the damping term in d_mu (sba_levmar.c:1170-1339); zero_S first clears S, whose
    // blocks of camera pairs without a common point the Schur pass does not write
    int schur(bool zero_S)
    {
        if (zero_S) BA_LAUNCH(zero_kernel, std::min(1024, (int) (((size_t) Sdim * Sdim + 255) / 256)), 256, P.S, (size_t) Sdim * Sdim);
        BA_LAUNCH(schur_partial_kernel, (P.nchunks * 32 + 127) / 128, 128, P);
        BA_LAUNCH(schur_final_kernel, (P.nblocks * 32 + 127) / 128, 128, P);
        return BSFM_OK;
    }
};

// visibility -> CRS and the camera-major permutation (sba_levmar.c:652-663), measurements
int Solve::visibility(const VisSource &vis, const double *x)
{
    Visibility V;
    if (vis.built) V = *vis.built;
    else TRY(build_visibility(vis, n, m, st, D, V));
    nvis = V.nvis;
    P.nvis = nvis;
    nobs = nvis * 2;
    if (nobs < P.nlm) {   // sba_levmar.c:647-650, :2235-2238
        fprintf(stderr, "SBA: %s() cannot solve a problem with fewer measurements [%d] than unknowns [%d]\n", fname, nobs, P.nlm);
        set_error("fewer measurements [%d] than unknowns [%d]", nobs, P.nlm);
        return SBA_ERROR_RC;
    }
    P.rowptr = V.rowptr; P.obs_cam = V.obs_cam; P.obs_pt = V.obs_pt; P.cam_ptr = V.cam_ptr; P.cam_obs = V.cam_obs;
    return D.upload(&P.x, x, (size_t) nobs);
}

// model, calibrated cameras, fisheye cameras, constraints, work arrays and the initial parameters
int Solve::upload(const bsfm_sfm_model_t *model, const bsfm_camera_params_t *init_params, bool fisheye, const double *p, const double *fixed_pts,
                  int use_constraints, const bsfm_camera_constraints_t *constraints,
                  int use_point_constraints, const bsfm_point_constraints_t *point_constraints, const DevicePointConstraints *dev_pc)
{
    TRY(D.upload(&P.R_init, model->R_init, (size_t) m * 9));
    if (model->f_fixed) TRY(D.upload(&P.f_fixed, model->f_fixed, (size_t) m));
    else { double *d; TRY(D.alloc(&d, (size_t) m)); BSFM_CUDA_TRY(cudaMemsetAsync(d, 0, (size_t) m * sizeof(double), st)); P.f_fixed = d; }
    // calibrated cameras (sfm.c:339-357): the table exists only when one is present, and selects the KI kernels
    std::vector<CamIntrinsics> h_intr;
    if (init_params) {
        bool any_known = false;
        for (int j = 0; j < m && !any_known; j++) any_known = init_params[j].known_intrinsics != 0;
        if (any_known) {
            h_intr.resize(m);
            for (int j = 0; j < m; j++) h_intr[j] = cam_intrinsics(init_params[j]);
            TRY(D.upload(&P.intr, h_intr.data(), (size_t) m));
        }
    }
    // the fisheye projection (sfm_project_point2_fisheye, sfm.c:448-492): its table exists only when the call asks for it,
    // and selects the FE kernels
    std::vector<CamFisheye> h_fe;
    if (fisheye) {
        h_fe.resize(m);
        for (int j = 0; j < m; j++) h_fe[j] = cam_fisheye(init_params[j]);
        TRY(D.upload(&P.fe, h_fe.data(), (size_t) m));
    }
    if (P.fe) {
        k_residual = P.intr ? residual_kernel<true, true> : residual_kernel<false, true>;
        k_jacobian = P.intr ? jacobian_kernel<true, true> : jacobian_kernel<false, true>;
    } else {
        k_residual = P.intr ? residual_kernel<true, false> : residual_kernel<false, false>;
        k_jacobian = P.intr ? jacobian_kernel<true, false> : jacobian_kernel<false, false>;
    }
    std::vector<char> h_cc; std::vector<double> h_cv, h_cw;
    if (use_constraints) {
        if (!constraints) { set_error("use_constraints set but constraints == NULL"); return BSFM_ERR_ARG; }
        h_cc.resize((size_t) m * cnp); h_cv.resize((size_t) m * cnp); h_cw.resize((size_t) m * cnp);
        for (int j = 0; j < m; j++)
            for (int q = 0; q < cnp; q++) {
                h_cc[(size_t) j * cnp + q] = constraints[j].constrained[q] ? 1 : 0;
                h_cv[(size_t) j * cnp + q] = constraints[j].constraints[q];
                h_cw[(size_t) j * cnp + q] = constraints[j].weights[q];
            }
        TRY(D.upload(&P.cam_constrained, h_cc.data(), h_cc.size()));
        TRY(D.upload(&P.cam_constraints, h_cv.data(), h_cv.size()));
        TRY(D.upload(&P.cam_weights, h_cw.data(), h_cw.size()));
    }
    std::vector<char> h_pc; std::vector<double> h_pv, h_pw;
    if (use_point_constraints && dev_pc) {
        P.pt_constrained = dev_pc->constrained; P.pt_constraints = dev_pc->constraints; P.pt_weights = dev_pc->weights;
    } else if (use_point_constraints) {
        if (!point_constraints) { set_error("use_point_constraints set but point_constraints == NULL"); return BSFM_ERR_ARG; }
        h_pc.resize(n); h_pv.resize((size_t) n * 3); h_pw.resize(n);
        for (int i = 0; i < n; i++) {
            h_pc[i] = point_constraints[i].constrained ? 1 : 0;
            for (int q = 0; q < 3; q++) h_pv[(size_t) i * 3 + q] = point_constraints[i].constraints[q];
            h_pw[i] = point_constraints[i].weight;
        }
        TRY(D.upload(&P.pt_constrained, h_pc.data(), h_pc.size()));
        TRY(D.upload(&P.pt_constraints, h_pv.data(), h_pv.size()));
        TRY(D.upload(&P.pt_weights, h_pw.data(), h_pw.size()));
    }

    // work arrays
    TRY(D.alloc(&d_p, (size_t) P.nvars)); TRY(D.alloc(&d_pdp, (size_t) P.nvars));
    TRY(D.alloc(&d_e, (size_t) nobs)); TRY(D.alloc(&d_enew, (size_t) nobs));
    TRY(D.alloc(&d_camR_a, (size_t) m * 36)); TRY(D.alloc(&d_camR_b, (size_t) m * 36));
    TRY(D.alloc(&P.jacA, (size_t) nvis * 2 * cnp)); TRY(D.alloc(&P.jacB, (size_t) nvis * 6));
    TRY(D.alloc(&P.W, (size_t) nvis * cnp * 3));
    TRY(D.alloc(&P.U, (size_t) m * cnp * cnp)); TRY(D.alloc(&P.V, (size_t) n * 9)); TRY(D.alloc(&P.Vinv, (size_t) n * 9));
    TRY(D.alloc(&P.eab, (size_t) P.nvars)); TRY(D.alloc(&P.dp, (size_t) P.nvars));
    TRY(D.alloc(&P.S, ((size_t) Sdim + 1) * Sdim));
    P.E = P.S + (size_t) Sdim * Sdim;      // RHS lives in matrix row Sdim (see ba_chol.cu)
    TRY(D.alloc(&d_Lmat, ((size_t) Sdim + 1) * Sdim));   // Cholesky factor (out of place)
    TRY(D.alloc(&d_linv, chol_ws_doubles(Sdim))); TRY(D.alloc(&d_da, (size_t) Sdim));
    red_blocks_obs = (nvis + 255) / 256; red_blocks_var = (P.nvars + 255) / 256;
    TRY(D.alloc(&P.partial, (size_t) 3 * std::max(red_blocks_obs, red_blocks_var) + 8));
    useg = std::max(1, std::min(32, (nvis / m + 1023) / 1024));   // ~1024 observations per U-accumulation CTA
    TRY(D.alloc(&P.u_part, (size_t) m * useg * 54));
    TRY(D.alloc(&P.ticket, 4));
    BSFM_CUDA_TRY(cudaMemsetAsync(P.ticket, 0, 4 * sizeof(unsigned int), st));
    TRY(D.alloc(&P.sc, 1));
    BSFM_CUDA_TRY(cudaMemsetAsync(P.sc, 0, sizeof(Scalars), st));
    TRY(D.alloc(&d_mu, 1));
    P.mu = d_mu;
    note_upload(p, (size_t) P.nlm * sizeof(double));
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_p, p, (size_t) P.nlm * sizeof(double), cudaMemcpyDefault, st));
    if (mot) {
        note_upload(fixed_pts, (size_t) n * 3 * sizeof(double));
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_p + P.nlm, fixed_pts, (size_t) n * 3 * sizeof(double), cudaMemcpyDefault, st));
        BSFM_CUDA_TRY(cudaMemsetAsync(P.dp, 0, (size_t) P.nvars * sizeof(double), st));   // the points' increments stay 0
    }
    return BSFM_OK;
}

// ---------------- LM controller (sba_levmar.c:603-2052) ----------------
int Solve::controller(int itmax, int verbose, const double opts[6], bool any_constraints, double *Vout)
{
    const double tau = fabs(opts[0]), eps1 = fabs(opts[1]), eps2 = fabs(opts[2]), eps2_sq = opts[2] * opts[2],
                 eps3_sq = opts[3] * opts[3], eps4_sq = opts[4] * opts[4], eps5 = opts[5];
    double pdp_eL2, p_L2 = 0.0, dF, dL, pen = 0.0;
    int nu = 2, nu2;
    const bool s_dense = (int64_t) P.nblocks == (int64_t) (m - mcon) * (m - mcon + 1) / 2;   // every block written by the Schur pass

    PT.begin(4);
    TRY(launch_residual(d_p, d_camR_a, d_e, nullptr, 0.0)); nfev = 1;
    if (any_constraints) BA_LAUNCH(penalty_kernel, 1, 32, P, d_p);
    PT.end();
    TRY(read_scalars());
    pen = any_constraints ? h_sc->penalty : 0.0;
    p_eL2 = h_sc->e_L2 + pen;    // sba_levmar.c:802-842
    if (verbose) printf(mot ? "initial mot-SBA error %g [%g]\n" : "initial motstr-SBA error %g [%g]\n", p_eL2, p_eL2 / nvis);
    init_p_eL2 = p_eL2;
    if (!std::isfinite(p_eL2)) stop = 7;

    HM.mark("initial residual");
    for (itno = 0; itno < itmax && !stop; ++itno) {
        PT.begin(1);
        TRY(normal_equations());
        if (Vout) BSFM_CUDA_TRY(cudaMemcpyAsync(Vout, P.V, (size_t) n * 9 * sizeof(double), cudaMemcpyDefault, st));   // :1039-1051
        BA_LAUNCH(grad_stats_kernel, red_blocks_var, 256, P, d_p);
        PT.end();
        TRY(read_scalars());
        eab_inf = h_sc->eab_inf; p_L2 = h_sc->p_L2; max_diag = h_sc->max_diag;
        if (any_constraints) pen = h_sc->penalty;

        if (eab_inf <= eps1) { dp_L2 = 0.0; stop = 1; break; }      // :1117-1121
        if (itno == 0) mu = tau * max_diag;                          // :1123-1128

        while (1) {   // damping loop :1131
            BSFM_CUDA_TRY(cudaMemsetAsync(&P.sc->singular_v, 0, 3 * sizeof(int), st));
            *h_mu = mu;
            BSFM_CUDA_TRY(cudaMemcpyAsync(d_mu, h_mu, sizeof(double), cudaMemcpyHostToDevice, st));
            if (mot) {
                // block-diagonal system: (U_j + mu I) da_j = ea_j per camera (sba_levmar.c:2487-2514)
                PT.begin(3);
                BA_LAUNCH(mot_solve_kernel, (m + 63) / 64, 64, P);
                PT.end();
                PT.begin(4);
            } else {
            PT.begin(2);
            BA_LAUNCH(vinv_kernel, (n + 255) / 256, 256, P);
            TRY(schur(!s_dense));   // camera pairs without a common point keep S_jk = 0
            PT.end();
            PT.begin(3);
            TRY(chol_solve(st, P.S, d_Lmat, Sdim, d_linv, d_da, P.sc, &band));
            PT.end();
            PT.begin(4);
            BA_LAUNCH(backsub_kernel, (std::max(n, m * cnp) + 127) / 128, 128, P, d_da);
            }
            BA_LAUNCH(update_kernel, red_blocks_var, 256, P, d_p, d_pdp);
            TRY(launch_residual(d_pdp, d_camR_b, d_enew, d_e, eps5));
            PT.end();
            TRY(read_scalars());

            bool take_moredamping = true;
            if (!mot && h_sc->singular_v) {
                fprintf(stderr, "SBA: singular matrix V*_i in sba_motstr_levmar_x(), increasing damping\n");   // :1156-1161
            } else {
                nlss += mot ? (m - mcon) : 1;      // the motion-only routine counts one system per camera (:2513)
                const bool issolved = !h_sc->chol_fail;
                if (issolved) {
                    dp_L2 = h_sc->dp_L2;
                    if (dp_L2 <= eps2_sq * p_L2) { stop = 2; break; }                              // :1450-1454
                    if (dp_L2 >= (p_L2 + eps2) / SBA_EPSILON_SQ) {                                 // :1456-1462
                        fprintf(stderr, "SBA: the matrix of the augmented normal equations is almost singular in %s(),\n"
                                        "     minimization should be restarted from the current solution with an increased damping term\n", fname);
                        set_error("augmented normal equations almost singular");
                        // the reference leaves through freemem_and_return with the last ACCEPTED p in place (it updates p
                        // in place on every accepted step, sba_levmar.c:1456-1462): fall through to the common tail
                        almost_singular = true;
                        break;
                    }
                    ++nfev;
                    pdp_eL2 = h_sc->e_L2;
                    if (verbose > 1) printf("mean reprojection error (trial) sq %g\n", pdp_eL2 / nvis);
                    if (!std::isfinite(pdp_eL2)) { stop = 7; break; }                              // :1479-1485
                    pdp_eL2 += pen;   // constraint terms evaluated at the OLD p (quirk 7, :1487-1522)
                    dL = h_sc->dL;
                    dF = p_eL2 - pdp_eL2;
                    if (verbose > 1) {
                        printf("\ndamping term %8g, gain ratio %8g, errors %8g / %8g = %g\n", mu, dL != 0.0 ? dF / dL : dF / DBL_EPSILON,
                               p_eL2 / nvis, pdp_eL2 / nvis, p_eL2 / pdp_eL2);
                        printf("pdp_eL2: %0.3f, nvis: %d\n", pdp_eL2, nvis);
                    }
                    if (dL > 0.0 && dF > 0.0) {                                                    // :1543
                        double tmp = (2.0 * dF / dL - 1.0);
                        tmp = 1.0 - tmp * tmp * tmp;
                        mu = mu * ((tmp >= SBA_ONE_THIRD) ? tmp : SBA_ONE_THIRD);
                        nu = 2;
                        const double max_pct_change = h_sc->max_pct;
                        if (!mot) {     // Snavely's stop-8 statistic exists only in the motion+structure routine
                            printf("max_pct_change: %0.3e\n", max_pct_change);                     // :1563 (unconditional)
                            fflush(stdout);
                        }
                        if (pdp_eL2 - 2.0 * sqrt(p_eL2 * pdp_eL2) < (eps4_sq - 1.0) * p_eL2) stop = 4;   // :1567, :2596
                        if (!mot && max_pct_change < eps5 && itno >= 4) { stop = 8; break; }       // :1569-1572 (step discarded)
                        std::swap(d_p, d_pdp); std::swap(d_e, d_enew); std::swap(d_camR_a, d_camR_b);
                        p_eL2 = pdp_eL2;
                        if (any_constraints) BA_LAUNCH(penalty_kernel, 1, 32, P, d_p);
                        take_moredamping = false;
                    }
                }
            }
            if (!take_moredamping) break;
            if (almost_singular) break;
            // moredamping :1584-1597
            mu *= nu;
            nu2 = nu << 1;
            if (nu2 <= nu) {
                fprintf(stderr, "SBA: too many failed attempts to increase the damping factor in %s()! Singular Hessian matrix?\n", fname);
                stop = 6;
                break;
            }
            nu = nu2;
        }
        if (almost_singular) break;
        if (p_eL2 <= eps3_sq) stop = 5;    // :1614
    }
    if (itno >= itmax) stop = 3;
    HM.mark("LM loop");
    return BSFM_OK;
}

// export pass (sba_levmar.c:1633-2026): Jacobian at the final p, U/V/W with constraints, UNDAMPED Schur complement
int Solve::export_blocks(double *Vout, double *Sout, double *Uout, double *Wout)
{
    TRY(normal_equations());
    if (Uout) BSFM_CUDA_TRY(cudaMemcpyAsync(Uout, P.U, (size_t) m * cnp * cnp * sizeof(double), cudaMemcpyDefault, st));
    if (Vout) BSFM_CUDA_TRY(cudaMemcpyAsync(Vout, P.V, (size_t) n * 9 * sizeof(double), cudaMemcpyDefault, st));
    vinv_export_kernel<<<(n + 255) / 256, 256, 0, st>>>(P);
    BSFM_KERNEL_CHECK();
    if (Wout) {
        double *d_wout;
        TRY(D.alloc(&d_wout, (size_t) m * cnp * 3 * (size_t) n));
        BSFM_CUDA_TRY(cudaMemcpyAsync(d_wout, Wout, (size_t) m * cnp * 3 * (size_t) n * sizeof(double), cudaMemcpyDefault, st));   // untouched entries keep the caller's values
        wout_scatter_kernel<<<(nvis + 255) / 256, 256, 0, st>>>(P, d_wout);
        BSFM_KERNEL_CHECK();
        BSFM_CUDA_TRY(cudaMemcpyAsync(Wout, d_wout, (size_t) m * cnp * 3 * (size_t) n * sizeof(double), cudaMemcpyDefault, st));
    }
    *h_mu = 0.0;
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_mu, h_mu, sizeof(double), cudaMemcpyHostToDevice, st));
    P.cam_pos = nullptr;      // S goes out in the caller's camera order, whichever order the solves factored it in
    TRY(schur(true));
    BSFM_CUDA_TRY(cudaMemcpyAsync(Sout, P.S, (size_t) Sdim * Sdim * sizeof(double), cudaMemcpyDefault, st));   // symmetric: transpose == itself (:2017-2025)
    return BSFM_OK;
}

}  // namespace

// Shared implementation of the two LM drivers (mot: see Solve).
// init_params (nullable, m entries): the calibrated-camera fields (known_intrinsics, K_known, k_known) are read.
// fisheye: project with sfm_project_point2_fisheye; init_params is required then, and its fisheye fields are read too.
// dev_pc (nullable): the point constraints as device tables, taken in place of point_constraints.
static int levmar_impl(int mot, const double *fixed_pts, int n, int m, int mcon, const VisSource &vis, double *p, int cnp, int pnp,
                       const double *x, const double *covx, int mnp,
                       const bsfm_sfm_model_t *model, const bsfm_camera_params_t *init_params, int fisheye, int jac_mode,
                       int itmax, int verbose, const double opts[6], double info[10],
                       int use_constraints, const bsfm_camera_constraints_t *constraints,
                       int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                       double *Vout, double *Sout, double *Uout, double *Wout, const DevicePointConstraints *dev_pc = nullptr)
{
    clear_error();
    TRY(require_device());
    if (n <= 0 || m <= 0 || mcon < 0 || mcon >= m || !vis.present() || !p || !x || !model || !opts || (mot && !fixed_pts)) {
        set_error("bsfm_sba_motstr_levmar_model: bad arguments (n=%d m=%d mcon=%d)", n, m, mcon);
        return BSFM_ERR_ARG;
    }
    if (fisheye && !init_params) {
        set_error("bsfm_sba_motstr_levmar_model: the fisheye projection reads init_params, which is NULL");
        return BSFM_ERR_ARG;
    }
    if (pnp != 3 || mnp != 2 || cnp < 6 || cnp > 9 || cnp != 6 + (model->est_focal_length ? 1 : 0) + (model->undistort ? 2 : 0)) {
        set_error("bsfm_sba_motstr_levmar_model: unsupported block sizes cnp=%d pnp=%d mnp=%d for the sfm camera model", cnp, pnp, mnp);
        return BSFM_ERR_UNSUPPORTED;
    }
    if (covx) { set_error("bsfm_sba_motstr_levmar_model: covx != NULL is not supported (Bundler always passes NULL, sfm.c:821)"); return BSFM_ERR_UNSUPPORTED; }
    if ((Sout || Uout || Wout) && mcon != 0) { set_error("bsfm_sba_motstr_levmar_model: Sout/Uout/Wout export assumes mcon == 0 (as the reference does, sba_levmar.c:2017-2022)"); return BSFM_ERR_UNSUPPORTED; }
    if ((int64_t) m * m > 0xffffffffLL) { set_error("too many cameras"); return BSFM_ERR_ARG; }
    {
        const char *jm = getenv("BSFM_BA_JAC");
        if (jm && !strcmp(jm, "analytic")) jac_mode = BSFM_BA_JAC_ANALYTIC;
        if (jm && !strcmp(jm, "fd")) jac_mode = BSFM_BA_JAC_FD;
    }
    const long long launches0 = g_kernel_launches.load();
    SolverCtx *ctx;
    TRY(solver_ctx(&ctx));
    const cudaStream_t st = ctx->st;
    BSFM_CUDA_TRY(cudaEventRecord(ctx->ev_begin, st));
    g_timing = Timing();
    Solve S(mot, n, m, mcon, cnp, model, jac_mode, *ctx);

    S.PT.begin(0);
    TRY(S.visibility(vis, x));
    TRY(build_schur_structure(S.P, st, S.D));
    if (!mot) TRY(apply_camera_order(S.P, cnp, st, S.D, S.band));      // large systems: S in the order that skips most of the factorisation
    S.HM.mark("Schur structure + camera order");
    TRY(S.upload(model, init_params, fisheye != 0, p, fixed_pts, use_constraints, constraints, use_point_constraints, point_constraints, dev_pc));
    S.PT.end();
    S.HM.mark("setup issued");

    TRY(S.controller(itmax, verbose, opts, use_constraints || use_point_constraints, Vout));
    if (Sout) TRY(S.export_blocks(Vout, Sout, Uout, Wout));

    BSFM_CUDA_TRY(cudaMemcpyAsync(p, S.d_p, (size_t) S.P.nlm * sizeof(double), cudaMemcpyDefault, st));
    BSFM_CUDA_TRY(cudaEventRecord(ctx->ev_end, st));
    BSFM_CUDA_TRY(cudaStreamSynchronize(st));
    if (info) {   // :2028-2049
        info[0] = S.init_p_eL2; info[1] = S.p_eL2; info[2] = S.eab_inf; info[3] = S.dp_L2;
        info[4] = S.mu / S.max_diag; info[5] = S.itno; info[6] = S.stop; info[7] = S.nfev; info[8] = S.njev; info[9] = S.nlss;
    }
    cudaEventElapsedTime(&g_timing.ms[5], ctx->ev_begin, ctx->ev_end);
    S.PT.collect(g_timing.ms);
    g_timing.iterations = S.itno;
    g_timing.launches = (int) (g_kernel_launches.load() - launches0);
    S.HM.mark("copy back + teardown");
    return (S.stop != 7 && !S.almost_singular) ? S.itno : SBA_ERROR_RC;
}

extern "C" int bsfm_sba_motstr_levmar_model_ki(int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                                               const double *x, const double *covx, int mnp,
                                               const bsfm_sfm_model_t *model, int jac_mode,
                                               int itmax, int verbose, const double opts[6], double info[10],
                                               int use_constraints, const bsfm_camera_constraints_t *constraints,
                                               int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                                               double *Vout, double *Sout, double *Uout, double *Wout,
                                               const bsfm_camera_params_t *init_params)
{
    return levmar_impl(0, nullptr, n, m, mcon, VisSource::mask(vmask), p, cnp, pnp, x, covx, mnp, model, init_params, 0, jac_mode, itmax, verbose,
                       opts, info, use_constraints, constraints, use_point_constraints, point_constraints, Vout, Sout, Uout, Wout);
}

extern "C" int bsfm_sba_motstr_levmar_model_fe(int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                                               const double *x, const double *covx, int mnp,
                                               const bsfm_sfm_model_t *model, int jac_mode,
                                               int itmax, int verbose, const double opts[6], double info[10],
                                               int use_constraints, const bsfm_camera_constraints_t *constraints,
                                               int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                                               double *Vout, double *Sout, double *Uout, double *Wout,
                                               const bsfm_camera_params_t *init_params, int optimize_for_fisheye)
{
    return levmar_impl(0, nullptr, n, m, mcon, VisSource::mask(vmask), p, cnp, pnp, x, covx, mnp, model, init_params, optimize_for_fisheye,
                       jac_mode, itmax, verbose, opts, info, use_constraints, constraints, use_point_constraints, point_constraints,
                       Vout, Sout, Uout, Wout);
}

extern "C" int bsfm_sba_motstr_levmar_model(int n, int m, int mcon, const char *vmask, double *p, int cnp, int pnp,
                                            const double *x, const double *covx, int mnp,
                                            const bsfm_sfm_model_t *model, int jac_mode,
                                            int itmax, int verbose, const double opts[6], double info[10],
                                            int use_constraints, const bsfm_camera_constraints_t *constraints,
                                            int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
                                            double *Vout, double *Sout, double *Uout, double *Wout)
{
    return bsfm_sba_motstr_levmar_model_ki(n, m, mcon, vmask, p, cnp, pnp, x, covx, mnp, model, jac_mode, itmax, verbose, opts, info,
                                           use_constraints, constraints, use_point_constraints, point_constraints, Vout, Sout, Uout, Wout,
                                           nullptr);
}

extern "C" int bsfm_sba_mot_levmar_model_ki(int n, int m, int mcon, const char *vmask, double *p, int cnp,
                                            const double *x, const double *covx, int mnp,
                                            const bsfm_sfm_model_t *model, const double *points, int jac_mode,
                                            int itmax, int verbose, const double opts[6], double info[10],
                                            int use_constraints, const bsfm_camera_constraints_t *constraints,
                                            const bsfm_camera_params_t *init_params)
{
    return levmar_impl(1, points, n, m, mcon, VisSource::mask(vmask), p, cnp, 3, x, covx, mnp, model, init_params, 0, jac_mode, itmax, verbose,
                       opts, info, use_constraints, constraints, 0, nullptr, nullptr, nullptr, nullptr, nullptr);
}

extern "C" int bsfm_sba_mot_levmar_model_fe(int n, int m, int mcon, const char *vmask, double *p, int cnp,
                                            const double *x, const double *covx, int mnp,
                                            const bsfm_sfm_model_t *model, const double *points, int jac_mode,
                                            int itmax, int verbose, const double opts[6], double info[10],
                                            int use_constraints, const bsfm_camera_constraints_t *constraints,
                                            const bsfm_camera_params_t *init_params, int optimize_for_fisheye)
{
    return levmar_impl(1, points, n, m, mcon, VisSource::mask(vmask), p, cnp, 3, x, covx, mnp, model, init_params, optimize_for_fisheye,
                       jac_mode, itmax, verbose, opts, info, use_constraints, constraints, 0, nullptr, nullptr, nullptr, nullptr, nullptr);
}

extern "C" int bsfm_sba_mot_levmar_model(int n, int m, int mcon, const char *vmask, double *p, int cnp,
                                         const double *x, const double *covx, int mnp,
                                         const bsfm_sfm_model_t *model, const double *points, int jac_mode,
                                         int itmax, int verbose, const double opts[6], double info[10],
                                         int use_constraints, const bsfm_camera_constraints_t *constraints)
{
    return bsfm_sba_mot_levmar_model_ki(n, m, mcon, vmask, p, cnp, x, covx, mnp, model, points, jac_mode, itmax, verbose, opts, info,
                                        use_constraints, constraints, nullptr);
}

// == sba_Axb_Chol, lib/sba-1.5/sba_lapack.c:374-485: x = A^-1 B for symmetric positive definite A (m x m).
// A, B, x may be host or device pointers; A and B are never modified (the reference overwrites them when
// iscolmaj == 1; a symmetric matrix reads the same in both orders, so the flag changes nothing else here).
// Returns 1 on success, 0 when a leading minor is not positive definite (the reference's return values), < 0 on a
// library error.  `reps` > 1 repeats the factorisation on a fresh copy of A; *ms_out = device time per repetition.
// `out` (bsfm_sba_Axb_Chol_factor): what the factorisation left behind, copied out whether or not it succeeded.
struct CholOutputs {
    double *L, *linv, *xinv;
    int *fail_code;
};
// first_col (bsfm_sba_Axb_Chol_factor_env): the caller's row envelope; a large system whose plan fits takes the band path
static int axb_chol_impl(const double *A, const double *B, double *x, int m, int reps, float *ms_out, const CholOutputs *out = nullptr,
                         const int32_t *first_col = nullptr)
{
    clear_error();
    TRY(require_device());
    if (!A || !B || !x || m <= 0 || reps < 1) { set_error("bsfm_sba_Axb_Chol: bad arguments"); return BSFM_ERR_ARG; }
    if (first_col)
        for (int i = 0; i < m; i++)
            if (first_col[i] < 0 || first_col[i] > i) { set_error("bsfm_sba_Axb_Chol_factor_env: first_col[%d] = %d is not in [0, %d]", i, first_col[i], i); return BSFM_ERR_ARG; }
    cudaStream_t st;
    BSFM_CUDA_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    struct StreamGuard { cudaStream_t s; ~StreamGuard() { cudaStreamDestroy(s); } } guard{st};
    DeviceArena D(st);   // after the guard: the arena waits for the stream and returns its blocks before the stream goes
    CholBand band;
    if (first_col && m > CHOL_LARGE_MIN) {
        int dev = 0, sms = 0;
        BSFM_CUDA_TRY(cudaGetDevice(&dev));
        BSFM_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        CholBandPlan plan;
        chol_band_plan(m, first_col, sms - 1, plan);
        if (plan.fits) TRY(upload_band_plan(plan, D, band));
    }
    double *d_src, *d_A, *d_L, *d_linv, *d_x; Scalars *d_sc;
    const size_t mm = (size_t) m * m;
    TRY(D.alloc(&d_src, mm + m)); TRY(D.alloc(&d_A, mm + m)); TRY(D.alloc(&d_L, mm + m));
    TRY(D.alloc(&d_linv, chol_ws_doubles(m))); TRY(D.alloc(&d_x, (size_t) m)); TRY(D.alloc(&d_sc, 1));
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_src, A, mm * sizeof(double), cudaMemcpyDefault, st));
    BSFM_CUDA_TRY(cudaMemcpyAsync(d_src + mm, B, (size_t) m * sizeof(double), cudaMemcpyDefault, st));
    BSFM_CUDA_TRY(cudaMemsetAsync(d_sc, 0, sizeof(Scalars), st));
    // every path writes the lower triangle of Lmat only: zeroed first, its upper part comes back as the zeros it was given
    if (out && out->L) BSFM_CUDA_TRY(cudaMemsetAsync(d_L, 0, (mm + m) * sizeof(double), st));
    cudaEvent_t e0, e1;
    BSFM_CUDA_TRY(cudaEventCreate(&e0)); BSFM_CUDA_TRY(cudaEventCreate(&e1));
    float total = 0.f;
    int rc = BSFM_OK;
    for (int r = 0; r < reps && rc == BSFM_OK; r++) {
        cudaMemcpyAsync(d_A, d_src, (mm + m) * sizeof(double), cudaMemcpyDeviceToDevice, st);
        cudaEventRecord(e0, st);
        rc = chol_solve(st, d_A, d_L, m, d_linv, d_x, d_sc, &band);
        cudaEventRecord(e1, st);
        if (cudaStreamSynchronize(st) != cudaSuccess) { set_error("bsfm_sba_Axb_Chol: %s", cudaGetErrorString(cudaGetLastError())); rc = BSFM_ERR_CUDA; }
        float t = 0.f; cudaEventElapsedTime(&t, e0, e1); total += t;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (rc != BSFM_OK) return rc;
    if (ms_out) *ms_out = total / reps;
    Scalars h;
    BSFM_CUDA_TRY(cudaMemcpy(&h, d_sc, sizeof h, cudaMemcpyDeviceToHost));
    if (out) {
        if (out->fail_code) *out->fail_code = h.chol_fail;
        if (out->L) BSFM_CUDA_TRY(cudaMemcpy(out->L, d_L, mm * sizeof(double), cudaMemcpyDefault));
        const size_t nlinv = (size_t) ((m + LNB - 1) / LNB) * LNB * LNB;
        if (out->linv) BSFM_CUDA_TRY(cudaMemcpy(out->linv, d_linv, nlinv * sizeof(double), cudaMemcpyDefault));
        // the large path (ba_chol_large.cu) keeps the panel inverses right behind the 32 x 32 ones
        if (out->xinv && m > CHOL_LARGE_MIN)
            BSFM_CUDA_TRY(cudaMemcpy(out->xinv, d_linv + nlinv, (size_t) ((m + LNBO - 1) / LNBO) * LNBO * LNBO * sizeof(double), cudaMemcpyDefault));
    }
    if (h.chol_fail) return 0;
    BSFM_CUDA_TRY(cudaMemcpy(x, d_x, (size_t) m * sizeof(double), cudaMemcpyDefault));
    return 1;
}
extern "C" int bsfm_sba_Axb_Chol_factor(const double *A, const double *B, double *x, int m, double *L, double *linv, double *xinv, int *fail_code)
{
    const CholOutputs out = {L, linv, xinv, fail_code};
    return axb_chol_impl(A, B, x, m, 1, nullptr, &out);
}
extern "C" int bsfm_sba_Axb_Chol_factor_env(const double *A, const double *B, double *x, int m, const int32_t *first_col, double *L, double *linv,
                                            double *xinv, int *fail_code)
{
    if (!first_col) { clear_error(); set_error("bsfm_sba_Axb_Chol_factor_env: first_col is NULL"); return BSFM_ERR_ARG; }
    const CholOutputs out = {L, linv, xinv, fail_code};
    return axb_chol_impl(A, B, x, m, 1, nullptr, &out, first_col);
}
extern "C" int bsfm_sba_Axb_Chol(const double *A, const double *B, double *x, int m, int iscolmaj)
{
    (void) iscolmaj;
    return axb_chol_impl(A, B, x, m, 1, nullptr);
}
extern "C" int bsfm_sba_Axb_Chol_timed(const double *A, const double *B, double *x, int m, int reps, float *ms_per_solve)
{
    return axb_chol_impl(A, B, x, m, reps, ms_per_solve);
}

extern "C" int bsfm_ba_last_timing(float ms[6], int *iterations, int *launches)
{
    if (ms) for (int q = 0; q < 6; q++) ms[q] = g_timing.ms[q];
    if (iterations) *iterations = g_timing.iterations;
    if (launches) *launches = g_timing.launches;
    return BSFM_OK;
}

// run_sfm's handling of the cameras (lib/sfm-driver/sfm.c:652-696 packing, :721-754 constraints, :876-929 unpacking) and
// its call of the solver (:705-714 options, :814-856), shared by run_sfm_impl and the outlier loop
struct SfmCameras {
    static constexpr double f_scale = 0.001, k_scale = 5.0;     // sfm.c:634-635 (TEST_FOCAL)
    const int m, cnp, est_focal_length, undistort;
    std::vector<double> R_init, f_fixed;
    std::vector<bsfm_camera_constraints_t> constraints;
    std::vector<char> cc; std::vector<double> cv, cw;
    bsfm_sfm_model_t model;

    SfmCameras(int num_cameras, int est_focal, int undist, int explicit_camera_centers)
        : m(num_cameras), cnp((est_focal ? 7 : 6) + (undist ? 2 : 0)), est_focal_length(est_focal), undistort(undist),
          R_init((size_t) num_cameras * 9), f_fixed(num_cameras)
    {
        model.est_focal_length = est_focal_length; model.undistort = undistort; model.explicit_camera_centers = explicit_camera_centers;
        model.f_scale = f_scale; model.k_scale = k_scale; model.R_init = R_init.data(); model.f_fixed = f_fixed.data();
    }
    // cameras -> params (m * cnp), R_init, f_fixed and, with use_constraints, the scaled constraints
    void pack(bsfm_camera_params_t *init_camera_params, double *params, int use_constraints)
    {
        for (int j = 0; j < m; j++) {                      // sfm.c:652-696
            int c;
            init_camera_params[j].f_scale = f_scale;
            init_camera_params[j].k_scale = k_scale;
            params[(size_t) cnp * j + 0] = init_camera_params[j].t[0];
            params[(size_t) cnp * j + 1] = init_camera_params[j].t[1];
            params[(size_t) cnp * j + 2] = init_camera_params[j].t[2];
            params[(size_t) cnp * j + 3] = 0.0; params[(size_t) cnp * j + 4] = 0.0; params[(size_t) cnp * j + 5] = 0.0;
            if (est_focal_length) { params[(size_t) cnp * j + 6] = init_camera_params[j].f * init_camera_params[j].f_scale; c = 7; }
            else c = 6;
            if (undistort) {
                const double scale = init_camera_params[j].k_scale;
                params[(size_t) cnp * j + c] = init_camera_params[j].k[0] * scale;
                params[(size_t) cnp * j + c + 1] = init_camera_params[j].k[1] * scale;
            }
            memcpy(&R_init[(size_t) j * 9], init_camera_params[j].R, 9 * sizeof(double));
            f_fixed[j] = init_camera_params[j].f;
        }
        if (!use_constraints) return;                      // sfm.c:721-754
        constraints.resize(m);
        cc.resize((size_t) m * cnp); cv.resize((size_t) m * cnp); cw.resize((size_t) m * cnp);
        for (int i = 0; i < m; i++) {
            char *c0 = &cc[(size_t) i * cnp]; double *v0 = &cv[(size_t) i * cnp]; double *w0 = &cw[(size_t) i * cnp];
            memcpy(c0, init_camera_params[i].constrained, cnp);
            memcpy(v0, init_camera_params[i].constraints, cnp * sizeof(double));
            memcpy(w0, init_camera_params[i].weights, cnp * sizeof(double));
            if (est_focal_length) { v0[6] *= f_scale; w0[6] *= (1.0 / (f_scale * f_scale)); }
            if (undistort) {
                // NOTE the reference indexes 7 and 8 unconditionally (sfm.c:745-751), i.e. it assumes est_focal_length;
                // with est_focal_length == 0 that would be out of bounds for cnp == 8, so the k pair at 6,7 is used there.
                const int k0 = est_focal_length ? 7 : 6;
                v0[k0] *= k_scale; w0[k0] *= (1.0 / (k_scale * k_scale));
                v0[k0 + 1] *= k_scale; w0[k0 + 1] *= (1.0 / (k_scale * k_scale));
            }
            constraints[i].constrained = c0; constraints[i].constraints = v0; constraints[i].weights = w0;
        }
    }
    // a BSFM_ERR_* of the solver: nothing was solved; the caller's cameras get back the scale fields pack() set to 0.001 / 5
    void restore_scales(bsfm_camera_params_t *init_camera_params) const
    {
        for (int j = 0; j < m; j++) { init_camera_params[j].f_scale = 1.0; init_camera_params[j].k_scale = 1.0; }
    }
    // host-side rot_update for the unpacking (sfm.c:876-929); same arithmetic as the device version
    void unpack(const double *params, bsfm_camera_params_t *init_camera_params) const
    {
        for (int j = 0; j < m; j++) {
            const double *dt = &params[(size_t) cnp * j + 0];
            const double *w = &params[(size_t) cnp * j + 3];
            int c;
            init_camera_params[j].t[0] = dt[0]; init_camera_params[j].t[1] = dt[1]; init_camera_params[j].t[2] = dt[2];
            {
                double *R = init_camera_params[j].R, Rnew[9];
                const double theta = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
                if (theta != 0.0) {
                    const double n0 = w[0] / theta, n1 = w[1] / theta, n2 = w[2] / theta;
                    const double nx[9] = {0.0, -n2, n1, n2, 0.0, -n0, -n1, n0, 0.0};
                    double nxsq[9], dR[9];
                    for (int r = 0; r < 3; r++) for (int cc2 = 0; cc2 < 3; cc2++)
                        nxsq[3 * r + cc2] = nx[3 * r] * nx[cc2] + nx[3 * r + 1] * nx[3 + cc2] + nx[3 * r + 2] * nx[6 + cc2];
                    const double sinth = sin(theta), costh = cos(theta);
                    for (int q = 0; q < 9; q++) dR[q] = (((q % 4 == 0) ? 1.0 : 0.0) + nx[q] * sinth) + nxsq[q] * (1.0 - costh);
                    for (int r = 0; r < 3; r++) for (int cc2 = 0; cc2 < 3; cc2++)
                        Rnew[3 * r + cc2] = dR[3 * r] * R[cc2] + dR[3 * r + 1] * R[3 + cc2] + dR[3 * r + 2] * R[6 + cc2];
                    memcpy(R, Rnew, sizeof Rnew);
                }
            }
            if (est_focal_length) { c = 7; init_camera_params[j].f = params[(size_t) cnp * j + 6] / init_camera_params[j].f_scale; }
            else c = 6;
            if (undistort) {
                const double scale = init_camera_params[j].k_scale;
                init_camera_params[j].k[0] = params[(size_t) cnp * j + c] / scale;
                init_camera_params[j].k[1] = params[(size_t) cnp * j + c + 1] / scale;
            }
            init_camera_params[j].f_scale = 1.0;
            init_camera_params[j].k_scale = 1.0;
        }
    }
    // the solve of sfm.c:814-856 on packed parameters p = (cameras, points), host or device; prints run_sfm's two lines
    // (:872-873) unless the solver returned a BSFM_ERR_*, which is passed on
    int solve(int num_pts, int ncons, const VisSource &vis, double *p, const double *projections, const bsfm_camera_params_t *init_camera_params,
              int use_constraints, int use_point_constraints, const bsfm_point_constraints_t *point_constraints,
              const DevicePointConstraints *dev_pc, int fix_points, int optimize_for_fisheye, double eps2,
              double *Vout, double *Sout, double *Uout, double *Wout, double info[10])
    {
        const double opts[6] = {1.0e-3, 1.0e-10, eps2, 1.0e-12, 0.0, 4.0e-2};   // sfm.c:705-714
        const char *verb_env = getenv("BSFM_BA_VERBOSE");
        const int verbosity = verb_env ? atoi(verb_env) : 3;          // VERBOSITY 3, MAX_ITERS 150 (sfm.c:814-815)
        const size_t num_camera_params = (size_t) cnp * m;
        int rc;
        if (fix_points)     // sfm.c:843-849: motion-only BA, the points come from init_pts and stay as they are
            rc = levmar_impl(1, p + num_camera_params, num_pts, m, ncons, vis, p, cnp, 3, projections,
                             nullptr, 2, &model, init_camera_params, optimize_for_fisheye, BSFM_BA_JAC_FD, 150, verbosity, opts, info,
                             use_constraints, use_constraints ? constraints.data() : nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr);
        else
            rc = levmar_impl(0, nullptr, num_pts, m, ncons, vis, p, cnp, 3, projections, nullptr, 2,
                             &model, init_camera_params, optimize_for_fisheye, BSFM_BA_JAC_FD, 150, verbosity, opts, info,
                             use_constraints, use_constraints ? constraints.data() : nullptr,
                             use_point_constraints, point_constraints, Vout, Sout, Uout, Wout, dev_pc);
        if (rc < -1) return rc;
        printf("[run_sfm] Number of iterations: %d\n", (int) info[5]);   // sfm.c:872-873
        printf("info[6] = %0.3f\n", info[6]);
        return BSFM_OK;
    }
};

// the point constraints of sfm.c:757-781 for points [0, num_pts)
static void sfm_point_constraints(const bsfm_v3_t *pt_constraints, double pt_constraint_weight, int num_pts, std::vector<bsfm_point_constraints_t> &out)
{
    out.resize(num_pts);
    for (int i = 0; i < num_pts; i++) {
        const double *q = pt_constraints[i].p;
        if (q[0] == 0.0 && q[1] == 0.0 && q[2] == 0.0) {
            out[i].constrained = 0;
            out[i].constraints[0] = out[i].constraints[1] = out[i].constraints[2] = 0.0;
            out[i].weight = 0.0;
        } else {
            out[i].constrained = 1;
            out[i].weight = pt_constraint_weight;
            out[i].constraints[0] = q[0]; out[i].constraints[1] = q[1]; out[i].constraints[2] = q[2];
        }
    }
}

// == run_sfm, lib/sfm-driver/sfm.c:592-1003, on either visibility source (bsfm_run_sfm, bsfm_run_sfm_crs)
static int run_sfm_impl(int num_pts, int num_cameras, int ncons, const VisSource &vis, double *projections,
                        int est_focal_length, int const_focal_length, int undistort, int explicit_camera_centers,
                        bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                        int use_constraints, int use_point_constraints, bsfm_v3_t *pt_constraints,
                        double pt_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                        double *Vout, double *Sout, double *Uout, double *Wout, double *info_out, bool fisheye_entry)
{
    clear_error();
    if (fix_points && (Vout || Sout || Uout || Wout)) { set_error("bsfm_run_sfm: fix_points=1 has no V/S/U/W export (nor has the reference, sfm.c:843-856)"); return BSFM_ERR_UNSUPPORTED; }
    if (optimize_for_fisheye && !fisheye_entry) { set_error("bsfm_run_sfm: optimize_for_fisheye=1 is outside this entry; bsfm_run_sfm_fe runs it"); return BSFM_ERR_UNSUPPORTED; }
    if (est_focal_length && const_focal_length) { set_error("bsfm_run_sfm: const_focal_length is not implemented (nor in the reference, sfm.c:518-521)"); return BSFM_ERR_UNSUPPORTED; }
    if (num_pts <= 0 || num_cameras <= 0 || !vis.present() || !projections || !init_camera_params || !init_pts) {
        set_error("bsfm_run_sfm: bad arguments"); return BSFM_ERR_ARG;
    }

    SfmCameras C(num_cameras, est_focal_length, undistort, explicit_camera_centers);
    const int cnp = C.cnp;
    const int num_camera_params = cnp * num_cameras;
    const size_t num_params = (size_t) num_camera_params + 3 * (size_t) num_pts;
    std::vector<double> params(num_params);
    C.pack(init_camera_params, params.data(), use_constraints);
    for (int i = 0; i < num_pts; i++)                            // sfm.c:698-703
        for (int q = 0; q < 3; q++) params[(size_t) num_camera_params + 3 * (size_t) i + q] = init_pts[i].p[q];
    double info[10] = {0};
    std::vector<bsfm_point_constraints_t> point_constraints;
    if (use_point_constraints) {                                 // sfm.c:757-781
        if (!pt_constraints) { set_error("bsfm_run_sfm: use_point_constraints without points_constraints"); return BSFM_ERR_ARG; }
        sfm_point_constraints(pt_constraints, pt_constraint_weight, num_pts, point_constraints);
    }
    const int rc = C.solve(num_pts, ncons, vis, params.data(), projections, init_camera_params, use_constraints, use_point_constraints,
                           use_point_constraints ? point_constraints.data() : nullptr, nullptr, fix_points, optimize_for_fisheye, eps2,
                           Vout, Sout, Uout, Wout, info);
    if (rc != BSFM_OK) { C.restore_scales(init_camera_params); return rc; }
    if (info_out) memcpy(info_out, info, sizeof info);
    C.unpack(params.data(), init_camera_params);
    for (int i = 0; i < num_pts; i++)
        for (int q = 0; q < 3; q++) init_pts[i].p[q] = params[(size_t) num_camera_params + 3 * (size_t) i + q];
    return BSFM_OK;
}

extern "C" int bsfm_run_sfm(int num_pts, int num_cameras, int ncons, char *vmask, double *projections,
                            int est_focal_length, int const_focal_length, int undistort, int explicit_camera_centers,
                            bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                            int use_constraints, int use_point_constraints, bsfm_v3_t *pt_constraints,
                            double pt_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                            double *Vout, double *Sout, double *Uout, double *Wout, double *info_out)
{
    return run_sfm_impl(num_pts, num_cameras, ncons, VisSource::mask(vmask), projections, est_focal_length, const_focal_length,
                        undistort, explicit_camera_centers, init_camera_params, init_pts, use_constraints, use_point_constraints,
                        pt_constraints, pt_constraint_weight, fix_points, optimize_for_fisheye, eps2, Vout, Sout, Uout, Wout, info_out, false);
}

extern "C" int bsfm_run_sfm_crs(int num_pts, int num_cameras, int ncons, const int32_t *vis_ptr, const int32_t *vis_cam, int nvis,
                                double *projections, int est_focal_length, int const_focal_length, int undistort,
                                int explicit_camera_centers, bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                                int use_constraints, int use_point_constraints, bsfm_v3_t *pt_constraints,
                                double pt_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                                double *Vout, double *Sout, double *Uout, double *Wout, double *info_out)
{
    return run_sfm_impl(num_pts, num_cameras, ncons, VisSource::crs(vis_ptr, vis_cam, nvis), projections, est_focal_length,
                        const_focal_length, undistort, explicit_camera_centers, init_camera_params, init_pts, use_constraints,
                        use_point_constraints, pt_constraints, pt_constraint_weight, fix_points, optimize_for_fisheye, eps2,
                        Vout, Sout, Uout, Wout, info_out, false);
}

extern "C" int bsfm_run_sfm_fe(int num_pts, int num_cameras, int ncons, char *vmask, double *projections,
                               int est_focal_length, int const_focal_length, int undistort, int explicit_camera_centers,
                               bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                               int use_constraints, int use_point_constraints, bsfm_v3_t *pt_constraints,
                               double pt_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                               double *Vout, double *Sout, double *Uout, double *Wout, double *info_out)
{
    return run_sfm_impl(num_pts, num_cameras, ncons, VisSource::mask(vmask), projections, est_focal_length, const_focal_length,
                        undistort, explicit_camera_centers, init_camera_params, init_pts, use_constraints, use_point_constraints,
                        pt_constraints, pt_constraint_weight, fix_points, optimize_for_fisheye, eps2, Vout, Sout, Uout, Wout, info_out, true);
}

extern "C" int bsfm_run_sfm_crs_fe(int num_pts, int num_cameras, int ncons, const int32_t *vis_ptr, const int32_t *vis_cam, int nvis,
                                   double *projections, int est_focal_length, int const_focal_length, int undistort,
                                   int explicit_camera_centers, bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                                   int use_constraints, int use_point_constraints, bsfm_v3_t *pt_constraints,
                                   double pt_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                                   double *Vout, double *Sout, double *Uout, double *Wout, double *info_out)
{
    return run_sfm_impl(num_pts, num_cameras, ncons, VisSource::crs(vis_ptr, vis_cam, nvis), projections, est_focal_length,
                        const_focal_length, undistort, explicit_camera_centers, init_camera_params, init_pts, use_constraints,
                        use_point_constraints, pt_constraints, pt_constraint_weight, fix_points, optimize_for_fisheye, eps2,
                        Vout, Sout, Uout, Wout, info_out, true);
}

// == the do / while of BundlerApp::RunSFM_SBA (src/Bundle.cpp:588-913): solve, outlier pass, removal, until a round removes
// at most min_outliers points.  The scene goes to the device once and is compacted there between rounds (ba_loop.cu); a
// round's solve and outlier pass share one Visibility.  Per round the host sends the packed cameras and their tables and
// reads back the cameras, the m x 5 statistics and three counts.
extern "C" int bsfm_run_sfm_outlier_loop(int num_pts, int num_cameras, int ncons, const int32_t *vis_ptr, const int32_t *vis_cam, int nvis,
                                         const double *projections, int est_focal_length, int const_focal_length, int undistort,
                                         int explicit_camera_centers, bsfm_camera_params_t *init_camera_params, bsfm_v3_t *init_pts,
                                         int use_constraints, int use_point_constraints, bsfm_v3_t *pt_constraints,
                                         double pt_constraint_weight, int fix_points, int optimize_for_fisheye, double eps2,
                                         int remove_outliers, int min_outliers, int min_points,
                                         double min_proj_error_threshold, double max_proj_error_threshold,
                                         int32_t *pt_round, double *pt_error, double *cam_stats,
                                         bsfm_sfm_round_t *rounds, int rounds_cap, double *mean_error)
{
    clear_error();
    TRY(require_device());
    if (est_focal_length && const_focal_length) { set_error("bsfm_run_sfm_outlier_loop: const_focal_length is not implemented (nor in the reference, sfm.c:518-521)"); return BSFM_ERR_UNSUPPORTED; }
    const VisSource caller = VisSource::crs(vis_ptr, vis_cam, nvis);
    if (num_pts <= 0 || num_cameras <= 0 || !caller.present() || (nvis > 0 && !projections) || !init_camera_params || !init_pts || !pt_round || !pt_error ||
        rounds_cap < 0 || (rounds_cap > 0 && !rounds) || !mean_error) {
        set_error("bsfm_run_sfm_outlier_loop: bad arguments"); return BSFM_ERR_ARG;
    }
    if (use_point_constraints && !pt_constraints) { set_error("bsfm_run_sfm_outlier_loop: use_point_constraints without points_constraints"); return BSFM_ERR_ARG; }

    const int m = num_cameras;
    SfmCameras C(m, est_focal_length, undistort, explicit_camera_centers);
    const int ncp = C.cnp * m;
    SolverCtx *ctx;
    TRY(solver_ctx(&ctx));
    const cudaStream_t st = ctx->st;
    struct TallyGuard { TallyGuard() { t_uploads = UploadTally(); t_uploads.on = true; } ~TallyGuard() { t_uploads.on = false; } } tally;
    DeviceArena D(st);      // the scene: lives until the loop ends

    // the caller's scene, checked like bsfm_run_sfm_crs checks it
    Visibility V0;
    TRY(build_visibility(caller, num_pts, m, st, D, V0));
    if (V0.nvis <= 0) { set_error("bsfm_run_sfm_outlier_loop: no point has a view"); return BSFM_ERR_ARG; }
    LoopFull full;
    double *d_proj0;
    TRY(D.upload(&d_proj0, projections, (size_t) nvis * 2));
    TRY(D.upload(&full.pts, init_pts, (size_t) num_pts * 3));
    TRY(D.alloc(&full.pt_round, (size_t) num_pts)); TRY(D.alloc(&full.pt_error, (size_t) num_pts));
    // protected points, by ORIGINAL index (Bundle.cpp:800-806), and the solver's point constraints, which it reads by the
    // index of the ROUND (the reference passes m_point_constraints to run_sfm as it is, Bundle.cpp:651, sfm.c:757-781):
    // neither array is ever compacted, a round's solve takes the first n entries of the tables
    DevicePointConstraints dpc = {nullptr, nullptr, nullptr};
    if (use_point_constraints) {
        std::vector<char> h_prot(num_pts), h_pc(num_pts);
        std::vector<double> h_pv((size_t) num_pts * 3), h_pw(num_pts);
        std::vector<bsfm_point_constraints_t> pc;
        sfm_point_constraints(pt_constraints, pt_constraint_weight, num_pts, pc);
        for (int i = 0; i < num_pts; i++) {
            h_prot[i] = pt_constraints[i].p[0] != 0.0;
            h_pc[i] = pc[i].constrained ? 1 : 0;
            for (int q = 0; q < 3; q++) h_pv[(size_t) i * 3 + q] = pc[i].constraints[q];
            h_pw[i] = pc[i].weight;
        }
        char *d_prot, *d_pc; double *d_pv, *d_pw;
        TRY(D.upload(&d_prot, h_prot.data(), h_prot.size())); TRY(D.upload(&d_pc, h_pc.data(), h_pc.size()));
        TRY(D.upload(&d_pv, h_pv.data(), h_pv.size())); TRY(D.upload(&d_pw, h_pw.data(), h_pw.size()));
        full.prot = d_prot;
        dpc.constrained = d_pc; dpc.constraints = d_pv; dpc.weights = d_pw;
        BSFM_CUDA_TRY(cudaStreamSynchronize(st));     // the host vectors go out of scope
    }
    LoopScene half[2];
    TRY(alloc_loop_scene(half[0], num_pts, nvis, ncp, use_point_constraints != 0, D));
    TRY(alloc_loop_scene(half[1], num_pts, nvis, ncp, use_point_constraints != 0, D));
    int counts[3];
    TRY(loop_compact_entry(num_pts, ncp, V0.rowptr, V0.obs_cam, d_proj0, full, half[0], counts, st, D));

    std::vector<double> cam_params(ncp), stats((size_t) m * 5);
    int cur = 0, nrounds = 0, total_outliers = 0, num_outliers = 0, rc = BSFM_OK;
    long long counted = 0;
    *mean_error = 0.0;
    do {
        if (num_pts - total_outliers < min_points) {          // Bundle.cpp:588-595
            printf("[RunSFM] Too few points remaining, exiting!\n");
            fflush(stdout);
            *mean_error = DBL_MAX;
            break;
        }
        LoopScene &S = half[cur];
        bsfm_sfm_round_t R;
        memset(&R, 0, sizeof R);
        R.num_pts = S.n; R.nvis = S.nvis;
        DeviceArena RD(st);     // the round: its Visibility, the outlier pass and the scans
        rc = [&]() -> int {
            Visibility V;
            TRY(build_visibility(VisSource::device_crs(S.vis_ptr, S.vis_cam, S.nvis), S.n, m, st, RD, V));
            C.pack(init_camera_params, cam_params.data(), use_constraints);
            note_upload(cam_params.data(), (size_t) ncp * sizeof(double));
            BSFM_CUDA_TRY(cudaMemcpyAsync(S.p, cam_params.data(), (size_t) ncp * sizeof(double), cudaMemcpyHostToDevice, st));
            const int src = C.solve(S.n, ncons, VisSource::visibility(&V), S.p, S.proj, init_camera_params, use_constraints, use_point_constraints,
                                    nullptr, use_point_constraints ? &dpc : nullptr, fix_points, optimize_for_fisheye, eps2,
                                    nullptr, nullptr, nullptr, nullptr, R.info);
            if (src != BSFM_OK) { C.restore_scales(init_camera_params); return src; }
            BSFM_CUDA_TRY(cudaMemcpyAsync(cam_params.data(), S.p, (size_t) ncp * sizeof(double), cudaMemcpyDeviceToHost, st));
            BSFM_CUDA_TRY(cudaStreamSynchronize(st));
            C.unpack(cam_params.data(), init_camera_params);

            OutlierCams T;
            OutlierPass pass;
            TRY(upload_outlier_cams(init_camera_params, m, optimize_for_fisheye, RD, T));
            TRY(outliers_core(V, S.n, m, T, S.p + ncp, S.proj, undistort, min_proj_error_threshold, max_proj_error_threshold, S.prot, st, RD, pass));
            BSFM_CUDA_TRY(cudaMemcpyAsync(stats.data(), pass.stats, stats.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
            TRY(loop_compact_round(m, ncp, nrounds, remove_outliers ? 1 : 0, S, pass, full, half[cur ^ 1], counts, st, RD));
            return BSFM_OK;
        }();
        if (rc != BSFM_OK) break;
        double tot = 0.0, cnt = 0.0;      // Bundle.cpp:790-791, :852-856: sum of the per-camera sums / number of observations
        for (int j = 0; j < m; j++) if (stats[5 * (size_t) j] > 0) { tot += stats[5 * (size_t) j + 1] * stats[5 * (size_t) j]; cnt += stats[5 * (size_t) j]; }
        R.global_mean = tot / cnt;
        *mean_error = R.global_mean;
        if (cam_stats) memcpy(cam_stats, stats.data(), stats.size() * sizeof(double));
        num_outliers = counts[2];
        R.num_outliers = num_outliers;
        R.removed = remove_outliers ? 1 : 0;
        R.h2d_bytes = t_uploads.bytes - counted; R.h2d_largest = t_uploads.largest;
        counted = t_uploads.bytes; t_uploads.largest = 0;
        if (nrounds < rounds_cap) rounds[nrounds] = R;
        nrounds++;
        if (!remove_outliers) break;                          // Bundle.cpp:911
        total_outliers += num_outliers;
        cur ^= 1;
    } while (num_outliers > min_outliers);                    // Bundle.cpp:913

    // what the completed rounds left, also on an error return
    const char *failed = rc != BSFM_OK ? last_error() : nullptr;
    char keep_msg[1024];
    if (failed) snprintf(keep_msg, sizeof keep_msg, "%s", failed);
    cudaMemcpyAsync(init_pts, full.pts, (size_t) num_pts * 3 * sizeof(double), cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(pt_round, full.pt_round, (size_t) num_pts * sizeof(int), cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(pt_error, full.pt_error, (size_t) num_pts * sizeof(double), cudaMemcpyDeviceToHost, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    if (rc != BSFM_OK) { set_error("%s", keep_msg); return rc; }
    if (e != cudaSuccess) { set_error("bsfm_run_sfm_outlier_loop: copying the results back: %s", cudaGetErrorString(e)); return BSFM_ERR_CUDA; }
    return nrounds;
}
