// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.hpp header).
// Flat C entry points so tests/ and bench.py's cpu_baseline leg can drive the oracle through ctypes.
// Built by oracle/Makefile into oracle/liboracle.so (serial + OpenMP variants live in the same library;
// `use_omp` selects the reference's `parallel for schedule(dynamic)` + `critical` structure).
#include "oracle_planner.hpp"
#include "oracle_minco.hpp"
#include "oracle_frontend.hpp"
#include <cstdio>
#include <dlfcn.h>

using namespace orc;

extern "C" {

// Same field order as isdf_config in include/isdf.h (tests assert sizeof equality).
struct orc_config {
    double vehicle_mass, grav_acc, horiz_drag, vert_drag, paras_drag, speed_eps;
    double vmax, omgmax, thetamax;
    double weight_v, weight_p, weight_omg, weight_theta;
    double smoothing_eps, safety_hor;
    double occupancy_resolution;
    int kernel_size, integral_intervs, threads_num, flags;
};

static Params to_params(const orc_config *c) {
    Params P;
    P.mass = c->vehicle_mass; P.grav = c->grav_acc; P.dh = c->horiz_drag; P.dv = c->vert_drag; P.cp = c->paras_drag;
    P.veps = c->speed_eps; P.vmax = c->vmax; P.omgmax = c->omgmax; P.thetamax = c->thetamax;
    P.weight_v = c->weight_v; P.weight_p = c->weight_p; P.weight_omg = c->weight_omg; P.weight_theta = c->weight_theta;
    P.smooth_fac = c->smoothing_eps; P.safety_hor = c->safety_hor; P.integral_res = c->integral_intervs;
    P.bd = c->kernel_size * c->occupancy_resolution;  // hpp:692
    P.threads = c->threads_num > 0 ? c->threads_num : 1;
    P.with_dynamics = (c->flags & 1) ? 1 : 0;
    P.with_collision = (c->flags & 2) ? 1 : 0;
    return P;
}

struct OrcShape { Shape s; Mesh mesh; };

void *orc_shape_create(int kind, const double *par, int npar, const double *rot_rowmajor, const double *trans) {
    OrcShape *o = new OrcShape();
    o->s.kind = kind;
    for (int i = 0; i < npar && i < 12; i++) o->s.par[i] = par[i];
    if (rot_rowmajor) for (int i = 0; i < 9; i++) o->s.Rotate.m[i] = rot_rowmajor[i];
    if (trans) o->s.trans = V3(trans[0], trans[1], trans[2]);
    return o;
}
void *orc_shape_create_named(const char *name, const double *rot_rowmajor, const double *trans) {
    OrcShape *o = new OrcShape();
    if (!make_named_shape(name, o->s)) { delete o; return nullptr; }
    if (rot_rowmajor) for (int i = 0; i < 9; i++) o->s.Rotate.m[i] = rot_rowmajor[i];
    if (trans) o->s.trans = V3(trans[0], trans[1], trans[2]);
    return o;
}
// V: nV x 3 row-major, F: nF x 3 row-major; poly_params may be NULL (no pre-transform)
void *orc_shape_create_mesh(const double *V, int nV, const int *F, int nF, const double *poly_params, int wn_mode) {
    OrcShape *o = new OrcShape();
    o->mesh.V.resize(nV);
    for (int i = 0; i < nV; i++) o->mesh.V[i] = V3(V[3 * i], V[3 * i + 1], V[3 * i + 2]);
    o->mesh.F.assign(F, F + 3 * (size_t)nF);
    if (poly_params) o->mesh.pretransform(poly_params);
    o->mesh.wn_mode = wn_mode;
    o->mesh.build();
    o->s.kind = SK_MESH;
    o->s.mesh = &o->mesh;
    return o;
}
// WN_REF: attach oracle/_ref/libref_fwn.so (the reference's own FastWindingNumberForSoups.h, compiled from /root/reference by
// `make ref`) to a mesh shape and switch its sign to the reference-faithful s = 1 - 2 w_FWN (Shape.cpp:110-111). Returns 0 on success.
int orc_shape_attach_ref_fwn(void *h, const char *libpath) {
    OrcShape *o = (OrcShape *)h;
    if (!o || o->s.kind != SK_MESH) return -1;
    void *dl = dlopen(libpath, RTLD_NOW | RTLD_LOCAL);
    if (!dl) return -2;
    auto create = (void *(*)(const double *, int, const int *, int, int))dlsym(dl, "ref_fwn_create");
    auto query = (void (*)(void *, const double *, int, double, double *))dlsym(dl, "ref_fwn_query");
    if (!create || !query) return -3;
    std::vector<double> V(3 * o->mesh.V.size());
    for (size_t i = 0; i < o->mesh.V.size(); i++) { V[3 * i] = o->mesh.V[i].x; V[3 * i + 1] = o->mesh.V[i].y; V[3 * i + 2] = o->mesh.V[i].z; }
    o->mesh.ref_fwn = create(V.data(), (int)o->mesh.V.size(), o->mesh.F.data(), o->mesh.ntri(), 2);   // order 2 (Shape.cpp:86)
    o->mesh.ref_fwn_query = query;
    o->mesh.wn_mode = WN_REF;
    return o->mesh.ref_fwn ? 0 : -4;
}
void orc_shape_destroy(void *h) { delete (OrcShape *)h; }
int orc_shape_kind(void *h) { return ((OrcShape *)h)->s.kind; }
void orc_shape_params(void *h, double *par12) { for (int i = 0; i < 12; i++) par12[i] = ((OrcShape *)h)->s.par[i]; }

// what: 0 = getonlySDF, 1 = getonlyGrad1, 2 = getSDFwithGrad1
void orc_shape_query(void *h, const double *p, int n, double *sdf, double *grad, int what) {
    const Shape &s = ((OrcShape *)h)->s;
    for (int i = 0; i < n; i++) {
        const V3 q(p[3 * i], p[3 * i + 1], p[3 * i + 2]);
        V3 g;
        if (what == 0) sdf[i] = s.sdf(q);
        else if (what == 1) g = s.grad(q);
        else sdf[i] = s.sdf_grad(q, g);
        if (what) { grad[3 * i] = g.x; grad[3 * i + 1] = g.y; grad[3 * i + 2] = g.z; }
    }
}
// mesh internals for known-answer tests
void orc_mesh_query(void *h, const double *p, int n, double *d2_bvh, double *d2_brute, double *closest, double *w_exact, double *w_bh) {
    const Mesh &m = ((OrcShape *)h)->mesh;
    for (int i = 0; i < n; i++) {
        const V3 q(p[3 * i], p[3 * i + 1], p[3 * i + 2]);
        V3 c; int t;
        if (d2_bvh) { d2_bvh[i] = m.closest(q, c, t); if (closest) { closest[3 * i] = c.x; closest[3 * i + 1] = c.y; closest[3 * i + 2] = c.z; } }
        if (d2_brute) d2_brute[i] = m.closest_brute(q, c, t);
        if (w_exact) w_exact[i] = m.winding_exact(q);
        if (w_bh) w_bh[i] = m.winding_bh(q);
    }
}

void orc_flat_forward(const orc_config *c, const double *v, const double *a, const double *j, double *quat, double *omg) {
    Params P = to_params(c); Flat F; F.reset(P.mass, P.grav, P.dh, P.dv, P.cp, P.veps);
    V3 o; F.forward(V3(v[0], v[1], v[2]), V3(a[0], a[1], a[2]), V3(j[0], j[1], j[2]), quat, o);
    omg[0] = o.x; omg[1] = o.y; omg[2] = o.z;
}
void orc_flat_backward(const orc_config *c, const double *v, const double *a, const double *j, const double *pos_grad,
                       const double *vel_grad, const double *quat_grad, const double *omg_grad, double *out12) {
    Params P = to_params(c); Flat F; F.reset(P.mass, P.grav, P.dh, P.dv, P.cp, P.veps);
    V3 gp, gv, ga, gj;
    F.backward(V3(v[0], v[1], v[2]), V3(a[0], a[1], a[2]), V3(j[0], j[1], j[2]), V3(pos_grad[0], pos_grad[1], pos_grad[2]),
               V3(vel_grad[0], vel_grad[1], vel_grad[2]), quat_grad, V3(omg_grad[0], omg_grad[1], omg_grad[2]), gp, gv, ga, gj);
    const V3 *o[4] = {&gp, &gv, &ga, &gj};
    for (int i = 0; i < 4; i++) { out12[3 * i] = o[i]->x; out12[3 * i + 1] = o[i]->y; out12[3 * i + 2] = o[i]->z; }
}

// batched twins (n inputs, contiguous rows) for the reference-pin tests against oracle/_ref/libref_flat.so
void orc_flat_forward_batch(const orc_config *c, int n, const double *v, const double *a, const double *j, double *quat, double *omg) {
    for (int i = 0; i < n; i++) orc_flat_forward(c, v + 3 * i, a + 3 * i, j + 3 * i, quat + 4 * i, omg + 3 * i);
}
void orc_flat_backward_batch(const orc_config *c, int n, const double *v, const double *a, const double *j, const double *pos_grad,
                             const double *vel_grad, const double *quat_grad, const double *omg_grad, double *out12) {
    for (int i = 0; i < n; i++)
        orc_flat_backward(c, v + 3 * i, a + 3 * i, j + 3 * i, pos_grad + 3 * i, vel_grad + 3 * i, quat_grad + 4 * i, omg_grad + 3 * i, out12 + 12 * i);
}

// Discrete path. occ: X*Y*Z bytes, z fastest. Accumulates nothing: outputs are overwritten.
int orc_eval_discrete(const orc_config *c, const uint8_t *occ, int X, int Y, int Z, const double *bmin, double res,
                      void *shape, int N, const double *T, const double *C, double *cost, double *gradC, double *gradT,
                      long long *npairs, int use_omp, int rank, int world) {
    Params P = to_params(c);
    Grid G; G.X = X; G.Y = Y; G.Z = Z; G.res = res; G.occ = occ;
    G.bmin = V3(bmin[0], bmin[1], bmin[2]);
    G.bmax = V3(bmin[0] + X * res, bmin[1] + Y * res, bmin[2] + Z * res);
    Traj tr; tr.N = N; tr.T = T; tr.C = C;
    EvalOut out;
    // use_omp: 0 serial (THE ORACLE), 1 the reference's loop structure, 2 the "fair CPU" arm (per-thread accumulators + exact culls)
    eval_discrete(P, occ ? &G : nullptr, shape ? &((OrcShape *)shape)->s : nullptr, tr, out, use_omp != 0, rank, world > 0 ? world : 1, use_omp == 2);
    *cost = out.cost;
    std::memcpy(gradC, out.gradC.data(), sizeof(double) * 18 * N);
    std::memcpy(gradT, out.gradT.data(), sizeof(double) * N);
    if (npairs) *npairs = out.n_pairs;
    return 0;
}

// Swept-volume path. tstar in/out (lastTstar). sdf_out / grel_out optional. given_* optional (tier-T1 tail parity).
// traj_duration (optional, in/out): the SweptVolumeManager's duration before the evaluation (NULL: 0, a fresh manager) and after it —
// the replay of quirk Q14 across a sequence of evaluations.
int orc_eval_swept_ex(const orc_config *c, void *shape, int N, const double *T, const double *C, int npts, const double *pts,
                      double *tstar, double *cost, double *gradC, double *gradT, double *sdf_out, double *grel_out,
                      long long *nsdf, int use_omp, const double *given_tstar, const double *given_sdf, const double *given_grel,
                      double *traj_duration) {
    Params P = to_params(c);
    Traj tr; tr.N = N; tr.T = T; tr.C = C;
    EvalOut out;
    SweptGiven gv{given_tstar, given_sdf, given_grel};
    const double prev = traj_duration ? *traj_duration : 0.0;
    eval_swept(P, ((OrcShape *)shape)->s, tr, npts, pts, tstar, out, use_omp != 0, sdf_out, grel_out, given_tstar ? &gv : nullptr, prev);
    *cost = out.cost;
    std::memcpy(gradC, out.gradC.data(), sizeof(double) * 18 * N);
    std::memcpy(gradT, out.gradT.data(), sizeof(double) * N);
    if (nsdf) *nsdf = out.n_sdf;
    if (traj_duration) { const double td = tr.total(); *traj_duration = td < 3 * 1e2 ? td : prev; }
    return 0;
}
int orc_eval_swept(const orc_config *c, void *shape, int N, const double *T, const double *C, int npts, const double *pts,
                   double *tstar, double *cost, double *gradC, double *gradT, double *sdf_out, double *grel_out,
                   long long *nsdf, int use_omp, const double *given_tstar, const double *given_sdf, const double *given_grel) {
    return orc_eval_swept_ex(c, shape, N, T, C, npts, pts, tstar, cost, gradC, gradT, sdf_out, grel_out, nsdf, use_omp, given_tstar, given_sdf,
                             given_grel, nullptr);
}

// Coarse in-range decisions of the swept-volume search (SweptVolume::coarse) for npts points: bits npts x words (point-major), margin and
// carried per point. traj_duration is the duration before the evaluation, as for orc_eval_swept_ex. Returns the number of coarse samples.
int orc_sv_coarse(const orc_config *c, void *shape, int N, const double *T, const double *C, int npts, const double *pts, double traj_duration,
                  uint32_t *bits, int words, double *margin, int *carried) {
    Params P = to_params(c);
    Traj tr; tr.N = N; tr.T = T; tr.C = C;
    int nc = 0;
#pragma omp parallel for schedule(dynamic, 4) reduction(max : nc)
    for (int k = 0; k < npts; k++) {
        SweptVolume sv; sv.P = &P; sv.S = &((OrcShape *)shape)->s; sv.tr = &tr; sv.F.reset(P.mass, P.grav, P.dh, P.dv, P.cp, P.veps);
        sv.traj_duration = traj_duration; sv.update();
        nc = std::max(nc, sv.coarse(V3(pts[3 * k], pts[3 * k + 1], pts[3 * k + 2]), bits + (size_t)words * k, words, margin[k], carried[k]));
    }
    return nc;
}

// Single swept-volume SDF query (getSDFofSweptVolume<true>(p, t, g, false), swm:710-747)
double orc_sdf_swept(const orc_config *c, void *shape, int N, const double *T, const double *C, const double *p, double *tstar, double *grel) {
    Params P = to_params(c);
    Traj tr; tr.N = N; tr.T = T; tr.C = C;
    SweptVolume sv; sv.P = &P; sv.S = &((OrcShape *)shape)->s; sv.tr = &tr; sv.F.reset(P.mass, P.grav, P.dh, P.dv, P.cp, P.veps); sv.update();
    V3 g; const double s = sv.sdf_swept(V3(p[0], p[1], p[2]), *tstar, g);
    grel[0] = g.x; grel[1] = g.y; grel[2] = g.z;
    return s;
}

// getPointsInAABB (pcs:148-170) exposed for grid tests; returns count, writes up to cap centres
int orc_points_in_aabb(const uint8_t *occ, int X, int Y, int Z, const double *bmin, double res, const double *centre,
                       double half, double *out, int cap) {
    Grid G; G.X = X; G.Y = Y; G.Z = Z; G.res = res; G.occ = occ;
    G.bmin = V3(bmin[0], bmin[1], bmin[2]); G.bmax = V3(bmin[0] + X * res, bmin[1] + Y * res, bmin[2] + Z * res);
    std::vector<V3> v; G.points_in_aabb(V3(centre[0], centre[1], centre[2]), half, half, half, v);
    for (int i = 0; i < (int)v.size() && i < cap; i++) { out[3 * i] = v[i].x; out[3 * i + 1] = v[i].y; out[3 * i + 2] = v[i].z; }
    return (int)v.size();
}

// getGridIndex / getGridCubeCenter / isInMap of the oracle grid for n points (same outputs as oracle/ref_grid_wrap.cpp's ref_grid_index)
int orc_grid_index(int X, int Y, int Z, const double *bmin, double res, int n, const double *pts, int *idx, double *centre, int *inmap) {
    Grid G; G.X = X; G.Y = Y; G.Z = Z; G.res = res; G.occ = nullptr;
    G.bmin = V3(bmin[0], bmin[1], bmin[2]); G.bmax = V3(bmin[0] + X * res, bmin[1] + Y * res, bmin[2] + Z * res);
    for (int q = 0; q < n; q++) {
        const V3 p(pts[3 * q], pts[3 * q + 1], pts[3 * q + 2]);
        G.grid_index(p, idx + 3 * q);
        const V3 c = G.centre(idx[3 * q], idx[3 * q + 1], idx[3 * q + 2]);
        centre[3 * q] = c.x; centre[3 * q + 1] = c.y; centre[3 * q + 2] = c.z;
        inmap[q] = G.in_map(p) ? 1 : 0;
    }
    return 0;
}

// obstacle list (plan_manager.cpp:232-254); wps: nQ x 3; returns count, writes up to cap points
int orc_gather_obstacle_points(const uint8_t *occ, int X, int Y, int Z, const double *bmin, double res, const double *wps, int nQ,
                               double half, const double *offset, double *out, int cap) {
    Grid G; G.X = X; G.Y = Y; G.Z = Z; G.res = res; G.occ = occ;
    G.bmin = V3(bmin[0], bmin[1], bmin[2]); G.bmax = V3(bmin[0] + X * res, bmin[1] + Y * res, bmin[2] + Z * res);
    std::vector<V3> w(nQ), v;
    for (int i = 0; i < nQ; i++) w[i] = V3(wps[3 * i], wps[3 * i + 1], wps[3 * i + 2]);
    G.gather_obstacle_points(w, half, V3(offset[0], offset[1], offset[2]), v);
    for (int i = 0; i < (int)v.size() && i < cap; i++) { out[3 * i] = v[i].x; out[3 * i + 1] = v[i].y; out[3 * i + 2] = v[i].z; }
    return (int)v.size();
}

// ---- MINCO S3NU (adjacent step, SURVEY §8f #1) --------------------------------------------------
// headPVA/tailPVA: 3x3 column-major (columns = pos, vel, acc). inPs: 3 x (N-1) column-major. coeffs out: 6N x 3 col-major.
int orc_minco_forward(int N, const double *headPVA, const double *tailPVA, const double *inPs, const double *T,
                      double *coeffs, double *energy, double *gradC_energy, double *gradT_energy) {
    MincoS3 m; m.set_conditions(headPVA, tailPVA, N);
    m.set_parameters(inPs, T);
    std::memcpy(coeffs, m.b.data(), sizeof(double) * 18 * N);
    if (energy) *energy = m.energy();
    if (gradC_energy) m.energy_grad_coeffs(gradC_energy);
    if (gradT_energy) m.energy_grad_times(gradT_energy);
    return 0;
}
int orc_minco_backward(int N, const double *headPVA, const double *tailPVA, const double *inPs, const double *T,
                       const double *gradC, const double *gradT, double *gradP_out, double *gradT_out) {
    MincoS3 m; m.set_conditions(headPVA, tailPVA, N);
    m.set_parameters(inPs, T);
    m.propagate_grad(gradC, gradT, gradP_out, gradT_out);
    return 0;
}

// Trajectory::getPos_Vel_Acc_Jerk / locatePieceIdx / getTotalDuration of the oracle (oracle_planner.hpp Traj) on a coefficient block:
// out nt x 12 (pos, vel, acc, jerk), piece nt, tloc nt — the same outputs as oracle/ref_minco_wrap.cpp's ref_traj_eval
void orc_traj_eval(int N, const double *T, const double *coeffs, int nt, const double *times, double *out, int *piece, double *tloc, double *total) {
    Traj tr; tr.N = N; tr.T = T; tr.C = coeffs;
    *total = tr.total();
    for (int q = 0; q < nt; q++) {
        V3 p, v, a, j;
        tr.pvaj(times[q], p, v, a, j);
        const V3 *src[4] = {&p, &v, &a, &j};
        for (int b = 0; b < 4; b++) { out[12 * q + 3 * b] = src[b]->x; out[12 * q + 3 * b + 1] = src[b]->y; out[12 * q + 3 * b + 2] = src[b]->z; }
        double t = times[q];
        piece[q] = tr.locate(t);
        tloc[q] = t;
    }
}

// ---- front end: attitude kernels (oracle_frontend.hpp) --------------------------------------------------------------------
void *orc_frontend_create(void *shape, double max_roll, double max_pitch, double ang_res, double front_end_safeh, double res, int ks,
                          const uint8_t *occ, int X, int Y, int Z, int *xk, int *yk) {
    FrontEnd *f = new FrontEnd();
    KernelCfg c; c.max_roll = max_roll; c.max_pitch = max_pitch; c.ang_res = ang_res; c.front_end_safeh = front_end_safeh; c.res = res; c.ks = ks;
    f->build_kernels(((OrcShape *)shape)->s, c);
    if (occ) f->build_map_kernel(occ, X, Y, Z);
    if (xk) *xk = f->xk;
    if (yk) *yk = f->yk;
    return f;
}
void orc_frontend_destroy(void *h) { delete (FrontEnd *)h; }
void orc_frontend_kernels(void *h, uint8_t *out) { FrontEnd *f = (FrontEnd *)h; std::copy(f->kernels.begin(), f->kernels.end(), out); }
// masks: n x 4 uint32, bit (i*yk + j) set = attitude (i, j) is collision-free at voxel ind
void orc_frontend_feasibility(void *h, int n, const int *ind, uint32_t *masks) {
    FrontEnd *f = (FrontEnd *)h;
#pragma omp parallel for schedule(dynamic, 64)
    for (int q = 0; q < n; q++) {
        uint32_t m[4] = {0, 0, 0, 0};
        for (int i = 0; i < f->xk; i++)
            for (int j = 0; j < f->yk; j++)
                if (f->conv(i, j, ind + 3 * q)) { const int b = i * f->yk + j; m[b >> 5] |= 1u << (b & 31); }
        for (int k = 0; k < 4; k++) masks[4 * (size_t)q + k] = m[k];
    }
}
void orc_frontend_check(void *h, int n, const int *ind, const double *father, double *child, uint8_t *ok) {
    FrontEnd *f = (FrontEnd *)h;
    for (int q = 0; q < n; q++) {
        double cr = father[2 * q], cp = father[2 * q + 1];
        ok[q] = f->check(father[2 * q], father[2 * q + 1], cr, cp, ind + 3 * q) ? 1 : 0;
        child[2 * q] = cr; child[2 * q + 1] = cp;
    }
}

void orc_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int orc_omp_max_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

}  // extern "C"
