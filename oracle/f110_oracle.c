/*
 * f110_oracle.c — CPU restatement of the f1tenth_gym per-tick hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is the parity oracle for the CUDA path in
 * f1tenth_gym_b200/csrc/.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load it; the product path never does.
 *
 * Parity status: PINNED.  tests/test_oracle_vs_golden.py checks this restatement against
 *   (1) the reference's own known-answer vectors (dynamic_models.py:257-258 f_ks_gt/f_st_gt,
 *       collision_models.py:306-324), and
 *   (2) golden trajectories produced by running the UNMODIFIED reference numba path in the
 *       build container (tests/golden/make_golden.py, fixtures committed under tests/golden/).
 *
 * Every function cites the reference file:line it follows (paths relative to
 * /root/reference/gym/f110_gym/envs/).  All arithmetic is IEEE fp64, compiled with
 * -ffp-contract=off so that no FMA contraction happens (numba emits none either).
 *
 * Written from the behaviour of the reference; not a source copy (the reference is Python).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <pthread.h>
#include <unistd.h>

#define ORC_NPARAM 18
/* parameter vector layout (order of the F110Env default dict, f110_env.py:130) */
enum { P_MU = 0, P_CSF, P_CSR, P_LF, P_LR, P_H, P_M, P_I, P_SMIN, P_SMAX, P_SVMIN, P_SVMAX,
       P_VSWITCH, P_AMAX, P_VMIN, P_VMAX, P_WIDTH, P_LENGTH };

typedef struct {
    int32_t height, width;
    double resolution, orig_x, orig_y, orig_c, orig_s;
    const double *dt;      /* [height*width] row-major, row 0 = bottom of the image */
    int32_t theta_dis;
    const double *sines;   /* [theta_dis] sin(linspace(0, 2pi, theta_dis)) laser_models.py:379-381 */
    const double *cosines;
    double eps, max_range;
} orc_map_t;

/* ------------------------------------------------------------------ dynamics */

/* dynamic_models.py:29-60 accl_constraints */
static double accl_constraints(double vel, double accl, double v_switch, double a_max,
                               double v_min, double v_max) {
    double pos_limit;
    if (vel > v_switch) pos_limit = a_max * v_switch / vel;
    else pos_limit = a_max;
    if ((vel <= v_min && accl <= 0) || (vel >= v_max && accl >= 0)) accl = 0.;
    else if (accl <= -a_max) accl = -a_max;
    else if (accl >= pos_limit) accl = pos_limit;
    return accl;
}

/* dynamic_models.py:62-87 steering_constraint */
static double steering_constraint(double steering_angle, double steering_velocity, double s_min,
                                  double s_max, double sv_min, double sv_max) {
    if ((steering_angle <= s_min && steering_velocity <= 0) ||
        (steering_angle >= s_max && steering_velocity >= 0)) steering_velocity = 0.;
    else if (steering_velocity <= sv_min) steering_velocity = sv_min;
    else if (steering_velocity >= sv_max) steering_velocity = sv_max;
    return steering_velocity;
}

/* dynamic_models.py:90-121 vehicle_dynamics_ks; x has 5 entries, f has 5 */
void orc_vehicle_dynamics_ks(const double *x, const double *u_init, const double *p, double *f) {
    double lwb = p[P_LF] + p[P_LR];
    double u0 = steering_constraint(x[2], u_init[0], p[P_SMIN], p[P_SMAX], p[P_SVMIN], p[P_SVMAX]);
    double u1 = accl_constraints(x[3], u_init[1], p[P_VSWITCH], p[P_AMAX], p[P_VMIN], p[P_VMAX]);
    f[0] = x[3] * cos(x[4]);
    f[1] = x[3] * sin(x[4]);
    f[2] = u0;
    f[3] = u1;
    f[4] = x[3] / lwb * tan(x[2]);
}

/* dynamic_models.py:123-176 vehicle_dynamics_st; x has 7 entries, f has 7 */
void orc_vehicle_dynamics_st(const double *x, const double *u_init, const double *p, double *f) {
    const double g = 9.81;
    double mu = p[P_MU], C_Sf = p[P_CSF], C_Sr = p[P_CSR], lf = p[P_LF], lr = p[P_LR], h = p[P_H],
           m = p[P_M], I = p[P_I];
    double u[2];
    u[0] = steering_constraint(x[2], u_init[0], p[P_SMIN], p[P_SMAX], p[P_SVMIN], p[P_SVMAX]);
    u[1] = accl_constraints(x[3], u_init[1], p[P_VSWITCH], p[P_AMAX], p[P_VMIN], p[P_VMAX]);
    if (fabs(x[3]) < 0.5) {
        /* :152-160 kinematic branch; constraints re-applied on the constrained input */
        double lwb = lf + lr;
        double fks[5];
        orc_vehicle_dynamics_ks(x, u, p, fks);
        for (int i = 0; i < 5; i++) f[i] = fks[i];
        double c2 = cos(x[2]);
        f[5] = u[1] / lwb * tan(x[2]) + x[3] / (lwb * (c2 * c2)) * u[0];
        f[6] = 0.;
    } else {
        /* :162-174; evaluation order = Python precedence, left to right */
        f[0] = x[3] * cos(x[6] + x[4]);
        f[1] = x[3] * sin(x[6] + x[4]);
        f[2] = u[0];
        f[3] = u[1];
        f[4] = x[5];
        f[5] = -mu * m / (x[3] * I * (lr + lf)) *
                   (lf * lf * C_Sf * (g * lr - u[1] * h) + lr * lr * C_Sr * (g * lf + u[1] * h)) * x[5]
               + mu * m / (I * (lr + lf)) * (lr * C_Sr * (g * lf + u[1] * h) - lf * C_Sf * (g * lr - u[1] * h)) * x[6]
               + mu * m / (I * (lr + lf)) * lf * C_Sf * (g * lr - u[1] * h) * x[2];
        f[6] = (mu / (x[3] * x[3] * (lr + lf)) * (C_Sr * (g * lf + u[1] * h) * lr - C_Sf * (g * lr - u[1] * h) * lf) - 1) * x[5]
               - mu / (x[3] * (lr + lf)) * (C_Sr * (g * lf + u[1] * h) + C_Sf * (g * lr - u[1] * h)) * x[6]
               + mu / (x[3] * (lr + lf)) * (C_Sf * (g * lr - u[1] * h)) * x[2];
    }
}

/* dynamic_models.py:178-221 pid; out[0]=accl, out[1]=sv */
void orc_pid(double speed, double steer, double current_speed, double current_steer, double max_sv,
             double max_a, double max_v, double min_v, double *out) {
    double sv, accl, kp;
    double steer_diff = steer - current_steer;
    if (fabs(steer_diff) > 1e-4) sv = (steer_diff / fabs(steer_diff)) * max_sv;
    else sv = 0.0;
    double vel_diff = speed - current_speed;
    if (current_speed > 0.) {
        if (vel_diff > 0) kp = 10.0 * max_a / max_v;
        else kp = 10.0 * max_a / (-min_v);
    } else {
        if (vel_diff > 0) kp = 2.0 * max_a / max_v;
        else kp = 2.0 * max_a / (-min_v);
    }
    accl = kp * vel_diff;
    out[0] = accl;
    out[1] = sv;
}

/* ------------------------------------------------------------------ lidar */

/* laser_models.py:55-104 xy_2_rc + distance_transform.  Off-map -> (r,c)=(-1,-1) and numba's
 * negative-index wraparound reads dt[-1,-1] = the last cell.
 * Deliberate deviation: an x_rot just below width*resolution passes the bounds test of :79, yet
 * x_rot/resolution can round to exactly `width` (likewise y_rot and `height`).  The reference then reads
 * the flat element r*W + W (the first cell of row r+1, or past the table in the top row, :102-104); here
 * such a cell is off-map and reads dt[-1,-1], as every CUDA kernel does (DESIGN.md §4). */
static inline double dt_lookup(const orc_map_t *mp, double x, double y) {
    double x_trans = x - mp->orig_x;
    double y_trans = y - mp->orig_y;
    double x_rot = x_trans * mp->orig_c + y_trans * mp->orig_s;
    double y_rot = -x_trans * mp->orig_s + y_trans * mp->orig_c;
    long r = mp->height - 1, c = mp->width - 1;
    if (!(x_rot < 0 || x_rot >= mp->width * mp->resolution || y_rot < 0 ||
          y_rot >= mp->height * mp->resolution)) {
        long cc = (long)(x_rot / mp->resolution);
        long rr = (long)(y_rot / mp->resolution);
        if (cc < mp->width && rr < mp->height) { c = cc; r = rr; }
    }
    return mp->dt[r * (long)mp->width + c];
}

/* laser_models.py:106-146 trace_ray.  nlook (optional) counts DT lookups (roofline denominator). */
static inline double trace_ray(const orc_map_t *mp, double x, double y, double theta_index,
                               int64_t *nlook) {
    int ti = (int)theta_index;
    /* Deliberate deviation: get_scan's first index can be exactly theta_dis (a yaw one ulp below fov/2 when
     * fov/2 < 2), and the reference then reads sines[theta_dis], one past its table.  Here it wraps to 0, as
     * every CUDA kernel does (DESIGN.md §4).  The sequence of later beams is unchanged. */
    if (ti >= mp->theta_dis) ti -= mp->theta_dis;
    double s = mp->sines[ti];
    double c = mp->cosines[ti];
    double dist_to_nearest = dt_lookup(mp, x, y);
    double total_dist = dist_to_nearest;
    int64_t n = 1;
    while (dist_to_nearest > mp->eps && total_dist <= mp->max_range) {
        x += dist_to_nearest * c;
        y += dist_to_nearest * s;
        dist_to_nearest = dt_lookup(mp, x, y);
        total_dist += dist_to_nearest;
        n++;
    }
    if (total_dist > mp->max_range) total_dist = mp->max_range;
    if (nlook) *nlook += n;
    return total_dist;
}

/* laser_models.py:148-186 get_scan.  theta_index_increment as computed in
 * ScanSimulator2D.__init__ (:367-368) is passed in by the caller. */
void orc_get_scan(const orc_map_t *mp, const double *pose, int num_beams, double fov,
                  double theta_index_increment, double *scan, int64_t *nlook) {
    double theta_dis = (double)mp->theta_dis;
    double theta_index = theta_dis * (pose[2] - fov / 2.) / (2. * M_PI);
    theta_index = fmod(theta_index, theta_dis);
    while (theta_index < 0) theta_index += theta_dis;
    for (int i = 0; i < num_beams; i++) {
        scan[i] = trace_ray(mp, pose[0], pose[1], theta_index, nlook);
        theta_index += theta_index_increment;
        while (theta_index >= theta_dis) theta_index -= theta_dis;
    }
}

/* laser_models.py:188-217 check_ttc_jit (error_model='numpy': x/0 -> inf/nan, no raise) */
int orc_check_ttc(const double *scan, int num_beams, double vel, const double *cosines,
                  const double *side_distances, double ttc_thresh) {
    if (vel != 0.0) {
        for (int i = 0; i < num_beams; i++) {
            double proj_vel = vel * cosines[i];
            double ttc = (scan[i] - side_distances[i]) / proj_vel;
            if ((ttc < ttc_thresh) && (ttc >= 0.0)) return 1;
        }
    }
    return 0;
}

/* laser_models.py:219-230 cross */
static inline double cross2(double ax, double ay, double bx, double by) { return ax * by - ay * bx; }

/* laser_models.py:249-280 get_range (+ are_collinear :232-247) */
static double get_range(const double *pose, double beam_theta, const double *va, const double *vb) {
    double ox = pose[0], oy = pose[1];
    double v1x = ox - va[0], v1y = oy - va[1];
    double v2x = vb[0] - va[0], v2y = vb[1] - va[1];
    double v3x = cos(beam_theta + M_PI / 2.), v3y = sin(beam_theta + M_PI / 2.);
    double denom = v2x * v3x + v2y * v3y;
    double distance = INFINITY;
    if (fabs(denom) > 0.0) {
        double d1 = cross2(v2x, v2y, v1x, v1y) / denom;
        double d2 = (v1x * v3x + v1y * v3y) / denom;
        if (d1 >= 0.0 && d2 >= 0.0 && d2 <= 1.0) distance = d1;
    } else {
        /* are_collinear(o, va, vb): ba = va - o ; ca = o - vb */
        double bax = va[0] - ox, bay = va[1] - oy;
        double cax = ox - vb[0], cay = oy - vb[1];
        if (fabs(cross2(bax, bay, cax, cay)) < 1e-8) {
            double da = sqrt((va[0] - ox) * (va[0] - ox) + (va[1] - oy) * (va[1] - oy));
            double db = sqrt((vb[0] - ox) * (vb[0] - ox) + (vb[1] - oy) * (vb[1] - oy));
            distance = da < db ? da : db;
        }
    }
    return distance;
}

static int argmin_abs_diff(const double *scan_angles, int n, double a) {
    int best = 0;
    double bv = fabs(scan_angles[0] - a);
    for (int i = 1; i < n; i++) {
        double v = fabs(scan_angles[i] - a);
        if (v < bv) { bv = v; best = i; }
    }
    return best;
}

/* laser_models.py:282-315 get_blocked_view_indices; vertices[4][2] */
void orc_blocked_view_indices(const double *pose, const double *vertices, const double *scan_angles,
                              int num_beams, int *min_ind, int *max_ind) {
    double ego_a = atan2(sin(pose[2]), cos(pose[2]));
    int lo = 0, hi = 0;
    for (int i = 0; i < 4; i++) {
        double vx = vertices[2 * i] - pose[0], vy = vertices[2 * i + 1] - pose[1];
        double norm = sqrt(vx * vx + vy * vy);
        double ux = vx / norm, uy = vy / norm;
        double angle = ego_a - atan2(uy, ux);
        if (angle > M_PI) angle = angle - 2 * M_PI;
        else if (angle < -M_PI) angle = angle + 2 * M_PI;
        int ind = argmin_abs_diff(scan_angles, num_beams, -angle);
        if (i == 0) { lo = hi = ind; }
        else { if (ind < lo) lo = ind; if (ind > hi) hi = ind; }
    }
    *min_ind = lo;
    *max_ind = hi;
}

/* laser_models.py:318-346 ray_cast; modifies scan in place */
void orc_ray_cast(const double *pose, double *scan, const double *scan_angles, int num_beams,
                  const double *vertices) {
    double lv[5][2];
    for (int i = 0; i < 4; i++) { lv[i][0] = vertices[2 * i]; lv[i][1] = vertices[2 * i + 1]; }
    lv[4][0] = vertices[0]; lv[4][1] = vertices[1];
    int min_ind, max_ind;
    orc_blocked_view_indices(pose, vertices, scan_angles, num_beams, &min_ind, &max_ind);
    for (int i = min_ind; i <= max_ind; i++) {
        for (int j = 0; j < 4; j++) {
            double r = get_range(pose, pose[2] + scan_angles[i], lv[j], lv[j + 1]);
            if (r < scan[i]) scan[i] = r;
        }
    }
}

/* ------------------------------------------------------------------ collision */

/* collision_models.py:218-260 get_trmtx + get_vertices -> (rl, rr, fr, fl) */
void orc_get_vertices(const double *pose, double length, double width, double *v /* [4][2] */) {
    double x = pose[0], y = pose[1], c = cos(pose[2]), s = sin(pose[2]);
    const double lx[4] = { -length / 2, -length / 2, length / 2, length / 2 };
    const double ly[4] = { width / 2, -width / 2, -width / 2, width / 2 };
    for (int i = 0; i < 4; i++) {
        /* row of H . [lx, ly, 0, 1]^T, then / w (w == 1) */
        v[2 * i] = ((c * lx[i] + (-s) * ly[i]) + 0. * 0.) + x * 1.;
        v[2 * i + 1] = ((s * lx[i] + c * ly[i]) + 0. * 0.) + y * 1.;
    }
}

/* collision_models.py:81-110 indexOfFurthestPoint + support */
static int furthest(const double *v, double dx, double dy) {
    int best = 0;
    double bv = v[0] * dx + v[1] * dy;
    for (int i = 1; i < 4; i++) {
        double t = v[2 * i] * dx + v[2 * i + 1] * dy;
        if (t > bv) { bv = t; best = i; }
    }
    return best;
}
static void support(const double *v1, const double *v2, double dx, double dy, double *out) {
    int i = furthest(v1, dx, dy);
    int j = furthest(v2, -dx, -dy);
    out[0] = v1[2 * i] - v2[2 * j];
    out[1] = v1[2 * i + 1] - v2[2 * j + 1];
}
/* collision_models.py:51-64 tripleProduct: b*(a.c) - a*(b.c) */
static void triple(const double *a, const double *b, const double *c, double *out) {
    double ac = a[0] * c[0] + a[1] * c[1];
    double bc = b[0] * c[0] + b[1] * c[1];
    out[0] = b[0] * ac - a[0] * bc;
    out[1] = b[1] * ac - a[1] * bc;
}

/* collision_models.py:113-182 collision (GJK on two 4-gons) */
int orc_collision(const double *v1, const double *v2) {
    int index = 0;
    double simplex[3][2];
    double p1x = (v1[0] + v1[2] + v1[4] + v1[6]) / 4, p1y = (v1[1] + v1[3] + v1[5] + v1[7]) / 4;
    double p2x = (v2[0] + v2[2] + v2[4] + v2[6]) / 4, p2y = (v2[1] + v2[3] + v2[5] + v2[7]) / 4;
    double d[2] = { p1x - p2x, p1y - p2y };
    if (d[0] == 0 && d[1] == 0) d[0] = 1.0;
    double a[2];
    support(v1, v2, d[0], d[1], a);
    simplex[0][0] = a[0]; simplex[0][1] = a[1];
    if (d[0] * a[0] + d[1] * a[1] <= 0) return 0;
    d[0] = -a[0]; d[1] = -a[1];
    int iter_count = 0;
    while (iter_count < 1000) {
        support(v1, v2, d[0], d[1], a);
        index += 1;
        simplex[index][0] = a[0]; simplex[index][1] = a[1];
        if (d[0] * a[0] + d[1] * a[1] <= 0) return 0;
        double ao[2] = { -a[0], -a[1] };
        if (index < 2) {
            double ab[2] = { simplex[0][0] - a[0], simplex[0][1] - a[1] };
            triple(ab, ao, ab, d);
            if (sqrt(d[0] * d[0] + d[1] * d[1]) < 1e-10) {
                /* perpendicular(ab) :34-48 */
                d[0] = ab[1]; d[1] = -1 * ab[0];
            }
            continue;
        }
        double ab[2] = { simplex[1][0] - a[0], simplex[1][1] - a[1] };
        double ac[2] = { simplex[0][0] - a[0], simplex[0][1] - a[1] };
        double acperp[2];
        triple(ab, ac, ac, acperp);
        if (acperp[0] * ao[0] + acperp[1] * ao[1] >= 0) {
            d[0] = acperp[0]; d[1] = acperp[1];
        } else {
            double abperp[2];
            triple(ac, ab, ab, abperp);
            if (abperp[0] * ao[0] + abperp[1] * ao[1] < 0) return 1;
            simplex[0][0] = simplex[1][0]; simplex[0][1] = simplex[1][1];
            d[0] = abperp[0]; d[1] = abperp[1];
        }
        simplex[1][0] = simplex[2][0]; simplex[1][1] = simplex[2][1];
        index -= 1;
        iter_count += 1;
    }
    return 0;
}

/* collision_models.py:184-212 collision_multiple; vertices [n][4][2] */
void orc_collision_multiple(const double *vertices, int n, double *collisions, double *collision_idx) {
    for (int i = 0; i < n; i++) { collisions[i] = 0.; collision_idx[i] = -1.; }
    for (int i = 0; i < n - 1; i++)
        for (int j = i + 1; j < n; j++)
            if (orc_collision(vertices + 8 * i, vertices + 8 * j)) {
                collisions[i] = 1.; collisions[j] = 1.;
                collision_idx[i] = j; collision_idx[j] = i;
            }
}

/* ------------------------------------------------------------------ Simulator (one env) */

typedef struct {
    int32_t num_agents, num_beams, integrator /* 1 RK4, 2 Euler (base_classes.py:40-42) */;
    int32_t ego_idx;
    double time_step, fov, theta_index_increment, lidar_dist, ttc_thresh;
    double sim_length, sim_width; /* Simulator.params['length'/'width'] (constructor dict, never updated) */
    const orc_map_t *map;
    const double *scan_angles, *cosines, *side_distances; /* [num_beams] base_classes.py:125-158 */
    double *params;      /* [A][18] */
    double *state;       /* [A][7]  x, y, steer, v, yaw, yaw_rate, slip */
    double *steer_buf;   /* [A][2]  index 0 = newest (np.append(raw, buf)) */
    int32_t *steer_cnt;  /* [A] */
    int32_t *in_collision; /* [A] wall (iTTC) flag */
    double *collisions;  /* [A] obs */
    double *collision_idx;
    double *agent_poses; /* [A][3] */
    double *scans;       /* [A][B] */
    /* F110Env level (f110_env.py:165-189) */
    double current_time;
    double *lap_times, *lap_counts, *toggle_list; /* [A] */
    int32_t *near_starts;                         /* [A] */
    double *start_xs, *start_ys, *start_thetas;   /* [A] */
    double start_rot[4];
    int64_t nlook;       /* DT lookups performed so far */
    /* batch driver (orc_step_batch) */
    const double *noise; /* [A][B] additive scan noise of the current step, or NULL */
    double *scans_pre;   /* [A][B] each agent's scan before the opponent ray-cast (after noise) */
    int32_t done;        /* result of the last orc_env_post_step */
} orc_sim_t;

orc_sim_t *orc_sim_create(int num_agents, int num_beams, int integrator, double time_step, double fov,
                          double theta_index_increment, double lidar_dist, const orc_map_t *map,
                          const double *scan_angles, const double *cosines,
                          const double *side_distances, const double *params /* [A][18] */) {
    orc_sim_t *s = (orc_sim_t *)calloc(1, sizeof(orc_sim_t));
    int A = num_agents, B = num_beams;
    s->num_agents = A; s->num_beams = B; s->integrator = integrator; s->ego_idx = 0;
    s->time_step = time_step; s->fov = fov; s->theta_index_increment = theta_index_increment;
    s->lidar_dist = lidar_dist; s->ttc_thresh = 0.005; /* base_classes.py:115 */
    s->map = map; s->scan_angles = scan_angles; s->cosines = cosines; s->side_distances = side_distances;
    s->params = (double *)malloc(sizeof(double) * A * ORC_NPARAM);
    memcpy(s->params, params, sizeof(double) * A * ORC_NPARAM);
    s->sim_length = params[P_LENGTH]; s->sim_width = params[P_WIDTH];
    s->state = (double *)calloc(A * 7, sizeof(double));
    s->steer_buf = (double *)calloc(A * 2, sizeof(double));
    s->steer_cnt = (int32_t *)calloc(A, sizeof(int32_t));
    s->in_collision = (int32_t *)calloc(A, sizeof(int32_t));
    s->collisions = (double *)calloc(A, sizeof(double));
    s->collision_idx = (double *)calloc(A, sizeof(double));
    s->agent_poses = (double *)calloc(A * 3, sizeof(double));
    s->scans = (double *)calloc((size_t)A * B, sizeof(double));
    s->scans_pre = (double *)calloc((size_t)A * B, sizeof(double));
    s->lap_times = (double *)calloc(A, sizeof(double));
    s->lap_counts = (double *)calloc(A, sizeof(double));
    s->toggle_list = (double *)calloc(A, sizeof(double));
    s->near_starts = (int32_t *)calloc(A, sizeof(int32_t));
    s->start_xs = (double *)calloc(A, sizeof(double));
    s->start_ys = (double *)calloc(A, sizeof(double));
    s->start_thetas = (double *)calloc(A, sizeof(double));
    for (int i = 0; i < A; i++) { s->near_starts[i] = 1; s->collision_idx[i] = -1.; }
    s->start_rot[0] = 1; s->start_rot[3] = 1;
    return s;
}

/* F110Env(ego_idx=...) (f110_env.py:145): the agent whose collision ends the episode and whose start pose sets the lap
 * frame.  orc_sim_create starts with agent 0.  Returns 0, or -1 (nothing changed) for an index outside [0, num_agents). */
int orc_sim_set_ego(orc_sim_t *s, int ego_idx) {
    if (ego_idx < 0 || ego_idx >= s->num_agents) return -1;
    s->ego_idx = ego_idx;
    return 0;
}

void orc_sim_destroy(orc_sim_t *s) {
    if (!s) return;
    free(s->params); free(s->state); free(s->steer_buf); free(s->steer_cnt); free(s->in_collision);
    free(s->collisions); free(s->collision_idx); free(s->agent_poses); free(s->scans); free(s->scans_pre);
    free(s->lap_times); free(s->lap_counts); free(s->toggle_list); free(s->near_starts);
    free(s->start_xs); free(s->start_ys); free(s->start_thetas);
    free(s);
}

/* accessors for ctypes */
double *orc_sim_state(orc_sim_t *s) { return s->state; }
double *orc_sim_scans(orc_sim_t *s) { return s->scans; }
double *orc_sim_scans_pre(orc_sim_t *s) { return s->scans_pre; }
double *orc_sim_collisions(orc_sim_t *s) { return s->collisions; }
double *orc_sim_collision_idx(orc_sim_t *s) { return s->collision_idx; }
double *orc_sim_lap_times(orc_sim_t *s) { return s->lap_times; }
double *orc_sim_lap_counts(orc_sim_t *s) { return s->lap_counts; }
double *orc_sim_toggle_list(orc_sim_t *s) { return s->toggle_list; }
double *orc_sim_params(orc_sim_t *s) { return s->params; }
int32_t *orc_sim_in_collision(orc_sim_t *s) { return s->in_collision; }
int32_t *orc_sim_steer_cnt(orc_sim_t *s) { return s->steer_cnt; }
double *orc_sim_steer_buf(orc_sim_t *s) { return s->steer_buf; }
int64_t orc_sim_nlook(orc_sim_t *s) { return s->nlook; }
double orc_sim_current_time(orc_sim_t *s) { return s->current_time; }

/* base_classes.py:183-204 RaceCar.reset + :614-630 Simulator.reset */
void orc_sim_reset(orc_sim_t *s, const double *poses /* [A][3] */) {
    for (int i = 0; i < s->num_agents; i++) {
        double *st = s->state + 7 * i;
        for (int k = 0; k < 7; k++) st[k] = 0.;
        st[0] = poses[3 * i]; st[1] = poses[3 * i + 1]; st[4] = poses[3 * i + 2];
        s->steer_cnt[i] = 0;
        s->in_collision[i] = 0;
    }
}

/* base_classes.py:256-413 RaceCar.update_pose for agent i; writes scans[i] */
static void update_pose(orc_sim_t *s, int i, double raw_steer, double vel) {
    double *st = s->state + 7 * i;
    const double *p = s->params + ORC_NPARAM * i;
    double *buf = s->steer_buf + 2 * i;
    double steer;
    /* :270-278 steering delay FIFO, depth 2 */
    if (s->steer_cnt[i] < 2) {
        steer = 0.;
        buf[1] = buf[0]; buf[0] = raw_steer;   /* np.append(raw_steer, buffer) */
        s->steer_cnt[i] += 1;
    } else {
        steer = buf[1];
        buf[1] = buf[0]; buf[0] = raw_steer;
    }
    double as[2];
    orc_pid(vel, steer, st[3], st[2], p[P_SVMAX], p[P_AMAX], p[P_VMAX], p[P_VMIN], as);
    double u[2] = { as[1], as[0] };   /* np.array([sv, accl]) */
    double dt = s->time_step;
    if (s->integrator == 1) {
        double k1[7], k2[7], k3[7], k4[7], xs[7];
        orc_vehicle_dynamics_st(st, u, p, k1);
        for (int k = 0; k < 7; k++) xs[k] = st[k] + dt * (k1[k] / 2);
        orc_vehicle_dynamics_st(xs, u, p, k2);
        for (int k = 0; k < 7; k++) xs[k] = st[k] + dt * (k2[k] / 2);
        orc_vehicle_dynamics_st(xs, u, p, k3);
        for (int k = 0; k < 7; k++) xs[k] = st[k] + dt * k3[k];
        orc_vehicle_dynamics_st(xs, u, p, k4);
        double w = dt * (1. / 6);   /* self.time_step*(1/6) is evaluated first (scalar) :373 */
        for (int k = 0; k < 7; k++) st[k] = st[k] + w * (((k1[k] + 2 * k2[k]) + 2 * k3[k]) + k4[k]);
    } else {
        double f[7];
        orc_vehicle_dynamics_st(st, u, p, f);
        for (int k = 0; k < 7; k++) st[k] = st[k] + dt * f[k];
    }
    /* :400-404 single-shot yaw wrap */
    if (st[4] > 2 * M_PI) st[4] = st[4] - 2 * M_PI;
    else if (st[4] < 0) st[4] = st[4] + 2 * M_PI;
    /* :406-410 scan pose */
    double scan_pose[3] = { st[0] + s->lidar_dist * cos(st[4]), st[1] + s->lidar_dist * sin(st[4]), st[4] };
    double *scan = s->scans + (size_t)i * s->num_beams;
    orc_get_scan(s->map, scan_pose, s->num_beams, s->fov, s->theta_index_increment, scan, &s->nlook);
    /* laser_models.py:450-452: the noise is part of the scan that check_ttc and the opponent ray-cast see */
    if (s->noise) {
        const double *nz = s->noise + (size_t)i * s->num_beams;
        for (int b = 0; b < s->num_beams; b++) scan[b] = scan[b] + nz[b];
    }
}

/* base_classes.py:553-612 Simulator.step.  control_inputs [A][2] = (steer, speed). */
void orc_sim_step(orc_sim_t *s, const double *control_inputs) {
    int A = s->num_agents, B = s->num_beams;
    for (int i = 0; i < A; i++) {
        update_pose(s, i, control_inputs[2 * i], control_inputs[2 * i + 1]);
        s->agent_poses[3 * i] = s->state[7 * i];
        s->agent_poses[3 * i + 1] = s->state[7 * i + 1];
        s->agent_poses[3 * i + 2] = s->state[7 * i + 4];
    }
    /* :536-550 check_collision — length/width are Simulator.params' (the constructor dict) */
    double verts[8 * 16] = { 0 };
    double *vp = A <= 16 ? verts : (double *)malloc(sizeof(double) * 8 * A);
    for (int i = 0; i < A; i++)
        orc_get_vertices(s->agent_poses + 3 * i, s->sim_length, s->sim_width, vp + 8 * i);
    orc_collision_multiple(vp, A, s->collisions, s->collision_idx);
    if (vp != verts) free(vp);
    /* :579-589 */
    for (int i = 0; i < A; i++) {
        double *st = s->state + 7 * i;
        double *scan = s->scans + (size_t)i * B;
        /* update_scan :428-449 -> check_ttc :229-254 */
        int hit = orc_check_ttc(scan, B, st[3], s->cosines, s->side_distances, s->ttc_thresh);
        if (hit) { st[3] = 0.; st[4] = 0.; st[5] = 0.; st[6] = 0.; }
        s->in_collision[i] = hit;
        memcpy(s->scans_pre + (size_t)i * B, scan, sizeof(double) * B);
        /* ray_cast_agents :206-227 (opponent vertices use this agent's own length/width) */
        const double *p = s->params + ORC_NPARAM * i;
        double pose[3] = { st[0], st[1], st[4] };
        for (int j = 0; j < A; j++) {
            if (j == i) continue;
            double ov[8];
            orc_get_vertices(s->agent_poses + 3 * j, p[P_LENGTH], p[P_WIDTH], ov);
            orc_ray_cast(pose, scan, s->scan_angles, B, ov);
        }
        if (hit) s->collisions[i] = 1.;
    }
}

/* f110_env.py:204-246 _check_done (after :294-298 time/state update). returns done. */
int orc_env_post_step(orc_sim_t *s) {
    int A = s->num_agents;
    const double left_t = 2, right_t = 2;
    s->current_time = s->current_time + s->time_step;
    int all_done = 1;
    for (int i = 0; i < A; i++) {
        double px = s->state[7 * i] - s->start_xs[i];
        double py = s->state[7 * i + 1] - s->start_ys[i];
        double dx = s->start_rot[0] * px + s->start_rot[1] * py;
        double ty = s->start_rot[2] * px + s->start_rot[3] * py;
        if (ty > left_t) ty -= left_t;
        else if (ty < -right_t) ty = -right_t - ty;
        else ty = 0;
        double dist2 = dx * dx + ty * ty;
        int close = dist2 <= 0.1;
        if (close && !s->near_starts[i]) { s->near_starts[i] = 1; s->toggle_list[i] += 1; }
        else if (!close && s->near_starts[i]) { s->near_starts[i] = 0; s->toggle_list[i] += 1; }
        s->lap_counts[i] = floor(s->toggle_list[i] / 2);
        if (s->toggle_list[i] < 4) s->lap_times[i] = s->current_time;
        if (!(s->toggle_list[i] >= 4)) all_done = 0;
    }
    return (s->collisions[s->ego_idx] != 0.) || all_done;
}

/* f110_env.py:306-349 F110Env.reset: counters, start frame, Simulator.reset, one zero-action step */
int orc_env_reset(orc_sim_t *s, const double *poses) {
    int A = s->num_agents;
    s->current_time = 0.0;
    for (int i = 0; i < A; i++) {
        s->near_starts[i] = 1; s->toggle_list[i] = 0.; s->collisions[i] = 0.;
        s->start_xs[i] = poses[3 * i]; s->start_ys[i] = poses[3 * i + 1]; s->start_thetas[i] = poses[3 * i + 2];
    }
    double th = -s->start_thetas[s->ego_idx];
    s->start_rot[0] = cos(th); s->start_rot[1] = -sin(th);
    s->start_rot[2] = sin(th); s->start_rot[3] = cos(th);
    orc_sim_reset(s, poses);
    double *zero = (double *)calloc(2 * A, sizeof(double));
    orc_sim_step(s, zero);
    free(zero);
    return orc_env_post_step(s);
}

/* The device auto-reset (include/f110_b200.h f110_autoreset) applied to one env: Simulator.reset to `poses`, the env
 * counters and start frame of F110Env.reset (f110_env.py:319-331).  Unlike orc_env_reset there is no zero-action step,
 * and `done` and the collision observation of the tick that ended the episode stay as they are. */
void orc_env_restart(orc_sim_t *s, const double *poses /* [A][3] */) {
    int A = s->num_agents;
    s->current_time = 0.0;
    for (int i = 0; i < A; i++) {
        s->near_starts[i] = 1; s->toggle_list[i] = 0.;
        s->start_xs[i] = poses[3 * i]; s->start_ys[i] = poses[3 * i + 1]; s->start_thetas[i] = poses[3 * i + 2];
    }
    double th = -s->start_thetas[s->ego_idx];
    s->start_rot[0] = cos(th); s->start_rot[1] = -sin(th);
    s->start_rot[2] = sin(th); s->start_rot[3] = cos(th);
    orc_sim_reset(s, poses);
}

/* ------------------------------------------------------------------ batched step (large-batch parity tests)
 * Steps n independent sims once each: sims[e] with actions + e*A*2 and, when `noise` is not NULL, the additive scan noise
 * noise + e*A*B; env_level != 0 also runs orc_env_post_step (result in `done`).  pthreads over envs, like orc_rollout. */
typedef struct {
    orc_sim_t **sims; int e0, e1, env_level; const double *actions, *noise;
} batch_job_t;

static void *batch_worker(void *arg) {
    batch_job_t *jb = (batch_job_t *)arg;
    for (int e = jb->e0; e < jb->e1; e++) {
        orc_sim_t *s = jb->sims[e];
        const size_t A = (size_t)s->num_agents, B = (size_t)s->num_beams;
        s->noise = jb->noise ? jb->noise + (size_t)e * A * B : NULL;
        orc_sim_step(s, jb->actions + (size_t)e * A * 2);
        s->noise = NULL;
        if (jb->env_level) s->done = orc_env_post_step(s);
    }
    return NULL;
}

/* nthreads <= 0 -> one thread per online core.  Every sim of one call must have the same num_agents / num_beams. */
void orc_step_batch(orc_sim_t **sims, int n, const double *actions /* [n][A][2] */, const double *noise /* [n][A][B] or NULL */,
                    int env_level, int nthreads) {
    if (n <= 0) return;
    if (nthreads <= 0) nthreads = (int)sysconf(_SC_NPROCESSORS_ONLN);
    if (nthreads > n) nthreads = n;
    if (nthreads < 1) nthreads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * nthreads);
    batch_job_t *jobs = (batch_job_t *)calloc(nthreads, sizeof(batch_job_t));
    for (int t = 0; t < nthreads; t++) {
        jobs[t].sims = sims; jobs[t].env_level = env_level; jobs[t].actions = actions; jobs[t].noise = noise;
        jobs[t].e0 = (int)((int64_t)n * t / nthreads);
        jobs[t].e1 = (int)((int64_t)n * (t + 1) / nthreads);
        pthread_create(&th[t], NULL, batch_worker, &jobs[t]);
    }
    for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
    free(th); free(jobs);
}

/* Copies one field of n sims into a contiguous array (per sim: A values, A*7 for the state, A*B for the scans, one for
 * done and current_time), so that a test can compare a whole batch with one array operation. */
enum { ORC_F_STATE = 0, ORC_F_SCANS, ORC_F_SCANS_PRE, ORC_F_COLLISIONS, ORC_F_COLLISION_IDX, ORC_F_IN_COLLISION,
       ORC_F_LAP_TIMES, ORC_F_LAP_COUNTS, ORC_F_TOGGLE_LIST, ORC_F_DONE, ORC_F_CURRENT_TIME, ORC_F_NLOOK };
void orc_gather(orc_sim_t **sims, int n, int field, double *out) {
    for (int e = 0; e < n; e++) {
        orc_sim_t *s = sims[e];
        const size_t A = (size_t)s->num_agents, B = (size_t)s->num_beams;
        switch (field) {
            case ORC_F_STATE: memcpy(out + e * A * 7, s->state, sizeof(double) * A * 7); break;
            case ORC_F_SCANS: memcpy(out + e * A * B, s->scans, sizeof(double) * A * B); break;
            case ORC_F_SCANS_PRE: memcpy(out + e * A * B, s->scans_pre, sizeof(double) * A * B); break;
            case ORC_F_COLLISIONS: memcpy(out + e * A, s->collisions, sizeof(double) * A); break;
            case ORC_F_COLLISION_IDX: memcpy(out + e * A, s->collision_idx, sizeof(double) * A); break;
            case ORC_F_IN_COLLISION: for (size_t i = 0; i < A; i++) out[e * A + i] = (double)s->in_collision[i]; break;
            case ORC_F_LAP_TIMES: memcpy(out + e * A, s->lap_times, sizeof(double) * A); break;
            case ORC_F_LAP_COUNTS: memcpy(out + e * A, s->lap_counts, sizeof(double) * A); break;
            case ORC_F_TOGGLE_LIST: memcpy(out + e * A, s->toggle_list, sizeof(double) * A); break;
            case ORC_F_DONE: out[e] = (double)s->done; break;
            case ORC_F_CURRENT_TIME: out[e] = s->current_time; break;
            case ORC_F_NLOOK: out[e] = (double)s->nlook; break;
        }
    }
}

/* ------------------------------------------------------------------ batched CPU-baseline driver
 * Used by bench.py (cpu_baseline / --impl reference).  Runs `num_envs` independent Simulators for
 * `ticks` ticks with the benchmark policy (SURVEY.md 8d): i.i.d. uniform random actions, auto-reset
 * to a sampled start pose when the ego collides.  pthreads over envs (the reference itself is
 * single-threaded; independent envs spread over the host cores is the fair mapping).  Returns total agent-steps performed. */
static inline uint64_t splitmix64(uint64_t *s) {
    uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static inline double u01(uint64_t *s) { return (double)(splitmix64(s) >> 11) * (1.0 / 9007199254740992.0); }

typedef struct {
    orc_sim_t **sims; int e0, e1, ticks; const double *start_poses; int num_start, pose_gap;
    uint64_t seed; int64_t total, nlook;
} rollout_job_t;

static void *rollout_worker(void *arg) {
    rollout_job_t *jb = (rollout_job_t *)arg;
    for (int e = jb->e0; e < jb->e1; e++) {
        orc_sim_t *s = jb->sims[e];
        int A = s->num_agents;
        uint64_t rng = jb->seed + 0x1234567ull * (uint64_t)(e + 1);
        double act[2 * 16], poses[3 * 16];
        int64_t n0 = s->nlook;
        for (int t = 0; t < jb->ticks; t++) {
            for (int i = 0; i < A; i++) {
                act[2 * i] = -0.4189 + 0.8378 * u01(&rng);
                act[2 * i + 1] = 8.0 * u01(&rng);
            }
            orc_sim_step(s, act);
            if (s->collisions[s->ego_idx] != 0.) {
                int k = (int)(u01(&rng) * jb->num_start);
                if (k >= jb->num_start) k = jb->num_start - 1;
                for (int i = 0; i < A; i++) {
                    int kk = ((k - jb->pose_gap * i) % jb->num_start + jb->num_start) % jb->num_start;
                    poses[3 * i] = jb->start_poses[3 * kk];
                    poses[3 * i + 1] = jb->start_poses[3 * kk + 1];
                    poses[3 * i + 2] = jb->start_poses[3 * kk + 2];
                }
                orc_sim_reset(s, poses);
            }
            jb->total += A;
        }
        jb->nlook += s->nlook - n0;
    }
    return NULL;
}

/* num_threads <= 0 -> one thread per online core */
int64_t orc_rollout(orc_sim_t **sims, int num_envs, int ticks, const double *start_poses /* [K][3] */,
                    int num_start, int pose_gap, uint64_t seed, int num_threads, int64_t *nlook_out) {
    if (num_threads <= 0) num_threads = (int)sysconf(_SC_NPROCESSORS_ONLN);
    if (num_threads > num_envs) num_threads = num_envs;
    if (num_threads < 1) num_threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * num_threads);
    rollout_job_t *jobs = (rollout_job_t *)calloc(num_threads, sizeof(rollout_job_t));
    for (int t = 0; t < num_threads; t++) {
        jobs[t].sims = sims; jobs[t].ticks = ticks; jobs[t].start_poses = start_poses;
        jobs[t].num_start = num_start; jobs[t].pose_gap = pose_gap; jobs[t].seed = seed;
        jobs[t].e0 = (int)((int64_t)num_envs * t / num_threads);
        jobs[t].e1 = (int)((int64_t)num_envs * (t + 1) / num_threads);
        pthread_create(&th[t], NULL, rollout_worker, &jobs[t]);
    }
    int64_t total = 0, nlook = 0;
    for (int t = 0; t < num_threads; t++) {
        pthread_join(th[t], NULL);
        total += jobs[t].total; nlook += jobs[t].nlook;
    }
    free(th); free(jobs);
    if (nlook_out) *nlook_out = nlook;
    return total;
}

int orc_num_cores(void) { return (int)sysconf(_SC_NPROCESSORS_ONLN); }

/* ------------------------------------------------------------------ pure-pursuit planner (SURVEY 8f row 4)
 * examples/waypoint_follow.py (paths relative to /root/reference/examples/):
 *   nearest_point_on_trajectory :15-47, first_point_on_trajectory_intersecting_circle :49-131,
 *   get_actuation :133-144, PurePursuitPlanner._get_current_waypoint :183-202, .plan :204-217.
 * wx, wy, wv: waypoint x, y, speed columns [n].  out[0] = speed, out[1] = steering angle. */
void orc_pure_pursuit(const double *wx, const double *wy, const double *wv, int n, double pose_x, double pose_y,
                      double pose_theta, double lookahead_distance, double vgain, double wheelbase,
                      double max_reacquire, double *out) {
    /* nearest_point_on_trajectory */
    int best = 0;
    double best_d = 0, best_t = 0;
    for (int i = 0; i < n - 1; i++) {
        double dx = wx[i + 1] - wx[i], dy = wy[i + 1] - wy[i];
        double l2 = dx * dx + dy * dy;
        double dot = (pose_x - wx[i]) * dx + (pose_y - wy[i]) * dy;
        double t = dot / l2;
        if (t < 0.0) t = 0.0;
        if (t > 1.0) t = 1.0;
        double px = wx[i] + t * dx, py = wy[i] + t * dy;
        double ex = pose_x - px, ey = pose_y - py;
        double d = sqrt(ex * ex + ey * ey);
        if (i == 0 || d < best_d) { best_d = d; best = i; best_t = t; }
    }
    double lx, ly, lv;
    int have = 0;
    if (best_d < lookahead_distance) {
        /* first_point_on_trajectory_intersecting_circle(position, L, wpts, i + t, wrap=True) */
        double tt = (double)best + best_t;
        int start_i = (int)tt;
        double start_t = fmod(tt, 1.0);
        int first_i = -1000000;
        for (int i = start_i; i < n - 1 && first_i == -1000000; i++) {
            double sx = wx[i], sy = wy[i];
            double Vx = (wx[i + 1] + 1e-6) - sx, Vy = (wy[i + 1] + 1e-6) - sy;
            double a = Vx * Vx + Vy * Vy;
            double b = 2.0 * (Vx * (sx - pose_x) + Vy * (sy - pose_y));
            double c = (sx * sx + sy * sy) + (pose_x * pose_x + pose_y * pose_y) - 2.0 * (sx * pose_x + sy * pose_y) -
                       lookahead_distance * lookahead_distance;
            double disc = b * b - 4 * a * c;
            if (disc < 0) continue;
            disc = sqrt(disc);
            double t1 = (-b - disc) / (2.0 * a), t2 = (-b + disc) / (2.0 * a);
            if (i == start_i) {
                if (t1 >= 0.0 && t1 <= 1.0 && t1 >= start_t) first_i = i;
                else if (t2 >= 0.0 && t2 <= 1.0 && t2 >= start_t) first_i = i;
            } else if (t1 >= 0.0 && t1 <= 1.0) first_i = i;
            else if (t2 >= 0.0 && t2 <= 1.0) first_i = i;
        }
        if (first_i == -1000000) {
            for (int i = -1; i < start_i && first_i == -1000000; i++) {
                int i0 = ((i % n) + n) % n, i1 = (((i + 1) % n) + n) % n;
                double sx = wx[i0], sy = wy[i0];
                double Vx = (wx[i1] + 1e-6) - sx, Vy = (wy[i1] + 1e-6) - sy;
                double a = Vx * Vx + Vy * Vy;
                double b = 2.0 * (Vx * (sx - pose_x) + Vy * (sy - pose_y));
                double c = (sx * sx + sy * sy) + (pose_x * pose_x + pose_y * pose_y) - 2.0 * (sx * pose_x + sy * pose_y) -
                           lookahead_distance * lookahead_distance;
                double disc = b * b - 4 * a * c;
                if (disc < 0) continue;
                disc = sqrt(disc);
                double t1 = (-b - disc) / (2.0 * a), t2 = (-b + disc) / (2.0 * a);
                if (t1 >= 0.0 && t1 <= 1.0) first_i = i;
                else if (t2 >= 0.0 && t2 <= 1.0) first_i = i;
            }
        }
        if (first_i != -1000000) {
            /* current_waypoint[0:2] = wpts[i2, :] (python negative index -1 -> last row); speed from row i */
            int i2 = first_i < 0 ? first_i + n : first_i;
            lx = wx[i2]; ly = wy[i2]; lv = wv[best]; have = 1;
        }
    } else if (best_d < max_reacquire) {
        lx = wx[best]; ly = wy[best]; lv = wv[best]; have = 1;
    }
    if (!have) { out[0] = 4.0; out[1] = 0.0; return; }
    /* get_actuation */
    double waypoint_y = sin(-pose_theta) * (lx - pose_x) + cos(-pose_theta) * (ly - pose_y);
    double speed = lv, steer;
    if (fabs(waypoint_y) < 1e-6) steer = 0.;
    else {
        double radius = 1 / (2.0 * waypoint_y / (lookahead_distance * lookahead_distance));
        steer = atan(wheelbase / radius);
    }
    out[0] = vgain * speed;
    out[1] = steer;
}
