// rb_world.cuh -- device-resident world: SoA tables in HBM (layout described in DESIGN.md §3).
//
// Bodies, colliders, persistent contact pairs and per-step constraint rows are structure-of-arrays
// of float4 "rows" (16-byte aligned, coalesced across the index).  Multi-row records are stored
// row-major: element (row r, index i) lives at table[r * cap + i], so a warp reading row r of 32
// consecutive records issues one 512-byte coalesced request.
#pragma once
#include "rb_math.cuh"

namespace rb {

constexpr int MAX_PTS = 4;              // MAX_MANIFOLD_POINTS, src/lib.rs:291
constexpr int MAX_RAW = 8;              // clipped quad/quad polygon
constexpr int COLOR_UNCOLORED = 255;    // contact_pair.rs:152
constexpr int COLOR_OVERFLOW = 128;     // contact_pair.rs:155
constexpr int DYN_COLOR_COUNT = 120;    // contact_pair.rs:159
constexpr int NUM_COLORS = 129;
constexpr int NO_BODY = -1;             // world-attached side (reference: u32::MAX)

constexpr int BODY_DYNAMIC = 0;
constexpr int BODY_FIXED = 1;
constexpr int BODY_KIN_POS = 2, BODY_KIN_VEL = 3;   // RigidBodyType::{KinematicPositionBased, KinematicVelocityBased} (rigid_body_components.rs:20-46)
constexpr int BODY_REMOVED = 7;          // removed (rb_world_remove_bodies) or quarantined: not simulated, its colliders are gone
constexpr int SHAPE_BALL = 0, SHAPE_CUBOID = 1;
constexpr int SHAPE_CAPSULE = 2;         // half extents = (half height of the segment, radius, axis 0 | 1 | 2)
constexpr int SHAPE_CONVEX = 3;          // convex polyhedron: half extents = (hull id, border radius, 0)
constexpr int HULL_MAX_VERTS = 32, HULL_MAX_FACES = 32, HULL_MAX_FACE_VERTS = 8, HULL_MAX_EDGES = 64;
constexpr int SHAPE_REMOVED = -1;        // collider of a removed body: in neither broad-phase list, in no pair
constexpr unsigned FLAG_GYRO = 1, FLAG_FAST_ROT = 2, FLAG_LTX = 4, FLAG_LTY = 8, FLAG_LTZ = 16, FLAG_LRX = 32,
                   FLAG_LRY = 64, FLAG_LRZ = 128, FLAG_NO_SLEEP = 256, FLAG_CCD = 512;

// Convex polyhedra shared by colliders (rb_world_add_hull); hull 0 is the unit cube, whose topology a cuboid borrows
// when it meets a polyhedron (rb_poly.cuh).  Read-only on the device.
struct HullTables {
    const int4* desc;      // per hull: first vertex, vertex count, first face, face count
    const int4* desc2;     // per hull: first edge, edge count, first loop entry, 0
    const float4* info;    // per hull: max |x|, |y|, |z| over the vertices (local AABB about the origin), bounding radius about the origin
    const float4* verts;   // xyz
    const float4* planes;  // outward unit normal, offset
    const int2* faces;     // start in the hull's loop entries, vertex count (counter-clockwise seen from outside)
    const int* loops;      // vertex indices (hull-local)
    const int4* edges;     // v0, v1, the face on which the edge runs v0 -> v1, the other face
};

// ---- persistent pair record rows (float4 each) ----
enum PairRow {
    PR_INFO = 0,   // int bits: x flags(bit0 has_recycle, bit1 pending colour, bit2 colouring scratch, bit3 force event emitted last step, bit4 sensor pair intersecting), y npts, z nsc, w colour
    PR_BODIES,     // int bits: x colour_body0, y colour_body1, z body1, w body2 (-1 none)
    PR_RT,         // recycle pos12.t xyz, w max_extent
    PR_RQ,         // recycle pos12.q
    PR_ROT1,       // recycle rot1
    PR_ROT2,       // recycle rot2
    PR_LN1,        // local_n1 xyz, w max_drift
    PR_LN2,        // local_n2 xyz, w restitution
    PR_NORMAL,     // world normal xyz, w friction
    PR_PA,         // [4] local_p1 xyz, w dist
    PR_PB = PR_PA + MAX_PTS,    // [4] local_p2 xyz, w fid1 bits
    PR_PD = PR_PB + MAX_PTS,    // [4] impulse, warmstart_impulse, warmstart_twist, fid2 bits
    PR_TW = PR_PD + MAX_PTS,    // [4] warmstart_tangent_world xyz
    PR_DP1 = PR_TW + MAX_PTS,   // [4] solver_dp1 xyz
    PR_DP2 = PR_DP1 + MAX_PTS,  // [4] solver_dp2 xyz
    PR_A1 = PR_DP2 + MAX_PTS,   // [4] anchor1 xyz, w cid bits
    PR_A2 = PR_A1 + MAX_PTS,    // [4] anchor2 xyz
    PR_ROWS = PR_A2 + MAX_PTS
};

// ---- per-step constraint record rows (float4 each), index = slot in the schedule ----
enum ConsRow {
    CR_DIR = 0,                 // dir1 xyz, w friction limit
    CR_T1,                      // tangent1 xyz, w twist r
    CR_DP1,                     // [4] dp1 xyz, w r (projected mass)
    CR_DP2 = CR_DP1 + MAX_PTS,  // [4] dp2 xyz, w dist0
    CR_LP1 = CR_DP2 + MAX_PTS,  // [4] builder local_p1 xyz, w restitution seed
    CR_LP2 = CR_LP1 + MAX_PTS,  // [4] builder local_p2 xyz
    CR_TDP1 = CR_LP2 + MAX_PTS, // tangent dp1 xyz, w r[0]
    CR_TDP2,                    // tangent dp2 xyz, w r[1]
    CR_LFC1,                    // local friction centre 1 xyz, w r[2]
    CR_LFC2,                    // local friction centre 2 xyz
    CR_TWD,                     // twist_dists[4]
    CR_IMP,                     // normal impulses[4]            (read-modify-write)
    CR_ACC,                     // normal impulse accumulators[4] (read-modify-write)
    CR_TI,                      // tangent impulse xy, accumulators zw (read-modify-write)
    CR_WI,                      // twist impulse x, accumulator y       (read-modify-write)
    // FrictionModel::Coulomb only (one coupled tangent part per point, contact_constraint_element.rs:14-36)
    CR_PTI,                     // [4] tangent impulse xy, accumulators zw of point k   (read-modify-write)
    CR_PTK = CR_PTI + MAX_PTS,  // [4] tangent K of point k: r0 r1 r2
    CR_ROWS = CR_PTK + MAX_PTS
};

struct Params {  // IntegrationParameters + derived per-substep coefficients (computed on the host)
    float dt, inv_dt_full, sub_dt, sub_inv_dt;
    float dyn_cfm, static_cfm, dyn_erp, static_erp;
    float max_corrective_velocity, warmstart_coeff;
    float prediction, recycle_dist, length_unit, fat_skin;
    float max_lin_vel, max_ang_vel;
    int num_substeps, num_pgs, num_relax, friction_in_bias, contact_recycling;
    int ccd;              // max_ccd_substeps != 0: motion clamping of fast bodies (substep.rs:404-409, :492-520)
    float linear_slop;    // allowed_linear_error(): target distance of the time of impact (ccd_solver.rs:184)
    int friction_model;   // 0 = Simplified (twist), 1 = Coulomb (integration_parameters.rs:16-30)
    int warmstart_joints; // joint rows carry their impulses (integration_parameters.rs:300); served by the generic joint path
};

// Device-side scalars (one struct in HBM, mirrored to pinned host memory on demand).
constexpr int ORDER_BUCKETS = 4096;   // item cost classes of the launch-order counting sort

struct State {
    int cur;               // which PairBuf is live (0/1)
    int npairs;
    int bp_dirty;          // a fat AABB changed: the pair set must be recomputed
    int sched_dirty;       // touching set changed: colours / islands / schedule must be rebuilt
    int ntodo;             // pairs that began touching this step
    int ncand;             // broad-phase candidates
    int ncons;             // solver-active manifolds
    int nitems;            // work items (item 0 = large islands)
    int nused_colors;      // colours in the contact stage order
    int njused_colors;     // colours in the joint stage order
    int nlarge_cons, nlarge_joints, nlarge_bodies;
    int error;             // RbStatus raised on the device (capacity, non-finite)
    int nislands;
    int bp_ran, sched_ran; // set when the corresponding section ran in the last step
    int any_bouncy;
    int need_big;          // some shared-memory item does not fit resident in the small launch shape (accumulated per step)
    int coop_streamed, coop_resident;   // shared-memory items of the last step: streamed from the pool / resident
    int norder;            // entries of World::item_order (non-empty items 1.., by decreasing cost)
    int cursor_rest, cursor_coop;   // dynamic work queues of the two kernels over item_order
    // broad phase: collider lists (rebuilt when lists_dirty) and scratch of the last run
    int lists_dirty;       // the static / dynamic collider lists must be rebuilt (scene upload, insertion, teleported fixed body)
    int ndyn, nstat, nwide; // movers, narrow static colliders (sorted by min-x), wide static colliders
    int stat_sorted;       // which of World::stat_key holds the sorted static keys
    int stat_count;        // all static colliders
    float stat_wsum;       // sum of their widths along x (classification threshold)
    unsigned stat_wn_bits; // widest narrow static collider along x (float bits)
    int bp_diff;           // the candidate pair set differs from the pair table
    int wake_any;          // a contact began with a sleeping body this step: run the wake pass
    int sleep_stamp;       // step counter of the sleep decision (isl_block holds the stamp of the last veto)
    unsigned mov_wz_bits, mov_wx_bits;   // widest mover along z / x of the last broad-phase run (float bits)
    int nquarantine;       // bodies quarantined since the host last read the list (non-finite state)
    int nccd;              // fast bodies queued for CCD motion clamping by the last solve (World::ccd_list)
    int ccd_total;         // fast bodies queued since the scene was uploaded (diagnostic)
    int nccd_bullets;      // ... of which bullets (ccd_enabled): they sweep in a second pass, against the already clamped poses
    int nev_coll, nev_force;   // buffered collision / contact-force events since the host last drained them
    int nconvex;           // polyhedron pairs whose manifold the warps compute together this step (World::convex_work)
};

struct PairBuf {
    unsigned long long* key;  // (collider1 << 32) | collider2, sorted ascending
    float4* rows;             // [PR_ROWS][pair_cap]
};

struct World {
    int nb, nc, nj;
    int pair_cap, cons_cap, item_cap, joint_cap;
    Params prm;
    State* st;
    // ---- bodies ----
    int* b_type;
    unsigned* b_flags;
    float4 *b_pos_t, *b_pos_q;        // RigidBodyPosition::position
    float4 *b_linvel, *b_angvel;
    float4 *b_next_t, *b_next_q;      // RigidBodyPosition::next_position of position-based kinematic bodies (the user's target)
    int* kinpos_list;                 // [nkinpos] the position-based kinematic bodies
    int nkinpos;
    float4* b_lcom_im;                // local_com xyz, w inv_mass
    float4 *b_ipi, *b_pi, *b_pframe;  // inverse principal inertia (w: max_extent), principal inertia, principal frame
    float4* b_misc;                   // linear damping, angular damping, gravity scale, ccd_thickness
    float4 *b_uforce, *b_utorque;
    float4* b_wcom;                   // world_com
    float4* b_eim;                    // effective_inv_mass
    float4* b_eii0;                   // effective_world_inv_inertia xx xy xz yy
    float2* b_eii1;                   //                              yz zz
    unsigned char* b_owned;           // multi-GPU sharding: 1 = simulated here, 2 = tracked halo, 0 = far foreign body
    // sleeping (RigidBodyActivation, rigid_body_components.rs:1296-1326)
    unsigned char* b_sleeping;        // 1 = asleep: not in the active set
    float* b_sleep_time;              // time_since_can_sleep
    float4 *b_sleep_prev_t, *b_sleep_prev_q;   // pose at the previous sleep check
    float* b_max_extent;              // mprops.max_extent: farthest shape point from the local centre of mass
    float* b_ccd_thick;               // RigidBodyCcd::ccd_thickness: thinnest extent over the body's colliders (FLT_MAX without colliders)
    int* b_col_head;                  // [nb] first collider of the body (-1 none); the chain continues through c_next
    int* c_next;                      // [nc] next collider of the same body (-1 end)
    int* ccd_list;                    // [nb] bodies queued for motion clamping (State::nccd entries)
    float4 *ccd_start_t, *ccd_start_q;   // [nb] their pose at the start of the step (RigidBodyPosition::position)
    int* wake_req;                    // [nb] by island root: wake this island (a contact began)
    int* isl_block;                   // [nb] by island root: stamp of the last step a body of the island was not sleep-eligible
    int sleep_enabled;                // some body may sleep: run the sleep decision
    int* quarantine;                  // [nb] bodies disabled because their state went non-finite (Quarantine::bodies)
    // solver bodies (global-memory path) + per-substep increments
    float4 *s_lin, *s_ang, *s_q, *s_t, *s_incr_lin, *s_incr_ang;
    float* state13;                   // packed [nb][13] t q lin ang (download / NCCL all-gather)
    // ---- colliders ----
    int* c_shape;
    int* c_parent;
    float4 *c_he, *c_rel_t, *c_rel_q;
    float4* c_mat;                    // friction, restitution, contact_skin
    int2* c_rules;
    uint2* c_groups;
    int* c_events;                    // ActiveEvents bits (1 = collision events, 2 = contact force events) | 4 = the collider is a sensor
    int has_sensors;                  // some collider is a sensor (Collider::is_sensor): intersection-only pairs exist
    float* c_force_thr;               // contact_force_event_threshold
    float4 *c_pos_t, *c_pos_q;
    float4 *c_aabb_min, *c_aabb_max, *c_fat_min, *c_fat_max;
    // ---- broad phase scratch ----
    int* dyn_list;                    // [nc] colliders that can move
    int* wide_list;                   // [WIDE_CAP] static colliders much wider than the rest
    unsigned long long* dyn_key[2];   // [nc] (sortable min-x << 32) | collider of the movers, radix-sort ping-pong
    unsigned long long* stat_key[2];  // [nc] ... of the narrow static colliders, sorted once
    float4 *dyn_smin, *dyn_smax;      // [nc] fat AABBs of the movers in sorted order (coalesced sweep)
    int* radix_hist;                  // [9][grid blocks][256] digit counts of the radix sorts
    unsigned long long* cand_key;     // [pair_cap] candidate pairs (collider1 << 32) | collider2
    unsigned long long* cand_key2;    // [pair_cap] radix-sort ping-pong
    unsigned long long* nocontact_keys;  // sorted body-pair keys of joints with contacts disabled
    int n_nocontact;
    int* remap_src;                   // [pair_cap] new pair -> old pair index or -1
    // ---- events (EventHandler): appended by the step, drained by the host ----
    int4* ev_coll;                    // [ev_cap] collider1, collider2, started, step
    float4* ev_force;                 // [3][ev_cap] (c1, c2, started, step as int bits) | total force xyz, magnitude | max direction xyz, max magnitude
    int ev_cap;
    int step_index;                   // index of the step being enqueued (1 = first step after the scene upload)
    // ---- pairs ----
    PairBuf pb[2];
    int* todo;                        // [pair_cap] pairs that began touching this step
    unsigned* color_mask;             // [nb][4] 128-bit colour masks per body
    int* body_min;                    // [nb] colouring scratch (INT_MAX when idle)
    unsigned long long* body_minkey;  // [nb] colouring scratch: smallest pending order key (~0 when idle)
    // ---- islands / schedule ----
    int* isl_label;                   // [nb] union-find parent / final root
    int* isl_nb;                      // [nb] bodies per root
    int* isl_ncons;                   // [nb] contact manifolds + joints per root
    int* isl_item;                    // [nb] work item of a root
    int* scan_tmp;                    // [nb + 1025]
    int* item_body_start;             // [item_cap + 1]
    int* item_cons_start;             // [item_cap + 1]
    int* item_joint_start;            // [item_cap + 1]
    int* item_cursor;                 // [3 * (item_cap + 1)] scatter cursors
    int* item_flags;                  // [item_cap + 1] per-item flags of the current step
    int* item_bodies;                 // [nb] global body ids grouped by item
    int* body_local;                  // [nb] index of a body inside its item
    int* body_item;                   // [nb] item of a body
    int* cons_pair_tmp;               // [cons_cap] pair index grouped by item (unsorted)
    int* cons_pair;                   // [cons_cap] pair index in schedule order
    int* item_color_off;              // [item_cap][NUM_COLORS + 1] offsets relative to item_cons_start
    int* adj_off;                     // [nb] per item body slot: start of its contact adjacency in adj_list
    int* adj_cnt;                     // [nb] ... and its length
    int* adj_list;                    // [2 * cons_cap] item-local slot * 2 + side, ascending (= colour stage order)
    int* item_order;                  // [item_cap] non-empty items 1.., most expensive first (launch order of the solve CTAs)
    int* order_hist;                  // [2 * ORDER_BUCKETS + 1] counting-sort scratch of item_order
    int* color_count;                 // [NUM_COLORS] global histogram
    int* color_pos;                   // [NUM_COLORS] stage position of a colour, -1 unused
    int* joint_tmp;                   // [joint_cap]
    int* joint_sched;                 // [joint_cap] joint index in schedule order
    int* item_jcolor_off;             // [item_cap][NUM_COLORS + 1]
    int* jcolor_pos;                  // [NUM_COLORS] (host computed, static per scene)
    // ---- constraints ----
    int4* cons_hdr;                   // [cons_cap] pair, id1, id2, num_contacts (ids item-local or global)
    float4* cons;                     // [CR_ROWS][cons_cap]
    float4* large_pool;               // [COOP_ROWS][cons_cap] constant rows of the grid-wide item 0 (lane-cooperative form)
    float4* large_mut;                // [MR_COUNT][cons_cap] its impulses
    float4* coop_pool;                // [2 * COOP_ROWS * cons_cap] L2-resident constant rows of streamed items, blocked by chunk
    int coop_small_floats;            // dynamic shared memory of the small launch shape (2 CTAs / SM), which must fit every shared-memory item
    long long* dbg_times;             // [32] phase timestamps of one item (debug_flags & 2)
    int debug_flags;                  // RB_DEBUG_FLAGS, honoured only by the -DRB_DEBUG build: 1 = skip the sweeps, 2 = record dbg_times
    int* host_hint;                   // pinned, host-mapped words read by the host without synchronising: [0] last step's State::need_big,
                                      // [1] first status raised on the device since the host last cleared it (RbStatus; 0 = none)
                                      // [2] a grid-wide island exists, [3] CCD clamps are queued (applied by the next k_collide or synchronising call)
    // ---- joints ----
    int4* j_info;                     // body1, body2, locked_axes, colour
    float4 *j_f1_t, *j_f1_q, *j_f2_t, *j_f2_q;   // local frames
    float2* j_soft;                   // natural frequency, damping ratio
    float* j_impulses;                // [nj][6]
    float4* j_rows;                   // [JR_ROWS][6 * joint_cap] per-substep rows
    int4* j_sched_ids;                // [joint_cap] joint, id1, id2, nrows in schedule order
    // limits and motors of the free axes (JointLimits / JointMotor, generic_joint.rs:142-232): only worlds in which some joint
    // has any take the generic joint path (solve_item<HbmRows<FM, 1>>, 12 row slots per joint instead of 6)
    int generic_joints;
    // Substep solve-groups (RigidBody::additional_solver_iterations; island_manager/substep_groups.rs): any_extra = some
    // body asks for extra substeps.  Then every island carries a key (max over its members, isl_key), the general solve
    // path is launched once per distinct key -- pass_key, with prm derived for num_solver_iterations + pass_key -- and each
    // launch takes the bodies / constraints / joints of the islands with that key (b_key, cons_key, j_key).
    int any_extra, pass_key;
    unsigned* isl_key;                // [nb] key of a root
    unsigned char *b_key, *cons_key, *j_key;   // [nb] [cons_cap] [joint_cap] key per body / scheduled constraint / scheduled joint
    HullTables hulls;                 // convex polyhedra (worlds with SHAPE_CONVEX colliders only; else null)
    int* convex_work;                 // [pair_cap] pairs of this step that need a polyhedron manifold (phase_convex_manifolds)
    float* convex_raw;                // [pair_cap][POLY_RAW_STRIDE] their raw manifolds, read back by the per-pair narrow phase
    uint2* j_axes;                    // limit_axes, motor_axes
    float2* j_limits;                 // [nj][6] min, max
    float4* j_motor_a;                // [nj][6] target_vel, target_pos, stiffness, damping
    float2* j_motor_b;                // [nj][6] max_force, model (int bits)
    float4* j_anglim;                 // [nj][3] AngularLimitParams: cos, sin of half the centre angle, half range
    float4* j_bnd;                    // [12 * joint_cap] per generic row: impulse bounds lo hi, dof (int bits), WritebackId kind (int bits)
    float *j_limit_impulses, *j_motor_impulses;   // [nj][6]
};

// joint row record (float4 rows), index = 6 * schedule slot + row
enum JointRowRec {
    JR_LIN = 0,   // lin_jac xyz, w impulse
    JR_A1,        // ang_jac1 xyz, w inv_lhs
    JR_A2,        // ang_jac2 xyz, w rhs
    JR_IA1,       // ii_ang_jac1 xyz, w rhs_wo_bias
    JR_IA2,       // ii_ang_jac2 xyz, w cfm_gain
    JR_ROWS
};

RB_HD float4& prow(const World& w, int buf, int row, int i) { return w.pb[buf].rows[(size_t)row * w.pair_cap + i]; }
RB_HD float4& crow(const World& w, int row, int i) { return w.cons[(size_t)row * w.cons_cap + i]; }
RB_HD float4& jrow(const World& w, int row, int i) { return w.j_rows[(size_t)row * (6 * w.joint_cap) + i]; }

RB_HD sym3 load_ii(const World& w, int b) {
    float4 a = w.b_eii0[b];
    float2 c = w.b_eii1[b];
    sym3 m; m.xx = a.x; m.xy = a.y; m.xz = a.z; m.yy = a.w; m.yz = c.x; m.zz = c.y;
    return m;
}

}  // namespace rb
