/*
 * collider_oracle.h -- CPU restatement of the boundaries: the signed-distance collider and the analytic collision objects
 * (DESIGN.md sections 2.4 and 2.9).  TEST INFRASTRUCTURE ONLY.
 *
 * The collider is SignedDistanceGrid, Projects/MGSP/boundary_condition.cuh:25-250, applied in the grid update as the MGSP form of
 * update_grid_velocity_query_max does (Projects/MGSP/mgmpm_kernels.cuh:323-399).  The objects are closed-form shapes in the
 * collider's material space, with its boundary types, friction and motion model: one response serves both, over the level
 * set's query or the shape's.  The grid update resolves the collider first, then the objects in list order.  Built into its
 * own library (oracle/libclaymore_collider_oracle.so, oracle/collider.mk) together with the oracle it extends
 * (claymore_oracle.c), whose grid update and sub-step it runs with the boundaries and a simulated-time clock.  The response is
 * pinned bit for bit against the reference's own detect_and_resolve_collision compiled for the host
 * (oracle/ref_collider_host.cpp).
 */
#ifndef COLLIDER_ORACLE_H
#define COLLIDER_ORACLE_H
#include "claymore_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* BoundaryT (boundary_condition.cuh:18-22) and the SignedDistanceGrid members (:28-35), layout of cb200_collider.  sdf: host
 * field, G^3 blocks of 4 channels x 64 cells (distance, gradient x, y, z), blocks row-major; rot_mat in vec3x3 storage
 * (element (i, j) at 3*i+j). */
enum { ORC_STICKY = 0, ORC_SLIP = 1, ORC_SEPARATE = 2 };
typedef struct orc_collider {
	const float* sdf;
	float rot_mat[9];
	float trans[3], trans_vel[3], omega[3];
	float dsdt, scale, friction;
	int type;
} orc_collider;

/* layout of cb200_collision_object: the shape (a, b: its two vectors, see claymore_b200.objects; a plane's normal of unit
 * length, as cb200_sim_set_collision_objects stores it) and the collider's motion fields */
enum { ORC_SHAPE_PLANE = 0, ORC_SHAPE_BOX = 1, ORC_SHAPE_SPHERE = 2, ORC_SHAPE_CYLINDER = 3 };
typedef struct orc_collision_object {
	int shape, type;
	float friction;
	float a[3], b[3];
	float rot_mat[9];
	float trans[3], trans_vel[3], omega[3];
	float dsdt, scale;
} orc_collision_object;

/* detect_and_resolve_collision (boundary_condition.cuh:159-249) of v[3] at grid node n[3] (= block*4 + cell) at time t */
void orc_collider_resolve(const orc_config* cfg, const orc_collider* col, float t, const int* node, float* v);
/* update_grid_velocity_query_max<.., Boundary>, Projects/MGSP/mgmpm_kernels.cuh:323-399, with the boundaries placed at `time`:
 * the collider col (NULL: none), then objs[0, n_objs).  The _collider form is the one with the collider alone. */
void orc_update_grid_velocity_query_max_collider(const orc_config* cfg, int block_count, float* grid, orc_partition part, float dt, const orc_collider* col, float time, float* max_vel);
void orc_update_grid_velocity_query_max_boundaries(const orc_config* cfg, int block_count, float* grid, orc_partition part, float dt, const orc_collider* col,
                                                   const orc_collision_object* objs, int n_objs, float time, float* max_vel);

/* The oracle's simulator with boundaries.  orc_csim_sim gives the orc_sim handle every orc_sim_* call of claymore_oracle.h
 * takes (of THIS library); orc_csim_step replaces orc_sim_step.  The boundaries are placed at the simulated time at the start
 * of each sub-step: the sum of the dt of the finished sub-steps, accumulated in double.  Without a collider and objects a
 * sub-step is orc_sim_step's.  sdf_host: distance, gradient x, y, z, each dense row-major over the (4G)^3 nodes
 * (init_from_signed_distance_file, boundary_condition.cuh:297-320); NULL keeps the field set before.  orc_csim_set_objects
 * copies the list; n = 0 clears it. */
typedef struct orc_csim orc_csim;
orc_csim* orc_csim_create(const orc_config* cfg, float dt_default, int max_blocks);
void orc_csim_destroy(orc_csim* c);
orc_sim* orc_csim_sim(orc_csim* c);
void orc_csim_set_collider(orc_csim* c, const orc_collider* params, const float* sdf_host);
void orc_csim_clear_collider(orc_csim* c);
void orc_csim_set_objects(orc_csim* c, const orc_collision_object* objs, int n);
void orc_csim_step(orc_csim* c, float time_left);
double orc_csim_time(orc_csim* c);

#ifdef __cplusplus
}
#endif
#endif
