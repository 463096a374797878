/*
 * collider_oracle.c -- see collider_oracle.h.  TEST INFRASTRUCTURE ONLY.
 * The oracle is compiled into this translation unit so that the grid update and sub-step below can use its simulator's state
 * (struct orc_sim) and its grid-update body; libclaymore_oracle.so itself is unchanged by it.
 */
#include "claymore_oracle.c"
#include "collider_oracle.h"

/* ---- signed-distance collider, Projects/MGSP/boundary_condition.cuh ------------------------------------------------------
 * Restated line by line on flat arrays; vec3x3 element (i, j) is stored at 3*i+j.  Fixed here: the object velocity takes a true
 * omega x r (vec3_cross_vec3 :92-95 adds all three products); the normal is normalised only when it is non-zero (:135 divides
 * 0 by 0); the +1 node of the trilinear stencil must lie in the domain; the max is |v|^2 (mgmpm_kernels.cuh:364-372 reports
 * 2|v|^2).  Kept: no hit inside the wall band (:138-143); get_material_velocity's vec_cross_mul_vec_3d (MatrixUtils.h:54-58). */
/* rot_angle_to_matrix :67-90 */
static void col_axis_rot(float a, int dim, float* r) {
	memset(r, 0, 9 * sizeof(float));
	if(dim == 0) {
		r[0] = 1;                   /* res(0, 0) = 1 */
		r[4] = r[8] = cosf(a);      /* res(1, 1) = res(2, 2) = cosf(omega) */
		r[7] = r[5] = sinf(a);      /* res(2, 1) = res(1, 2) = sinf(omega) */
		r[5] = -r[5];               /* res(1, 2) = -res(1, 2) */
	} else if(dim == 1) {
		r[4] = 1;
		r[0] = r[8] = cosf(a);
		r[6] = r[2] = sinf(a);
		r[6] = -r[6];
	} else {
		r[8] = 1;
		r[0] = r[4] = cosf(a);
		r[3] = r[1] = sinf(a);
		r[1] = -r[1];
	}
}
/* matrix_matrix_multiplication_3d, Library/MnBase/Math/Matrix/MatrixUtils.h:147-157 */
static void col_mat_mul(const float* a, const float* b, float* c) {
	for(int j = 0; j < 3; ++j)
		for(int i = 0; i < 3; ++i) c[3 * j + i] = a[i] * b[3 * j] + a[3 + i] * b[3 * j + 1] + a[6 + i] * b[3 * j + 2];
}
/* get_signed_distance_and_normal :98-137 + query_sdf :138-143 */
static int col_query(const orc_config* cfg, const void* ctx, const float* x, float* normal) {
	const orc_collider* col = (const orc_collider*) ctx;
	const int G = cfg_gsize(cfg), bc = cfg->boundary;
	const float dx = cfg_dx(cfg);
	const float lo = (float) bc * dx * 4.f, hi = (float) (G - bc) * 4.f * dx; /* :139 */
	for(int d = 0; d < 3; ++d)
		if(x[d] < lo || x[d] >= hi) return 0; /* :139-141 */
	int gc[3];
	float w1[3][2];
	for(int d = 0; d < 3; ++d) {
		gc[d] = (int) (x[d] / dx);                  /* :100 g_cid = (x / G_DX).cast<int>() */
		if(gc[d] + 1 >= 4 * G) return 0;            /* node g_cid + 1 out of the field (no wall band there) */
		const float dl = x[d] - (float) gc[d] * dx; /* :109 */
		w1[d][0] = 1 - dl / dx;                     /* :112 */
		w1[d][1] = dl / dx;                         /* :113 */
	}
	float sd = 0.f;
	normal[0] = normal[1] = normal[2] = 0.f;
	for(int i = 0; i < 2; ++i)
		for(int j = 0; j < 2; ++j)
			for(int k = 0; k < 2; ++k) {
				const float w = w1[0][i] * w1[1][j] * w1[2][k]; /* :118 */
				const int px = gc[0] + i, py = gc[1] + j, pz = gc[2] + k;
				const float* blk = col->sdf + tbl(cfg, px >> 2, py >> 2, pz >> 2) * 256 + ((px & 3) * 16 + (py & 3) * 4 + (pz & 3));
				sd += w * blk[0];          /* :128 */
				normal[0] += w * blk[64];  /* :129 */
				normal[1] += w * blk[128]; /* :130 */
				normal[2] += w * blk[192]; /* :131 */
			}
	const float nn = normal[0] * normal[0] + normal[1] * normal[1] + normal[2] * normal[2];
	if(nn > 0.f) { /* :135 normal /= sqrtf(normal.l2NormSqr()) */
		const float len = sqrtf(nn);
		for(int d = 0; d < 3; ++d) normal[d] /= len;
	}
	return sd <= 0.f; /* :142 */
}

/* hit test (phi <= 0) and material-space normal (0 where there is none) of one shape at the material-space point x, restated
 * from the header's definitions */
static int object_query(const orc_config* cfg, const void* ctx, const float* x, float* n) {
	const orc_collision_object* o = (const orc_collision_object*) ctx;
	const float *a = o->a, *b = o->b;
	n[0] = n[1] = n[2] = 0.f;
	if(o->shape == ORC_SHAPE_PLANE) {
		if((x[0] - a[0]) * b[0] + (x[1] - a[1]) * b[1] + (x[2] - a[2]) * b[2] > 0.f) return 0;
		for(int d = 0; d < 3; ++d) n[d] = b[d];
		return 1;
	}
	if(o->shape == ORC_SHAPE_BOX) {
		for(int d = 0; d < 3; ++d)
			if(!(a[d] <= x[d] && x[d] <= b[d])) return 0;
		int axis = 0;
		float best = 0.f, sgn = 1.f;
		for(int d = 0; d < 3; ++d) {
			const float ql = a[d] - x[d], qh = x[d] - b[d];
			const float q = ql > qh ? ql : qh;
			if(d == 0 || q > best) {
				best = q;
				axis = d;
				sgn = ql > qh ? -1.f : 1.f;
			}
		}
		n[axis] = sgn;
		return 1;
	}
	const float d0 = x[0] - a[0], d1 = x[1] - a[1], d2 = x[2] - a[2], r = b[0];
	if(o->shape == ORC_SHAPE_SPHERE) {
		const float dd = d0 * d0 + d1 * d1 + d2 * d2;
		if(dd > r * r) return 0;
		if(dd > 0.f) {
			const float len = sqrtf(dd);
			n[0] = d0 / len;
			n[1] = d1 / len;
			n[2] = d2 / len;
		}
		return 1;
	}
	const float rho2 = d0 * d0 + d2 * d2, h = b[1];
	if(rho2 > r * r || fabsf(d1) > h) return 0;
	const float rho = sqrtf(rho2);
	if(h - fabsf(d1) < r - rho) {
		n[1] = d1 < 0.f ? -1.f : 1.f;
	} else if(rho > 0.f) {
		n[0] = d0 / rho;
		n[2] = d2 / rho;
	}
	return 1;
}

/* the motion fields orc_collider and orc_collision_object share */
typedef struct boundary_motion {
	const float *rot_mat, *trans, *trans_vel, *omega;
	float dsdt, scale, friction;
	int type;
} boundary_motion;
#define BOUNDARY_MOTION(p) {(p)->rot_mat, (p)->trans, (p)->trans_vel, (p)->omega, (p)->dsdt, (p)->scale, (p)->friction, (p)->type}
typedef int (*boundary_query)(const orc_config* cfg, const void* ctx, const float* x, float* normal);

/* detect_and_resolve_collision :159-249 over the query of a level set (col_query) or of a shape (object_query) */
static void boundary_resolve(const orc_config* cfg, const boundary_motion* col, boundary_query query, const void* ctx, float t, const int* node, float* vel) {
	const float dx = cfg_dx(cfg);
	float xm[3], x0[3], x[3], cur[9], prev[9], r[9];
	for(int d = 0; d < 3; ++d) xm[d] = (float) node[d] * dx - (col->trans[d] + col->trans_vel[d] * t); /* :160 */
	{
		const float s = 1.f / (1.f + col->dsdt * t);
		for(int d = 0; d < 3; ++d) x0[d] = xm[d] * s; /* :165 */
		memcpy(cur, col->rot_mat, sizeof(cur));        /* :163 */
		for(int d = 0; d < 3; ++d) {                   /* :167-177 */
			col_axis_rot(col->omega[d] * t, d, r);
			memcpy(prev, cur, sizeof(cur));
			col_mat_mul(prev, r, cur);
		}
		for(int d = 0; d < 3; ++d) x[d] = cur[3 * d] * x0[0] + cur[3 * d + 1] * x0[1] + cur[3 * d + 2] * x0[2]; /* :178 mat_t_mul_vec_3d */
	}
	for(int d = 0; d < 3; ++d) x[d] = x[d] * col->scale + col->trans[d]; /* :181 */
	float on[3];
	if(!query(cfg, ctx, x, on)) return; /* :185-186 */
	const float* w = col->omega;
	float vo[3] = {w[1] * xm[2] - w[2] * xm[1], w[2] * xm[0] - w[0] * xm[2], w[0] * xm[1] - w[1] * xm[0]}; /* :188, a true cross product */
	for(int d = 0; d < 3; ++d) vo[d] += xm[d] * (col->dsdt / col->scale); /* :189 */
	{
		const float rr[3] = {x[0] - col->trans[0], x[1] - col->trans[1], x[2] - col->trans[2]}; /* :60 */
		float mv[3] = {w[1] * rr[2] + w[2] * rr[1], w[2] * rr[0] + w[0] * rr[2], w[0] * rr[1] + w[1] * rr[0]}; /* :62 */
		for(int d = 0; d < 3; ++d) mv[d] += col->trans_vel[d]; /* :63 */
		for(int d = 0; d < 3; ++d) vo[d] += (cur[d] * mv[0] + cur[3 + d] * mv[1] + cur[6 + d] * mv[2]) * col->scale + col->trans_vel[d]; /* :192-193 */
	}
	for(int d = 0; d < 3; ++d) vel[d] -= vo[d]; /* :195 */
	if(col->type == ORC_STICKY) {
		vel[0] = vel[1] = vel[2] = 0.f; /* :199 */
	} else if(col->type == ORC_SLIP) {
		float n[3];
		for(int d = 0; d < 3; ++d) n[d] = cur[d] * on[0] + cur[3 + d] * on[1] + cur[6 + d] * on[2]; /* :204 */
		const float vn = n[0] * vel[0] + n[1] * vel[1] + n[2] * vel[2]; /* :207 */
		for(int d = 0; d < 3; ++d) vel[d] -= n[d] * vn;                 /* :208 */
		if(col->friction > 0.0f && vn < 0) {                            /* :209-210 */
			const float len = sqrtf(vel[0] * vel[0] + vel[1] * vel[1] + vel[2] * vel[2]);
			if(-vn * col->friction < len)
				for(int d = 0; d < 3; ++d) vel[d] += vel[d] / len * (vn * col->friction); /* :213 */
			else
				vel[0] = vel[1] = vel[2] = 0.f;
		}
	} else if(col->type == ORC_SEPARATE) {
		if(on[0] == 0.0f && on[1] == 0.0f && on[2] == 0.0f) { /* :222-225 */
			vel[0] = vel[1] = vel[2] = 0.f;
			return;
		}
		float n[3];
		for(int d = 0; d < 3; ++d) n[d] = cur[d] * on[0] + cur[3 + d] * on[1] + cur[6 + d] * on[2]; /* :228 */
		const float vn = n[0] * vel[0] + n[1] * vel[1] + n[2] * vel[2];
		if(vn < 0) { /* :232 */
			for(int d = 0; d < 3; ++d) vel[d] -= n[d] * vn;
			if(col->friction != 0) { /* :234 */
				const float len = sqrtf(vel[0] * vel[0] + vel[1] * vel[1] + vel[2] * vel[2]);
				if(-vn * col->friction < len)
					for(int d = 0; d < 3; ++d) vel[d] += vel[d] / len * (vn * col->friction);
				else
					vel[0] = vel[1] = vel[2] = 0.f;
			}
		}
	}
	for(int d = 0; d < 3; ++d) vel[d] += vo[d]; /* :247 */
}

void orc_collider_resolve(const orc_config* cfg, const orc_collider* col, float t, const int* node, float* vel) {
	const boundary_motion m = BOUNDARY_MOTION(col);
	boundary_resolve(cfg, &m, col_query, col, t, node, vel);
}

static void object_resolve(const orc_config* cfg, const orc_collision_object* o, float t, const int* node, float* vel) {
	const boundary_motion m = BOUNDARY_MOTION(o);
	boundary_resolve(cfg, &m, object_query, o, t, node, vel);
}

/* ref: Projects/MGSP/mgmpm_kernels.cuh:323-399: the GMPM grid update (:357-360, claymore_oracle.c), then the boundaries
 * (:362-363): the collider, then the objects in list order */
typedef struct boundaries {
	const orc_config* cfg;
	const orc_collider* col;
	const orc_collision_object* objs;
	int n_objs;
	float time;
} boundaries;
static void boundaries_resolve(const void* ctx, const int* node, float* v) {
	const boundaries* b = (const boundaries*) ctx;
	if(b->col) orc_collider_resolve(b->cfg, b->col, b->time, node, v);
	for(int i = 0; i < b->n_objs; ++i) object_resolve(b->cfg, &b->objs[i], b->time, node, v);
}
void orc_update_grid_velocity_query_max_boundaries(const orc_config* cfg, int block_count, float* grid, orc_partition part, float dt, const orc_collider* col,
                                                   const orc_collision_object* objs, int n_objs, float time, float* max_vel) {
	const boundaries b = {cfg, col, objs, n_objs, time};
	boundaries_update(cfg, block_count, grid, part, dt, boundaries_resolve, &b, max_vel);
}
void orc_update_grid_velocity_query_max_collider(const orc_config* cfg, int block_count, float* grid, orc_partition part, float dt, const orc_collider* col, float time, float* max_vel) {
	orc_update_grid_velocity_query_max_boundaries(cfg, block_count, grid, part, dt, col, NULL, 0, time, max_vel);
}

/* ---- the oracle's simulator with boundaries ------------------------------------------------------------------------------ */
struct orc_csim {
	orc_sim* s;
	double sim_time;   /* sum of the dt of every finished sub-step */
	int has_collider;
	orc_collider col;
	float* sdf;        /* owned block-layout field of the collider */
	orc_collision_object* objs;  /* owned copy of the objects */
	int n_objs;
};
orc_csim* orc_csim_create(const orc_config* cfg, float dt_default, int max_blocks) {
	orc_csim* c = (orc_csim*) calloc(1, sizeof(orc_csim));
	c->s = orc_sim_create(cfg, dt_default, max_blocks);
	return c;
}
void orc_csim_destroy(orc_csim* c) {
	if(!c) return;
	orc_sim_destroy(c->s);
	free(c->sdf);
	free(c->objs);
	free(c);
}
orc_sim* orc_csim_sim(orc_csim* c) { return c->s; }
double orc_csim_time(orc_csim* c) { return c->sim_time; }

/* init_boundary (mgsp_benchmark.cuh:257-266) + fill_signed_distance_field (boundary_condition.cuh:253-295) */
void orc_csim_set_collider(orc_csim* c, const orc_collider* params, const float* sdf_host) {
	const orc_config* cfg = &c->s->cfg;
	if(sdf_host) {
		const int G = cfg_gsize(cfg), N = 4 * G;
		const size_t nodes = (size_t) N * N * N;
		if(!c->sdf) c->sdf = (float*) malloc(sizeof(float) * (size_t) G * G * G * 256);
		for(int ch = 0; ch < 4; ++ch)
			for(int i = 0; i < N; ++i)
				for(int j = 0; j < N; ++j)
					for(int k = 0; k < N; ++k)
						c->sdf[tbl(cfg, i >> 2, j >> 2, k >> 2) * 256 + ch * 64 + (i & 3) * 16 + (j & 3) * 4 + (k & 3)] = sdf_host[ch * nodes + ((size_t) i * N + j) * N + k];
	}
	c->col = *params;
	c->col.sdf = c->sdf;
	c->has_collider = c->sdf != NULL;
}
void orc_csim_clear_collider(orc_csim* c) {
	c->has_collider = 0;
	free(c->sdf);
	c->sdf = NULL;
}

void orc_csim_set_objects(orc_csim* c, const orc_collision_object* objs, int n) {
	free(c->objs);
	c->objs = NULL;
	c->n_objs = n;
	if(n > 0) {
		c->objs = (orc_collision_object*) malloc(sizeof(orc_collision_object) * n);
		memcpy(c->objs, objs, sizeof(orc_collision_object) * n);
	}
}

/* orc_sim_step (claymore_oracle.c; ref: gmpm_simulator.cuh:324-580) with the grid update of the MGSP form, the boundaries placed
 * at the simulated time at the start of the sub-step, and the clock advanced by the dt the sub-step ran with */
void orc_csim_step(orc_csim* c, float time_left) {
	orc_sim* s = c->s;
	const float dt = s->dt;
	float mv = 0.f; /* :337-362 */
	orc_update_grid_velocity_query_max_boundaries(&s->cfg, s->nbc, s->grids[0], s->parts[s->rollid], dt, c->has_collider ? &c->col : NULL, c->objs, c->n_objs,
	                                              (float) c->sim_time, &mv);
	sim_step_after_grid_update(s, mv, time_left);
	c->sim_time += (double) dt;
}
