/*
 * objects_oracle.c -- CPU restatement of the analytic collision objects (DESIGN.md section 2.9).  TEST INFRASTRUCTURE ONLY.
 *
 * Compiled together with the collider oracle (oracle/collider_oracle.c, which itself compiles claymore_oracle.c) into one
 * library by tests/objects_oracle_binding.py, so that the sub-step restated here can use the oracle simulator's state and the
 * collider's helpers.  The shapes are restated from the header's definitions; the response (object velocity, projection,
 * friction) follows orc_collider_resolve line by line with the level-set query replaced by the shape's.
 */
#include "collider_oracle.c"

enum { ORC_PLANE = 0, ORC_BOX = 1, ORC_SPHERE = 2, ORC_CYLINDER = 3 };
/* layout of cb200_collision_object */
typedef struct orc_object {
	int shape, type;
	float friction;
	float a[3], b[3];
	float rot_mat[9];
	float trans[3], trans_vel[3], omega[3];
	float dsdt, scale;
} orc_object;

/* hit test and material-space normal (0 where there is none) of one shape at the material-space point x */
static int obj_query(const orc_object* o, const float* x, float* n) {
	const float *a = o->a, *b = o->b;
	n[0] = n[1] = n[2] = 0.f;
	if(o->shape == ORC_PLANE) {
		if((x[0] - a[0]) * b[0] + (x[1] - a[1]) * b[1] + (x[2] - a[2]) * b[2] > 0.f) return 0;
		for(int d = 0; d < 3; ++d) n[d] = b[d];
		return 1;
	}
	if(o->shape == ORC_BOX) {
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
	if(o->shape == ORC_SPHERE) {
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

/* orc_collider_resolve with the shape's query */
void orc_object_resolve(const orc_config* cfg, const orc_object* col, float t, const int* node, float* vel) {
	const float dx = cfg_dx(cfg);
	float xm[3], x0[3], x[3], cur[9], prev[9], r[9];
	for(int d = 0; d < 3; ++d) xm[d] = (float) node[d] * dx - (col->trans[d] + col->trans_vel[d] * t);
	{
		const float s = 1.f / (1.f + col->dsdt * t);
		for(int d = 0; d < 3; ++d) x0[d] = xm[d] * s;
		memcpy(cur, col->rot_mat, sizeof(cur));
		for(int d = 0; d < 3; ++d) {
			col_axis_rot(col->omega[d] * t, d, r);
			memcpy(prev, cur, sizeof(cur));
			col_mat_mul(prev, r, cur);
		}
		for(int d = 0; d < 3; ++d) x[d] = cur[3 * d] * x0[0] + cur[3 * d + 1] * x0[1] + cur[3 * d + 2] * x0[2];
	}
	for(int d = 0; d < 3; ++d) x[d] = x[d] * col->scale + col->trans[d];
	float on[3];
	if(!obj_query(col, x, on)) return;
	const float* w = col->omega;
	float vo[3] = {w[1] * xm[2] - w[2] * xm[1], w[2] * xm[0] - w[0] * xm[2], w[0] * xm[1] - w[1] * xm[0]};
	for(int d = 0; d < 3; ++d) vo[d] += xm[d] * (col->dsdt / col->scale);
	{
		const float rr[3] = {x[0] - col->trans[0], x[1] - col->trans[1], x[2] - col->trans[2]};
		float mv[3] = {w[1] * rr[2] + w[2] * rr[1], w[2] * rr[0] + w[0] * rr[2], w[0] * rr[1] + w[1] * rr[0]};
		for(int d = 0; d < 3; ++d) mv[d] += col->trans_vel[d];
		for(int d = 0; d < 3; ++d) vo[d] += (cur[d] * mv[0] + cur[3 + d] * mv[1] + cur[6 + d] * mv[2]) * col->scale + col->trans_vel[d];
	}
	for(int d = 0; d < 3; ++d) vel[d] -= vo[d];
	if(col->type == ORC_STICKY) {
		vel[0] = vel[1] = vel[2] = 0.f;
	} else if(col->type == ORC_SLIP) {
		float n[3];
		for(int d = 0; d < 3; ++d) n[d] = cur[d] * on[0] + cur[3 + d] * on[1] + cur[6 + d] * on[2];
		const float vn = n[0] * vel[0] + n[1] * vel[1] + n[2] * vel[2];
		for(int d = 0; d < 3; ++d) vel[d] -= n[d] * vn;
		if(col->friction > 0.0f && vn < 0) {
			const float len = sqrtf(vel[0] * vel[0] + vel[1] * vel[1] + vel[2] * vel[2]);
			if(-vn * col->friction < len)
				for(int d = 0; d < 3; ++d) vel[d] += vel[d] / len * (vn * col->friction);
			else
				vel[0] = vel[1] = vel[2] = 0.f;
		}
	} else {
		if(on[0] == 0.0f && on[1] == 0.0f && on[2] == 0.0f) {
			vel[0] = vel[1] = vel[2] = 0.f;
			return;
		}
		float n[3];
		for(int d = 0; d < 3; ++d) n[d] = cur[d] * on[0] + cur[3 + d] * on[1] + cur[6 + d] * on[2];
		const float vn = n[0] * vel[0] + n[1] * vel[1] + n[2] * vel[2];
		if(vn < 0) {
			for(int d = 0; d < 3; ++d) vel[d] -= n[d] * vn;
			if(col->friction != 0) {
				const float len = sqrtf(vel[0] * vel[0] + vel[1] * vel[1] + vel[2] * vel[2]);
				if(-vn * col->friction < len)
					for(int d = 0; d < 3; ++d) vel[d] += vel[d] / len * (vn * col->friction);
				else
					vel[0] = vel[1] = vel[2] = 0.f;
			}
		}
	}
	for(int d = 0; d < 3; ++d) vel[d] += vo[d];
}

/* the level-set collider (col, nullable), then objs[0, n) in list order */
void orc_objects_resolve(const orc_config* cfg, const orc_collider* col, const orc_object* objs, int n, float t, const int* node, float* v) {
	if(col) orc_collider_resolve(cfg, col, t, node, v);
	for(int i = 0; i < n; ++i) orc_object_resolve(cfg, &objs[i], t, node, v);
}

/* orc_update_grid_velocity_query_max_collider with the objects after the collider */
void orc_update_grid_velocity_query_max_objects(const orc_config* cfg, int block_count, float* grid, orc_partition part, float dt, const orc_collider* col, const orc_object* objs, int n, float time, float* max_vel) {
	const int g = cfg_gsize(cfg), bc = cfg->boundary;
	float mx = *max_vel;
#pragma omp parallel for num_threads(g_threads) schedule(static) reduction(max : mx)
	for(int b = 0; b < block_count; ++b) {
		const int* k = part.active_keys + 3 * b;
		const int ob = ((k[0] < bc || k[0] >= g - bc) << 2) | ((k[1] < bc || k[1] >= g - bc) << 1) | (k[2] < bc || k[2] >= g - bc);
		float* blk = grid + (long) b * 256;
		for(int c = 0; c < BLOCK_VOL; ++c) {
			const float mass = blk[c];
			float vsq = 0.f;
			if(node_has_mass(mass)) {
				const float mi = 1.f / mass;
				float v[3];
				v[0] = (ob & 4) ? 0.f : blk[64 + c] * mi;
				v[1] = (ob & 2) ? 0.f : blk[128 + c] * mi;
				v[1] += cfg->gravity * dt;
				v[2] = (ob & 1) ? 0.f : blk[192 + c] * mi;
				const int node[3] = {4 * k[0] + ((c & 0x30) >> 4), 4 * k[1] + ((c & 0xc) >> 2), 4 * k[2] + (c & 0x3)};
				orc_objects_resolve(cfg, col, objs, n, time, node, v);
				blk[64 + c] = v[0];
				blk[128 + c] = v[1];
				blk[192 + c] = v[2];
				vsq += v[0] * v[0];
				vsq += v[1] * v[1];
				vsq += v[2] * v[2];
			}
			if(isnan(vsq)) vsq = INFINITY;
			if(vsq > mx) mx = vsq;
		}
	}
	*max_vel = mx;
}

/* ---- the collider oracle's simulator with objects -------------------------------------------------------------------------
 * orc_csim_step with the objects form of the grid update: the level-set collider of c (if set), then objs[0, n), placed at the
 * simulated time at the start of the sub-step.  The caller keeps the list (plane normals of unit length, as the engine stores
 * them). */
void orc_csim_step_objects(orc_csim* c, const orc_object* objs, int n, float time_left) {
	orc_sim* s = c->s;
	const orc_config* cfg = &s->cfg;
	const int R = s->rollid, Rn = R ^ 1;
	float mv = 0.f;
	orc_update_grid_velocity_query_max_objects(cfg, s->nbc, s->grids[0], s->parts[R], s->dt, c->has_collider ? &c->col : NULL, objs, n, (float) c->sim_time, &mv);
	s->max_vel = sqrtf(mv);
	s->next_dt = compute_dt(cfg, s->max_vel, time_left, s->dt_default);
	orc_clear_grid(s->nbc, s->grids[1]);
	for(int m = 0; m < s->nmodels; ++m) {
		memset(s->bins[Rn][m].cell_particle_counts, 0, sizeof(int) * (size_t) s->ebc * BLOCK_VOL);
		orc_g2p2g(cfg, s->dt, s->next_dt, s->pbc, s->bins[R][m], s->bins[Rn][m], s->parts[Rn], s->parts[R], s->grids[0], s->grids[1]);
	}
	for(int m = 0; m < s->nmodels; ++m) {
		orc_particle_buffer pb = s->bins[Rn][m];
		memset(pb.particle_bucket_sizes, 0, sizeof(int) * (s->ebc + 1));
		orc_cell_bucket_to_block(cfg, s->ebc, pb.cell_particle_counts, pb.cellbuckets, pb.particle_bucket_sizes, pb.blockbuckets);
	}
	memset(s->marks, 0, sizeof(int) * s->nbc);
	orc_mark_active_grid_blocks(s->nbc, s->grids[1], s->marks);
	memset(s->sources, 0, sizeof(int) * (s->ebc + 1));
	for(int m = 0; m < s->nmodels; ++m) orc_mark_active_particle_blocks(s->ebc + 1, s->bins[Rn][m].particle_bucket_sizes, s->sources);
	orc_exclusive_scan(s->ebc + 1, s->sources, s->destinations);
	const int new_pbc = s->destinations[s->ebc];
	*s->parts[Rn].count = new_pbc;
	orc_exclusive_scan_inverse(s->ebc, s->destinations, s->sources);
	orc_reset_table(cfg, s->parts[Rn]);
	check_blocks(s, new_pbc, "particle");
	orc_update_partition(cfg, new_pbc, s->sources, s->parts[R], s->parts[Rn]);
	for(int m = 0; m < s->nmodels; ++m) {
		orc_update_buckets(cfg, new_pbc, s->sources, s->bins[Rn][m], s->bins[R][m]);
		s->bins[R][m].particle_bucket_sizes[new_pbc] = 0;
		orc_compute_bin_capacity(new_pbc + 1, s->bins[R][m].particle_bucket_sizes, s->bin_sizes);
		orc_exclusive_scan(new_pbc + 1, s->bin_sizes, s->bins[R][m].bin_offsets);
		if(s->bins[R][m].bin_offsets[new_pbc] > s->bin_capacity[m]) {
			fprintf(stderr, "oracle: bin capacity exceeded\n");
			abort();
		}
	}
	orc_register_neighbor_blocks(cfg, new_pbc, s->parts[Rn]);
	const int prev_nbc = s->nbc;
	const int new_nbc = *s->parts[Rn].count;
	check_blocks(s, new_nbc, "neighbour");
	orc_clear_grid(s->ebc > new_nbc ? s->ebc : new_nbc, s->grids[0]);
	orc_copy_selected_grid_blocks(cfg, prev_nbc, s->parts[R].active_keys, s->parts[Rn], s->marks, s->grids[1], s->grids[0]);
	orc_register_exterior_blocks(cfg, new_pbc, s->parts[Rn]);
	const int new_ebc = *s->parts[Rn].count;
	check_blocks(s, new_ebc, "exterior");
	s->pbc = new_pbc;
	s->nbc = new_nbc;
	s->ebc = new_ebc;
	s->rollid = Rn;
	c->sim_time += (double) s->dt;
	s->dt = s->next_dt;
}
