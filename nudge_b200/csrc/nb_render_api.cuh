// nudge_b200 — renderer read-back (SURVEY.md §8 f4): what the demo's draw loop computes on the host for every collider
// (example/main.cpp:224-268: rotation = body ∘ collider, position = body.rotation * collider.position + body.position, then the
// column-major model matrix of example/main.cpp:74-110 with scale = box half extents or sphere radius), computed where the state
// lives.  One 4x4 float matrix per collider, boxes first, then spheres — the layout an instanced draw call (or glLoadMatrixf) takes.
// The output may be a device pointer (a mapped GL / Vulkan buffer: no host round trip at all) or a host pointer (pinned for an
// asynchronous copy).  Algorithmic bytes: 32 (collider transform) + 32 (body transform, gathered) + 16 (size) read, 64 written.
// Included at the end of nb_api.cu.
#pragma once

__global__ void __launch_bounds__(NB_BLOCK) k_instance_matrices(u32 nboxes, u32 nspheres, const nb_transform* body_xf,
		const nb_transform* box_xf, const nb_box_collider* box_data, const nb_transform* sph_xf, const nb_sphere_collider* sph_data, float4* out) {
	__shared__ float4 tile[NB_BLOCK * 4];
	const u32 K = nboxes + nspheres;
	for (u32 base = blockIdx.x * blockDim.x; base < K; base += gridDim.x * blockDim.x) {
		const u32 i = base + threadIdx.x;
		if (i < K) {
			const bool is_box = i < nboxes;
			const xform c = is_box ? ld_xform(box_xf, i) : ld_xform(sph_xf, i - nboxes);
			const xform b = ld_xform(body_xf, asu(c.p.w));
			float sx, sy, sz;
			if (is_box) { const float4 s = reinterpret_cast<const float4*>(box_data)[i]; sx = s.x; sy = s.y; sz = s.z; }
			else sx = sy = sz = sph_data[i - nboxes].radius;
			// rotation = body.rotation * collider.rotation (example/main.cpp:53-58, same operation order)
			const float ax = b.q.x, ay = b.q.y, az = b.q.z, aw = b.q.w, bx = c.q.x, by = c.q.y, bz = c.q.z, bw = c.q.w;
			const float qx = bx*aw + ax*bw + ay*bz - az*by;
			const float qy = by*aw + ay*bw + az*bx - ax*bz;
			const float qz = bz*aw + az*bw + ax*by - ay*bx;
			const float qw = aw*bw - ax*bx - ay*by - az*bz;
			// position = body.rotation applied to collider.position, plus body.position (example/main.cpp:60-72, 238-242)
			float tx = ay*c.p.z - az*c.p.y, ty = az*c.p.x - ax*c.p.z, tz = ax*c.p.y - ay*c.p.x;
			tx += tx; ty += ty; tz += tz;
			float px = c.p.x + aw*tx + ay*tz - az*ty;
			float py = c.p.y + aw*ty + az*tx - ax*tz;
			float pz = c.p.z + aw*tz + ax*ty - ay*tx;
			px += b.p.x; py += b.p.y; pz += b.p.z;
			// scaled rotation matrix, column major (example/main.cpp:74-110)
			const float kx = qx + qx, ky = qy + qy, kz = qz + qz;
			const float xx = kx*qx, yy = ky*qy, zz = kz*qz, xy = kx*qy, xz = kx*qz, yz = ky*qz, wx = kx*qw, wy = ky*qw, wz = kz*qw;
			float4* t = tile + 4 * threadIdx.x;
			t[0] = make_float4((1.0f - yy - zz) * sx, (xy + wz) * sx, (xz - wy) * sx, 0.0f);
			t[1] = make_float4((xy - wz) * sy, (1.0f - xx - zz) * sy, (yz + wx) * sy, 0.0f);
			t[2] = make_float4((xz + wy) * sz, (yz - wx) * sz, (1.0f - xx - yy) * sz, 0.0f);
			t[3] = make_float4(px, py, pz, 1.0f);
		}
		__syncthreads();
		const u32 rows = 4 * min(blockDim.x, K - base);   // consecutive threads write consecutive 16-byte words
		for (u32 r = threadIdx.x; r < rows; r += blockDim.x) out[(size_t)4 * base + r] = tile[r];
		__syncthreads();
	}
}

extern "C" {

// Writes min(colliders, capacity) matrices (16 floats each) to `out` and the collider count to *count.  out_is_device != 0: `out` is a
// device pointer, the call is asynchronous on `stream`.  Otherwise `out` is host memory and the call returns when it is filled.
int nb_instance_matrices(nb_context* ctx, float* out, uint32_t capacity, int out_is_device, uint32_t* count, void* stream) {
	NB_RANGE("nb_instance_matrices");
	cudaStream_t st = (cudaStream_t)stream;
	const u32 K = ctx->nboxes + ctx->nspheres;
	if (count) *count = K;
	if (!out) { ctx->error = "null output"; return NB_ERR_ARGUMENT; }
	if (capacity < K) { ctx->error = "instance buffer smaller than the collider count"; return NB_ERR_CAPACITY; }
	if (!K) return NB_OK;
	float4* dst = reinterpret_cast<float4*>(out);
	if (!out_is_device) {
		ALLOC(ctx->instances, 4 * ((size_t)ctx->cfg.max_boxes + ctx->cfg.max_spheres));
		dst = ctx->instances;
	}
	launch_grid(mk_launch(ctx, st), k_instance_matrices, GRID(K), ctx->nboxes, ctx->nspheres, ctx->xf, ctx->box_xf, ctx->box_data, ctx->sph_xf, ctx->sph_data, dst);
	CK(cudaGetLastError());
	if (!out_is_device) {
		CK(cudaMemcpyAsync(out, dst, (size_t)K * 64, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
	}
	return NB_OK;
}

}  // extern "C"
