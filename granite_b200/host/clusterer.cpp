#include "clusterer.hpp"
#include "shard_plan.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <numeric>
#include <utility>
#include <stdexcept>

namespace Granite
{
LightClusterer::LightClusterer() = default;

LightClusterer::~LightClusterer()
{
	if (staging)
		cudaFreeHost(staging);
}

void LightClusterer::set_resolution(unsigned x, unsigned y, unsigned z)
{
	// the binning kernel works on 8x4-tile blocks (clusterer.cpp:1516-1517 asserts & 7)
	if ((x & 7) || (y & 7) || (z & 63))
		throw std::logic_error("LightClusterer: resolution must be a multiple of (8, 8, 64).");
	resolution_x = x;
	resolution_y = y;
	resolution_z = z;
}

// "cluster-transforms" holds, packed for the CURRENT light count n so one copy uploads it all:
//   [n x PositionalFragmentInfo][n x mat_affine][128 x u32 type mask][max(n,1) x uvec2 Z ranges]
// (the reference uploads lights / model / type_mask with three update_buffer calls into the
// fixed-offset ClustererBindlessTransforms and the Z ranges through a fresh host-visible buffer,
// clusterer.cpp:1178-1207, 1280-1284).
static size_t packed_offset_model(size_t n) { return n * sizeof(PositionalFragmentInfo); }
static size_t packed_offset_type_mask(size_t n) { return packed_offset_model(n) + n * sizeof(mat_affine); }
static size_t packed_offset_z_ranges(size_t n) { return packed_offset_type_mask(n) + sizeof(uint32_t) * (ClustererMaxLightsBindless / 32); }
static size_t packed_size(size_t n) { return packed_offset_z_ranges(n) + sizeof(uvec2) * (n ? n : 1); }
// with shadows enabled two more arrays follow: [n x mat4 shadow transform][n x device pointer to the light's map]
static size_t packed_offset_shadow_maps(size_t n) { return packed_size(n) + n * sizeof(mat4); }
static size_t packed_size_with_shadows(size_t n) { return packed_offset_shadow_maps(n) + n * sizeof(void *); }

size_t LightClusterer::transforms_offset_model() const { return packed_offset_model((size_t)parameters.num_lights); }
size_t LightClusterer::transforms_offset_type_mask() const { return packed_offset_type_mask((size_t)parameters.num_lights); }
size_t LightClusterer::transforms_size() const
{
	return enable_shadows ? packed_size_with_shadows(ClustererMaxLightsBindless) : packed_size(ClustererMaxLightsBindless);
}

// clusterer.cpp:467-474: the spot light's own view (looking down its axis) and a projection that just covers the cone,
// near = 0.5 % of the range, biased from clip space to texture coordinates
mat4 LightClusterer::spot_shadow_transform(const PositionalFragmentInfo &light, float xy_range)
{
	const float range = std::tan(xy_range);
	const mat4 view = mat4_cast(look_at_arbitrary_up(light.direction)) * translate(-light.position);
	const mat4 proj = perspective(range * 2.0f, 1.0f, 0.005f / light.inv_radius, 1.0f / light.inv_radius);
	return translate(vec3(0.5f, 0.5f, 0.0f)) * scale(vec3(0.5f, 0.5f, 1.0f)) * proj * view;
}

// clusterer.cpp:518-521 with math/transforms.cpp:223-224: the six faces share one 90-degree projection (mirrored in x);
// the shader only needs the two rows that turn the distance along the major axis into the stored depth
mat4 LightClusterer::point_shadow_transform(const PositionalFragmentInfo &light)
{
	const float pi = 3.1415926535897932384626433832795f; // muglm::pi<float>()
	const mat4 proj = scale(vec3(-1.0f, 1.0f, 1.0f)) * perspective(0.5f * pi, 1.0f, 0.005f / light.inv_radius, 1.0f / light.inv_radius);
	mat4 m(0.0f);
	m[0] = vec4(proj[2].z, proj[2].w, proj[3].z, proj[3].w);
	return m;
}

GrbLightShadows LightClusterer::get_light_shadows() const
{
	GrbLightShadows s = {};
	if (!enable_shadows || !transforms_buffer)
		return s;
	auto *base = transforms_buffer->get<uint8_t>();
	const size_t n = (size_t)parameters.num_lights;
	s.transforms = reinterpret_cast<const float *>(base + packed_size(n));
	s.maps = reinterpret_cast<const void *const *>(base + packed_offset_shadow_maps(n));
	s.resolution = (int32_t)shadow_resolution;
	s.pcf_wide = shadow_pcf_wide ? 1 : 0;
	return s;
}

void LightClusterer::add_render_passes(RenderGraph &graph)
{
	add_render_passes_bindless(graph);
}

// renderer/lights/clusterer.cpp:1575-1613
void LightClusterer::add_render_passes_bindless(RenderGraph &graph)
{
	BufferInfo att;
	att.usage = VK_BUFFER_USAGE_STORAGE_BUFFER_BIT | VK_BUFFER_USAGE_TRANSFER_DST_BIT;
	// every buffer here is rewritten each frame; alternating two copies lets the build of frame
	// N+1 run while frame N's lighting still reads the previous structure
	if (async_compute)
		att.flags |= ATTACHMENT_INFO_PINGPONG_BIT;

	// On the async-compute queue the build of frame N+1 overlaps the (HBM-bound) post chain of
	// frame N: it only waits for frame N's lighting pass to release the cluster buffers.
	auto &pass = graph.add_pass("clustering-bindless", async_compute ? RENDER_GRAPH_QUEUE_ASYNC_COMPUTE_BIT : RENDER_GRAPH_QUEUE_COMPUTE_BIT);
	att.size = resolution_x * resolution_y * (ClustererMaxLightsBindless / 8);
	res_bitmask = &pass.add_storage_output("cluster-bitmask", att);
	att.size = resolution_z * sizeof(ivec2);
	res_range = &pass.add_storage_output("cluster-range", att);
	att.size = transforms_size();
	res_transforms = &pass.add_transfer_output("cluster-transforms", att);
	att.size = sizeof(vec4) * 4 * 8 * ClustererMaxLightsBindless;
	res_cull = &pass.add_storage_output("cluster-cull-setup", att);
	att.size = sizeof(vec4) * 6 * ClustererMaxLightsBindless;
	res_spots = &pass.add_storage_output("cluster-transformed-spot", att);

	if (enable_volumetric_decals)
	{
		// clusterer.cpp:1585-1592: the decals' own bitmask and Z-range buffers, same grid
		att.size = resolution_x * resolution_y * (MaxDecalsBindless / 8);
		res_bitmask_decal = &pass.add_storage_output("cluster-bitmask-decal", att);
		att.size = resolution_z * sizeof(ivec2);
		res_range_decal = &pass.add_storage_output("cluster-range-decal", att);
		// per-frame inputs and scratch: [n x mat4 mvp][n x vec4 screen box][max(n,1) x uvec2 Z range]
		att.size = MaxDecalsBindless * (sizeof(mat4) + sizeof(vec4) + sizeof(uvec2));
		res_decal_scratch = &pass.add_transfer_output("cluster-decal-transforms", att);
	}

	pass.set_build_render_pass([this](Vulkan::CommandBuffer &cmd) {
		build_cluster_bindless_gpu(cmd);
		build_decal_clusters_gpu(cmd);
	});
}

// renderer/lights/clusterer.cpp:83-93
void LightClusterer::setup_render_pass_dependencies(RenderGraph &, RenderPass &target)
{
	target.add_storage_read_only_input("cluster-bitmask");
	target.add_storage_read_only_input("cluster-range");
	target.add_storage_read_only_input("cluster-transforms");
	// the shadow atlas is managed outside the graph (clusterer.cpp:92); a no-op while nothing registers it
	target.add_external_lock("bindless-shadowmaps", VK_PIPELINE_STAGE_FRAGMENT_SHADER_BIT, VK_ACCESS_2_SHADER_SAMPLED_READ_BIT);
}

// renderer/lights/clusterer.cpp:107-116
void LightClusterer::setup_render_pass_resources(RenderGraph &graph)
{
	bitmask_buffer = graph.maybe_get_physical_buffer_resource(res_bitmask);
	range_buffer = graph.maybe_get_physical_buffer_resource(res_range);
	transforms_buffer = graph.maybe_get_physical_buffer_resource(res_transforms);
	cull_buffer = graph.maybe_get_physical_buffer_resource(res_cull);
	spot_buffer = graph.maybe_get_physical_buffer_resource(res_spots);
	bitmask_decal_buffer = res_bitmask_decal ? graph.maybe_get_physical_buffer_resource(res_bitmask_decal) : nullptr;
	range_decal_buffer = res_range_decal ? graph.maybe_get_physical_buffer_resource(res_range_decal) : nullptr;
	decal_scratch_buffer = res_decal_scratch ? graph.maybe_get_physical_buffer_resource(res_decal_scratch) : nullptr;
}

GrbClusterBuffers LightClusterer::get_cluster_buffers() const
{
	GrbClusterBuffers b = {};
	if (!transforms_buffer || !bitmask_buffer || !range_buffer || !cull_buffer || !spot_buffer)
		return b;
	auto *base = transforms_buffer->get<uint8_t>();
	b.lights = reinterpret_cast<const GrbPositionalLight *>(base);
	b.model = reinterpret_cast<const float *>(base + transforms_offset_model());
	b.type_mask = reinterpret_cast<const uint32_t *>(base + transforms_offset_type_mask());
	b.z_ranges = reinterpret_cast<const uint32_t *>(base + packed_offset_z_ranges((size_t)parameters.num_lights));
	b.transformed_spots = spot_buffer->get<float>();
	b.cull_setup = cull_buffer->get<float>();
	b.bitmask = bitmask_buffer->get<uint32_t>();
	b.cluster_range = range_buffer->get<uint32_t>();
	b.resolution_z = (int32_t)resolution_z;
	return b;
}

// renderer/lights/clusterer.cpp:700-703
float LightClusterer::get_z_slice_extent(const RenderContext &ctx) const
{
	return min(0.5f, ctx.get_render_parameters().z_far / float(resolution_z));
}

// renderer/lights/clusterer.cpp:1265-1275
uvec2 LightClusterer::compute_uint_range(vec2 range) const
{
	float extent = get_z_slice_extent(*context);
	range.x = range.x / extent;
	range.y = range.y / extent;
	if (range.y < 0.0f)
		return uvec2(0xffffffffu, 0u);
	range.x = max(range.x, 0.0f);
	uvec2 urange((uint32_t)range.x, (uint32_t)range.y);
	urange.y = std::min<uint32_t>(urange.y, resolution_z - 1);
	return urange;
}

void LightClusterer::refresh(const RenderContext &ctx)
{
	context = &ctx;
	refresh_bindless_prepare(ctx);
	refresh_decals(ctx);
}

// clusterer.cpp:1348-1369: view-depth range of the decal's unit cube
vec2 LightClusterer::decal_z_range(const RenderContext &ctx, const mat_affine &transform)
{
	const auto &rp = ctx.get_render_parameters();
	float lo = std::numeric_limits<float>::infinity(), hi = -std::numeric_limits<float>::infinity();
	for (unsigned i = 0; i < 8; i++)
	{
		const vec4 corner((i & 1) ? 0.5f : -0.5f, (i & 2) ? 0.5f : -0.5f, (i & 4) ? 0.5f : -0.5f, 1.0f);
		// SIMD::mul(vec4, mat_affine, vec4): one dot product per row, added pairwise as DPPS does
		vec3 world;
		float *w = &world.x;
		for (int r = 0; r < 3; r++)
			w[r] = (transform[r].x * corner.x + transform[r].y * corner.y) + (transform[r].z * corner.z + transform[r].w * corner.w);
		const float z = dot(world - rp.camera_position, rp.camera_front);
		lo = std::min(lo, z);
		hi = std::max(hi, z);
	}
	return vec2(lo, hi);
}

// The visible decals front to back (clusterer.cpp:1124-1131, 1167-1171), their mvps (clusterer.cpp:1406-1410) and Z-slice
// ranges (clusterer.cpp:1371-1389).
void LightClusterer::refresh_decals(const RenderContext &ctx)
{
	decal_mvps.clear();
	decal_index_range.clear();
	if (!enable_volumetric_decals)
		return;
	const auto &rp = ctx.get_render_parameters();
	std::vector<std::pair<float, unsigned>> order;
	if (scene_decals)
	{
		const Frustum &frustum = ctx.get_visibility_frustum();
		const AABB unit(vec3(-0.5f), vec3(0.5f));
		for (unsigned i = 0; i < (unsigned)scene_decals->size(); i++)
		{
			const AABB world = unit.transform((*scene_decals)[i]);
			if (frustum_culling && !frustum.intersects_fast(world))
				continue;
			order.emplace_back(dot(rp.camera_front, world.get_center()), i);
		}
		std::stable_sort(order.begin(), order.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
	}
	if (order.size() > MaxDecalsBindless)
		order.resize(MaxDecalsBindless);
	for (auto &o : order)
	{
		const mat_affine &t = (*scene_decals)[o.second];
		const mat4 world(vec4(t[0].x, t[1].x, t[2].x, 0.0f), vec4(t[0].y, t[1].y, t[2].y, 0.0f), vec4(t[0].z, t[1].z, t[2].z, 0.0f),
		                 vec4(t[0].w, t[1].w, t[2].w, 1.0f)); // mat_affine::to_mat4
		decal_mvps.push_back(rp.view_projection * world);
		decal_index_range.push_back(compute_uint_range(decal_z_range(ctx, t)));
	}
	// the Z-range kernel still runs with one empty entry so that the range buffer is cleared (clusterer.cpp:1384-1386)
	if (decal_index_range.empty())
		decal_index_range.push_back(uvec2(~0u, 0u));
}

// update_bindless_mask_buffer_decal_gpu + update_bindless_range_buffer_decal_gpu (clusterer.cpp:1570-1572)
void LightClusterer::build_decal_clusters_gpu(Vulkan::CommandBuffer &cmd)
{
	if (!enable_volumetric_decals || !decal_scratch_buffer || !bitmask_decal_buffer || !range_decal_buffer)
		return;
	const size_t n = decal_mvps.size();
	auto *base = decal_scratch_buffer->get<uint8_t>();
	auto *d_mvps = reinterpret_cast<float *>(base);
	auto *d_boxes = reinterpret_cast<float *>(base + MaxDecalsBindless * sizeof(mat4));
	auto *d_ranges = reinterpret_cast<uint32_t *>(base + MaxDecalsBindless * (sizeof(mat4) + sizeof(vec4)));
	auto stream = reinterpret_cast<cudaStream_t>(cmd.get_stream());
	// pageable copies: the runtime stages them before returning, so the vectors may change right after
	if (n)
		Vulkan::cuda_ok(cudaMemcpyAsync(d_mvps, decal_mvps.data(), n * sizeof(mat4), cudaMemcpyHostToDevice, stream), "decal upload");
	Vulkan::cuda_ok(cudaMemcpyAsync(d_ranges, decal_index_range.data(), decal_index_range.size() * sizeof(uvec2), cudaMemcpyHostToDevice, stream),
	                "decal range upload");
	cmd.check(grb_cluster_decal_binning(&parameters, d_mvps, (int32_t)n, d_boxes, bitmask_decal_buffer->get<uint32_t>(), cmd.get_stream_handle()),
	          "grb_cluster_decal_binning");
	GrbClusterBuffers buf = {};
	buf.z_ranges = d_ranges;
	buf.cluster_range = range_decal_buffer->get<uint32_t>();
	buf.resolution_z = (int32_t)resolution_z;
	cmd.check(grb_cluster_z_range(&buf, (int32_t)decal_index_range.size(), cmd.get_stream_handle()), "grb_cluster_z_range(decals)");
}

// renderer/threaded_scene.cpp:137-150 (front-to-back order), clusterer.cpp:656-698 (scan),
// :803-826 (parameters), :1322-1346 (per-light Z ranges).
void LightClusterer::refresh_bindless_prepare(const RenderContext &ctx)
{
	const auto &rp = ctx.get_render_parameters();
	lights.clear();
	model.clear();
	shadow_transforms.clear();
	shadow_maps.clear();
	volume_index_range.clear();
	type_mask.assign(ClustererMaxLightsBindless / 32, 0u);

	// Sort key: view depth of the light centre.  (The reference's key reads one vec4 past the
	// end of the node transform -- SURVEY.md §7 -- the intended key is this one.)  stable_sort
	// keeps input order on ties so the light order, hence bit positions and fp accumulation
	// order, is deterministic.
	auto &order = sort_order;
	auto &keys = sort_keys;
	if (scene_lights && !device_lights)
	{
		const size_t n = scene_lights->size();
		// gather_positional_lights (renderer/scene.cpp:333-358): only lights whose world-space AABB
		// passes the visibility frustum reach the sort.  Last frame's order is the starting point:
		// with coherent motion it is already sorted and the sort below is skipped (ties keep input
		// order, so sorting from the previous order and sorting from scratch agree).
		const Frustum &frustum = ctx.get_visibility_frustum();
		visible.resize(n);
		size_t n_visible = 0;
		for (size_t i = 0; i < n; i++)
		{
			const auto &l = (*scene_lights)[i];
			visible[i] = !frustum_culling || frustum.intersects_fast(l.light->get_static_aabb().transform(l.transform));
			n_visible += visible[i] ? 1 : 0;
		}
		bool same_set = order.size() == n_visible;
		for (size_t i = 0; same_set && i < order.size(); i++)
			same_set = order[i] < n && visible[order[i]];
		if (!same_set)
		{
			order.clear();
			for (size_t i = 0; i < n; i++)
				if (visible[i])
					order.push_back((unsigned)i);
		}
		keys.resize(n);
		for (size_t i = 0; i < n; i++)
			keys[i] = dot((*scene_lights)[i].transform.get_translation(), rp.camera_front);
		auto by_key_then_input = [&](unsigned a, unsigned b) { return keys[a] < keys[b] || (keys[a] == keys[b] && a < b); };
		if (!std::is_sorted(order.begin(), order.end(), by_key_then_input))
			std::sort(order.begin(), order.end(), by_key_then_input);
	}
	else
		order.clear();

	unsigned index = 0;
	for (unsigned src : order)
	{
		if (index >= ClustererMaxLightsBindless)
			break;
		auto &l = (*scene_lights)[src];
		if (l.light->get_type() == PositionalLight::Type::Spot)
		{
			auto &spot = static_cast<SpotLight &>(*l.light);
			lights.push_back(spot.get_shader_info(l.transform));
			model.push_back(spot.build_model_matrix(l.transform));
			if (enable_shadows)
				shadow_transforms.push_back(spot_shadow_transform(lights.back(), spot.get_xy_range()));
		}
		else
		{
			auto &point = static_cast<PointLight &>(*l.light);
			lights.push_back(point.get_shader_info(l.transform));
			// set_point_model_transform (clusterer.cpp:647-650): row 0 = (position, radius)
			mat_affine m(vec4(0.0f), vec4(0.0f), vec4(0.0f));
			m[0] = vec4(lights.back().position, 1.0f / lights.back().inv_radius);
			model.push_back(m);
			type_mask[index >> 5] |= 1u << (index & 31u);
			if (enable_shadows)
				shadow_transforms.push_back(point_shadow_transform(lights.back()));
		}
		if (enable_shadows)
			shadow_maps.push_back(l.light->get_shadow_map());
		index++;
	}
	if (device_lights)
		index = (unsigned)std::min<int32_t>(device_lights->list.count, ClustererMaxLightsBindless);

	std::memset(&parameters, 0, sizeof(parameters));
	parameters.num_lights = (int32_t)index;
	parameters.num_lights_32 = (int32_t)((index + 31) / 32);
	float z_slice_size = get_z_slice_extent(ctx);
	parameters.clip_scale[0] = rp.projection[0][0];
	parameters.clip_scale[1] = -rp.projection[1][1];
	parameters.clip_scale[2] = rp.inv_projection[0][0];
	parameters.clip_scale[3] = -rp.inv_projection[1][1];
	mat4 transform = translate(vec3(0.5f, 0.5f, 0.0f)) * scale(vec3(0.5f, 0.5f, 1.0f)) * rp.view_projection;
	std::memcpy(parameters.transform, transform.data(), sizeof(parameters.transform));
	for (int i = 0; i < 3; i++)
	{
		parameters.camera_front[i] = rp.camera_front[i];
		parameters.camera_base[i] = rp.camera_position[i];
	}
	parameters.xy_scale[0] = float(resolution_x);
	parameters.xy_scale[1] = float(resolution_y);
	parameters.resolution_xy[0] = (int32_t)resolution_x;
	parameters.resolution_xy[1] = (int32_t)resolution_y;
	parameters.inv_resolution_xy[0] = 1.0f / float(resolution_x);
	parameters.inv_resolution_xy[1] = 1.0f / float(resolution_y);
	parameters.z_scale = 1.0f / z_slice_size;
	parameters.z_max_index = (int32_t)resolution_z - 1;

	if (device_lights)
	{
		// the camera terms of the device prep; the per-light work is the clustering pass's
		std::memset(&device_view, 0, sizeof(device_view));
		for (int i = 0; i < 3; i++)
		{
			device_view.camera_position[i] = rp.camera_position[i];
			device_view.camera_front[i] = rp.camera_front[i];
		}
		const vec4 *planes = ctx.get_visibility_frustum().get_planes();
		for (int p = 0; p < 6; p++)
			for (int c = 0; c < 4; c++)
				device_view.planes[4 * p + c] = planes[p][c];
		device_view.z_slice_extent = z_slice_size;
		device_view.z_max_index = (int32_t)resolution_z - 1;
		device_view.frustum_culling = frustum_culling ? 1 : 0;
		return;
	}

	// update_bindless_range_buffer_gpu: per-light slice range on the host
	volume_index_range.resize(index);
	for (unsigned i = 0; i < index; i++)
	{
		vec2 range;
		if (type_mask[i >> 5] & (1u << (i & 31)))
			range = point_light_z_range(ctx, lights[i].position, 1.0f / lights[i].inv_radius);
		else
			range = spot_light_z_range(ctx, model[i]);
		volume_index_range[i] = compute_uint_range(range);
	}
	// still run the Z-range kernel with one empty entry so the range buffer is cleared
	if (volume_index_range.empty())
		volume_index_range.push_back(uvec2(~0u, 0u));
}

// renderer/lights/clusterer.cpp:1564-1573: update_bindless_data (upload), then the kernels.
void LightClusterer::build_cluster_bindless_gpu(Vulkan::CommandBuffer &cmd)
{
	if (!context || !transforms_buffer)
	{
		Vulkan::log_error("LightClusterer: refresh() / setup_render_pass_resources() must run before the clustering pass.\n");
		return;
	}
	if (device_lights)
	{
		// the device prep writes this frame's copy of "cluster-transforms" in place of the staging upload
		auto stream = reinterpret_cast<cudaStream_t>(cmd.get_stream());
		const DeviceLightSource &src = *device_lights;
		if (src.ready)
			Vulkan::cuda_ok(cudaStreamWaitEvent(stream, static_cast<cudaEvent_t>(src.ready), 0), "cudaStreamWaitEvent(lights ready)");
		const GrbClusterBuffers buf = get_cluster_buffers();
		auto *records = const_cast<GrbPositionalLight *>(buf.lights);
		auto *model = const_cast<float *>(buf.model);
		auto *type_mask = const_cast<uint32_t *>(buf.type_mask);
		auto *z_ranges = const_cast<uint32_t *>(buf.z_ranges);
		void *s = cmd.get_stream_handle();
		GrbLightList list = src.list;
		const int32_t *input_count = src.input_count;
		GrbLightShadowIdList ids = src.shadow_ids;
		if (src.exchange)
			src.exchange(cmd, list, input_count, ids);
		if (enable_shadows)
		{
			// the shadow tables where the lighting pass reads them: packed_size(slots) and packed_offset_shadow_maps(slots)
			const GrbLightShadows out = get_light_shadows();
			auto *transforms = const_cast<float *>(out.transforms);
			auto *maps = const_cast<const void **>(out.maps);
			if (src.by_id)
				cmd.check(grb_light_prep_shadow_ids(&list, input_count, &ids, src.map_table, src.map_table_size, &device_view, records, model, type_mask,
				                                    z_ranges, transforms, maps, src.count, src.scratch, src.scratch_bytes, s),
				          "grb_light_prep_shadow_ids");
			else if (input_count)
				cmd.check(grb_light_prep_shadowed_counted(&list, input_count, &src.shadows, &device_view, records, model, type_mask, z_ranges,
				                                          transforms, maps, src.count, src.scratch, src.scratch_bytes, s),
				          "grb_light_prep_shadowed_counted");
			else
				cmd.check(grb_light_prep_shadowed(&list, &src.shadows, &device_view, records, model, type_mask, z_ranges, transforms, maps, src.count,
				                                  src.scratch, src.scratch_bytes, s),
				          "grb_light_prep_shadowed");
		}
		else if (input_count)
			cmd.check(grb_light_prep_counted(&list, input_count, &device_view, records, model, type_mask, z_ranges, src.count, src.scratch,
			                                 src.scratch_bytes, s),
			          "grb_light_prep_counted");
		else
			cmd.check(grb_light_prep(&list, &device_view, records, model, type_mask, z_ranges, src.count, src.scratch, src.scratch_bytes, s),
			          "grb_light_prep");
		if (src.after_prep)
			src.after_prep(cmd);
		if (src.consumed)
			Vulkan::cuda_ok(cudaEventRecord(static_cast<cudaEvent_t>(src.consumed), stream), "cudaEventRecord(lights consumed)");
		launch_cluster_kernels(cmd, src.count, std::max<int32_t>(parameters.num_lights, 1));
		return;
	}
	const unsigned n = (unsigned)parameters.num_lights;
	const size_t lights_bytes = n * sizeof(PositionalFragmentInfo);
	const size_t model_bytes = n * sizeof(mat_affine);
	const size_t mask_bytes = sizeof(uint32_t) * (ClustererMaxLightsBindless / 32);
	const size_t range_bytes = volume_index_range.size() * sizeof(uvec2);
	const size_t shadow_bytes = enable_shadows ? n * (sizeof(mat4) + sizeof(void *)) : 0;
	const size_t need = lights_bytes + model_bytes + mask_bytes + range_bytes + shadow_bytes;
	auto stream = reinterpret_cast<cudaStream_t>(cmd.get_stream());
	// Two pinned staging slots used alternately; a slot is reused only after the copies that
	// read it have completed (its event), so frames pipeline without a host-device sync.
	const size_t slot_size =
	    ClustererMaxLightsBindless * (sizeof(PositionalFragmentInfo) + sizeof(mat_affine) + sizeof(uvec2) + sizeof(mat4) + sizeof(void *)) + mask_bytes;
	if (!staging)
	{
		if (!Vulkan::cuda_ok(cudaMallocHost(&staging, slot_size * 2), "cudaMallocHost"))
		{
			staging = nullptr;
			return;
		}
		staging_size = slot_size * 2;
		for (auto &e : staging_events)
		{
			cudaEvent_t ev;
			Vulkan::cuda_ok(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming), "cudaEventCreate(staging)");
			e = ev;
		}
	}
	if (need > slot_size)
		return;
	const unsigned slot = staging_slot;
	staging_slot ^= 1u;
	if (staging_event_pending[slot])
	{
		Vulkan::ScopedHostTimer timer("(flow control: wait for staging slot)");
		cudaEventSynchronize(reinterpret_cast<cudaEvent_t>(staging_events[slot]));
	}
	auto *s = static_cast<uint8_t *>(staging) + slot * slot_size;
	std::memcpy(s, lights.data(), lights_bytes);
	std::memcpy(s + lights_bytes, model.data(), model_bytes);
	std::memcpy(s + lights_bytes + model_bytes, type_mask.data(), mask_bytes);
	std::memcpy(s + lights_bytes + model_bytes + mask_bytes, volume_index_range.data(), range_bytes);
	if (enable_shadows && n)
	{
		std::memcpy(s + packed_size(n), shadow_transforms.data(), n * sizeof(mat4));
		std::memcpy(s + packed_offset_shadow_maps(n), shadow_maps.data(), n * sizeof(void *));
	}

	// the staging slot already has the packed device layout: one H2D copy
	if (!Vulkan::cuda_ok(cudaMemcpyAsync(transforms_buffer->get_device_pointer(), s, need, cudaMemcpyHostToDevice, stream), "light upload"))
		return;
	Vulkan::cuda_ok(cudaEventRecord(reinterpret_cast<cudaEvent_t>(staging_events[slot]), stream), "cudaEventRecord(staging)");
	staging_event_pending[slot] = true;
	launch_cluster_kernels(cmd, nullptr, (int32_t)volume_index_range.size());
}

// K1 -> K4 over the packed lights of this frame; device_count: the list was packed on the device (counted K3)
void LightClusterer::launch_cluster_kernels(Vulkan::CommandBuffer &cmd, const int32_t *device_count, int32_t num_ranges)
{
	const auto &rp = context->get_render_parameters();
	GrbCamera cam = {};
	std::memcpy(cam.view, rp.view.data(), 64);
	std::memcpy(cam.view_projection, rp.view_projection.data(), 64);
	std::memcpy(cam.inv_view_projection, rp.inv_view_projection.data(), 64);
	for (int i = 0; i < 3; i++)
	{
		cam.camera_position[i] = rp.camera_position[i];
		cam.camera_front[i] = rp.camera_front[i];
	}
	cam.z_near = rp.z_near;
	cam.z_far = rp.z_far;
	GrbClusterBuffers buf = get_cluster_buffers();

	// update_bindless_mask_buffer_gpu: K1 -> K2 -> K3 (stream order replaces the barriers)
	cmd.check(grb_cluster_spot_transform(&cam, &parameters, &buf, cmd.get_stream_handle()), "grb_cluster_spot_transform");
	cmd.check(grb_cluster_cull_setup(&cam, &parameters, &buf, cmd.get_stream_handle()), "grb_cluster_cull_setup");
	int tile_y0 = 0, tile_y1 = 0;
	if (lit_y1 > lit_y0 && lit_height > 0)
	{
		const GrbRows tiles = cluster_tile_rows(lit_y0, lit_y1, lit_height, int(resolution_y));
		tile_y0 = tiles.y0;
		tile_y1 = tiles.y1;
	}
	auto binning = [&](int32_t y0, int32_t y1) {
		if (device_count)
			cmd.check(grb_cluster_binning_rows_counted(&parameters, &buf, device_count, y0, y1, cmd.get_stream_handle()), "grb_cluster_binning_rows_counted");
		else
			cmd.check(grb_cluster_binning_rows(&parameters, &buf, y0, y1, cmd.get_stream_handle()), "grb_cluster_binning");
	};
	if (!lit_tile_ranges.empty())
		for (const GrbRows &r : lit_tile_ranges)
			binning(r.y0, r.y1);
	else
		binning(tile_y0, tile_y1);
	// update_bindless_range_buffer_gpu: K4
	cmd.check(grb_cluster_z_range(&buf, num_ranges, cmd.get_stream_handle()), "grb_cluster_z_range");
}
} // namespace Granite
