// scene_viewer.cpp -- application-side harness + its C API (include/granite_b200_host.h).
// Mirrors the parts of SceneViewerApplication that assemble and drive the hot path:
// add_main_pass_deferred (application/scene_viewer_application.cpp:876-991), bake_render_graph
// (:1167-1318), render_frame (:1540-1611).  The G-buffer (and motion vectors) the reference
// rasterises are uploaded from host memory by the "gbuffer" pass at the head of the graph.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/granite_b200_host.h"
#include "clusterer.hpp"
#include "nccl_collectives.hpp"
#include "post/aa.hpp"
#include "post/fxaa.hpp"
#include "post/smaa.hpp"
#include "post/hdr.hpp"
#include "renderer.hpp"

using namespace Granite;

namespace
{
thread_local std::string t_error;

int32_t fail(const std::string &msg)
{
	t_error = msg;
	return -1;
}

struct FixedExposure : HDRDynamicExposureInterface
{
	float exposure = 1.0f;
	float get_exposure() const override { return exposure; }
};

// The "bindless-shadowmaps" lock of a shadowed viewer (clusterer.cpp's external lock on the lighting pass): the caller
// renders the maps of device lights on its own streams, so the lighting pass waits on the caller's `ready` and records
// the caller's `consumed` behind its last read.  Both null (host lights, or no events given): no CUDA call at all.
struct ShadowMapEvents : RenderPassExternalLockInterface
{
	cudaEvent_t ready = nullptr, consumed = nullptr;
	const char *get_ident() const override { return "bindless-shadowmaps"; }
	Vulkan::Event external_acquire_event() override { return ready; }
	void external_release_event(Vulkan::Event, Vulkan::Stream stream) override
	{
		if (consumed)
			Vulkan::cuda_ok(cudaEventRecord(consumed, stream), "cudaEventRecord(shadow maps consumed)");
	}
};
} // namespace

struct GrbhViewer
{
	GrbhViewerConfig config;
	std::unique_ptr<Vulkan::Device> device;
	RenderGraph graph;
	RenderContext context;
	LightingParameters lighting;
	LightClusterer cluster;
	TemporalJitter jitter;
	FixedExposure exposure;
	TaskComposer composer;
	std::unique_ptr<NcclCollectives> collectives;
	std::vector<GrbRows> bands;
	unsigned rank = 0;
	// row-sharded frames presented from one rank (-1: off): the "present" pass gathers the bands there, and
	// `presented` is where this frame's whole image lies on that rank (the channel's slot, or the gathered output)
	int present_rank = -1;
	const void *presented = nullptr;
	// grbh_viewer_move_row_shards ran since the last frame: the resident G-buffer, the last output and the last depth
	// image hold the old layout's rows until a frame (which must bring the host G-buffer) renders on the new one
	bool bands_moved = false;
	// row-sharded frames lit in stripes of this many rows (0: off; grbh_viewer_set_lighting_stripes), and what this
	// frame's lighting pass left for its "lighting-exchange" pass
	unsigned lighting_stripes = 0;
	struct StripeExchange
	{
		bool peer = false;
		RenderGraphCollectives::PeerSlot slot;
	} stripe_exchange;
	// A peer channel that one source rank S fills for every rank, with credits (DESIGN.md section 5, "Feeding a sharded
	// frame from one rank")
	struct SourceHandover
	{
		RenderGraphCollectives::PeerChannel channel;
		RenderGraphCollectives::PeerSlot slot;
		bool credit_owed = false;
		// Peer memory: S waits for every rank's credit of the last epoch (the last read of every slot, by stream order);
		// any other rank waits for S's flag of this epoch and owes a credit.  false: no peer memory (the caller's NCCL path).
		bool begin(Vulkan::CommandBuffer &cmd, RenderGraphCollectives &coll, size_t bytes, unsigned source, unsigned rank)
		{
			credit_owed = false;
			if (!coll.peer_exchange_begin_frame(channel, bytes, slot))
				return false;
			credit_owed = rank != source;
			if (credit_owed)
				cmd.check(grb_peer_wait(slot.flags[rank] + source, 1, slot.epoch, cmd.get_stream_handle()), "grb_peer_wait");
			else
				cmd.check(grb_peer_wait(slot.flags[source], (int32_t)slot.count, slot.epoch - 1u, cmd.get_stream_handle()), "grb_peer_wait");
			return true;
		}
		// A receiving rank, behind its last read of slot.images[rank]: grb_peer_publish.  No-op when no credit is owed.
		void credit(Vulkan::CommandBuffer &cmd, unsigned rank)
		{
			if (credit_owed)
				cmd.check(grb_peer_publish(slot.flags, (int32_t)slot.count, (int32_t)rank, slot.epoch, slot.counter, cmd.get_stream_handle()), "grb_peer_publish");
			credit_owed = false;
		}
	};
	// row-sharded frames fed from the one rank that rasterises the whole frame (-1: off;
	// grbh_viewer_set_gbuffer_source_rank): its "gbuffer" pass pushes every rank's input rows into that rank's slot
	int gbuffer_source = -1;
	SourceHandover gbuffer_handover{ RenderGraphCollectives::PeerChannel::GBuffer };
	// the caller's ring of output images (grbh_viewer_set_output_images), wrapped once each for the ring's life (the
	// graph's cross-stream tracking keys on the wrapper), and the image, events of the next frame's acquire (-1: none)
	std::vector<std::unique_ptr<Vulkan::ImageView>> output_ring;
	int output_index = -1;
	cudaEvent_t output_acquired = nullptr, output_rendered = nullptr;
	// this frame's acquired image on the presenting rank: the "present" pass copies the assembled frame into it
	Vulkan::ImageView *present_target = nullptr;

	std::vector<std::unique_ptr<PositionalLight>> light_storage;
	PositionalLightList scene_lights;
	// the caller's light list in device memory (grbh_viewer_set_lights_device) and the prep's scratch, allocated once
	// for GRBH_MAX_DEVICE_LIGHTS input lights with the kept count in its first bytes; `device_prep_rendered`: a frame
	// has packed the bound list since it was bound
	LightClusterer::DeviceLightSource device_lights;
	ShadowMapEvents shadow_map_events;
	void *light_scratch = nullptr;
	size_t light_scratch_bytes = 0;
	bool device_prep_rendered = false;
	// row-sharded frames whose device light list comes from one rank (-1: off; grbh_viewer_set_light_source_rank): that
	// rank's clustering pass pushes the list's live entries into every other rank's slot of the light channel, and every
	// other rank binds a receiving list (grbh_viewer_set_lights_device_from_source) whose prep reads its slot
	int light_source = -1;
	SourceHandover light_handover{ RenderGraphCollectives::PeerChannel::Lights };
	// without peer memory: this rank's light slot (the source fills it, a broadcast carries it to every rank) and, past
	// its end, the flag words and counter of the source's push; allocated on the first such frame
	void *light_slot = nullptr;
	uint32_t light_slot_epoch = 0;
	// this rank's shadow map table for device lights whose maps come by id (grbh_viewer_set_light_shadow_map_table): the
	// caller's pointers, uploaded into the device table (GRBH_MAX_DEVICE_LIGHTS entries) on the clustering pass's stream
	// by the first frame after a change, and the map events that go with the table
	bool has_shadow_table = false, shadow_table_changed = false;
	std::vector<const void *> shadow_table;
	void *shadow_table_device = nullptr;
	cudaEvent_t table_maps_ready = nullptr, table_maps_consumed = nullptr;
	void upload_shadow_table(Vulkan::CommandBuffer &cmd)
	{
		if (!shadow_table_changed)
			return;
		// from pageable memory: the driver stages the bytes before the call returns (it may wait for the stream first; a
		// table changes rarely), and the copy follows every earlier frame's prep on this stream, so frames already
		// recorded keep the table they were recorded with
		if (!shadow_table.empty() &&
		    !Vulkan::cuda_ok(cudaMemcpyAsync(shadow_table_device, shadow_table.data(), sizeof(void *) * shadow_table.size(), cudaMemcpyHostToDevice,
		                                     reinterpret_cast<cudaStream_t>(cmd.get_stream())),
		                     "shadow map table upload"))
			throw std::runtime_error("clustering: the upload of the shadow map table failed");
		shadow_table_changed = false;
	}
	std::vector<mat_affine> scene_decals;

	mat4 projection = mat4(1.0f), view = mat4(1.0f);
	bool baked = false;
	std::string output_name;
	bool ui_layer_cleared = false;
	const GrbhHostGBuffer *pending_upload = nullptr;
	// this frame's G-buffer in device memory (grbh_viewer_render_frame_device), and how many passes still read it: the
	// last of them records its `consumed` event
	const GrbhDeviceGBuffer *pending_device = nullptr;
	int device_reads_left = 0;
	unsigned profiled_frames = 0;
	std::map<std::string, std::pair<double, int>> timings;
	std::vector<cudaEvent_t> pending_outputs; // one per async readback still in flight (oldest first)
	std::vector<cudaEvent_t> free_output_events;

	RenderTextureResource *res_emissive = nullptr, *res_albedo = nullptr, *res_normal = nullptr, *res_pbr = nullptr, *res_depth = nullptr,
	                      *res_mv = nullptr;

	bool uses_taa() const
	{
		return config.post_aa == GRBH_AA_TAA_LOW || config.post_aa == GRBH_AA_TAA_MEDIUM || config.post_aa == GRBH_AA_TAA_HIGH ||
		       config.post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA;
	}
	// "resolutionScale": the scene is rendered at ceil(scale * display size) (render_graph.cpp's relative-size rule)
	bool upscales() const { return config.resolution_scale > 0.0f && config.resolution_scale < 1.0f; }
	float scene_scale() const { return upscales() ? config.resolution_scale : 1.0f; }
	int render_width() const { return upscales() ? std::max(int(std::ceil(config.resolution_scale * float(config.width))), 1) : config.width; }
	int render_height() const { return upscales() ? std::max(int(std::ceil(config.resolution_scale * float(config.height))), 1) : config.height; }
	bool uses_fxaa() const { return config.post_aa == GRBH_AA_FXAA || config.post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA; }
	bool uses_smaa() const { return config.post_aa >= GRBH_AA_SMAA_LOW && config.post_aa <= GRBH_AA_SMAA_ULTRA; }
	int smaa_quality() const { return uses_smaa() ? config.post_aa - GRBH_AA_SMAA_LOW : -1; }

	// FSR 1 after the post chain: the plan's render rows are rows of the render-size image
	ShardUpscale shard_upscale() const
	{
		ShardUpscale up;
		if (upscales())
		{
			up.width = (unsigned)render_width();
			up.height = (unsigned)render_height();
			up.rcas = config.resolution_scale_sharpen != 0;
		}
		return up;
	}
	ShardPlan shard_plan() const
	{
		return compute_shard_plan((unsigned)config.width, (unsigned)config.height, bands, rank, uses_fxaa(), smaa_quality(), uses_taa(), shard_upscale());
	}
	// rows of the render-resolution inputs this rank must hold: its band + the halo the bloom
	// threshold (and FXAA through the tonemap, TAA's neighbourhood, FSR's window) reaches into
	GrbRows input_rows() const { return shard_plan().lighting; }
	bool striped() const { return lighting_stripes > 0 && bands.size() > 1; }
	StripePlan stripe_plan() const
	{
		return compute_stripe_plan((unsigned)config.width, (unsigned)config.height, bands, rank, uses_fxaa(), smaa_quality(), uses_taa(), lighting_stripes,
		                           (unsigned)config.cluster_res[1]);
	}
	// rank r's stripes: every bands.size()-th stripe from stripe r
	GrbStripes stripes_of(unsigned r) const
	{
		return GrbStripes{ (int32_t)(r * lighting_stripes), (int32_t)lighting_stripes, (int32_t)(bands.size() * lighting_stripes) };
	}
	// the G-buffer rows this rank must hold
	std::vector<GrbRows> upload_ranges() const { return striped() ? stripe_plan().upload : std::vector<GrbRows>{ input_rows() }; }
	// the same for rank q of the current bands
	std::vector<GrbRows> upload_ranges_of(unsigned q) const
	{
		if (striped())
			return compute_stripe_plan((unsigned)config.width, (unsigned)config.height, bands, q, uses_fxaa(), smaa_quality(), uses_taa(), lighting_stripes,
			                           (unsigned)config.cluster_res[1])
			    .upload;
		return { compute_shard_plan((unsigned)config.width, (unsigned)config.height, bands, q, uses_fxaa(), smaa_quality(), uses_taa(), shard_upscale()).lighting };
	}
	bool sharded_presenting() const { return bands.size() > 1 && present_rank >= 0; }
	// the final pass's attachment format, which a ring image stands in for: EASU without RCAS stores UNORM codes
	VkFormat output_format() const
	{
		if (config.hdr10_output)
			return VK_FORMAT_A2B10G10R10_UNORM_PACK32;
		return upscales() && !config.resolution_scale_sharpen ? VK_FORMAT_R8G8B8A8_UNORM : VK_FORMAT_R8G8B8A8_SRGB;
	}
	// a ring on a presenting layout belongs to the presenting rank only
	std::string check_ring_rank(size_t count) const
	{
		if (count > 0 && sharded_presenting() && rank != (unsigned)present_rank)
			return "rank " + std::to_string(rank) + " does not present (grbh_viewer_set_present_rank " + std::to_string(present_rank) +
			       "): only the presenting rank may hold output images";
		return "";
	}
	std::string check_output_images(const GrbImage *images, int32_t count) const;
	void set_output_ring(const GrbImage *images, int32_t count);
	bool fed_from_source() const { return bands.size() > 1 && gbuffer_source >= 0; }
	bool lights_from_source() const { return bands.size() > 1 && light_source >= 0; }
	void exchange_lights(Vulkan::CommandBuffer &cmd, GrbLightList &list, const int32_t *&count, GrbLightShadowIdList &ids);

	// the G-buffer planes of the attachments (grb_gbuffer_copy_rows order), the G-buffer ones and / or motion vectors
	GrbGBufferPlanes attachment_planes(bool gbuffer_planes, bool mv)
	{
		GrbGBufferPlanes a = {};
		RenderTextureResource *res[GRB_GBUFFER_PLANES] = { res_emissive, res_albedo, res_normal, res_pbr, res_depth, res_mv };
		for (int p = 0; p < GRB_GBUFFER_PLANES; p++)
			if (res[p] && (p == 5 ? mv : gbuffer_planes))
				a.plane[p] = graph.get_physical_texture_resource(*res[p]).as_grb();
		return a;
	}
	static GrbGBufferPlanes caller_planes(const GrbhDeviceGBuffer &g, bool gbuffer_planes, bool mv)
	{
		GrbGBufferPlanes a = {};
		if (gbuffer_planes)
		{
			a.plane[0] = g.emissive;
			a.plane[1] = g.albedo;
			a.plane[2] = g.normal;
			a.plane[3] = g.pbr;
			a.plane[4] = g.depth;
		}
		if (mv)
			a.plane[5] = g.mv;
		return a;
	}
	// a device G-buffer the viewer can read: every plane it needs, at the render size, in the attachment's format, with
	// a pitch that holds a row and is a multiple of the texel.  "" when it is; no device needed.
	std::string check_device_gbuffer(const GrbhDeviceGBuffer &g) const;
	void wait_ready(cudaStream_t stream, const GrbhDeviceGBuffer &g)
	{
		if (g.ready)
			Vulkan::cuda_ok(cudaStreamWaitEvent(stream, static_cast<cudaEvent_t>(g.ready), 0), "cudaStreamWaitEvent(ready)");
	}
	void record_consumed(cudaStream_t stream, const GrbhDeviceGBuffer &g)
	{
		if (g.consumed)
			Vulkan::cuda_ok(cudaEventRecord(static_cast<cudaEvent_t>(g.consumed), stream), "cudaEventRecord(consumed)");
	}
	// the "gbuffer" / "mv" pass with a device G-buffer on one rank's own: the rank's rows of the planes the pass writes
	void copy_device_rows(Vulkan::CommandBuffer &cmd, bool mv)
	{
		auto stream = reinterpret_cast<cudaStream_t>(cmd.get_stream());
		wait_ready(stream, *pending_device);
		const GrbGBufferPlanes src = caller_planes(*pending_device, !mv, mv), dst = attachment_planes(!mv, mv);
		const std::vector<GrbRows> rows = upload_ranges();
		cmd.check(grb_gbuffer_copy_rows(&src, &dst, rows.data(), (int32_t)rows.size(), cmd.get_stream_handle()), "grb_gbuffer_copy_rows");
		if (--device_reads_left == 0)
			record_consumed(stream, *pending_device);
	}
	void feed_from_source(Vulkan::CommandBuffer &cmd);

	// the presenting rank with an acquired output image: the assembled frame (`presented`, laid out as `frame`) into
	// it, behind the present pass on its stream, between the caller's two events
	void copy_presented(Vulkan::CommandBuffer &cmd, const GrbImage &frame)
	{
		if (!present_target)
			return;
		auto stream = reinterpret_cast<cudaStream_t>(cmd.get_stream());
		if (output_acquired)
			Vulkan::cuda_ok(cudaStreamWaitEvent(stream, output_acquired, 0), "cudaStreamWaitEvent(acquired)");
		const GrbImage dst = present_target->as_grb();
		if (!Vulkan::cuda_ok(cudaMemcpy2DAsync(dst.data, (size_t)dst.row_pitch, presented, (size_t)frame.row_pitch, (size_t)frame.width * 4,
		                                       (size_t)frame.height, cudaMemcpyDeviceToDevice, stream),
		                     "present: copy into the output image"))
			throw std::runtime_error("present: the copy into the acquired output image failed");
		if (output_rendered)
			Vulkan::cuda_ok(cudaEventRecord(output_rendered, stream), "cudaEventRecord(rendered)");
	}

	// the device-to-host copy of this rank's rows of the final image (the whole frame on the presenting rank), on the
	// stream of the pass that produced it
	cudaStream_t enqueue_readback(uint32_t *dst, GrbRows &rows);

	void upload_rows(Vulkan::CommandBuffer &cmd, RenderTextureResource *res, const void *host, unsigned texel)
	{
		if (!res || !host)
			return;
		auto &view_ = graph.get_physical_texture_resource(*res);
		size_t pitch = (size_t)render_width() * texel;
		for (const GrbRows &r : upload_ranges())
		{
			auto *dst = static_cast<uint8_t *>(view_.get_image().get_device_pointer()) + (size_t)r.y0 * pitch;
			auto *src = static_cast<const uint8_t *>(host) + (size_t)r.y0 * pitch;
			Vulkan::cuda_ok(cudaMemcpyAsync(dst, src, pitch * (size_t)(r.y1 - r.y0), cudaMemcpyHostToDevice, reinterpret_cast<cudaStream_t>(cmd.get_stream())),
			                "G-buffer upload");
		}
	}

	void bake_render_graph();
	void render_frame(const GrbhHostGBuffer *host, double frame_time);
	int32_t measure_row_cost_sharded(uint32_t *out, int groups);
};

void GrbhViewer::bake_render_graph()
{
	auto physical_buffers = graph.consume_physical_buffers();
	graph.reset();
	graph.set_device(device.get());
	graph.enable_timestamps(config.timestamps != 0);

	ResourceDimensions dim;
	dim.width = (unsigned)config.width;
	dim.height = (unsigned)config.height;
	dim.format = VK_FORMAT_R8G8B8A8_SRGB; // headless swapchain format (application_headless.cpp:207)
	graph.set_backbuffer_dimensions(dim);
	if (!bands.empty())
		graph.set_row_shards(bands, rank, collectives.get(), uses_fxaa(), smaa_quality(), uses_taa(), shard_upscale());

	// scene.add_render_passes(graph) -> LightClusterer::add_render_passes
	cluster.set_resolution((unsigned)config.cluster_res[0], (unsigned)config.cluster_res[1], (unsigned)config.cluster_res[2]);
	cluster.set_scene_lights(&scene_lights);
	cluster.set_base_render_context(&context);
	cluster.set_async_compute(getenv("GRB_NO_ASYNC_CLUSTER") == nullptr);
	cluster.set_enable_volumetric_decals(config.volumetric_decals != 0);
	cluster.set_scene_decals(&scene_decals);
	cluster.set_enable_shadows(config.clustered_lights_shadows != 0);
	if (config.clustered_lights_shadows)
		graph.add_external_lock_interface("bindless-shadowmaps", &shadow_map_events);
	cluster.set_shadow_resolution(config.clustered_lights_shadow_resolution > 0 ? (unsigned)config.clustered_lights_shadow_resolution : 512u);
	if (bands.size() > 1)
	{
		const GrbRows lit = input_rows();
		cluster.set_lit_pixel_rows(lit.y0, lit.y1, render_height());
	}
	else
		cluster.set_lit_pixel_rows(0, 0, 0);
	cluster.set_lit_tile_ranges(striped() ? stripe_plan().tile_rows : std::vector<GrbRows>{});
	if (lights_from_source() || config.clustered_lights_shadows)
		device_lights.exchange = [this](Vulkan::CommandBuffer &cmd, GrbLightList &list, const int32_t *&count, GrbLightShadowIdList &ids) {
			upload_shadow_table(cmd);
			if (lights_from_source())
				exchange_lights(cmd, list, count, ids);
		};
	else
		device_lights.exchange = nullptr;
	if (lights_from_source())
		device_lights.after_prep = [this](Vulkan::CommandBuffer &cmd) { light_handover.credit(cmd, rank); };
	else
		device_lights.after_prep = nullptr;
	cluster.add_render_passes(graph);
	lighting.cluster = &cluster;
	context.set_lighting_parameters(&lighting);

	// Post chain on its own stream (the reference's async-compute post, scene_viewer_application.cpp:
	// 1238-1247) unless disabled; its input image then alternates between two copies per frame.
	const bool async_post = getenv("GRB_NO_ASYNC_POST") == nullptr;
	RenderGraph::set_async_post(async_post);

	// ---- add_main_pass_deferred ----
	AttachmentInfo emissive, albedo, normal, pbr, depth;
	emissive.format = config.render_target_fp16 ? VK_FORMAT_R16G16B16A16_SFLOAT : VK_FORMAT_B10G11R11_UFLOAT_PACK32; // scene_viewer_application.cpp:882-884
	albedo.format = VK_FORMAT_R8G8B8A8_SRGB;
	normal.format = VK_FORMAT_A2B10G10R10_UNORM_PACK32;
	pbr.format = VK_FORMAT_R8G8_UNORM;
	depth.format = VK_FORMAT_D32_SFLOAT;

	// pipelined I/O: uploads on the async-compute stream into ping-pong images, so the copy of the
	// next frame's inputs overlaps this frame's lighting
	// scene_viewer_application.cpp:758-761, 888-889: the scene attachments scale with "resolutionScale"; everything
	// downstream is sized relative to them
	for (auto *info : { &emissive, &albedo, &normal, &pbr, &depth })
		info->size_x = info->size_y = scene_scale();
	const bool pipelined = config.pipelined_io != 0;
	if (pipelined)
		for (auto *info : { &emissive, &albedo, &normal, &pbr, &depth })
			info->flags |= ATTACHMENT_INFO_PINGPONG_BIT;
	auto &gbuffer = graph.add_pass("gbuffer", pipelined ? RENDER_GRAPH_QUEUE_ASYNC_COMPUTE_BIT : RENDER_GRAPH_QUEUE_GRAPHICS_BIT);
	res_emissive = &gbuffer.add_color_output("emissive", emissive);
	res_albedo = &gbuffer.add_color_output("albedo", albedo);
	res_normal = &gbuffer.add_color_output("normal", normal);
	res_pbr = &gbuffer.add_color_output("pbr", pbr);
	res_depth = &gbuffer.set_depth_stencil_output("depth-transient", depth);
	// fed from one rank: the motion vectors come through the same channel, so this pass writes them too
	res_mv = nullptr;
	if (fed_from_source() && uses_taa())
	{
		AttachmentInfo mv;
		mv.format = VK_FORMAT_R16G16_SFLOAT;
		mv.size_x = mv.size_y = scene_scale();
		res_mv = &gbuffer.add_color_output("mv-main", mv);
	}
	gbuffer.set_build_render_pass([this](Vulkan::CommandBuffer &cmd) {
		if (fed_from_source())
		{
			feed_from_source(cmd);
			return;
		}
		if (pending_device)
		{
			copy_device_rows(cmd, false);
			return;
		}
		if (!pending_upload)
			return; // inputs already resident from an earlier frame
		upload_rows(cmd, res_emissive, pending_upload->emissive, config.render_target_fp16 ? 8 : 4);
		upload_rows(cmd, res_albedo, pending_upload->albedo, 4);
		upload_rows(cmd, res_normal, pending_upload->normal, 4);
		upload_rows(cmd, res_pbr, pending_upload->pbr, 2);
		upload_rows(cmd, res_depth, pending_upload->depth, 4);
	});

	auto &lighting_pass = graph.add_pass("lighting", RENDER_GRAPH_QUEUE_GRAPHICS_BIT);
	// The reference lets HDR-main alias emissive (add_color_output(..., "emissive")) and blends in
	// place.  Here HDR-main is its own image and emissive a read-only input: same bytes moved,
	// and the uploaded G-buffer stays intact, so a resident G-buffer can be lit again next frame.
	AttachmentInfo hdr_info = emissive;
	if (async_post)
		hdr_info.flags |= ATTACHMENT_INFO_PINGPONG_BIT;
	auto &hdr_main = lighting_pass.add_color_output("HDR-main", hdr_info);
	auto &in_emissive = lighting_pass.add_attachment_input("emissive");
	auto &in_albedo = lighting_pass.add_attachment_input("albedo");
	auto &in_normal = lighting_pass.add_attachment_input("normal");
	auto &in_pbr = lighting_pass.add_attachment_input("pbr");
	auto &in_depth = lighting_pass.add_attachment_input("depth-transient");
	lighting_pass.set_depth_stencil_input("depth-transient");
	// work schedule of the lighting kernel: row costs of this frame order the next frame's rows
	BufferInfo schedule_info;
	schedule_info.size = (size_t)grb_lighting_schedule_bytes(render_height());
	schedule_info.usage = VK_BUFFER_USAGE_STORAGE_BUFFER_BIT;
	auto &schedule = lighting_pass.add_storage_output("lighting-schedule", schedule_info);
	auto light_iface = std::make_shared<DeferredLightingPass>(context, &cluster);
	light_iface->set_resources(graph, in_albedo, in_normal, in_pbr, in_depth, hdr_main, &in_emissive);
	light_iface->set_schedule(schedule);
	light_iface->set_shard_halo(uses_fxaa() ? 12u : 8u);
	lighting_pass.set_render_pass_interface(light_iface);

	std::string light_output = "HDR-main";
	if (striped())
	{
		// Lighting in stripes (DESIGN.md section 5, "Lighting in stripes"): the lighting pass lights this rank's stripes
		// and pushes the rows other ranks' lighting rows hold into their slots; "lighting-exchange" waits for every
		// rank's push and copies the rows this rank received into HDR-main.  It rewrites HDR-main in place, so every
		// reader of the lit image (TAA, threshold, tonemap, ui / pq10) follows it through the graph's dependencies.
		light_iface->set_stripes(stripes_of(rank), [this](Vulkan::CommandBuffer &cmd, Vulkan::ImageView &hdr) {
			const GrbImage image = hdr.as_grb();
			stripe_exchange.peer = graph.get_collectives()->peer_exchange_begin_frame(
			    RenderGraphCollectives::PeerChannel::HdrStripes, (size_t)image.row_pitch * (size_t)image.height, stripe_exchange.slot);
			if (!stripe_exchange.peer)
				return;
			const RenderGraphCollectives::PeerSlot &slot = stripe_exchange.slot;
			const std::vector<GrbRows> lighting_rows = graph.get_shard_plan_rows(&ShardPlan::lighting);
			cmd.check(grb_hdr_rows_to_peers(&image, slot.images, slot.flags, lighting_rows.data(), (int32_t)slot.count, (int32_t)rank, slot.epoch,
			                                slot.counter, stripes_of(rank), cmd.get_stream_handle()),
			          "grb_hdr_rows_to_peers");
		});
		auto &exchange = graph.add_pass("lighting-exchange", RENDER_GRAPH_QUEUE_GRAPHICS_BIT);
		auto &lit = exchange.add_color_output("HDR-lit", hdr_info, "HDR-main");
		exchange.set_build_render_pass([this, &lit](Vulkan::CommandBuffer &cmd) {
			auto &view_ = graph.get_physical_texture_resource(lit);
			if (stripe_exchange.peer)
			{
				const RenderGraphCollectives::PeerSlot &slot = stripe_exchange.slot;
				auto stream = reinterpret_cast<cudaStream_t>(cmd.get_stream());
				cmd.check(grb_peer_wait(slot.flags[rank], (int32_t)slot.count, slot.epoch, stream), "grb_peer_wait");
				const GrbImage image = view_.as_grb();
				const size_t pitch = (size_t)image.row_pitch;
				auto *dst = static_cast<uint8_t *>(image.data);
				const auto *src = static_cast<const uint8_t *>(slot.images[rank]);
				for (const GrbRows &r : stripe_plan().receive)
					Vulkan::cuda_ok(cudaMemcpyAsync(dst + (size_t)r.y0 * pitch, src + (size_t)r.y0 * pitch, pitch * (size_t)(r.y1 - r.y0),
					                                cudaMemcpyDeviceToDevice, stream),
					                "lighting-exchange copy");
				return;
			}
			// without peer memory: every rank's stripes to every rank, in place
			std::vector<std::vector<GrbRows>> lists;
			for (unsigned r = 0; r < bands.size(); r++)
			{
				const GrbStripes s = stripes_of(r);
				lists.emplace_back();
				for (int y = s.first; y < config.height; y += s.period)
					lists.back().push_back(GrbRows{ y, std::min(y + s.rows, config.height) });
			}
			if (!graph.get_collectives()->all_gather_row_lists(cmd, view_, lists))
				throw std::runtime_error("lighting-exchange: the all-gather of the stripes failed");
		});
		light_output = "HDR-lit";
	}

	// ---- AA before the post chain (TAA) ----
	PostAAType before = PostAAType::None;
	switch (config.post_aa)
	{
	case GRBH_AA_TAA_LOW: before = PostAAType::TAA_Low; break;
	case GRBH_AA_TAA_MEDIUM: before = PostAAType::TAA_Medium; break;
	case GRBH_AA_TAA_HIGH:
	case GRBH_AA_TAA_HIGH_PLUS_FXAA: before = PostAAType::TAA_High; break;
	default: break;
	}
	if (uses_taa() && !fed_from_source())
	{
		// add_mv_pass: the motion-vector image is an input of this path
		AttachmentInfo mv;
		mv.format = VK_FORMAT_R16G16_SFLOAT;
		mv.size_x = mv.size_y = scene_scale();
		if (pipelined)
			mv.flags |= ATTACHMENT_INFO_PINGPONG_BIT;
		auto &mv_pass = graph.add_pass("mv", pipelined ? RENDER_GRAPH_QUEUE_ASYNC_COMPUTE_BIT : RENDER_GRAPH_QUEUE_GRAPHICS_BIT);
		res_mv = &mv_pass.add_color_output("mv-main", mv);
		mv_pass.set_build_render_pass([this](Vulkan::CommandBuffer &cmd) {
			if (pending_device)
				copy_device_rows(cmd, true);
			else if (pending_upload)
				upload_rows(cmd, res_mv, pending_upload->mv, 4);
		});
	}
	bool resolved = setup_before_post_chain_antialiasing(before, graph, jitter, scene_scale(), light_output, "depth-transient", "mv-main", "HDR-resolved");
	if (resolved && async_post)
		graph.get_texture_resource("HDR-resolved").get_attachment_info().flags |= ATTACHMENT_INFO_PINGPONG_BIT;

	// ---- HDR10 swapchain: no bloom / tonemap, the scene goes to the PQ encoder (scene_viewer_application.cpp:1233-1288) ----
	std::string chain_input = resolved ? "HDR-resolved" : light_output;
	std::string ui_source;
	if (config.hdr10_output)
	{
		// "ui": the application's widgets over a layer cleared to (0, 0, 0, 1) (scene_viewer_application.cpp:1296-1302).
		// Widget rendering is the application's; this viewer draws none, so the layer is its clear colour.
		AttachmentInfo ui_info;
		ui_info.format = VK_FORMAT_R8G8B8A8_UNORM;
		ui_info.size_class = SizeClass::InputRelative;
		ui_info.size_relative_name = chain_input;
		auto &ui = graph.add_pass("ui", RENDER_GRAPH_QUEUE_GRAPHICS_BIT);
		auto &ui_layer = ui.add_color_output("ui-temporary", ui_info);
		ui.add_texture_input(chain_input);
		ui.set_get_clear_color([](unsigned, VkClearColorValue *value) {
			if (value)
			{
				value->float32[0] = value->float32[1] = value->float32[2] = 0.0f;
				value->float32[3] = 1.0f;
			}
			return true;
		});
		ui_layer_cleared = false;
		ui.set_build_render_pass([this, &ui_layer](Vulkan::CommandBuffer &cmd) {
			if (ui_layer_cleared)
				return; // nothing draws into the layer afterwards
			auto &view_ = graph.get_physical_texture_resource(ui_layer);
			const std::vector<uint32_t> clear((size_t)config.width * (size_t)config.height, 0xff000000u);
			Vulkan::cuda_ok(cudaMemcpyAsync(view_.get_image().get_device_pointer(), clear.data(), clear.size() * 4, cudaMemcpyHostToDevice,
			                                reinterpret_cast<cudaStream_t>(cmd.get_stream())),
			                "ui layer clear");
			Vulkan::cuda_ok(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(cmd.get_stream())), "ui layer clear");
			ui_layer_cleared = true;
		});

		HDR10PQEncodingConfig hdr10_config = {};
		hdr10_config.hdr_pre_exposure = 500.0f; // scene_viewer_application.cpp:1284-1285
		hdr10_config.ui_pre_exposure = 400.0f;
		VkHdrMetadataEXT md = {};
		md.displayPrimaryRed = { 0.708f, 0.292f }; // BT.2020, D65
		md.displayPrimaryGreen = { 0.170f, 0.797f };
		md.displayPrimaryBlue = { 0.131f, 0.046f };
		md.whitePoint = { 0.3127f, 0.3290f };
		md.maxContentLightLevel = config.hdr10_max_content_light_level > 0.0f ? config.hdr10_max_content_light_level : 1000.0f;
		setup_hdr10_pq_encoding(graph, "ui-output", chain_input, "ui-temporary", hdr10_config, md);
		ui_source = "ui-output";
	}
	else
	{
		// ---- HDR chain ----
		HDROptions opts;
		opts.dynamic_exposure = config.dynamic_exposure != 0;
		if (config.hdr_bloom)
			setup_hdr_postprocess_compute(graph, context.get_frame_parameters(), chain_input, "tonemapped", opts, &exposure);
		else
		{
			// BASELINE config 1: a single tonemap pass.  tonemap.frag always samples uBloom; with
			// bloom off that image is the zero-initialised one nothing ever writes.
			AttachmentInfo quarter;
			quarter.format = VK_FORMAT_R16G16B16A16_SFLOAT;
			quarter.size_class = SizeClass::InputRelative;
			quarter.size_relative_name = chain_input;
			quarter.size_x = 0.25f;
			quarter.size_y = 0.25f;
			auto &off = graph.add_pass("bloom-disabled", RENDER_GRAPH_QUEUE_COMPUTE_BIT);
			off.add_storage_texture_output("upsample-0", quarter);
			off.add_texture_input(chain_input);
			off.set_build_render_pass([](Vulkan::CommandBuffer &) {});
			AttachmentInfo tonemap_info;
			tonemap_info.size_class = SizeClass::InputRelative;
			tonemap_info.size_relative_name = chain_input;
			auto &tonemap = graph.add_pass("tonemap", RenderGraph::get_default_post_graphics_queue());
			auto &out = tonemap.add_color_output("tonemapped", tonemap_info);
			auto &hdr_res = tonemap.add_texture_input(chain_input);
			auto &bloom_res = tonemap.add_texture_input("upsample-0");
			tonemap.set_build_render_pass([this, &out, &hdr_res, &bloom_res](Vulkan::CommandBuffer &cmd) {
				GrbImage hdr = graph.get_physical_texture_resource(hdr_res).as_grb();
				GrbImage bloom = graph.get_physical_texture_resource(bloom_res).as_grb();
				auto &ov = graph.get_physical_texture_resource(out);
				GrbImage o = ov.as_grb();
				cmd.check(grb_tonemap(&hdr, &bloom, nullptr, exposure.get_exposure(), &o, graph.is_sharded() ? graph.get_shard_plan().tonemap : GrbRows{ 0, 0 },
				                      cmd.get_stream_handle()),
				          "grb_tonemap");
			});
		}
		ui_source = "tonemapped";

		// ---- AA after the post chain (FXAA) ----
		if (uses_fxaa())
		{
			setup_fxaa_postprocess(graph, ui_source, "post-aa-output");
			ui_source = "post-aa-output";
		}
		else if (uses_smaa())
		{
			const PostAAType type = config.post_aa == GRBH_AA_SMAA_LOW ? PostAAType::SMAA_Low :
			                        (config.post_aa == GRBH_AA_SMAA_MEDIUM ? PostAAType::SMAA_Medium :
			                                                                 (config.post_aa == GRBH_AA_SMAA_HIGH ? PostAAType::SMAA_High : PostAAType::SMAA_Ultra));
			if (setup_after_post_chain_antialiasing(type, graph, jitter, scene_scale(), ui_source, "depth-transient", "post-aa-output"))
				ui_source = "post-aa-output";
		}
	}
	// scene_viewer_application.cpp:1263-1268: FSR 1 from the scaled-down image to the swapchain size
	if (upscales() && setup_after_post_chain_upscaling(graph, ui_source, "post-scale-output", config.resolution_scale_sharpen != 0))
		ui_source = "post-scale-output";
	presented = nullptr;
	if (sharded_presenting())
	{
		// on the stream of the pass that writes the final image, so that the readback on the presenting rank (same
		// stream) orders its frames' pushes behind its earlier readbacks (DESIGN.md section 5, "Presenting a sharded frame")
		auto &source = graph.get_texture_resource(ui_source);
		auto &present = graph.add_pass("present", graph.get_writer_queue(source));
		auto &frame = present.add_color_output("presented", source.get_attachment_info(), ui_source);
		present.set_build_render_pass([this, &frame](Vulkan::CommandBuffer &cmd) {
			auto &view_ = graph.get_physical_texture_resource(frame);
			const GrbImage image = view_.as_grb();
			void *stream = cmd.get_stream_handle();
			const unsigned P = (unsigned)present_rank;
			RenderGraphCollectives::PeerSlot slot;
			if (graph.get_collectives()->peer_exchange_begin_frame(RenderGraphCollectives::PeerChannel::Present, (size_t)image.row_pitch * (size_t)image.height,
			                                                       slot))
			{
				// the credit: P's push of the last frame ran after P's readback of the frame before, the last one that
				// used this frame's slot
				cmd.check(grb_peer_wait(slot.flags[rank] + P, 1, slot.epoch - 1u, stream), "grb_peer_wait");
				cmd.check(grb_present_rows_to_peer(&image, slot.images[P], slot.flags, (int32_t)slot.count, (int32_t)rank, slot.epoch, slot.counter,
				                                   bands[rank], stream),
				          "grb_present_rows_to_peer");
				if (rank == P)
				{
					cmd.check(grb_peer_wait(slot.flags[rank], (int32_t)slot.count, slot.epoch, stream), "grb_peer_wait");
					presented = slot.images[P];
					copy_presented(cmd, image);
				}
				return;
			}
			// without peer memory: every rank's band to every rank, in place (the output image is full-size everywhere)
			graph.get_collectives()->all_gather_rows(cmd, view_, bands);
			presented = image.data;
			copy_presented(cmd, image);
		});
		ui_source = "presented";
	}
	output_name = ui_source;
	graph.set_backbuffer_source(ui_source);
	graph.bake();
	// keep feed-back buffers (average luminance) across re-bakes
	graph.install_physical_buffers(std::move(physical_buffers));
	baked = true;
}

std::string GrbhViewer::check_device_gbuffer(const GrbhDeviceGBuffer &g) const
{
	const int w = render_width(), h = render_height();
	struct Plane
	{
		const char *name;
		const GrbImage *image;
		int32_t format, texel;
		bool required;
	};
	const Plane planes[] = {
		{ "emissive", &g.emissive, config.render_target_fp16 ? GRB_FORMAT_R16G16B16A16_SFLOAT : GRB_FORMAT_B10G11R11_UFLOAT_PACK32, config.render_target_fp16 ? 8 : 4,
		  true },
		{ "albedo", &g.albedo, GRB_FORMAT_R8G8B8A8_SRGB, 4, true },
		{ "normal", &g.normal, GRB_FORMAT_A2B10G10R10_UNORM_PACK32, 4, true },
		{ "pbr", &g.pbr, GRB_FORMAT_R8G8_UNORM, 2, true },
		{ "depth", &g.depth, GRB_FORMAT_D32_SFLOAT, 4, true },
		{ "mv", &g.mv, GRB_FORMAT_R16G16_SFLOAT, 4, uses_taa() },
	};
	for (const Plane &p : planes)
	{
		const GrbImage &im = *p.image;
		const std::string name = std::string("the ") + p.name + " plane";
		if (!p.required)
			continue; // motion vectors without TAA: nothing reads them
		if (!im.data)
			return name + " is missing" + (std::string(p.name) == "mv" ? " (TAA reads the motion vectors)" : "");
		if (im.width != w || im.height != h)
			return name + " is " + std::to_string(im.width) + " x " + std::to_string(im.height) + "; the viewer renders at " + std::to_string(w) + " x " +
			       std::to_string(h) + " (grbh_viewer_get_render_size)";
		if (im.format != p.format)
			return name + " has format " + std::to_string(im.format) + "; the attachment's is " + std::to_string(p.format);
		if (im.row_pitch < w * p.texel || im.row_pitch % p.texel != 0)
			return name + "'s row_pitch " + std::to_string(im.row_pitch) + " must be a multiple of its texel size (" + std::to_string(p.texel) +
			       " bytes) and at least width x texel (" + std::to_string(w * p.texel) + ")";
	}
	return "";
}

std::string GrbhViewer::check_output_images(const GrbImage *images, int32_t count) const
{
	if (count < 0 || (count > 0 && !images))
		return "bad arguments (count " + std::to_string(count) + (images ? ")" : ", images NULL)");
	const int w = config.width, h = config.height;
	const int32_t format = config.hdr10_output ? GRB_FORMAT_A2B10G10R10_UNORM_PACK32 : GRB_FORMAT_R8G8B8A8_SRGB;
	for (int32_t i = 0; i < count; i++)
	{
		const GrbImage &im = images[i];
		const std::string name = "output image " + std::to_string(i);
		if (!im.data)
			return name + " has no memory";
		if (im.width != w || im.height != h)
			return name + " is " + std::to_string(im.width) + " x " + std::to_string(im.height) + "; the display size is " + std::to_string(w) + " x " +
			       std::to_string(h);
		if (im.format != format)
			return name + " has format " + std::to_string(im.format) + "; the viewer's output format is " + std::to_string(format) +
			       (config.hdr10_output ? " (A2B10G10R10_UNORM_PACK32: HDR10 output)" : " (R8G8B8A8_SRGB)");
		if (im.row_pitch < w * 4 || im.row_pitch % 16 != 0)
			return name + "'s row_pitch " + std::to_string(im.row_pitch) + " must be a multiple of 16 bytes and at least width x 4 (" + std::to_string(w * 4) + ")";
		if (reinterpret_cast<uintptr_t>(im.data) % 16 != 0)
			return name + "'s base address is not 16-byte aligned";
	}
	// each image's bytes from its first texel to its last, as the final kernels may write them
	auto span = [&](const GrbImage &im) {
		const uintptr_t b = reinterpret_cast<uintptr_t>(im.data);
		return std::make_pair(b, b + (uintptr_t)im.row_pitch * (uintptr_t)(h - 1) + (uintptr_t)w * 4);
	};
	for (int32_t i = 0; i < count; i++)
		for (int32_t j = i + 1; j < count; j++)
		{
			const auto a = span(images[i]), b = span(images[j]);
			if (a.first < b.second && b.first < a.second)
				return "output images " + std::to_string(i) + " and " + std::to_string(j) + " overlap";
		}
	return check_ring_rank((size_t)count);
}

void GrbhViewer::set_output_ring(const GrbImage *images, int32_t count)
{
	// the caller may free an image of the old ring once its last frame's `rendered` event has completed: nothing of
	// it stays in the graph's tracking
	for (const auto &view_ : output_ring)
		graph.forget_image(view_->get_image());
	output_ring.clear();
	output_index = -1;
	output_acquired = output_rendered = nullptr;
	Vulkan::ImageCreateInfo info;
	info.width = (unsigned)config.width;
	info.height = (unsigned)config.height;
	info.format = output_format();
	for (int32_t i = 0; i < count; i++)
		output_ring.emplace_back(new Vulkan::ImageView(std::make_shared<Vulkan::Image>(*device, info, images[i].data, (unsigned)images[i].row_pitch)));
}

// Feeding from the rank S that rasterised the whole frame.  Peer path: S pushes each rank q's input rows into q's slot
// and copies its own; every other rank copies its rows out of its slot.  Without peer memory: S copies every rank's
// input rows into its own attachments, and per-plane NCCL broadcasts from S write them into every rank's in place.
void GrbhViewer::feed_from_source(Vulkan::CommandBuffer &cmd)
{
	const unsigned S = (unsigned)gbuffer_source;
	auto stream = reinterpret_cast<cudaStream_t>(cmd.get_stream());
	void *handle = cmd.get_stream_handle();
	const GrbGBufferPlanes attachments = attachment_planes(true, true);
	const GrbhDeviceGBuffer *in = rank == S ? pending_device : nullptr;
	if (rank == S && !in)
		throw std::runtime_error("gbuffer: the source rank needs the whole frame's G-buffer every frame");
	GrbGBufferPlanes src = {};
	if (in)
	{
		wait_ready(stream, *in);
		src = caller_planes(*in, true, uses_taa());
	}
	uint64_t bytes = 0;
	if (!cmd.check(grb_gbuffer_slot_layout(&attachments, nullptr, nullptr, &bytes), "grb_gbuffer_slot_layout"))
		return;
	RenderGraphCollectives *coll = graph.get_collectives();
	if (gbuffer_handover.begin(cmd, *coll, (size_t)bytes, S, rank))
	{
		const RenderGraphCollectives::PeerSlot &slot = gbuffer_handover.slot;
		const std::vector<GrbRows> own = upload_ranges();
		if (rank == S)
		{
			std::vector<GrbRows> rows;
			std::vector<int32_t> counts;
			for (unsigned q = 0; q < slot.count; q++)
			{
				const std::vector<GrbRows> r = q == S ? std::vector<GrbRows>{} : upload_ranges_of(q);
				rows.insert(rows.end(), r.begin(), r.end());
				counts.push_back((int32_t)r.size());
			}
			cmd.check(grb_gbuffer_rows_to_peers(&src, slot.images, slot.flags, rows.data(), counts.data(), (int32_t)slot.count, (int32_t)S, slot.epoch,
			                                    slot.counter, handle),
			          "grb_gbuffer_rows_to_peers");
			cmd.check(grb_gbuffer_copy_rows(&src, &attachments, own.data(), (int32_t)own.size(), handle), "grb_gbuffer_copy_rows");
			record_consumed(stream, *in);
			return;
		}
		GrbGBufferPlanes received = {};
		cmd.check(grb_gbuffer_slot_layout(&attachments, slot.images[rank], &received, &bytes), "grb_gbuffer_slot_layout");
		cmd.check(grb_gbuffer_copy_rows(&received, &attachments, own.data(), (int32_t)own.size(), handle), "grb_gbuffer_copy_rows");
		gbuffer_handover.credit(cmd, rank);
		return;
	}
	// without peer memory: the union of every rank's input rows, broadcast from S
	std::vector<GrbRows> all;
	for (unsigned q = 0; q < bands.size(); q++)
	{
		const std::vector<GrbRows> r = upload_ranges_of(q);
		all.insert(all.end(), r.begin(), r.end());
	}
	std::sort(all.begin(), all.end(), [](const GrbRows &a, const GrbRows &b) { return a.y0 < b.y0; });
	std::vector<GrbRows> merged;
	for (const GrbRows &r : all)
	{
		if (r.y1 <= r.y0)
			continue;
		if (!merged.empty() && r.y0 <= merged.back().y1)
			merged.back().y1 = std::max(merged.back().y1, r.y1);
		else
			merged.push_back(r);
	}
	if (rank == S)
	{
		cmd.check(grb_gbuffer_copy_rows(&src, &attachments, merged.data(), (int32_t)merged.size(), handle), "grb_gbuffer_copy_rows");
		record_consumed(stream, *in);
	}
	std::vector<std::vector<GrbRows>> lists(bands.size());
	lists[S] = merged;
	for (RenderTextureResource *res : { res_emissive, res_albedo, res_normal, res_pbr, res_depth, res_mv })
		if (res && !coll->all_gather_row_lists(cmd, graph.get_physical_texture_resource(*res), lists))
			throw std::runtime_error("gbuffer: the broadcast of the G-buffer rows from the source rank failed");
}

// The light channel of a row-sharded frame whose device lights come from rank S (DESIGN.md section 5, "Lights from
// device memory", "From one rank"), on the clustering pass's stream after the lights' `ready`.  Peer path: S pushes its
// list's live entries into every rank's slot, then preps its own list; every other rank preps its slot (the list and
// count returned here) and raises its credit behind the prep (`after_prep`).  Without peer memory: S fills its own
// slot with the same kernel and a broadcast from S carries the whole slot into every rank's, in stream order with the
// prep that reads it.  A shadowed viewer's slot also holds each live light's shadow transform and map id (the shadowed
// slot of grb_light_shadow_slot_layout); every rank resolves the ids through its own map table.
void GrbhViewer::exchange_lights(Vulkan::CommandBuffer &cmd, GrbLightList &list, const int32_t *&count, GrbLightShadowIdList &ids)
{
	const unsigned S = (unsigned)light_source;
	const bool shadowed = config.clustered_lights_shadows != 0;
	void *handle = cmd.get_stream_handle();
	uint64_t bytes = 0;
	if (shadowed ? !cmd.check(grb_light_shadow_slot_layout(nullptr, nullptr, nullptr, &bytes), "grb_light_shadow_slot_layout")
	             : !cmd.check(grb_light_slot_layout(nullptr, nullptr, nullptr, &bytes), "grb_light_slot_layout"))
		return;
	// S's push of its list (and shadow ids) into `slots`
	auto push = [&](void *const *slots, uint32_t *const *flags, int32_t peers, int32_t index, uint32_t epoch, uint32_t *counter) {
		if (shadowed)
			cmd.check(grb_light_list_shadowed_to_peers(&list, &ids, count, slots, flags, peers, index, epoch, counter, handle), "grb_light_list_shadowed_to_peers");
		else
			cmd.check(grb_light_list_to_peers(&list, count, slots, flags, peers, index, epoch, counter, handle), "grb_light_list_to_peers");
	};
	RenderGraphCollectives *coll = graph.get_collectives();
	void *received = nullptr;
	if (light_handover.begin(cmd, *coll, (size_t)bytes, S, rank))
	{
		const RenderGraphCollectives::PeerSlot &slot = light_handover.slot;
		if (rank == S)
		{
			push(slot.images, slot.flags, (int32_t)slot.count, (int32_t)S, slot.epoch, slot.counter);
			return;
		}
		received = slot.images[rank];
	}
	else
	{
		if (!light_slot)
		{
			// zeroed on the pass's stream, ahead of the first push and broadcast (the push's counter must start at 0)
			void *p = nullptr;
			if (!Vulkan::cuda_ok(cudaMalloc(&p, (size_t)bytes + 256), "cudaMalloc(light slot)") ||
			    !Vulkan::cuda_ok(cudaMemsetAsync(p, 0, (size_t)bytes + 256, cmd.get_stream()), "cudaMemsetAsync(light slot)"))
			{
				cudaFree(p);
				throw std::runtime_error("clustering: allocating the light slot failed");
			}
			light_slot = p;
		}
		if (rank == S)
		{
			void *slots[1] = { light_slot };
			uint32_t *flags[1] = { reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(light_slot) + bytes) };
			push(slots, flags, 1, 0, ++light_slot_epoch, flags[0] + 8);
		}
		if (!coll->broadcast_bytes(cmd.get_stream(), light_slot, (size_t)bytes, S))
			throw std::runtime_error("clustering: the broadcast of the light list from the source rank failed");
		if (rank == S)
			return;
		received = light_slot;
	}
	// this frame's slot as a list of this rank's own capacity: the prep clamps the pushed count to it
	GrbLightList slot_list = {};
	int32_t *slot_count = nullptr;
	if (!cmd.check(grb_light_slot_layout(received, &slot_list, &slot_count, &bytes), "grb_light_slot_layout"))
		return;
	slot_list.count = list.count;
	slot_list.cutoff_range = list.cutoff_range;
	list = slot_list;
	count = slot_count;
	if (shadowed)
	{
		float *transforms = nullptr;
		int32_t *map_ids = nullptr;
		if (!cmd.check(grb_light_shadow_slot_layout(received, &transforms, &map_ids, &bytes), "grb_light_shadow_slot_layout"))
			return;
		ids.transforms = transforms;
		ids.map_ids = map_ids;
	}
}

cudaStream_t GrbhViewer::enqueue_readback(uint32_t *dst, GrbRows &r)
{
	if (bands_moved)
		throw std::runtime_error("output readback: the bands moved (grbh_viewer_move_row_shards) since the last frame; render a frame first");
	auto &output = graph.get_texture_resource(output_name);
	// the graph-owned output image, or the caller's image the last frame went into (any pitch)
	const Vulkan::Image &image = graph.get_physical_texture_resource(output).get_image();
	const void *base = image.get_device_pointer();
	size_t src_pitch = image.get_row_pitch();
	r = bands.size() > 1 ? bands[rank] : GrbRows{ 0, config.height };
	if (sharded_presenting() && rank == (unsigned)present_rank)
	{
		if (!presented)
			throw std::runtime_error("output readback: no frame has been presented since the last bake");
		base = presented; // the same size and pitch as the graph-owned output image
		r = GrbRows{ 0, config.height };
	}
	const size_t pitch = (size_t)config.width * 4;
	auto stream = reinterpret_cast<cudaStream_t>(graph.get_writer_stream(output));
	if (!Vulkan::cuda_ok(cudaMemcpy2DAsync(reinterpret_cast<uint8_t *>(dst) + (size_t)r.y0 * pitch, pitch, static_cast<const uint8_t *>(base) + (size_t)r.y0 * src_pitch,
	                                       src_pitch, pitch, (size_t)(r.y1 - r.y0), cudaMemcpyDeviceToHost, stream),
	                     "output readback"))
		throw std::runtime_error("cudaMemcpyAsync failed");
	return stream;
}

// The row cost of a row-sharded frame: each rank measures the rows it produced (its band, or its render rows under
// FSR 1), whose depth it holds and whose cluster tiles it binned, into a zero-filled whole-frame vector; an integer
// all-reduce then sums the ranks' disjoint pieces.  The kernel charges each 4-row group for its own pixels only and
// sums with integer atomics, so with every cut on a multiple of 4 rows the result is the unsharded viewer's, bit for
// bit.  Collective: every rank calls it after the same frame.
int32_t GrbhViewer::measure_row_cost_sharded(uint32_t *out, int groups)
{
	if (bands_moved)
		return fail("grbh_viewer_measure_row_cost: the bands moved (grbh_viewer_move_row_shards) since the last frame; render a frame first");
	for (const GrbRows &r : graph.get_shard_plan_rows(&ShardPlan::render_own))
		if (!striped() && r.y0 % 4 != 0)
			return fail("grbh_viewer_measure_row_cost: a row-sharded measurement needs every cut on a multiple of 4 rows (render row " +
			            std::to_string(r.y0) + ")");
	RenderGraphCollectives *coll = graph.get_collectives();
	device->wait_idle();
	// the rows whose depth this rank holds and whose tiles it binned: its stripes (multiples of 8 rows), or its band
	const std::vector<GrbRows> measured = striped() ? stripe_plan().lit : std::vector<GrbRows>{ shard_plan().render_own };
	GrbImage depth = graph.get_physical_texture_resource(*res_depth).as_grb();
	GrbCamera cam;
	if (grbh_viewer_get_camera(this, &cam, nullptr, nullptr) != 0)
		return -1;
	GrbClusterParameters params = cluster.get_cluster_parameters_bindless();
	GrbClusterBuffers buffers = cluster.get_cluster_buffers();
	auto stream = reinterpret_cast<cudaStream_t>(device->get_stream());
	uint32_t *dev = nullptr;
	if (!Vulkan::cuda_ok(cudaMalloc(&dev, sizeof(uint32_t) * groups), "cudaMalloc"))
		return fail("cudaMalloc failed");
	bool ok = Vulkan::cuda_ok(cudaMemsetAsync(dev, 0, sizeof(uint32_t) * groups, stream), "cudaMemsetAsync");
	int32_t rc = GRB_OK;
	for (size_t i = 0; ok && rc == GRB_OK && i < measured.size(); i++)
		rc = grb_lighting_row_cost(&depth, &cam, &params, &buffers, measured[i], dev + measured[i].y0 / 4, stream);
	const std::string kernel_error = rc != GRB_OK ? grb_last_error_string() : "";
	// every rank joins the reduction, also one whose own part failed, so that no peer waits in it alone
	const bool reduced = coll && coll->all_reduce_sum_u32(stream, dev, (size_t)groups);
	const bool synced = Vulkan::cuda_ok(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
	ok = ok && rc == GRB_OK && reduced && synced && Vulkan::cuda_ok(cudaMemcpy(out, dev, sizeof(uint32_t) * groups, cudaMemcpyDeviceToHost), "cudaMemcpy");
	cudaFree(dev);
	if (!ok)
		return fail(!kernel_error.empty() ? kernel_error
		                                  : (reduced ? "grbh_viewer_measure_row_cost: copy failed" : "grbh_viewer_measure_row_cost: the all-reduce over the ranks failed"));
	return groups;
}

void GrbhViewer::render_frame(const GrbhHostGBuffer *host, double frame_time)
{
	FrameParameters frame = context.get_frame_parameters();
	frame.frame_time = frame_time;
	frame.elapsed_time += frame_time;
	context.set_frame_parameters(frame);

	// an acquired ring image: the backbuffer itself, or on the presenting rank the target of the present pass's copy
	Vulkan::ImageView *acquired = output_index >= 0 ? output_ring[(size_t)output_index].get() : nullptr;
	output_index = -1;
	const bool bind = acquired && !sharded_presenting();
	{
		Vulkan::ScopedHostTimer timer("frame.setup_attachments");
		graph.setup_attachments(*device, bind ? acquired : nullptr);
		cluster.setup_render_pass_resources(graph);
	}

	// update_scene: jitter.step, context.set_camera, LightClusterer::refresh
	{
		Vulkan::ScopedHostTimer timer("frame.camera + cluster refresh");
		// scene_viewer_application.cpp:1431-1432: the frame is rendered (and clustered, and lit) with the
		// jittered projection; the reprojection keeps the unjittered history (temporal.cpp:239-243)
		jitter.step(projection, view);
		context.set_camera(jitter.get_jittered_projection(), view);
		cluster.refresh(context);
	}

	pending_upload = host;
	present_target = bind ? nullptr : acquired;
	if (bind)
		graph.set_backbuffer_events(output_acquired, output_rendered);
	{
		Vulkan::ScopedHostTimer timer("frame.enqueue_render_passes");
		try
		{
			graph.enqueue_render_passes(*device, composer);
		}
		catch (...)
		{
			pending_upload = nullptr;
			present_target = nullptr;
			throw;
		}
	}
	pending_upload = nullptr;
	present_target = nullptr;
	profiled_frames++;
	device_prep_rendered = cluster.has_device_lights();

	if (config.timestamps == 1)
		for (auto &iv : device->collect_time_intervals())
		{
			auto &slot = timings[iv.first];
			slot.first += iv.second;
			slot.second++;
		}
}

// ----------------------------------------------------------------------------- C API
#define GRBH_TRY try {
#define GRBH_CATCH                                  \
	}                                               \
	catch (const std::exception &e)                 \
	{                                               \
		return fail(e.what());                      \
	}                                               \
	catch (...)                                     \
	{                                               \
		return fail("unknown C++ exception");       \
	}

extern "C" const char *grbh_last_error(void)
{
	return t_error.c_str();
}

extern "C" uint16_t grbh_float_to_half(float v)
{
	return muglm::floatToHalf(v);
}

extern "C" int32_t grbh_viewer_create(const GrbhViewerConfig *config, GrbhViewer **out)
{
	if (!config || !out || config->width <= 0 || config->height <= 0)
		return fail("grbh_viewer_create: bad config");
	if (config->hdr10_output && (config->post_aa == GRBH_AA_FXAA || config->post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA))
		return fail("grbh_viewer_create: FXAA reads the tonemapped 8-bit image; an HDR10 output has none (use TAA)");
	if (config->hdr10_output && config->post_aa >= GRBH_AA_SMAA_LOW && config->post_aa <= GRBH_AA_SMAA_ULTRA)
		return fail("grbh_viewer_create: SMAA reads the tonemapped 8-bit image; an HDR10 output has none (use TAA)");
	if (config->resolution_scale > 0.0f && config->resolution_scale < 1.0f && config->hdr10_output)
		return fail("grbh_viewer_create: FSR 1 upscaling reads the tonemapped 8-bit image; an HDR10 output has none");
	if (config->render_target_fp16 && config->hdr10_output)
		return fail("grbh_viewer_create: the HDR10 / PQ encoder reads a B10G11R11 scene image; render_target_fp16 is not supported with it");
	if (!(config->resolution_scale >= 0.0f && config->resolution_scale <= 1.0f))
		return fail("grbh_viewer_create: resolution_scale must be within [0, 1] (0 or 1 = off)");
	GRBH_TRY
	auto v = std::make_unique<GrbhViewer>();
	v->config = *config;
	if (v->config.cluster_res[0] == 0)
	{
		v->config.cluster_res[0] = 128; // scene_viewer_application.cpp:407
		v->config.cluster_res[1] = 64;
		v->config.cluster_res[2] = 4096;
	}
	// cuda_device < 0: host-only viewer (camera / light preparation without touching a GPU)
	if (config->cuda_device >= 0)
		v->device = std::make_unique<Vulkan::Device>(config->cuda_device, static_cast<Vulkan::Stream>(config->cuda_stream));
	v->lighting.directional.color = vec3(6.0f, 5.5f, 4.5f); // scene_viewer_application.cpp:380
	v->lighting.directional.direction = normalize(vec3(0.3f, 0.8f, 0.5f));
	*out = v.release();
	return 0;
	GRBH_CATCH
}

extern "C" void grbh_viewer_destroy(GrbhViewer *viewer)
{
	if (!viewer)
		return;
	if (viewer->device)
		viewer->device->wait_idle();
	Vulkan::HostProfile::report(viewer->profiled_frames);
	for (auto e : viewer->pending_outputs)
		cudaEventDestroy(e);
	for (auto e : viewer->free_output_events)
		cudaEventDestroy(e);
	viewer->graph.reset();
	if (viewer->light_scratch)
		cudaFree(viewer->light_scratch);
	if (viewer->light_slot)
		cudaFree(viewer->light_slot);
	if (viewer->shadow_table_device)
		cudaFree(viewer->shadow_table_device);
	if (viewer->device)
		Granite::release_smaa_lookup_textures(*viewer->device); // device images: must go before the device does
	delete viewer;
}

extern "C" int32_t grbh_viewer_set_camera(GrbhViewer *v, const float *projection16, const float *view16)
{
	if (!v || !projection16 || !view16)
		return fail("grbh_viewer_set_camera: null");
	std::memcpy(v->projection.data(), projection16, 64);
	std::memcpy(v->view.data(), view16, 64);
	v->context.set_camera(v->projection, v->view);
	return 0;
}

extern "C" int32_t grbh_viewer_set_directional(GrbhViewer *v, const float *color3, const float *direction3)
{
	if (!v || !color3 || !direction3)
		return fail("grbh_viewer_set_directional: null");
	v->lighting.directional.color = vec3(color3[0], color3[1], color3[2]);
	v->lighting.directional.direction = vec3(direction3[0], direction3[1], direction3[2]);
	return 0;
}

extern "C" int32_t grbh_viewer_set_exposure(GrbhViewer *v, float exposure)
{
	if (!v)
		return fail("null viewer");
	v->exposure.exposure = exposure;
	return 0;
}

extern "C" int32_t grbh_viewer_set_lights(GrbhViewer *v, const GrbhLights *l)
{
	if (!v || !l || l->count < 0)
		return fail("grbh_viewer_set_lights: bad arguments");
	GRBH_TRY
	v->cluster.set_device_lights(nullptr);
	v->device_prep_rendered = false;
	v->device_lights.shadows = {};
	v->device_lights.by_id = false;
	v->device_lights.shadow_ids = {};
	v->device_lights.input_count = nullptr;
	v->shadow_map_events.ready = v->shadow_map_events.consumed = nullptr;
	v->light_storage.clear();
	v->scene_lights.clear();
	for (int i = 0; i < l->count; i++)
	{
		vec3 color(l->color[3 * i], l->color[3 * i + 1], l->color[3 * i + 2]);
		vec3 pos(l->position[3 * i], l->position[3 * i + 1], l->position[3 * i + 2]);
		PositionalLightInfo info;
		if (l->is_point[i])
		{
			auto p = std::make_unique<PointLight>();
			p->set_maximum_range(l->cutoff_range);
			p->set_color(color);
			info.transform = mat_affine(vec4(1, 0, 0, pos.x), vec4(0, 1, 0, pos.y), vec4(0, 0, 1, pos.z));
			info.light = p.get();
			v->light_storage.push_back(std::move(p));
		}
		else
		{
			auto s = std::make_unique<SpotLight>();
			s->set_maximum_range(l->cutoff_range);
			s->set_color(color);
			s->set_spot_parameters(l->inner_cone[i], l->outer_cone[i]);
			const float *r = l->rotation + 9 * i; // column-major 3x3
			info.transform = mat_affine(vec4(r[0], r[3], r[6], pos.x), vec4(r[1], r[4], r[7], pos.y), vec4(r[2], r[5], r[8], pos.z));
			info.light = s.get();
			v->light_storage.push_back(std::move(s));
		}
		v->scene_lights.push_back(info);
	}
	return 0;
	GRBH_CATCH
}

namespace
{
// false (and the error set) unless [data, data + bytes) starts and ends in device memory of the viewer's device
bool is_viewer_device_memory(GrbhViewer *v, const std::string &fn, const char *name, const void *data, size_t bytes)
{
	const uint8_t *base = static_cast<const uint8_t *>(data);
	for (const uint8_t *p : { base, base + bytes - 1 })
	{
		cudaPointerAttributes attr = {};
		const cudaError_t err = cudaPointerGetAttributes(&attr, p);
		if (err != cudaSuccess)
			cudaGetLastError();
		if (err != cudaSuccess || (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged) ||
		    attr.device != v->device->get_device_index())
		{
			fail(fn + name + " is not device memory of the viewer's device (" + std::to_string(v->device->get_device_index()) + ")");
			return false;
		}
	}
	return true;
}

// grbh_viewer_set_lights_device[_shadowed] once the arguments that need no CUDA call have passed
int32_t bind_device_lights(GrbhViewer *v, const GrbhDeviceLights *l, const GrbhDeviceLightShadows *sh, const std::string &fn)
{
	cudaSetDevice(v->device->get_device_index());
	if (l->count > 0)
	{
		const struct
		{
			const char *name;
			const void *data;
			size_t bytes;
		} arrays[] = { { "color", l->color, 12 }, { "position", l->position, 12 }, { "is_point", l->is_point, 1 },
			           { "rotation", l->rotation, 36 }, { "inner_cone", l->inner_cone, 4 }, { "outer_cone", l->outer_cone, 4 } };
		for (const auto &a : arrays)
		{
			if (!a.data)
				return fail(fn + "null " + a.name);
			// the first and the last byte of each array are device memory of the viewer's device
			if (!is_viewer_device_memory(v, fn, a.name, a.data, a.bytes * (size_t)l->count))
				return -1;
		}
		if (sh && (!is_viewer_device_memory(v, fn, "shadow transforms", sh->transforms, 64 * (size_t)l->count) ||
		           !is_viewer_device_memory(v, fn, "shadow maps", sh->maps, 8 * (size_t)l->count)))
			return -1;
	}
	if (!v->light_scratch)
	{
		const uint64_t bytes = grb_light_prep_scratch_bytes(GRBH_MAX_DEVICE_LIGHTS);
		if (bytes == 0)
			return fail(fn + "grb_light_prep_scratch_bytes failed: " + grb_last_error_string());
		if (!Vulkan::cuda_ok(cudaMalloc(&v->light_scratch, (size_t)bytes + 256), "cudaMalloc(light prep scratch)"))
		{
			v->light_scratch = nullptr;
			return fail(fn + "cudaMalloc of the prep scratch failed");
		}
		v->light_scratch_bytes = (size_t)bytes;
	}
	auto &d = v->device_lights;
	d.list.count = l->count;
	d.list.color = l->color;
	d.list.position = l->position;
	d.list.is_point = l->is_point;
	d.list.rotation = l->rotation;
	d.list.inner_cone = l->inner_cone;
	d.list.outer_cone = l->outer_cone;
	d.list.cutoff_range = l->cutoff_range;
	d.shadows.transforms = sh ? sh->transforms : nullptr;
	d.shadows.maps = sh ? reinterpret_cast<const void *const *>(sh->maps) : nullptr;
	d.by_id = false;
	d.shadow_ids = {};
	d.input_count = nullptr; // a new list: every entry is live until grbh_viewer_set_light_count_device
	d.ready = l->ready;
	d.consumed = l->consumed;
	d.count = static_cast<int32_t *>(v->light_scratch);
	d.scratch = static_cast<uint8_t *>(v->light_scratch) + 256;
	d.scratch_bytes = v->light_scratch_bytes;
	v->shadow_map_events.ready = sh ? static_cast<cudaEvent_t>(sh->maps_ready) : nullptr;
	v->shadow_map_events.consumed = sh ? static_cast<cudaEvent_t>(sh->maps_consumed) : nullptr;
	v->cluster.set_device_lights(&d);
	v->device_prep_rendered = false;
	return 0;
}

// "" unless the device light list of this rank comes from another rank (grbh_viewer_set_light_source_rank)
std::string not_light_source(const GrbhViewer *v)
{
	if (v->light_source < 0 || v->rank == (unsigned)v->light_source)
		return "";
	return "rank " + std::to_string(v->rank) + " receives its device lights from light source rank " + std::to_string(v->light_source) +
	       " (grbh_viewer_set_light_source_rank); it binds grbh_viewer_set_lights_device_from_source";
}
} // namespace

extern "C" int32_t grbh_viewer_set_lights_device(GrbhViewer *v, const GrbhDeviceLights *l)
{
	const std::string fn = "grbh_viewer_set_lights_device: ";
	if (!v || !l)
		return fail(fn + "null viewer or light list");
	if (l->count < 0 || l->count > GRBH_MAX_DEVICE_LIGHTS)
		return fail(fn + "count " + std::to_string(l->count) + " is outside 0.." + std::to_string(GRBH_MAX_DEVICE_LIGHTS));
	if (v->config.clustered_lights_shadows)
		return fail(fn + "the viewer was created with clustered_lights_shadows; its device lights need their shadows "
		                 "(grbh_viewer_set_lights_device_shadowed)");
	const std::string receiver = not_light_source(v);
	if (!receiver.empty())
		return fail(fn + receiver);
	if (!v->device)
		return fail(fn + "host-only viewer (no CUDA device)");
	GRBH_TRY
	return bind_device_lights(v, l, nullptr, fn);
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_lights_device_shadowed(GrbhViewer *v, const GrbhDeviceLights *l, const GrbhDeviceLightShadows *shadows)
{
	const std::string fn = "grbh_viewer_set_lights_device_shadowed: ";
	if (!v || !l || !shadows)
		return fail(fn + "null viewer, light list or shadow list");
	if (l->count < 0 || l->count > GRBH_MAX_DEVICE_LIGHTS)
		return fail(fn + "count " + std::to_string(l->count) + " is outside 0.." + std::to_string(GRBH_MAX_DEVICE_LIGHTS));
	if (!v->config.clustered_lights_shadows)
		return fail(fn + "the viewer was created without clustered_lights_shadows (grbh_viewer_set_lights_device)");
	if (l->count > 0 && (!shadows->transforms || !shadows->maps))
		return fail(fn + "null shadow transforms or shadow maps table");
	if (v->light_source >= 0)
	{
		const std::string receiver = not_light_source(v);
		return fail(fn + (receiver.empty() ? "the light source rank binds shadowed device lights by map id, whose maps every rank resolves in its own "
		                                     "table (grbh_viewer_set_lights_device_shadow_ids)"
		                                   : receiver));
	}
	if (!v->device)
		return fail(fn + "host-only viewer (no CUDA device)");
	GRBH_TRY
	return bind_device_lights(v, l, shadows, fn);
	GRBH_CATCH
}

namespace
{
// the bound device list's shadows come by map id, through this rank's table and under the table's map events
void bind_shadow_ids(GrbhViewer *v, const GrbhDeviceLightShadowIds *ids)
{
	auto &d = v->device_lights;
	d.by_id = true;
	d.shadow_ids.transforms = ids ? ids->transforms : nullptr;
	d.shadow_ids.map_ids = ids ? ids->map_ids : nullptr;
	v->shadow_map_events.ready = v->table_maps_ready;
	v->shadow_map_events.consumed = v->table_maps_consumed;
}
} // namespace

extern "C" int32_t grbh_viewer_set_light_shadow_map_table(GrbhViewer *v, const void *const *maps, int32_t count, void *maps_ready, void *maps_consumed)
{
	const std::string fn = "grbh_viewer_set_light_shadow_map_table: ";
	if (!v)
		return fail(fn + "null viewer");
	if (count < 0 || count > GRBH_MAX_DEVICE_LIGHTS)
		return fail(fn + "count " + std::to_string(count) + " is outside 0.." + std::to_string(GRBH_MAX_DEVICE_LIGHTS));
	if (count > 0 && !maps)
		return fail(fn + "null map array with count > 0");
	if (!v->config.clustered_lights_shadows)
		return fail(fn + "the viewer was created without clustered_lights_shadows");
	if (!v->device)
		return fail(fn + "host-only viewer (no CUDA device)");
	GRBH_TRY
	cudaSetDevice(v->device->get_device_index());
	for (int32_t i = 0; i < count; i++)
		if (maps[i] && !is_viewer_device_memory(v, fn, ("map " + std::to_string(i)).c_str(), maps[i], 1))
			return -1;
	if (!v->shadow_table_device)
	{
		void *p = nullptr;
		if (!Vulkan::cuda_ok(cudaMalloc(&p, sizeof(void *) * GRBH_MAX_DEVICE_LIGHTS), "cudaMalloc(shadow map table)"))
			return fail(fn + "cudaMalloc of the device table failed");
		v->shadow_table_device = p;
	}
	v->shadow_table.assign(maps, maps + count);
	v->shadow_table_changed = true;
	v->has_shadow_table = true;
	v->table_maps_ready = static_cast<cudaEvent_t>(maps_ready);
	v->table_maps_consumed = static_cast<cudaEvent_t>(maps_consumed);
	auto &d = v->device_lights;
	d.map_table = static_cast<const void *const *>(v->shadow_table_device);
	d.map_table_size = count;
	if (d.by_id && v->cluster.has_device_lights())
	{
		v->shadow_map_events.ready = v->table_maps_ready;
		v->shadow_map_events.consumed = v->table_maps_consumed;
	}
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_lights_device_shadow_ids(GrbhViewer *v, const GrbhDeviceLights *l, const GrbhDeviceLightShadowIds *ids)
{
	const std::string fn = "grbh_viewer_set_lights_device_shadow_ids: ";
	if (!v || !l || !ids)
		return fail(fn + "null viewer, light list or shadow id list");
	if (l->count < 0 || l->count > GRBH_MAX_DEVICE_LIGHTS)
		return fail(fn + "count " + std::to_string(l->count) + " is outside 0.." + std::to_string(GRBH_MAX_DEVICE_LIGHTS));
	if (!v->config.clustered_lights_shadows)
		return fail(fn + "the viewer was created without clustered_lights_shadows (grbh_viewer_set_lights_device)");
	if (l->count > 0 && (!ids->transforms || !ids->map_ids))
		return fail(fn + "null shadow transforms or map ids");
	const std::string receiver = not_light_source(v);
	if (!receiver.empty())
		return fail(fn + receiver);
	if (!v->device)
		return fail(fn + "host-only viewer (no CUDA device)");
	if (!v->has_shadow_table)
		return fail(fn + "no shadow map table is set on this rank (grbh_viewer_set_light_shadow_map_table first)");
	GRBH_TRY
	cudaSetDevice(v->device->get_device_index());
	if (l->count > 0 && (!is_viewer_device_memory(v, fn, "shadow transforms", ids->transforms, 64 * (size_t)l->count) ||
	                     !is_viewer_device_memory(v, fn, "map ids", ids->map_ids, 4 * (size_t)l->count)))
		return -1;
	const int32_t rc = bind_device_lights(v, l, nullptr, fn);
	if (rc != 0)
		return rc;
	bind_shadow_ids(v, ids);
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_light_count_device(GrbhViewer *v, const int32_t *count)
{
	const std::string fn = "grbh_viewer_set_light_count_device: ";
	if (!v)
		return fail(fn + "null viewer");
	const std::string receiver = not_light_source(v);
	if (!receiver.empty())
		return fail(fn + receiver + ", whose count comes with the list");
	if (!v->device)
		return fail(fn + "host-only viewer (no CUDA device)");
	if (!v->cluster.has_device_lights())
		return fail(fn + "no device light list is bound (grbh_viewer_set_lights_device[_shadowed] first)");
	if ((uintptr_t)count & 3)
		return fail(fn + "the count is not 4-byte aligned");
	GRBH_TRY
	if (count)
	{
		cudaSetDevice(v->device->get_device_index());
		if (!is_viewer_device_memory(v, fn, "count", count, sizeof(int32_t)))
			return -1;
	}
	v->device_lights.input_count = count;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_lights_device_from_source(GrbhViewer *v, int32_t capacity, float cutoff_range)
{
	const std::string fn = "grbh_viewer_set_lights_device_from_source: ";
	if (!v)
		return fail(fn + "null viewer");
	if (v->light_source < 0)
		return fail(fn + "the viewer has no light source rank (grbh_viewer_set_light_source_rank)");
	if (v->rank == (unsigned)v->light_source)
		return fail(fn + "rank " + std::to_string(v->rank) + " is the light source rank; it binds its list with grbh_viewer_set_lights_device");
	if (capacity < 0 || capacity > GRBH_MAX_DEVICE_LIGHTS)
		return fail(fn + "capacity " + std::to_string(capacity) + " is outside 0.." + std::to_string(GRBH_MAX_DEVICE_LIGHTS));
	if (!v->device)
		return fail(fn + "host-only viewer (no CUDA device)");
	GRBH_TRY
	// a list with no arrays of its own: every frame's clustering pass points the prep at the slot the source filled
	GrbhDeviceLights none = {};
	none.count = 0;
	none.cutoff_range = cutoff_range;
	const int32_t rc = bind_device_lights(v, &none, nullptr, fn);
	if (rc != 0)
		return rc;
	v->device_lights.list.count = capacity;
	// a shadowed viewer's slot holds the shadow transforms and map ids too: resolved through this rank's table
	if (v->config.clustered_lights_shadows)
		bind_shadow_ids(v, nullptr);
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_light_shadow_maps(GrbhViewer *v, const void *const *device_maps, int32_t count)
{
	if (!v || count < 0 || (count > 0 && !device_maps))
		return fail("grbh_viewer_set_light_shadow_maps: bad arguments");
	if ((size_t)count != v->scene_lights.size())
		return fail("grbh_viewer_set_light_shadow_maps: one entry per light of the last grbh_viewer_set_lights call");
	if (!v->config.clustered_lights_shadows)
		return fail("grbh_viewer_set_light_shadow_maps: the viewer was created without clustered_lights_shadows");
	for (int i = 0; i < count; i++)
		v->scene_lights[(size_t)i].light->set_shadow_map(device_maps[i]);
	return 0;
}

extern "C" int32_t grbh_viewer_get_shadow_transforms(GrbhViewer *v, float *out16_per_light, int32_t capacity)
{
	if (!v)
		return fail("null viewer");
	// host prep only (no GPU work), like grbh_viewer_get_light_prep
	v->cluster.set_scene_lights(&v->scene_lights);
	v->cluster.set_enable_shadows(true);
	v->cluster.refresh(v->context);
	v->cluster.set_enable_shadows(v->config.clustered_lights_shadows != 0);
	const auto &t = v->cluster.get_shadow_transforms();
	if ((int64_t)t.size() > capacity)
		return fail("grbh_viewer_get_shadow_transforms: capacity too small");
	if (out16_per_light && !t.empty())
		std::memcpy(out16_per_light, t.data(), 64 * t.size());
	return (int32_t)t.size();
}

extern "C" int32_t grbh_viewer_set_smaa_lookup_textures(GrbhViewer *v, const uint8_t *area_rg8, const uint8_t *search_r8)
{
	if (!v || !area_rg8 || !search_r8)
		return fail("grbh_viewer_set_smaa_lookup_textures: bad arguments");
	if (!v->device)
		return fail("grbh_viewer_set_smaa_lookup_textures: host-only viewer (no CUDA device)");
	GRBH_TRY
	if (!Granite::set_smaa_lookup_textures(*v->device, area_rg8, search_r8))
		return fail("grbh_viewer_set_smaa_lookup_textures: upload failed");
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_load_gtx(const char *path, int32_t *format, int32_t *width, int32_t *height, uint8_t *texels, int64_t capacity)
{
	if (!path || !format || !width || !height)
		return fail("grbh_load_gtx: bad arguments");
	GRBH_TRY
	Granite::GtxImage img;
	std::string error;
	if (!Granite::load_gtx(path, img, error))
		return fail(error.c_str());
	*format = (int32_t)img.format;
	*width = (int32_t)img.width;
	*height = (int32_t)img.height;
	if (texels)
	{
		if (capacity < (int64_t)img.texels.size())
			return fail("grbh_load_gtx: texel buffer too small");
		std::memcpy(texels, img.texels.data(), img.texels.size());
	}
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_rec709_to_display_primaries(const float *primaries_xy8, float *out16)
{
	if (!primaries_xy8 || !out16)
		return fail("grbh_rec709_to_display_primaries: bad arguments");
	VkHdrMetadataEXT md = {};
	md.displayPrimaryRed = { primaries_xy8[0], primaries_xy8[1] };
	md.displayPrimaryGreen = { primaries_xy8[2], primaries_xy8[3] };
	md.displayPrimaryBlue = { primaries_xy8[4], primaries_xy8[5] };
	md.whitePoint = { primaries_xy8[6], primaries_xy8[7] };
	const muglm::mat4 m = Granite::compute_rec709_to_display_primaries(md);
	std::memcpy(out16, m.data(), 64);
	return GRB_OK;
}

extern "C" int32_t grbh_nccl_unique_id(uint8_t out128[128])
{
	std::string err;
	if (!NcclCollectives::get_unique_id(out128, err))
		return fail(err);
	return 0;
}

extern "C" int32_t grbh_viewer_init_collectives(GrbhViewer *v, const uint8_t id128[128], int32_t rank, int32_t world_size)
{
	if (!v || !id128 || rank < 0 || world_size <= 0 || rank >= world_size)
		return fail("grbh_viewer_init_collectives: bad arguments");
	if (!v->device)
		return fail("grbh_viewer_init_collectives: host-only viewer (cuda_device < 0) has no device to communicate from");
	GRBH_TRY
	cudaSetDevice(v->device->get_device_index());
	auto c = std::make_unique<NcclCollectives>();
	std::string err;
	if (!c->init(id128, (unsigned)rank, (unsigned)world_size, err))
		return fail(err);
	v->collectives = std::move(c);
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_row_shards(GrbhViewer *v, const GrbRows *bands, int32_t count, int32_t rank)
{
	if (!v || count < 0 || (count && !bands) || (count && (rank < 0 || rank >= count)))
		return fail("grbh_viewer_set_row_shards: bad arguments");
	GRBH_TRY
	if (count > 1 && v->upscales())
	{
		// every rank must produce render rows for the exchanges (shard_plan.hpp)
		try
		{
			compute_shard_plan((unsigned)v->config.width, (unsigned)v->config.height, std::vector<GrbRows>(bands, bands + count), (unsigned)rank,
			                   v->uses_fxaa(), v->smaa_quality(), v->uses_taa(), v->shard_upscale());
		}
		catch (const std::invalid_argument &e)
		{
			return fail(std::string("grbh_viewer_set_row_shards: ") + e.what());
		}
	}
	if (v->present_rank >= std::max(count, 1))
		return fail("grbh_viewer_set_row_shards: the presenting rank " + std::to_string(v->present_rank) + " would have no band among " +
		            std::to_string(count) + " (call grbh_viewer_set_present_rank first)");
	if (v->gbuffer_source >= std::max(count, 1))
		return fail("grbh_viewer_set_row_shards: the G-buffer source rank " + std::to_string(v->gbuffer_source) + " would have no band among " +
		            std::to_string(count) + " (call grbh_viewer_set_gbuffer_source_rank first)");
	if (v->light_source >= std::max(count, 1))
		return fail("grbh_viewer_set_row_shards: the light source rank " + std::to_string(v->light_source) + " would have no band among " +
		            std::to_string(count) + " (call grbh_viewer_set_light_source_rank first)");
	v->bands.assign(bands, bands + count);
	v->rank = (unsigned)rank;
	v->baked = false;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_present_rank(GrbhViewer *v, int32_t rank)
{
	if (!v)
		return fail("null viewer");
	const int32_t count = std::max((int32_t)v->bands.size(), 1); // an unsharded viewer is one band
	if (rank < -1 || rank >= count)
		return fail("grbh_viewer_set_present_rank: rank must be -1 (off) or within [0, " + std::to_string(count) +
		            ") (the bands of the last grbh_viewer_set_row_shards)");
	v->present_rank = rank;
	v->baked = false;
	return 0;
}

extern "C" int32_t grbh_viewer_set_gbuffer_source_rank(GrbhViewer *v, int32_t rank)
{
	if (!v)
		return fail("null viewer");
	const int32_t count = std::max((int32_t)v->bands.size(), 1); // an unsharded viewer is one band
	if (rank < -1 || rank >= count)
		return fail("grbh_viewer_set_gbuffer_source_rank: rank must be -1 (off) or within [0, " + std::to_string(count) +
		            ") (the bands of the last grbh_viewer_set_row_shards)");
	if (rank >= 0 && v->config.pipelined_io)
		return fail("grbh_viewer_set_gbuffer_source_rank: not with pipelined_io (the G-buffer channel already keeps two slots in flight)");
	v->gbuffer_source = rank;
	v->baked = false;
	return 0;
}

extern "C" int32_t grbh_viewer_set_light_source_rank(GrbhViewer *v, int32_t rank)
{
	const std::string fn = "grbh_viewer_set_light_source_rank: ";
	if (!v)
		return fail(fn + "null viewer");
	if (rank >= 0 && v->config.clustered_lights_shadows && !v->has_shadow_table)
		return fail(fn + "not with clustered_lights_shadows (a light's shadow map pointer is valid on its own rank only) unless a shadow map table "
		                 "is set (grbh_viewer_set_light_shadow_map_table)");
	const int32_t count = std::max((int32_t)v->bands.size(), 1); // an unsharded viewer is one band
	if (rank < -1 || rank >= count)
		return fail(fn + "rank must be -1 (off) or within [0, " + std::to_string(count) + ") (the bands of the last grbh_viewer_set_row_shards)");
	if (v->baked)
		return fail(fn + "the viewer is baked; set the light source rank before grbh_viewer_bake");
	v->light_source = rank;
	return 0;
}

extern "C" int32_t grbh_viewer_get_input_rows(GrbhViewer *v, GrbRows *out, int32_t capacity)
{
	if (!v || capacity < 0)
		return fail("grbh_viewer_get_input_rows: bad arguments");
	GRBH_TRY
	const std::vector<GrbRows> rows = v->upload_ranges();
	if (out && (int64_t)rows.size() > capacity)
		return fail("grbh_viewer_get_input_rows: the rank reads " + std::to_string(rows.size()) + " row ranges, capacity is " + std::to_string(capacity));
	if (out)
		std::copy(rows.begin(), rows.end(), out);
	return (int32_t)rows.size();
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_lighting_stripes(GrbhViewer *v, int32_t stripe_rows)
{
	if (!v)
		return fail("null viewer");
	if (stripe_rows < 0 || stripe_rows % 8 != 0)
		return fail("grbh_viewer_set_lighting_stripes: stripe_rows must be 0 (off) or a positive multiple of 8 (got " + std::to_string(stripe_rows) + ")");
	if (stripe_rows > 0 && v->upscales())
		return fail("grbh_viewer_set_lighting_stripes: lighting in stripes is not supported with FSR 1 upscaling (resolution_scale < 1)");
	v->lighting_stripes = (unsigned)stripe_rows;
	v->baked = false;
	return 0;
}

extern "C" int32_t grbh_viewer_move_row_shards(GrbhViewer *v, const GrbRows *bands, int32_t count)
{
	if (!v || !bands || count <= 0)
		return fail("grbh_viewer_move_row_shards: bad arguments");
	if (v->bands.size() <= 1)
		return fail("grbh_viewer_move_row_shards: the viewer is not row-sharded (grbh_viewer_set_row_shards with more than one band)");
	if ((size_t)count != v->bands.size())
		return fail("grbh_viewer_move_row_shards: " + std::to_string(count) + " bands for a viewer of " + std::to_string(v->bands.size()) +
		            " (the band count of a viewer is fixed; re-bake to change it)");
	GRBH_TRY
	// the checks that need no device come first, so that a host-only viewer reaches them
	const std::vector<GrbRows> moved(bands, bands + count);
	try
	{
		// under FSR 1 every rank must also produce render rows for the exchanges (shard_plan.hpp)
		check_band_layout((unsigned)v->config.width, (unsigned)v->config.height, moved, v->shard_upscale());
	}
	catch (const std::invalid_argument &e)
	{
		return fail(std::string("grbh_viewer_move_row_shards: ") + e.what());
	}
	// the band count and the rank stay, so the presenting rank (< the band count) keeps its band
	if (!v->baked)
		return fail("grbh_viewer_move_row_shards: viewer not baked (before bake, grbh_viewer_set_row_shards sets the bands)");
	v->graph.move_row_shards(moved); // the graph's bands only: no reset, no bake, no allocation, same collectives
	v->bands = moved;
	const GrbRows lit = v->input_rows();
	v->cluster.set_lit_pixel_rows(lit.y0, lit.y1, v->render_height());
	v->bands_moved = true;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_shard_plan(int32_t width, int32_t height, const GrbRows *bands, int32_t count, int32_t rank, int32_t fxaa, GrbRows *out9)
{
	if (width <= 0 || height <= 0 || count < 0 || (count && !bands) || !out9 || (count && (rank < 0 || rank >= count)))
		return fail("grbh_shard_plan: bad arguments");
	GRBH_TRY
	std::vector<GrbRows> b(bands, bands + count);
	ShardPlan p = compute_shard_plan((unsigned)width, (unsigned)height, b, (unsigned)rank, fxaa != 0);
	const GrbRows all[8] = { p.own, p.fxaa, p.tonemap, p.upsample0, p.downsample0, p.threshold, p.lighting, p.lum_grid };
	for (int i = 0; i < 8; i++)
		out9[i] = all[i];
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_shard_plan_smaa(int32_t width, int32_t height, const GrbRows *bands, int32_t count, int32_t rank, int32_t quality, GrbRows *out6)
{
	if (width <= 0 || height <= 0 || count < 0 || (count && !bands) || !out6 || (count && (rank < 0 || rank >= count)) || quality < 0 || quality > 3)
		return fail("grbh_shard_plan_smaa: bad arguments");
	GRBH_TRY
	std::vector<GrbRows> b(bands, bands + count);
	ShardPlan p = compute_shard_plan((unsigned)width, (unsigned)height, b, (unsigned)rank, false, quality);
	const GrbRows all[6] = { p.smaa_blend, p.smaa_weights, p.smaa_edges, p.smaa_edge_window, p.tonemap, p.lighting };
	for (int i = 0; i < 6; i++)
		out6[i] = all[i];
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_shard_plan_taa(int32_t width, int32_t height, const GrbRows *bands, int32_t count, int32_t rank, int32_t fxaa, GrbRows *out3)
{
	if (width <= 0 || height <= 0 || count < 0 || (count && !bands) || !out3 || (count && (rank < 0 || rank >= count)))
		return fail("grbh_shard_plan_taa: bad arguments");
	GRBH_TRY
	std::vector<GrbRows> b(bands, bands + count);
	ShardPlan p = compute_shard_plan((unsigned)width, (unsigned)height, b, (unsigned)rank, fxaa != 0, -1, true);
	out3[0] = p.own;
	out3[1] = p.taa;
	out3[2] = p.lighting;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_shard_plan_fsr(int32_t width, int32_t height, int32_t render_width, int32_t render_height, const GrbRows *bands, int32_t count,
                                       int32_t rank, int32_t post_aa, int32_t rcas, GrbRows *out12)
{
	const bool known_aa = post_aa == GRBH_AA_NONE || post_aa == GRBH_AA_FXAA || (post_aa >= GRBH_AA_SMAA_LOW && post_aa <= GRBH_AA_SMAA_ULTRA) ||
	                      (post_aa >= GRBH_AA_TAA_LOW && post_aa <= GRBH_AA_TAA_HIGH) || post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA;
	if (width <= 0 || height <= 0 || render_width <= 0 || render_height <= 0 || render_width > width || render_height > height || count < 0 ||
	    (count && !bands) || !out12 || (count && (rank < 0 || rank >= count)) || !known_aa)
		return fail("grbh_shard_plan_fsr: bad arguments");
	GRBH_TRY
	std::vector<GrbRows> b(bands, bands + count);
	const bool fxaa = post_aa == GRBH_AA_FXAA || post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA;
	const bool taa = (post_aa >= GRBH_AA_TAA_LOW && post_aa <= GRBH_AA_TAA_HIGH) || post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA;
	const int smaa = post_aa >= GRBH_AA_SMAA_LOW && post_aa <= GRBH_AA_SMAA_ULTRA ? post_aa - GRBH_AA_SMAA_LOW : -1;
	ShardUpscale up; // the display size itself: no upscale (the viewer runs no FSR pass then)
	if (render_width < width || render_height < height)
	{
		up.width = (unsigned)render_width;
		up.height = (unsigned)render_height;
		up.rcas = rcas != 0;
	}
	ShardPlan p;
	try
	{
		p = compute_shard_plan((unsigned)width, (unsigned)height, b, (unsigned)rank, fxaa, smaa, taa, up);
	}
	catch (const std::invalid_argument &e)
	{
		return fail(std::string("grbh_shard_plan_fsr: ") + e.what());
	}
	const GrbRows all[12] = { p.own, p.easu,     p.easu_window, p.render_own,   p.fxaa,       p.tonemap,
		                      p.taa, p.lighting, p.smaa_blend,  p.smaa_weights, p.smaa_edges, p.smaa_edge_window };
	for (int i = 0; i < 12; i++)
		out12[i] = all[i];
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_shard_plan_stripes(int32_t width, int32_t height, const GrbRows *bands, int32_t count, int32_t rank, int32_t post_aa,
                                           int32_t stripe_rows, int32_t cluster_rows, GrbRows *out, int32_t capacity, int32_t *counts)
{
	const bool known_aa = post_aa == GRBH_AA_NONE || post_aa == GRBH_AA_FXAA || (post_aa >= GRBH_AA_SMAA_LOW && post_aa <= GRBH_AA_SMAA_ULTRA) ||
	                      (post_aa >= GRBH_AA_TAA_LOW && post_aa <= GRBH_AA_TAA_HIGH) || post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA;
	if (width <= 0 || height <= 0 || count < 0 || (count && !bands) || (count && (rank < 0 || rank >= count)) || (!count && rank != 0) || !known_aa ||
	    cluster_rows <= 0 || capacity < 0 || (capacity && !out) || !counts)
		return fail("grbh_shard_plan_stripes: bad arguments");
	GRBH_TRY
	std::vector<GrbRows> b(bands, bands + count);
	const bool fxaa = post_aa == GRBH_AA_FXAA || post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA;
	const bool taa = (post_aa >= GRBH_AA_TAA_LOW && post_aa <= GRBH_AA_TAA_HIGH) || post_aa == GRBH_AA_TAA_HIGH_PLUS_FXAA;
	const int smaa = post_aa >= GRBH_AA_SMAA_LOW && post_aa <= GRBH_AA_SMAA_ULTRA ? post_aa - GRBH_AA_SMAA_LOW : -1;
	StripePlan sp;
	try
	{
		sp = compute_stripe_plan((unsigned)width, (unsigned)height, b, (unsigned)rank, fxaa, smaa, taa, stripe_rows > 0 ? (unsigned)stripe_rows : 0u,
		                         (unsigned)cluster_rows);
	}
	catch (const std::invalid_argument &e)
	{
		return fail(std::string("grbh_shard_plan_stripes: ") + e.what());
	}
	std::vector<const std::vector<GrbRows> *> lists = { &sp.lit, &sp.receive, &sp.upload, &sp.tile_rows };
	for (const auto &p : sp.push)
		lists.push_back(&p);
	size_t total = 0;
	for (const auto *l : lists)
		total += l->size();
	if (total > (size_t)capacity)
		return fail("grbh_shard_plan_stripes: the plan has " + std::to_string(total) + " ranges, capacity is " + std::to_string(capacity));
	size_t at = 0;
	for (size_t i = 0; i < lists.size(); i++)
	{
		counts[i] = (int32_t)lists[i]->size();
		for (const GrbRows &r : *lists[i])
			out[at++] = r;
	}
	return (int32_t)total;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_bake(GrbhViewer *v)
{
	if (!v)
		return fail("null viewer");
	const std::string ring_rank = v->check_ring_rank(v->output_ring.size());
	if (!ring_rank.empty())
		return fail("grbh_viewer_bake: " + ring_rank + " (grbh_viewer_set_output_images with count 0 drops them)");
	if (!v->device)
		return fail("grbh_viewer_bake: host-only viewer (cuda_device < 0) cannot bake");
	GRBH_TRY
	cudaSetDevice(v->device->get_device_index());
	// attachments are set up by the first render_frame (calling setup_attachments here as well
	// would swap the history images once too often and fake a previous frame)
	v->bake_render_graph();
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_output_images(GrbhViewer *v, const GrbImage *images, int32_t count)
{
	const char *fn = "grbh_viewer_set_output_images: ";
	if (!v)
		return fail(std::string(fn) + "null viewer");
	const std::string bad = v->check_output_images(images, count);
	if (!bad.empty())
		return fail(fn + bad);
	if (count > 0 && !v->device)
		return fail(std::string(fn) + "host-only viewer (cuda_device < 0) has no device for the images to be on");
	GRBH_TRY
	for (int32_t i = 0; i < count; i++)
	{
		// the first and the last byte of each image are device memory of the viewer's device
		const uint8_t *base = static_cast<const uint8_t *>(images[i].data);
		for (const uint8_t *p : { base, base + (size_t)images[i].row_pitch * (size_t)(images[i].height - 1) + (size_t)images[i].width * 4 - 1 })
		{
			cudaPointerAttributes attr = {};
			const cudaError_t err = cudaPointerGetAttributes(&attr, p);
			if (err != cudaSuccess)
				cudaGetLastError();
			if (err != cudaSuccess || (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged) ||
			    attr.device != v->device->get_device_index())
				return fail(std::string(fn) + "output image " + std::to_string(i) + " is not device memory of the viewer's device (" +
				            std::to_string(v->device->get_device_index()) + ")");
		}
	}
	v->set_output_ring(images, count);
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_acquire_output(GrbhViewer *v, int32_t index, void *acquired, void *rendered)
{
	const char *fn = "grbh_viewer_acquire_output: ";
	if (!v)
		return fail(std::string(fn) + "null viewer");
	if (v->output_ring.empty())
		return fail(std::string(fn) + "no output images are set (grbh_viewer_set_output_images)");
	if (index < 0 || (size_t)index >= v->output_ring.size())
		return fail(std::string(fn) + "index " + std::to_string(index) + " is out of range: the ring holds " + std::to_string(v->output_ring.size()) +
		            " images");
	v->output_index = index;
	v->output_acquired = static_cast<cudaEvent_t>(acquired);
	v->output_rendered = static_cast<cudaEvent_t>(rendered);
	return 0;
}

// While a ring of output images is set, every frame renders into an acquired one
static bool frame_without_acquire(const GrbhViewer *v, const char *fn)
{
	if (v->output_ring.empty() || v->output_index >= 0)
		return false;
	fail(std::string(fn) + "a ring of output images is set (grbh_viewer_set_output_images): grbh_viewer_acquire_output must precede every frame");
	return true;
}

extern "C" int32_t grbh_viewer_render_frame(GrbhViewer *v, const GrbhHostGBuffer *host, double frame_time)
{
	if (v && frame_without_acquire(v, "grbh_viewer_render_frame: "))
		return -1;
	if (v && v->fed_from_source())
		return fail("grbh_viewer_render_frame: the frame is fed from the G-buffer source rank (grbh_viewer_set_gbuffer_source_rank); every rank calls "
		            "grbh_viewer_render_frame_device");
	if (!v || !v->baked)
		return fail("grbh_viewer_render_frame: viewer not baked");
	if (v->config.pipelined_io && !host)
		return fail("grbh_viewer_render_frame: pipelined_io viewers need the host G-buffer every frame");
	if (v->bands_moved && (!host || (v->uses_taa() && !host->mv)))
		return fail(std::string("grbh_viewer_render_frame: the bands moved (grbh_viewer_move_row_shards) since the last frame and the resident "
		                        "G-buffer holds the old rows; this frame must bring the host G-buffer") +
		            (v->uses_taa() ? " with its motion vectors" : ""));
	GRBH_TRY
	cudaSetDevice(v->device->get_device_index());
	v->render_frame(host, frame_time);
	v->bands_moved = false;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_render_frame_device(GrbhViewer *v, const GrbhDeviceGBuffer *gbuffer, double frame_time)
{
	const char *fn = "grbh_viewer_render_frame_device: ";
	if (!v)
		return fail(std::string(fn) + "null viewer");
	if (frame_without_acquire(v, fn))
		return -1;
	if (v->fed_from_source())
	{
		const bool source = v->rank == (unsigned)v->gbuffer_source;
		if (source && !gbuffer)
			return fail(std::string(fn) + "this rank is the G-buffer source rank (grbh_viewer_set_gbuffer_source_rank): it passes the whole frame's G-buffer every frame");
		if (!source && gbuffer)
			return fail(std::string(fn) + "the frame is fed from G-buffer source rank " + std::to_string(v->gbuffer_source) +
			            " (grbh_viewer_set_gbuffer_source_rank); every other rank passes NULL");
	}
	if (gbuffer)
	{
		const std::string bad = v->check_device_gbuffer(*gbuffer);
		if (!bad.empty())
			return fail(fn + bad);
	}
	if (!v->device)
		return fail(std::string(fn) + "host-only viewer (cuda_device < 0) has no device to read a G-buffer on");
	if (!v->baked)
		return fail(std::string(fn) + "viewer not baked");
	if (!v->fed_from_source())
	{
		if (v->config.pipelined_io && !gbuffer)
			return fail(std::string(fn) + "pipelined_io viewers need a G-buffer every frame");
		if (v->bands_moved && !gbuffer)
			return fail(std::string(fn) + "the bands moved (grbh_viewer_move_row_shards) since the last frame and the resident G-buffer holds the old rows; "
			                              "this frame must bring a G-buffer");
	}
	GRBH_TRY
	cudaSetDevice(v->device->get_device_index());
	v->pending_device = gbuffer;
	v->device_reads_left = v->uses_taa() ? 2 : 1;
	try
	{
		v->render_frame(nullptr, frame_time);
	}
	catch (...)
	{
		v->pending_device = nullptr;
		throw;
	}
	v->pending_device = nullptr;
	v->bands_moved = false;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_read_output(GrbhViewer *v, uint32_t *dst, GrbRows *rows_out)
{
	if (!v || !v->baked || !dst)
		return fail("grbh_viewer_read_output: bad arguments");
	GRBH_TRY
	GrbRows r;
	cudaStream_t stream = v->enqueue_readback(dst, r);
	if (!Vulkan::cuda_ok(cudaStreamSynchronize(stream), "cudaStreamSynchronize"))
		return fail("cudaStreamSynchronize failed");
	if (rows_out)
		*rows_out = r;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_read_output_async(GrbhViewer *v, uint32_t *dst, GrbRows *rows_out)
{
	if (!v || !v->baked || !dst)
		return fail("grbh_viewer_read_output_async: bad arguments");
	GRBH_TRY
	GrbRows r;
	cudaStream_t stream = v->enqueue_readback(dst, r);
	cudaEvent_t e;
	if (!v->free_output_events.empty())
	{
		e = v->free_output_events.back();
		v->free_output_events.pop_back();
	}
	else
		cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
	cudaEventRecord(e, stream);
	v->pending_outputs.push_back(e);
	if (rows_out)
		*rows_out = r;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_wait_outputs(GrbhViewer *v, int32_t max_pending)
{
	if (!v || max_pending < 0)
		return fail("grbh_viewer_wait_outputs: bad arguments");
	GRBH_TRY
	while ((int32_t)v->pending_outputs.size() > max_pending)
	{
		cudaEvent_t e = v->pending_outputs.front();
		if (!Vulkan::cuda_ok(cudaEventSynchronize(e), "cudaEventSynchronize"))
			return fail("cudaEventSynchronize failed");
		v->pending_outputs.erase(v->pending_outputs.begin());
		v->free_output_events.push_back(e);
	}
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_collect_timeline(GrbhViewer *v, char *names, int32_t names_capacity, float *begin_ms, float *end_ms, int32_t capacity)
{
	if (!v || !v->device)
		return fail("null viewer");
	GRBH_TRY
	auto tl = v->device->collect_timeline();
	std::string all;
	int i = 0;
	for (auto &e : tl)
	{
		if (i < capacity)
		{
			if (begin_ms)
				begin_ms[i] = e.begin_ms;
			if (end_ms)
				end_ms[i] = e.end_ms;
		}
		all += e.tag + "\n";
		i++;
	}
	if (names && names_capacity > 0)
		std::snprintf(names, (size_t)names_capacity, "%s", all.c_str());
	return i;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_join_streams(GrbhViewer *v)
{
	if (!v || !v->device)
		return fail("null viewer");
	v->device->join_side_streams();
	return 0;
}

extern "C" int32_t grbh_viewer_sync(GrbhViewer *v)
{
	if (!v)
		return fail("null viewer");
	if (!v->device)
		return fail("grbh_viewer_sync: host-only viewer (no CUDA device)");
	GRBH_TRY
	v->device->wait_idle();
	cudaError_t err = cudaGetLastError();
	if (err != cudaSuccess)
		return fail(cudaGetErrorString(err));
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_get_taa_reprojection(GrbhViewer *v, float *out16)
{
	if (!v || !out16)
		return fail("grbh_viewer_get_taa_reprojection: bad arguments");
	GRBH_TRY
	// the matrix the taa-resolve pass pushed for the LAST rendered frame (temporal.cpp:239-243)
	mat4 reproj = translate(vec3(0.5f, 0.5f, 0.0f)) * scale(vec3(0.5f, 0.5f, 1.0f)) * v->jitter.get_history_view_proj(1) *
	              v->jitter.get_history_inv_view_proj(0);
	std::memcpy(out16, reproj.data(), 16 * sizeof(float));
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_get_image(GrbhViewer *v, const char *name, GrbImage *out)
{
	if (!v || !name || !out || !v->baked)
		return fail("grbh_viewer_get_image: bad arguments");
	GRBH_TRY
	if (!v->graph.has_texture_resource(name))
		return fail(std::string("no such resource: ") + name);
	auto &res = v->graph.get_texture_resource(name);
	*out = v->graph.get_physical_texture_resource(res).as_grb();
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_get_buffer(GrbhViewer *v, const char *name, void **ptr, uint64_t *size)
{
	if (!v || !name || !ptr || !v->baked)
		return fail("grbh_viewer_get_buffer: bad arguments");
	GRBH_TRY
	if (!v->graph.has_texture_resource(name))
		return fail(std::string("no such resource: ") + name);
	auto &buf = v->graph.get_physical_buffer_resource(v->graph.get_buffer_resource(name));
	*ptr = buf.get_device_pointer();
	if (size)
		*size = buf.get_create_info().size;
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_get_cluster(GrbhViewer *v, GrbClusterParameters *params, GrbClusterBuffers *buffers)
{
	if (!v || !v->baked)
		return fail("grbh_viewer_get_cluster: viewer not baked");
	if (params)
		*params = v->cluster.get_cluster_parameters_bindless();
	if (buffers)
		*buffers = v->cluster.get_cluster_buffers();
	return 0;
}

extern "C" int32_t grbh_viewer_get_light_prep(GrbhViewer *v, GrbPositionalLight *records, float *model_rows, uint32_t *type_mask, uint32_t *z_ranges,
                                              int32_t capacity)
{
	if (!v)
		return fail("null viewer");
	if (v->cluster.has_device_lights())
	{
		if (!v->device_prep_rendered)
			return fail("grbh_viewer_get_light_prep: no frame has been rendered since the device lights were bound");
		GRBH_TRY
		cudaSetDevice(v->device->get_device_index());
		v->device->wait_idle();
		const GrbClusterBuffers buf = v->cluster.get_cluster_buffers();
		int32_t n = 0;
		if (!Vulkan::cuda_ok(cudaMemcpy(&n, v->device_lights.count, sizeof(n), cudaMemcpyDeviceToHost), "cudaMemcpy(count)"))
			return fail("grbh_viewer_get_light_prep: reading the device count failed");
		if (n > capacity)
			return fail("grbh_viewer_get_light_prep: capacity too small");
		const std::pair<void *, std::pair<const void *, size_t>> copies[] = {
			{ records, { buf.lights, sizeof(GrbPositionalLight) * (size_t)n } },
			{ model_rows, { buf.model, 48 * (size_t)n } },
			{ type_mask, { buf.type_mask, sizeof(uint32_t) * (size_t)((n + 31) / 32) } },
			{ z_ranges, { buf.z_ranges, sizeof(uint32_t) * 2 * (size_t)std::max(n, 1) } },
		};
		for (const auto &c : copies)
			if (c.first && c.second.second &&
			    !Vulkan::cuda_ok(cudaMemcpy(c.first, c.second.first, c.second.second, cudaMemcpyDeviceToHost), "cudaMemcpy(light prep)"))
				return fail("grbh_viewer_get_light_prep: reading the device prep failed");
		return n;
		GRBH_CATCH
	}
	// host prep only (no GPU work): usable on a machine without a device
	v->cluster.set_scene_lights(&v->scene_lights);
	if (v->config.cluster_res[0])
		v->cluster.set_resolution((unsigned)v->config.cluster_res[0], (unsigned)v->config.cluster_res[1], (unsigned)v->config.cluster_res[2]);
	v->cluster.refresh(v->context);
	int n = (int)v->cluster.get_active_light_count();
	if (n > capacity)
		return fail("grbh_viewer_get_light_prep: capacity too small");
	if (records)
		std::memcpy(records, v->cluster.get_light_records().data(), sizeof(GrbPositionalLight) * n);
	if (model_rows)
		std::memcpy(model_rows, v->cluster.get_model_transforms().data(), 48 * (size_t)n);
	if (type_mask)
		std::memcpy(type_mask, v->cluster.get_type_mask().data(), sizeof(uint32_t) * ((n + 31) / 32));
	if (z_ranges)
		std::memcpy(z_ranges, v->cluster.get_z_ranges().data(), sizeof(uint32_t) * 2 * v->cluster.get_z_ranges().size());
	return n;
}

extern "C" int32_t grbh_viewer_get_light_shadow_prep(GrbhViewer *v, float *transforms16, uint64_t *maps, int32_t capacity)
{
	if (!v)
		return fail("null viewer");
	if (v->cluster.has_device_lights())
	{
		if (!v->config.clustered_lights_shadows)
			return fail("grbh_viewer_get_light_shadow_prep: the viewer was created without clustered_lights_shadows");
		if (!v->device_prep_rendered)
			return fail("grbh_viewer_get_light_shadow_prep: no frame has been rendered since the device lights were bound");
		GRBH_TRY
		cudaSetDevice(v->device->get_device_index());
		v->device->wait_idle();
		const GrbLightShadows sh = v->cluster.get_light_shadows();
		int32_t n = 0;
		if (!Vulkan::cuda_ok(cudaMemcpy(&n, v->device_lights.count, sizeof(n), cudaMemcpyDeviceToHost), "cudaMemcpy(count)"))
			return fail("grbh_viewer_get_light_shadow_prep: reading the device count failed");
		if (n > capacity)
			return fail("grbh_viewer_get_light_shadow_prep: capacity too small");
		if (n && ((transforms16 && !Vulkan::cuda_ok(cudaMemcpy(transforms16, sh.transforms, 64 * (size_t)n, cudaMemcpyDeviceToHost), "cudaMemcpy(shadow transforms)")) ||
		          (maps && !Vulkan::cuda_ok(cudaMemcpy(maps, sh.maps, 8 * (size_t)n, cudaMemcpyDeviceToHost), "cudaMemcpy(shadow maps)"))))
			return fail("grbh_viewer_get_light_shadow_prep: reading the device prep failed");
		return n;
		GRBH_CATCH
	}
	// host prep only (no GPU work), like grbh_viewer_get_shadow_transforms
	GRBH_TRY
	v->cluster.set_scene_lights(&v->scene_lights);
	v->cluster.set_enable_shadows(true);
	v->cluster.refresh(v->context);
	v->cluster.set_enable_shadows(v->config.clustered_lights_shadows != 0);
	const auto &t = v->cluster.get_shadow_transforms();
	const auto &m = v->cluster.get_shadow_maps();
	if ((int64_t)t.size() > capacity)
		return fail("grbh_viewer_get_light_shadow_prep: capacity too small");
	if (transforms16 && !t.empty())
		std::memcpy(transforms16, t.data(), 64 * t.size());
	for (size_t i = 0; maps && i < m.size(); i++)
		maps[i] = (uint64_t)(uintptr_t)m[i];
	return (int32_t)t.size();
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_set_decals(GrbhViewer *v, const float *world_rows12, int32_t count)
{
	if (!v || count < 0 || (count > 0 && !world_rows12))
		return fail("grbh_viewer_set_decals: bad arguments");
	GRBH_TRY
	v->scene_decals.clear();
	for (int i = 0; i < count; i++)
	{
		const float *r = world_rows12 + 12 * (size_t)i;
		v->scene_decals.push_back(mat_affine(vec4(r[0], r[1], r[2], r[3]), vec4(r[4], r[5], r[6], r[7]), vec4(r[8], r[9], r[10], r[11])));
	}
	return 0;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_get_decal_prep(GrbhViewer *v, float *mvps16, uint32_t *z_ranges2, int32_t capacity)
{
	if (!v)
		return fail("null viewer");
	GRBH_TRY
	if (v->config.cluster_res[0])
		v->cluster.set_resolution((unsigned)v->config.cluster_res[0], (unsigned)v->config.cluster_res[1], (unsigned)v->config.cluster_res[2]);
	v->cluster.set_scene_lights(&v->scene_lights);
	v->cluster.set_scene_decals(&v->scene_decals);
	v->cluster.set_enable_volumetric_decals(true);
	v->cluster.refresh(v->context);
	v->cluster.set_enable_volumetric_decals(v->config.volumetric_decals != 0);
	const int n = (int)v->cluster.get_active_decal_count();
	if (n > capacity)
		return fail("grbh_viewer_get_decal_prep: capacity too small");
	if (mvps16 && n)
		std::memcpy(mvps16, v->cluster.get_decal_mvps().data(), 64 * (size_t)n);
	if (z_ranges2 && n)
		std::memcpy(z_ranges2, v->cluster.get_decal_z_ranges().data(), 8 * (size_t)n);
	return n;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_get_render_size(GrbhViewer *v, int32_t *width, int32_t *height)
{
	if (!v || !width || !height)
		return fail("grbh_viewer_get_render_size: null");
	*width = v->render_width();
	*height = v->render_height();
	return 0;
}

extern "C" int32_t grbh_viewer_get_camera(GrbhViewer *v, GrbCamera *out, float *projection16, float *inv_projection16)
{
	if (!v || !out)
		return fail("grbh_viewer_get_camera: null");
	const auto &rp = v->context.get_render_parameters();
	std::memcpy(out->view, rp.view.data(), 64);
	std::memcpy(out->view_projection, rp.view_projection.data(), 64);
	std::memcpy(out->inv_view_projection, rp.inv_view_projection.data(), 64);
	for (int i = 0; i < 3; i++)
	{
		out->camera_position[i] = rp.camera_position[i];
		out->camera_front[i] = rp.camera_front[i];
	}
	out->z_near = rp.z_near;
	out->z_far = rp.z_far;
	if (projection16)
		std::memcpy(projection16, rp.projection.data(), 64);
	if (inv_projection16)
		std::memcpy(inv_projection16, rp.inv_projection.data(), 64);
	return 0;
}

extern "C" int32_t grbh_viewer_measure_row_cost(GrbhViewer *v, uint32_t *out, int32_t capacity)
{
	if (!v || !v->baked || !v->device || !out)
		return fail("grbh_viewer_measure_row_cost: needs a baked device viewer");
	GRBH_TRY
	const int groups = (v->render_height() + 3) / 4;
	if (capacity < groups)
		return fail("grbh_viewer_measure_row_cost: capacity too small");
	const bool sharded = v->graph.is_sharded() && v->graph.get_shard_count() > 1;
	if (sharded)
		return v->measure_row_cost_sharded(out, groups);
	v->device->wait_idle();
	GrbImage depth = v->graph.get_physical_texture_resource(*v->res_depth).as_grb();
	GrbCamera cam;
	if (grbh_viewer_get_camera(v, &cam, nullptr, nullptr) != 0)
		return -1;
	GrbClusterParameters params = v->cluster.get_cluster_parameters_bindless();
	GrbClusterBuffers buffers = v->cluster.get_cluster_buffers();
	uint32_t *dev = nullptr;
	if (!Vulkan::cuda_ok(cudaMalloc(&dev, sizeof(uint32_t) * groups), "cudaMalloc"))
		return fail("cudaMalloc failed");
	int32_t rc = grb_lighting_row_cost(&depth, &cam, &params, &buffers, GrbRows{ 0, 0 }, dev, v->device->get_stream());
	bool ok = rc == GRB_OK && Vulkan::cuda_ok(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(v->device->get_stream())), "cudaStreamSynchronize") &&
	          Vulkan::cuda_ok(cudaMemcpy(out, dev, sizeof(uint32_t) * groups, cudaMemcpyDeviceToHost), "cudaMemcpy");
	cudaFree(dev);
	if (!ok)
		return fail(rc != GRB_OK ? grb_last_error_string() : "grbh_viewer_measure_row_cost: copy failed");
	return groups;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_get_pass_names(GrbhViewer *v, char *buffer, int32_t capacity)
{
	if (!v || !v->baked)
		return fail("viewer not baked");
	GRBH_TRY
	std::string all;
	for (auto &n : v->graph.get_baked_pass_names())
		all += n + "\n";
	if (buffer && capacity > 0)
		std::snprintf(buffer, (size_t)capacity, "%s", all.c_str());
	return (int32_t)all.size() + 1;
	GRBH_CATCH
}

extern "C" int32_t grbh_viewer_collect_timings(GrbhViewer *v, char *names, int32_t names_capacity, float *total_ms, int32_t *counts, int32_t capacity)
{
	if (!v)
		return fail("null viewer");
	std::string all;
	int i = 0;
	for (auto &kv : v->timings)
	{
		if (i < capacity)
		{
			if (total_ms)
				total_ms[i] = (float)kv.second.first;
			if (counts)
				counts[i] = kv.second.second;
		}
		all += kv.first + "\n";
		i++;
	}
	if (names && names_capacity > 0)
		std::snprintf(names, (size_t)names_capacity, "%s", all.c_str());
	v->timings.clear();
	return i;
}
