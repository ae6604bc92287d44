/*
 * granite_b200_host.h -- C entry points of libgranite_b200_host.so: the application-side
 * harness that drives the C++ host layer (granite_b200/host/: RenderGraph, LightClusterer,
 * DeferredLightRenderer, setup_hdr_postprocess_compute, setup_taa_resolve,
 * setup_fxaa_postprocess) the way SceneViewerApplication does in the reference
 * (application/scene_viewer_application.cpp:876-991 add_main_pass_deferred, :1167-1318
 * bake_render_graph, :1540-1611 render_frame).  The G-buffer, which the reference rasterises,
 * is an INPUT here: a "gbuffer" pass at the head of the graph uploads it from host memory
 * (grbh_viewer_render_frame) or copies it from device memory (grbh_viewer_render_frame_device).
 *
 * This is what bench.py's end-to-end measurement and the graph-level tests call.  All
 * functions return 0 on success, negative on failure (grbh_last_error()).
 */
#ifndef GRANITE_B200_HOST_H_
#define GRANITE_B200_HOST_H_

#include <stdint.h>

#include "granite_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct GrbhViewer GrbhViewer;

typedef enum GrbhPostAA
{
	GRBH_AA_NONE = 0,
	GRBH_AA_FXAA = 1,
	/* SMAA 1x after the tonemap, presets Low .. Ultra; needs grbh_viewer_set_smaa_lookup_textures before the first frame */
	GRBH_AA_SMAA_LOW = 3,
	GRBH_AA_SMAA_MEDIUM = 4,
	GRBH_AA_SMAA_HIGH = 5,
	GRBH_AA_SMAA_ULTRA = 6,
	GRBH_AA_TAA_LOW = 8,
	GRBH_AA_TAA_MEDIUM = 9,
	GRBH_AA_TAA_HIGH = 10,
	/* BASELINE config 5: TAA (pre-tonemap) and FXAA (post-tonemap) chained explicitly */
	GRBH_AA_TAA_HIGH_PLUS_FXAA = 100
} GrbhPostAA;

typedef struct GrbhViewerConfig
{
	int32_t cuda_device;
	int32_t width, height;
	int32_t post_aa;            /* GrbhPostAA */
	int32_t hdr_bloom;          /* 1: full bloom chain; 0: tonemap only (BASELINE config 1) */
	int32_t dynamic_exposure;   /* HDROptions::dynamic_exposure */
	int32_t cluster_res[3];     /* LightClusterer::set_resolution; viewer default 128,64,4096 */
	int32_t timestamps;         /* RenderGraph::enable_timestamps */
	void *cuda_stream;          /* NULL: the device creates its own stream */
	int32_t pipelined_io;       /* 1: the G-buffer upload runs on a side stream into images that alternate
	                             * per frame, so frame N+1's host->device copy overlaps frame N's compute
	                             * (every frame must then bring its G-buffer: render_frame(NULL) is an error) */
	int32_t hdr10_output;       /* 1: HDR10 swapchain (scene_viewer_application.cpp:1233-1288): no bloom / tonemap; the lit
	                             * (and TAA-resolved) scene goes through a "ui" pass (cleared to 0,0,0,1: no widgets) and the
	                             * "pq10" pass into an A2B10G10R10 image of ST.2084 codes, BT.2020 primaries, D65 */
	float hdr10_max_content_light_level; /* VkHdrMetadataEXT::maxContentLightLevel in nits; <= 0: 1000 */
	int32_t clustered_lights_shadows;           /* config "clusteredLightsShadows" (scene_viewer_application.cpp:214-215): the lighting
	                                             * pass samples the per-light shadow maps of grbh_viewer_set_light_shadow_maps */
	int32_t clustered_lights_shadow_resolution; /* "clusteredLightsShadowsResolution" (:216-217); <= 0: 512 */
	float resolution_scale;          /* "resolutionScale" (scene_viewer_application.cpp:247-248): 0 or 1 = off.  < 1: width x height
	                                  * is the DISPLAY size; the G-buffer the caller supplies (and every pass up to the post-chain
	                                  * output) has ceil(scale * size) texels (:758-761, 888-889), and FSR 1 upscales the result
	                                  * to the display size (:1263-1268).  Not with HDR10 output.  Row-sharded: the bands are
	                                  * display rows; grbh_shard_plan_fsr gives the render rows each rank computes. */
	int32_t resolution_scale_sharpen; /* "resolutionScaleSharpen" (:249-250): the RCAS pass after the upscale */
	int32_t render_target_fp16;       /* "renderTargetFp16" (:235-236, 880-884): emissive / HDR-main are R16G16B16A16_SFLOAT (8 bytes per
	                                   * texel -- GrbhHostGBuffer::emissive then points at RGBA16F texels); lighting, bloom threshold,
	                                   * tonemap and TAA read / write that format (TAA's own output stays B10G11R11).  Not with HDR10. */
	int32_t volumetric_decals;        /* LightClusterer::set_enable_volumetric_decals (clusterer.cpp:153-156): the decals of
	                                   * grbh_viewer_set_decals are binned into "cluster-bitmask-decal" / "cluster-range-decal" */
} GrbhViewerConfig;

/* Raw light list as the application owns it (before the clusterer sorts/packs it). */
typedef struct GrbhLights
{
	int32_t count;
	const float *color;       /* count x 3 */
	const float *position;    /* count x 3 */
	const uint8_t *is_point;  /* count */
	const float *rotation;    /* count x 9, column-major node rotation (spots) */
	const float *inner_cone;  /* count */
	const float *outer_cone;  /* count */
	float cutoff_range;       /* PositionalLight::set_maximum_range */
} GrbhLights;

/* The same light list in device memory on the viewer's device (grbh_viewer_set_lights_device): the clustering pass culls,
 * sorts and packs it on the GPU every frame, so lights that a GPU pass moves never go through the host. */
#define GRBH_MAX_DEVICE_LIGHTS 65536
typedef struct GrbhDeviceLights
{
	int32_t count;            /* 0 .. GRBH_MAX_DEVICE_LIGHTS */
	const float *color;       /* device, count x 3 */
	const float *position;    /* device, count x 3 */
	const uint8_t *is_point;  /* device, count */
	const float *rotation;    /* device, count x 9, column-major (as GrbhLights) */
	const float *inner_cone;  /* device, count */
	const float *outer_cone;  /* device, count */
	float cutoff_range;
	void *ready;    /* cudaEvent_t or NULL: the clustering pass waits on it before it reads */
	void *consumed; /* cudaEvent_t or NULL: recorded right after the prep's last read */
} GrbhDeviceLights;

/* The shadows of a device light list (grbh_viewer_set_lights_device_shadowed), in the lights' input order.  The viewer
 * never computes a shadow transform for device lights: each is the matrix the caller rendered that light's map with
 * (INTEGRATION.md gives the reference's shadow cameras). */
typedef struct GrbhDeviceLightShadows
{
	const float *transforms; /* device, count x 16, column-major: what GrbLightShadows::transforms holds per light */
	const uint64_t *maps;    /* device, count map pointers (0 = no shadow), as grbh_viewer_set_light_shadow_maps takes */
	void *maps_ready;        /* cudaEvent_t or NULL: the lighting pass waits on it before it samples the maps */
	void *maps_consumed;     /* cudaEvent_t or NULL: recorded on the lighting pass's stream behind its last read of the maps */
} GrbhDeviceLightShadows;

/* The shadows of a device light list by map id (grbh_viewer_set_lights_device_shadow_ids), in the lights' input order:
 * each light's transform, as in GrbhDeviceLightShadows, and the index of its map in this rank's shadow map table
 * (grbh_viewer_set_light_shadow_map_table).  An id outside 0..table count - 1 means no shadow. */
typedef struct GrbhDeviceLightShadowIds
{
	const float *transforms; /* device, count x 16, column-major */
	const int32_t *map_ids;  /* device, count map ids */
} GrbhDeviceLightShadowIds;

/* Host-memory G-buffer of the full frame (pinned memory makes the uploads asynchronous).
 * Only the rows this rank needs (its band + halo) are copied.  mv may be NULL without TAA. */
typedef struct GrbhHostGBuffer
{
	const uint32_t *albedo;
	const uint32_t *normal;
	const uint16_t *pbr;
	const float *depth;
	const uint32_t *emissive;
	const uint32_t *mv; /* R16G16_SFLOAT */
} GrbhHostGBuffer;

/* A G-buffer in device memory on the viewer's device, at the render size (grbh_viewer_get_render_size), each plane in
 * its attachment's format: emissive B10G11R11_UFLOAT (R16G16B16A16_SFLOAT with render_target_fp16), albedo
 * R8G8B8A8_SRGB, normal A2B10G10R10_UNORM_PACK32, pbr R8G8_UNORM, depth D32_SFLOAT, mv R16G16_SFLOAT (needed under TAA
 * only).  row_pitch: any multiple of the texel size of at least width x texel (padded images, strided tensors).  Only
 * the rows of grbh_viewer_get_input_rows are read.
 * ready: an event the "gbuffer" pass waits on before it reads, or NULL (the caller orders its writes before the frame).
 * consumed: a caller-created event, or NULL; the viewer records it right after its last read of the caller's memory,
 * so the caller may overwrite its buffers once it has completed. */
typedef struct GrbhDeviceGBuffer
{
	GrbImage emissive, albedo, normal, pbr, depth, mv;
	void *ready;    /* cudaEvent_t */
	void *consumed; /* cudaEvent_t */
} GrbhDeviceGBuffer;

const char *grbh_last_error(void);

int32_t grbh_viewer_create(const GrbhViewerConfig *config, GrbhViewer **out);
void grbh_viewer_destroy(GrbhViewer *viewer);

/* RenderContext::set_camera(projection, view) (renderer/render_context.cpp:54-87). */
int32_t grbh_viewer_set_camera(GrbhViewer *viewer, const float *projection16, const float *view16);
int32_t grbh_viewer_set_directional(GrbhViewer *viewer, const float *color3, const float *direction3);
int32_t grbh_viewer_set_lights(GrbhViewer *viewer, const GrbhLights *lights);
/* Binds a light list in device memory from the next frame until the next grbh_viewer_set_lights[_device] call
 * (grbh_viewer_set_lights goes back to host lights).  Every frame's clustering pass reads the arrays after `ready`, so
 * the caller may update them in place between frames; it culls, sorts and packs them on the GPU into the same bytes
 * the host prep of the same lights gives, and the kept count never comes back to the host.  The arrays must be device
 * memory of the viewer's device and stay alive while frames that read them are in flight.  Refused: a host-only viewer,
 * a count outside 0..GRBH_MAX_DEVICE_LIGHTS, a viewer created with clustered_lights_shadows (whose device lights go
 * through grbh_viewer_set_lights_device_shadowed), a rank other than the light source rank of
 * grbh_viewer_set_light_source_rank. */
int32_t grbh_viewer_set_lights_device(GrbhViewer *viewer, const GrbhDeviceLights *lights);
/* grbh_viewer_set_lights_device for a viewer created with clustered_lights_shadows: the clustering pass also moves each
 * kept light's shadow transform and map pointer into cluster order, so frames equal those of host lights given the same
 * maps.  The tables are read by the clustering pass under the lights' ready / consumed events; the maps' texels by the
 * lighting pass under maps_ready / maps_consumed.  Refused: a null argument, a count outside 0..GRBH_MAX_DEVICE_LIGHTS,
 * a viewer created without clustered_lights_shadows, null tables with count > 0, a host-only viewer, arrays or tables
 * that are not device memory of the viewer's device. */
int32_t grbh_viewer_set_lights_device_shadowed(GrbhViewer *viewer, const GrbhDeviceLights *lights, const GrbhDeviceLightShadows *shadows);
/* This rank's shadow map table for shadowed device lights whose maps come by id: maps is a HOST array of `count` device
 * map pointers of this rank (null = no shadow; maps as grbh_viewer_set_light_shadow_maps takes them), copied into a
 * device table the viewer owns.  A replaced table takes effect from the next frame: the upload is ordered on the
 * clustering pass's stream, so frames already recorded keep the table they were recorded with.  maps_ready /
 * maps_consumed (cudaEvent_t or NULL) go to the lighting pass as for grbh_viewer_set_lights_device_shadowed: it waits on
 * the first before it samples the maps and records the second behind its last read.  The caller owns the maps on every
 * rank (renders them there, or copies static maps there once); no texel crosses between ranks.  Refused: a null
 * viewer, a count outside 0..GRBH_MAX_DEVICE_LIGHTS, a null array with count > 0, a viewer created without
 * clustered_lights_shadows, a host-only viewer, a non-null entry that is not device memory of the viewer's device. */
int32_t grbh_viewer_set_light_shadow_map_table(GrbhViewer *viewer, const void *const *maps, int32_t count, void *maps_ready, void *maps_consumed);
/* grbh_viewer_set_lights_device_shadowed with each light's map named by id: the clustering pass moves each kept light's
 * transform into cluster order and resolves its id through this rank's table (an id outside the table: no shadow), so
 * frames equal those of host lights given table[id].  On one GPU, on each rank and on the light source rank of
 * grbh_viewer_set_light_source_rank, whose push carries the transforms and ids to every other rank.
 * grbh_viewer_set_light_count_device applies to it.  Refused: a null argument, a count outside
 * 0..GRBH_MAX_DEVICE_LIGHTS, a viewer created without clustered_lights_shadows, null arrays with count > 0, a rank that
 * receives its lights from the light source rank, a host-only viewer, no table set on this rank, arrays that are not
 * device memory of the viewer's device. */
int32_t grbh_viewer_set_lights_device_shadow_ids(GrbhViewer *viewer, const GrbhDeviceLights *lights, const GrbhDeviceLightShadowIds *ids);
/* Gives the device light list bound now (shadowed or not) a length that lives on the device: its `count` becomes the
 * capacity, and every frame's clustering pass reads *count under the lights' ready / consumed events, so a GPU pass may
 * rewrite it between frames with no host read.  Entries [0, live) are the lights, live = min(max(*count, 0), capacity)
 * (a value written on the device cannot be refused, so it is clamped); entries [live, capacity) are never read.  The
 * frame equals the frame of the first `live` lights bound without a count.  count: device memory of the viewer's device,
 * 4-byte aligned, alive while frames that read it are in flight; NULL goes back to every bound entry being live.
 * grbh_viewer_set_lights[_device[_shadowed]] clear it: a new binding is a new list.  On a row-sharded viewer with a
 * light source rank (grbh_viewer_set_light_source_rank) the count goes with the list to every other rank, so the ranks
 * need no copies of it to keep equal.  Refused: a null viewer, a rank other than the light source rank, a host-only
 * viewer, no device light list bound, a count that is not 4-byte aligned or not device memory of the viewer's device. */
int32_t grbh_viewer_set_light_count_device(GrbhViewer *viewer, const int32_t *count);
int32_t grbh_viewer_set_exposure(GrbhViewer *viewer, float exposure);
/* Shadow maps of the lights of the last grbh_viewer_set_lights call, in THAT order: `count` device pointers (host array),
 * each D16_UNORM of resolution^2 texels (spot) or 6 x resolution^2 (point, faces +X -X +Y -Y +Z -Z); null = no shadow.
 * The caller renders and owns them (the reference's LightClusterer::render_shadow is rasterisation, outside the path). */
int32_t grbh_viewer_set_light_shadow_maps(GrbhViewer *viewer, const void *const *device_maps, int32_t count);
/* ClustererBindlessTransforms::shadow[i] of the visible lights in cluster order, as the clusterer uploads them (host
 * preparation only, no GPU work): capacity x 16 floats.  Returns the light count. */
int32_t grbh_viewer_get_shadow_transforms(GrbhViewer *viewer, float *out16_per_light, int32_t capacity);
/* The shadow tables of the light prep in cluster order (for parity tests): capacity x 16 floats and capacity map pointers
 * (either may be NULL).  Host lights: the host prep's, no GPU work.  Device lights: the last rendered frame's device prep,
 * after waiting for the device to go idle, as grbh_viewer_get_light_prep.  Returns the kept light count. */
int32_t grbh_viewer_get_light_shadow_prep(GrbhViewer *viewer, float *transforms16, uint64_t *maps, int32_t capacity);

/* The two lookup textures SMAA samples (the payloads of the reference's assets/textures/smaa/area.gtx: 160x560 R8G8_UNORM,
 * and search.gtx: 64x16 R8_UNORM), uploaded once to the viewer's device.  grbh_load_gtx reads such a container from a
 * file: returns the VkFormat and fills width / height; texels (capacity bytes) receives the level-0 payload. */
int32_t grbh_viewer_set_smaa_lookup_textures(GrbhViewer *viewer, const uint8_t *area_rg8, const uint8_t *search_r8);
int32_t grbh_load_gtx(const char *path, int32_t *format, int32_t *width, int32_t *height, uint8_t *texels, int64_t capacity);

/* Rec.709 -> display primaries, the matrix setup_hdr10_pq_encoding pushes (renderer/post/hdr.cpp:580-593, 651).
 * primaries_xy8: red, green, blue, white chromaticities (VkHdrMetadataEXT order); out16: column-major mat4. */
int32_t grbh_rec709_to_display_primaries(const float *primaries_xy8, float *out16);

/* Row sharding (multi-GPU): bands[r] = backbuffer rows of rank r.  Must precede bake (a baked viewer moves its cuts with
 * grbh_viewer_move_row_shards below).  With FSR 1 upscaling, a layout in
 * which some rank would produce no render rows (grbh_shard_plan_fsr) is refused, and so is a layout with fewer bands
 * than the presenting rank of grbh_viewer_set_present_rank needs. */
int32_t grbh_nccl_unique_id(uint8_t out128[128]);
int32_t grbh_viewer_init_collectives(GrbhViewer *viewer, const uint8_t id128[128], int32_t rank, int32_t world_size);
int32_t grbh_viewer_set_row_shards(GrbhViewer *viewer, const GrbRows *bands, int32_t count, int32_t rank);
/* Presents row-sharded frames from one rank (the one that owns the swapchain): a "present" pass at the end of every
 * frame pushes each rank's band of the final image into that rank's memory (NVLink peer stores, or an NCCL all-gather
 * without peer memory), and grbh_viewer_read_output / _async on that rank return the whole frame, rows {0, height}.
 * Other ranks still return their bands.  rank: -1 = off (the default), otherwise within [0, band count) of the last
 * grbh_viewer_set_row_shards; an unsharded viewer counts as one band, so 0 is accepted there and changes nothing.
 * Every rank must set the same value.  Must precede bake.  Readers of the presented frame must be stream-ordered
 * behind the frame (these readbacks are): DESIGN.md section 5, "Presenting a sharded frame". */
int32_t grbh_viewer_set_present_rank(GrbhViewer *viewer, int32_t rank);
/* Row-sharded frames lit in stripes of stripe_rows rows (a positive multiple of 8; 0 = off, the default): rank r of W
 * lights the stripes k with k mod W == r, rows [k * stripe_rows, min((k + 1) * stripe_rows, height)), whatever the
 * bands, so every rank gets its share of the light-dense and of the sparse rows without a measurement.  Each rank then
 * pushes the rows other ranks' lighting rows hold into their HDR-main (through NVLink peer memory, or NCCL broadcasts
 * without it), and a "lighting-exchange" pass after "lighting" waits for them.  The bands keep deciding who runs the
 * post chain on which rows; grbh_viewer_move_row_shards and grbh_viewer_set_present_rank work unchanged.  Call before
 * grbh_viewer_bake, with the same value on every rank.  The frame equals the unsharded frame bit for bit.  Refused under
 * FSR 1 (resolution_scale < 1) and for a value that is not a multiple of 8; on an unsharded viewer it changes nothing. */
int32_t grbh_viewer_set_lighting_stripes(GrbhViewer *viewer, int32_t stripe_rows);
/* Moves the band cuts of a baked row-sharded viewer; takes effect from the next grbh_viewer_render_frame.
 * bands: `count` rows ranges that tile [0, height) in order, count = the band count the viewer was baked with; the rank
 * stays.  Under FSR 1 a layout in which some rank would produce no render rows is refused, as by
 * grbh_viewer_set_row_shards.  A refused layout returns an error and leaves the viewer as it was.  Nothing is re-baked
 * or allocated: attachments, the TAA history, the bloom feedback, the average luminance, the lighting schedule and the
 * peer channels carry over, and the next frame is the one an unsharded viewer renders (DESIGN.md section 5, "Moving the
 * bands between frames"; with FXAA and no upscale, bit-exact only for cuts on multiples of 16 rows).
 * The resident G-buffer holds the old layout's rows, so the first grbh_viewer_render_frame after a move must bring the
 * host G-buffer (with its motion vectors under TAA): a NULL one is refused there, and so are output readbacks and
 * grbh_viewer_measure_row_cost until that frame has been rendered.  Readbacks enqueued before the move keep the rows
 * they reported.
 * Collective contract: every rank calls it with the same bands, between the same two grbh_viewer_render_frame calls
 * (the checks give every rank the same answer for the same input).  Ranks that disagree on the layout run mismatched
 * exchanges. */
int32_t grbh_viewer_move_row_shards(GrbhViewer *viewer, const GrbRows *bands, int32_t count);
/* Row-sharded frames fed from the one rank that rasterises the whole frame: rank -1 = off (the default), otherwise
 * within [0, band count) of the last grbh_viewer_set_row_shards (an unsharded viewer counts as one band and changes
 * nothing).  Every rank then calls grbh_viewer_render_frame_device every frame, that rank with the whole frame's
 * G-buffer and every other rank with NULL; grbh_viewer_render_frame is refused.  The source rank's "gbuffer" pass pushes
 * each rank's input rows (grbh_viewer_get_input_rows of that rank, from the current bands) into that rank's slot of a
 * double-buffered peer channel and each rank copies them into its attachments (DESIGN.md section 5, "Feeding a sharded
 * frame from one rank"); without peer memory the rows go out in NCCL broadcasts.  Call before bake, with the same value
 * on every rank.  Refused with pipelined_io. */
int32_t grbh_viewer_set_gbuffer_source_rank(GrbhViewer *viewer, int32_t rank);
/* Row-sharded frames whose device light list comes from one rank: rank -1 = off (the default), otherwise within [0, band
 * count) of the last grbh_viewer_set_row_shards (an unsharded viewer counts as one band: it accepts 0, and that changes
 * nothing).  That rank S binds its list as today (grbh_viewer_set_lights_device, grbh_viewer_set_light_count_device);
 * every other rank binds a receiving list (grbh_viewer_set_lights_device_from_source), and both are refused on the
 * ranks they do not belong to.  Every frame S's clustering pass, after the lights' `ready`, pushes the list's live
 * entries and its live count into every other rank's slot of a double-buffered light channel (through NVLink peer
 * memory, or a broadcast of the whole slot without it), then preps its own list; every other rank preps its slot with
 * the counted prep.  So every rank renders the same list and the same count from one binding, with no host read of the
 * count (DESIGN.md section 5, "Lights from device memory").
 * Collective contract: every rank sets the same value before bake.  Every binding on S (with or without a count) is
 * matched by a receiving binding of the same capacity and cutoff on every other rank, between the same two frames;
 * grbh_viewer_set_lights (host lights) is called on every rank or on none.
 * Shadowed viewers (clustered_lights_shadows): a map pointer is valid on its own rank only, so the maps go by id.  Every
 * rank first sets its own shadow map table (grbh_viewer_set_light_shadow_map_table); S binds with
 * grbh_viewer_set_lights_device_shadow_ids (grbh_viewer_set_lights_device_shadowed is refused there), and every other
 * rank's receiving binding then preps the transforms and ids S pushed with the list, resolving each id through its own
 * table, so grbh_viewer_get_light_shadow_prep returns this rank's pointers.  Collective contract, on top of the one
 * above: every rank's table has the same count, and for each id every rank's map has the same texels.
 * Refused: a shadowed viewer without a shadow map table, a rank out of range, a call after bake. */
int32_t grbh_viewer_set_light_source_rank(GrbhViewer *viewer, int32_t rank);
/* The receiving binding of a rank other than the light source rank: from the next frame, the clustering pass preps the
 * list the source rank pushed this frame, as a list of `capacity` entries with cutoff_range, so the frame is sized from
 * `capacity` exactly as on the source rank.  The pushed count is clamped to `capacity`.  grbh_viewer_get_light_prep
 * reads this rank's own prep.  On a shadowed viewer the prep also reads the slot's shadow transforms and map ids and
 * resolves the ids through this rank's table.  Refused: a null viewer, a viewer with no light source rank, the light source rank itself,
 * a capacity outside 0..GRBH_MAX_DEVICE_LIGHTS, a host-only viewer. */
int32_t grbh_viewer_set_lights_device_from_source(GrbhViewer *viewer, int32_t capacity, float cutoff_range);
/* The row ranges of the render-size G-buffer this rank reads: its lighting rows (grbh_shard_plan*), or the upload list
 * of grbh_shard_plan_stripes under lighting in stripes; {0, render height} unsharded.  These are the rows a sort-first
 * rasteriser on this rank must produce: a device G-buffer needs only these rows to be valid.  Returns the count;
 * out = NULL only counts.  Pure host math of the current bands. */
int32_t grbh_viewer_get_input_rows(GrbhViewer *viewer, GrbRows *out, int32_t capacity);

/* Work estimate of the lighting pass per group of 4 rows of the render-size image (the backbuffer without FSR 1) for
 * the frame last rendered: grb_lighting_row_cost() on the viewer's depth image and light cluster, copied to the host.
 * out: ceil(render height / 4) values; returns that count.  Feed the sums per band unit to a weighted partition to
 * get bands of equal lighting work (granite_b200/viewer.py: band_partition_measured).
 * A row-sharded viewer measures on each rank the rows it produced (its band, or its render rows under FSR 1) and sums
 * the ranks' pieces with an exact integer all-reduce over its collectives: every rank returns the same whole-frame
 * vector, equal bit for bit to the unsharded viewer's.  That form is collective (every rank calls it after the same
 * frame) and needs every cut on a multiple of 4 rows. */
int32_t grbh_viewer_measure_row_cost(GrbhViewer *viewer, uint32_t *out, int32_t capacity);

/* The row plan of one rank of a row-sharded frame (granite_b200/host/shard_plan.hpp): out8 =
 * {own, fxaa, tonemap, upsample0, downsample0, threshold, lighting, lum_grid}.  Pure host math. */
int32_t grbh_shard_plan(int32_t width, int32_t height, const GrbRows *bands, int32_t count, int32_t rank, int32_t fxaa, GrbRows *out8);
/* The SMAA rows of the same plan for preset `quality` 0..3 (Low .. Ultra): out6 = {blend, weights, edges (the rows
 * this rank produces), edge window (the rows its weight pass reads, delivered by the ranks that own them), tonemap,
 * lighting}.  Whole images when count <= 1.  Pure host math. */
int32_t grbh_shard_plan_smaa(int32_t width, int32_t height, const GrbRows *bands, int32_t count, int32_t rank, int32_t quality, GrbRows *out6);
/* The TAA rows of the same plan with a TAA resolve before the post chain (and FXAA after it when fxaa != 0): out3 =
 * {own (the history rows this rank produces), taa (the rows it resolves: the lighting rows of the plan without TAA),
 * lighting (taa +- 1 row)}.  Whole images when count <= 1.  Pure host math. */
int32_t grbh_shard_plan_taa(int32_t width, int32_t height, const GrbRows *bands, int32_t count, int32_t rank, int32_t fxaa, GrbRows *out3);
/* The plan with FSR 1 upscaling after the post chain: width x height is the display size the bands cut, render_width x
 * render_height (each 1 .. the display's) the size every pass before FSR runs at; post_aa a GrbhPostAA; rcas != 0: the
 * sharpen pass follows the upscale.  out12 = {own (display rows), easu (the display rows EASU writes: own, +-1 row with
 * RCAS), easu window (the render rows EASU reads: the rows of the final render-resolution image), render own (the render
 * rows this rank produces for the exchanges), fxaa (the easu window from a multiple of 16 rows), tonemap, taa, lighting,
 * smaa blend, smaa weights, smaa edges, smaa edge window}; everything after `easu` in render rows, the SMAA rows whole images without SMAA.  A render size equal to the
 * display size is no upscale: the rows of grbh_shard_plan / _smaa / _taa, with easu = easu window = render own = own.
 * Whole images when count <= 1.  Fails when some rank would produce no render rows.  Pure host math. */
int32_t grbh_shard_plan_fsr(int32_t width, int32_t height, int32_t render_width, int32_t render_height, const GrbRows *bands, int32_t count,
                            int32_t rank, int32_t post_aa, int32_t rcas, GrbRows *out12);

/* The rows of one rank of a row-sharded frame that lights in stripes of stripe_rows rows (a positive multiple of 8):
 * rank r of `count` lights the stripes k with k mod count == r, rows [k * stripe_rows, min((k + 1) * stripe_rows,
 * height)), whatever the bands; the bands and post_aa (a GrbhPostAA) give every rank's lighting rows L_q as in
 * grbh_shard_plan / _smaa / _taa.  cluster_rows: the light cluster's tile rows.  The ranges go to `out` list after list,
 * and counts[i] receives the length of list i:
 *   0  lit:       the rank's stripes S_r, clipped to the image
 *   1  receive:   the rows of L_r that other ranks light
 *   2  upload:    S_r u L_r merged, the G-buffer rows that must be resident
 *   3  tile rows: the cluster tile rows the lighting of S_r reads (the clusterer's pixel-row to tile-row rounding with
 *                 one tile row of margin, per stripe, merged)
 *   4 + q         push to q: the rows of S_r inside L_q (none for q = rank)
 * counts holds max(count, 1) + 4 entries.  One band or none: the whole image, nothing pushed or received.  Returns the
 * number of ranges; fails when that exceeds capacity, or for a stripe height that is not a positive multiple of 8.
 * Pure host math. */
int32_t grbh_shard_plan_stripes(int32_t width, int32_t height, const GrbRows *bands, int32_t count, int32_t rank, int32_t post_aa,
                                int32_t stripe_rows, int32_t cluster_rows, GrbRows *out, int32_t capacity, int32_t *counts);

/* bake_render_graph: declares the passes, bakes, allocates attachments. */
int32_t grbh_viewer_bake(GrbhViewer *viewer);

/* One frame: (optionally) upload the host G-buffer rows, refresh the clusterer, record every
 * pass on the stream.  Asynchronous; ordering with later calls is stream order. */
int32_t grbh_viewer_render_frame(GrbhViewer *viewer, const GrbhHostGBuffer *host_gbuffer, double frame_time);
/* The same frame from a G-buffer in device memory: bit for bit the frame grbh_viewer_render_frame renders from a host
 * G-buffer holding the same bytes.  The "gbuffer" and "mv" passes copy this rank's input rows into the attachments
 * (grb_gbuffer_copy_rows; on the side stream into the alternating images with pipelined_io).  NULL: light the resident
 * G-buffer again, as grbh_viewer_render_frame(NULL) (refused with pipelined_io and on the first frame after
 * grbh_viewer_move_row_shards).  Refused: a missing plane (mv under TAA), a plane not at the render size or not in its
 * attachment's format, a pitch too small or not a multiple of the texel size, a host-only viewer; and under
 * grbh_viewer_set_gbuffer_source_rank a NULL G-buffer on the source rank or a G-buffer on any other. */
int32_t grbh_viewer_render_frame_device(GrbhViewer *viewer, const GrbhDeviceGBuffer *gbuffer, double frame_time);
/* A ring of `count` caller-owned device images that frames render into, in place of the graph-owned output image (the
 * reference's swapchain / headless image ring).  Each image: the display size (width x height, also under FSR 1), the
 * viewer's output format (R8G8B8A8_SRGB; A2B10G10R10_UNORM_PACK32 with hdr10_output), base 16-byte aligned, row_pitch a
 * multiple of 16 and >= width * 4, device memory of the viewer's device, no two overlapping.  The bytes written are the
 * ones grbh_viewer_read_output returns without a ring, bit for bit (FSR 1 without RCAS stores UNORM codes, as there).
 * count = 0: back to the graph-owned image.  May be called between frames; takes effect at the next
 * grbh_viewer_acquire_output (an acquire of the old ring is dropped).  An image of the old ring may be freed once the
 * `rendered` event of its last frame has completed.
 * One GPU, or a row-sharded rank without a presenting rank: the acquired image is the backbuffer, and the final pass
 * writes into it directly (on a row-sharded rank only the band's rows; the others stay as they are).
 * A presenting row-sharded viewer (grbh_viewer_set_present_rank): only the presenting rank may hold images (refused here
 * and at bake on every other rank); its backbuffer stays graph-owned, and after the "present" pass, on its stream, the
 * assembled frame is copied into the acquired image (DESIGN.md section 5, "Presenting a sharded frame"). */
int32_t grbh_viewer_set_output_images(GrbhViewer *viewer, const GrbImage *images, int32_t count);
/* The next frame renders into images[index] of the ring.  acquired: an event (cudaEvent_t, or NULL) the frame waits on
 * before its first write to that image (the caller's last reads of it are done).  rendered: a caller-created event (or
 * NULL) the viewer records after the frame's last write to it.  Both on the stream of the pass that writes the image.
 * While a ring is set, every grbh_viewer_render_frame / _device must follow an acquire; a frame without one is refused
 * before anything is recorded. */
int32_t grbh_viewer_acquire_output(GrbhViewer *viewer, int32_t index, void *acquired, void *rendered);
/* Copies this rank's rows of the final image (R8G8B8A8) to host memory laid out as the full
 * frame (row pitch = width*4) and waits for it. rows_out receives the band (the whole frame on
 * the presenting rank, grbh_viewer_set_present_rank).  With a ring of output images: the image
 * the last frame went into. */
int32_t grbh_viewer_read_output(GrbhViewer *viewer, uint32_t *dst_full_frame, GrbRows *rows_out);
/* Asynchronous form: enqueues the device->host copy of this frame's rows behind the frame and
 * returns; grbh_viewer_wait_outputs(viewer, k) blocks until at most k such copies are pending
 * (k = 0: all done).  With pipelined_io this keeps PCIe busy in both directions while the GPU
 * computes the next frame. */
int32_t grbh_viewer_read_output_async(GrbhViewer *viewer, uint32_t *dst_full_frame, GrbRows *rows_out);
int32_t grbh_viewer_wait_outputs(GrbhViewer *viewer, int32_t max_pending);
int32_t grbh_viewer_sync(GrbhViewer *viewer);
/* Makes the viewer's main stream (config.cuda_stream) wait for everything recorded so far on its
 * side streams (async cluster build, async post chain), so an event recorded on the main stream
 * afterwards covers the whole frame. */
int32_t grbh_viewer_join_streams(GrbhViewer *viewer);

/* Introspection for tests: device views of graph resources by name (valid until next bake). */
int32_t grbh_viewer_get_image(GrbhViewer *viewer, const char *resource_name, GrbImage *out);
int32_t grbh_viewer_get_buffer(GrbhViewer *viewer, const char *resource_name, void **device_ptr, uint64_t *size);
int32_t grbh_viewer_get_cluster(GrbhViewer *viewer, GrbClusterParameters *params, GrbClusterBuffers *buffers);
/* Copies the sorted/packed host-side light data of the last refresh (for host-prep parity tests).  With device lights
 * bound it copies the device prep of the last rendered frame instead -- the kept count, its records, model rows, type
 * mask words and Z ranges (one (~0u, 0) range when the count is 0) -- after waiting for the device to go idle. */
int32_t grbh_viewer_get_light_prep(GrbhViewer *viewer, GrbPositionalLight *records, float *model_rows, uint32_t *type_mask, uint32_t *z_ranges,
                                   int32_t capacity);
int32_t grbh_viewer_get_camera(GrbhViewer *viewer, GrbCamera *out, float *projection16, float *inv_projection16);
/* clip(now) -> UV(previous frame) as the taa-resolve pass of the last rendered frame used it
 * (renderer/post/temporal.cpp:239-243: unjittered history matrices). */
int32_t grbh_viewer_get_taa_reprojection(GrbhViewer *viewer, float *out16);
/* Names of the baked passes, '\n' separated. Returns the length needed. */
/* The scene's volumetric decals: `count` world transforms, 12 floats each (mat_affine rows) of unit cubes in decal space. */
int32_t grbh_viewer_set_decals(GrbhViewer *viewer, const float *world_rows12, int32_t count);
/* Host preparation of the decal binning (no GPU work): the visible decals front to back -- view_projection * world
 * (capacity x 16 floats) and their Z-slice ranges (capacity x 2 words).  Returns the count. */
int32_t grbh_viewer_get_decal_prep(GrbhViewer *viewer, float *mvps16, uint32_t *z_ranges2, int32_t capacity);
/* Size of the G-buffer the viewer expects (= width x height unless resolution_scale < 1). */
int32_t grbh_viewer_get_render_size(GrbhViewer *viewer, int32_t *width, int32_t *height);
int32_t grbh_viewer_get_pass_names(GrbhViewer *viewer, char *buffer, int32_t capacity);
/* Per-pass GPU time of the frames since the last call (needs config.timestamps):
 * writes up to `capacity` (name, total ms, count) triples. Returns the number of passes. */
int32_t grbh_viewer_collect_timings(GrbhViewer *viewer, char *names, int32_t names_capacity, float *total_ms, int32_t *counts, int32_t capacity);
/* GPU timeline of the passes recorded since the last call (config.timestamps == 2: intervals are
 * kept, not aggregated): (name, begin ms, end ms) relative to the first interval. Returns the count. */
int32_t grbh_viewer_collect_timeline(GrbhViewer *viewer, char *names, int32_t names_capacity, float *begin_ms, float *end_ms, int32_t capacity);
uint16_t grbh_float_to_half(float v);

#ifdef __cplusplus
}
#endif
#endif
