/*
 * oracle.h -- TEST INFRASTRUCTURE ONLY (see oracle_math.h header for the rules).
 *
 * Public entry points of the CPU oracle (liboracle.so, plain C ABI so the
 * Python tests can call it through ctypes on numpy buffers).  Every function
 * cites the reference file:line it restates (paths relative to the Granite
 * tree, commit 7c59ad8089).  Parity status (pinned to the reference's own shaders run on the CPU): see oracle_math.h.
 */
#ifndef ORACLE_H_
#define ORACLE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* renderer/lights/light_info.hpp:35-44 == assets/shaders/lights/clusterer_data.h:10-18 */
typedef struct
{
	float color[3];
	uint16_t spot_scale_bias[2];
	float position[3];
	uint16_t offset_radius[2];
	float direction[3];
	float inv_radius;
} orc_light_t;

/* Subset of math/render_parameters.hpp:90-108 that the light path reads. */
typedef struct
{
	float transform[16];
	float clip_scale[4];
	float camera_base[3];
	float camera_front[3];
	float xy_scale[2];
	int32_t resolution_xy[2];
	float inv_resolution_xy[2];
	int32_t num_lights;
	int32_t num_lights_32;
	int32_t z_max_index;
	float z_scale;
} orc_cluster_params_t;

/* Subset of math/render_parameters.hpp:37-59 (RenderParameters). Column-major mat4. */
typedef struct
{
	float projection[16];
	float view[16];
	float view_projection[16];
	float inv_projection[16];
	float inv_view[16];
	float inv_view_projection[16];
	float camera_position[3];
	float camera_front[3];
	float z_near;
	float z_far;
} orc_camera_t;

/* ---- host math (checked against oracle/_ref = the reference's math/muglm) ---- */
void orc_perspective(float fovy, float aspect, float z_near, float z_far, float *out16);  /* math/muglm/muglm.cpp:319-345 */
void orc_mat4_mul(const float *a, const float *b, float *out16);
void orc_mat4_inverse(const float *m, float *out16);                                      /* math/muglm/muglm.cpp inverse(mat4) */
uint16_t orc_float_to_half(float v);                                                      /* math/muglm/muglm_impl.hpp:860-907 */
void orc_camera_setup(const float *projection, const float *view, orc_camera_t *out);     /* renderer/render_context.cpp:54-87 */

/* ---- host light prep ---- */
/* renderer/lights/lights.cpp:63-70,203-220 (PointLight, unit node scale). */
void orc_point_light_info(const float *color, const float *position, float cutoff_range, orc_light_t *out);
/* renderer/lights/lights.cpp:77-146 (SpotLight): also returns the model matrix rows (3 x vec4). */
void orc_spot_light_info(const float *color, const float *position, const float *rot_cols9,
                         float inner_cone, float outer_cone, float cutoff_range,
                         orc_light_t *out, float *model_rows12);
/* renderer/lights/clusterer.cpp:803-826. resolution (128,64,4096) for the viewer. */
void orc_cluster_params(const orc_camera_t *cam, int num_lights, int res_x, int res_y, int res_z,
                        orc_cluster_params_t *out);
/* renderer/lights/clusterer.cpp:1265-1275,1322-1346 + lights.cpp:330-370.
 * z_ranges: max(num_lights,1) uvec2 entries. */
void orc_light_z_ranges(const orc_camera_t *cam, const orc_light_t *lights, const float *model_rows,
                        const uint32_t *type_mask, int num_lights, int res_z, uint32_t *z_ranges);

/* ClustererBindlessTransforms::shadow[index] (clusterer.cpp:467-474 spot, :518-521 point), column-major mat4. */
void orc_spot_shadow_transform(const orc_light_t *light, float xy_range, float *out16);
void orc_point_shadow_transform(const orc_light_t *light, float *out16);

/* ---- light visibility: renderer/scene.cpp:333-358 gather_positional_lights ---- */
void orc_frustum_planes(const float *inv_view_projection16, float *planes24);                 /* math/frustum.cpp:109-156 */
void orc_transform_aabb(const float *rows12, const float *lo3, const float *hi3, float *out_lo3, float *out_hi3); /* math/simd.hpp:386-419 */
int orc_frustum_cull(const float *lo3, const float *hi3, const float *planes24);              /* math/simd.hpp:34-60, 1 = visible */
int orc_light_visible(const float *planes24, int is_point, const float *color3, float cutoff_range, float outer_cone,
                      const float *rows12);                                                    /* lights.cpp:77-89,196-201 */

/* ---- clusterer kernels ---- */
/* K1 clusterer_bindless_spot_transform.comp:33-73. out: 6 vec4 per light. */
void orc_spot_transform(const orc_camera_t *cam, const float *model_rows, int num_lights, float *transformed_spots);
/* K2 clusterer_bindless_setup.comp:252-322. out: 32 vec4 per light (zero-initialised by the graph). */
void orc_cull_setup(const orc_camera_t *cam, const orc_cluster_params_t *p, const orc_light_t *lights,
                    const uint32_t *type_mask, const float *transformed_spots, float *cull_setup);
/* K3 clusterer_bindless_binning.comp:125-179 (SUBGROUPS=1, subgroup size 32 => 8x4 coarse tile).
 * bitmask: res_x*res_y*num_lights_32 words.  Bits >= num_lights are defined 0. */
void orc_binning(const orc_cluster_params_t *p, const uint32_t *type_mask, const float *cull_setup, uint32_t *bitmask);
/* K4 clusterer_bindless_z_range.comp:20-51. out: res_z uvec2. */
void orc_z_range(const uint32_t *z_ranges, int num_ranges, int res_z, uint32_t *cluster_range);

/* ---- volumetric-decal binning (SURVEY 8(f) rank 4): clusterer_bindless_binning_decal.comp, SUBGROUPS = 0 ---- */
void orc_decal_mvp(const float *view_projection16, const float *world_rows12, float *out16);      /* clusterer.cpp:1408-1409 */
void orc_decal_z_range(const orc_camera_t *cam, const float *world_rows12, float *lo_hi2);       /* clusterer.cpp:1348-1369 */
void orc_decal_screen_bb(const float *mvp16, float *bb4);                                         /* .comp:39-70 */
/* bitmask: res_x * res_y * ((num_decals + 31) / 32) words */
void orc_decal_binning(int res_x, int res_y, const float *inv_resolution_xy2, int num_decals, const float *mvps16, uint32_t *bitmask);

/* ---- deferred lighting (K6 directional + K5 clustered, two additive blends) ---- */
typedef struct
{
	int width, height;
	const uint32_t *albedo;   /* R8G8B8A8_SRGB */
	const uint32_t *normal;   /* A2B10G10R10_UNORM */
	const uint16_t *pbr;      /* R8G8_UNORM */
	const float *depth;       /* D32_SFLOAT, reverse-Z, 0 = sky */
	const uint32_t *emissive; /* B10G11R11_UFLOAT (HDR-main aliases emissive) */
	float dir_color[3];
	float dir_direction[3];
} orc_gbuffer_t;

/* renderer/renderer.cpp:1004-1156; directional.frag:40-65; clustering.frag:29-44;
 * clusterer_bindless.h:29-84; point.h; spot.h; pbr.h; lighting.h.
 * out_tile_index / out_z_index (optional, may be NULL): per-pixel cluster indices (bit-exact contract).
 * out_light_count (optional): lights evaluated per pixel. */
void orc_deferred_lighting(const orc_gbuffer_t *g, const orc_camera_t *cam, const orc_cluster_params_t *p,
                           const orc_light_t *lights, const uint32_t *type_mask,
                           const uint32_t *bitmask, const uint32_t *cluster_range,
                           uint32_t *hdr_out, int32_t *out_tile_index, int32_t *out_z_index,
                           int32_t *out_light_count, int y0, int y1);

/* Shadowed positional lights (POSITIONAL_LIGHTS_SHADOW with the PCF sampler; point.h:45-74, spot.h:51-77,
 * pcf.h:98-99).  transforms: 16 floats per light = ClustererBindlessTransforms::shadow[index], column-major
 * (spot: bias * proj * view, clusterer.cpp:467-474; point: column 0 = (proj[2].zw, proj[3].zw), clusterer.cpp:518-521).
 * maps[index]: D16_UNORM, resolution^2 texels (spot) or 6 faces of resolution^2 in Vulkan layer order
 * +X -X +Y -Y +Z -Z (point); NULL = the light casts no shadow. */
typedef struct
{
	const float *transforms;
	const uint16_t *const *maps;
	int resolution;
	int pcf_wide; /* SHADOW_MAP_PCF_KERNEL_WIDE: spot lights filter with the 6 x 6 kernel of pcf.h:7-80 (point lights are unaffected) */
} orc_shadows_t;
void orc_deferred_lighting_shadowed(const orc_gbuffer_t *g, const orc_camera_t *cam, const orc_cluster_params_t *p,
                                    const orc_light_t *lights, const uint32_t *type_mask,
                                    const uint32_t *bitmask, const uint32_t *cluster_range, const orc_shadows_t *shadows,
                                    uint32_t *hdr_out, int y0, int y1);
/* The same pass for an R16G16B16A16_SFLOAT HDR target ("renderTargetFp16", scene_viewer_application.cpp:880-884):
 * g->emissive points at RGBA16F texels; each blend rounds to fp16 (RNE); alpha passes through.  shadows may be NULL. */
void orc_deferred_lighting_fp16(const orc_gbuffer_t *g, const orc_camera_t *cam, const orc_cluster_params_t *p,
                                const orc_light_t *lights, const uint32_t *type_mask,
                                const uint32_t *bitmask, const uint32_t *cluster_range, const orc_shadows_t *shadows,
                                uint16_t *hdr_out_rgba16f, int y0, int y1);
/* the two comparison samplers on their own (Vulkan specification's filtering, fp32 weights) */
float orc_shadow_sample_2d(const uint16_t *map, int res, float clip_x, float clip_y, float clip_z, float clip_w);
float orc_shadow_sample_cube(const uint16_t *map, int res, float dx, float dy, float dz, float ref);
float orc_shadow_sample_2d_wide(const uint16_t *map, int res, float clip_x, float clip_y, float clip_z, float clip_w); /* pcf.h:7-80 */
/* texel (i, j) of cube face f, i or j possibly one step outside the face (-> the adjacent face); 0 at a corner */
int orc_shadow_cube_texel(int res, int f, int i, int j, size_t *texel);

/* One additive blend into a B10G11R11 attachment (renderer.cpp:1009-1011): dst = q(unpack(dst) + src) where
 * mask != 0.  Used by the tests that run the reference's own fragment shaders (oracle/_ref). */
void orc_blend_add_r11g11b10(uint32_t *dst, const float *src_rgb, const uint8_t *mask, int64_t count);
void orc_blend_add_rgba16f(uint16_t *dst, const float *src_rgb, const uint8_t *mask, int64_t count);

/* ---- HDR chain ---- */
/* K7 bloom_threshold.comp:23-45.  lum3: {avg_log, avg_lin, avg_inv_lin} or NULL (DYNAMIC_EXPOSURE=0). */
void orc_bloom_threshold(const uint32_t *hdr, int w_in, int h_in, const float *lum3,
                         uint16_t *out, int w, int h);
/* K8 bloom_downsample.comp:21-42.  history may be NULL (FEEDBACK=0). */
void orc_bloom_downsample(const uint16_t *in, int w_in, int h_in, const uint16_t *history, float lerp,
                          uint16_t *out, int w, int h);
/* K9 bloom_upsample.comp:15-33 */
void orc_bloom_upsample(const uint16_t *in, int w_in, int h_in, uint16_t *out, int w, int h);
/* K10 luminance.comp:23-68 + hdr.cpp:68-98.  lum3 in/out.  grid (optional): size_x*size_y sampled values. */
void orc_luminance(const uint16_t *d3, int w, int h, float lerp, float min_loglum, float max_loglum,
                   float *lum3, float *grid);
/* K11 tonemap.frag:55-66 + hdr.cpp:283-306.  lum3 NULL => DYNAMIC_EXPOSURE=0. out RGBA8: sRGB-encoded when
 * target_srgb, else the R8G8B8A8_UNORM store of the linear value. */
void orc_tonemap(const uint32_t *hdr, int w, int h, const uint16_t *bloom, int bw, int bh,
                 const float *lum3, float exposure, int target_srgb, uint32_t *out, int y0, int y1);
/* K12 fxaa.frag:20-67 + fxaa.cpp:28-56. in: RGBA8 read as UNORM. target_srgb => decode_srgb before store. */
void orc_fxaa(const uint32_t *in, int w, int h, int target_srgb, uint32_t *out, int y0, int y1);
/* K13 taa_resolve.frag:43-83 + reprojection.h.  history may be NULL (REPROJECTION_HISTORY=0).
 * mv: RG16F. out_color: B10G11R11. out_history: RGBA16F (alpha written as 1.0... see .c). */
void orc_taa_resolve(const uint32_t *hdr, const float *depth, const uint16_t *mv, const uint16_t *history,
                     int w, int h, const float *reproj16, int quality,
                     uint32_t *out_color, uint16_t *out_history, int y0, int y1);

/* K7 / K11 / K13 reading an R16G16B16A16_SFLOAT HDR image ("renderTargetFp16": HDR-main is RGBA16F; TAA's own output stays
 * B10G11R11, temporal.cpp:209-212).  Same functions, the HDR texel decode differs. */
void orc_bloom_threshold_fp16(const uint16_t *hdr_rgba16f, int w_in, int h_in, const float *lum3, uint16_t *out, int w, int h);
void orc_tonemap_fp16(const uint16_t *hdr_rgba16f, int w, int h, const uint16_t *bloom, int bw, int bh,
                      const float *lum3, float exposure, int target_srgb, uint32_t *out, int y0, int y1);
void orc_taa_resolve_fp16(const uint16_t *hdr_rgba16f, const float *depth, const uint16_t *mv, const uint16_t *history,
                          int w, int h, const float *reproj16, int quality,
                          uint32_t *out_color, uint16_t *out_history, int y0, int y1);

/* K14 pq10_encode.frag:20-52 + hdr.cpp:595-658 (setup_hdr10_pq_encoding): HDR10 / ST.2084 output encoding.
 * hdr: B10G11R11 linear scene colour; ui: R8G8B8A8_UNORM (alpha = how much of the scene shows through);
 * primary16: column-major mat4 whose upper 3x3 converts Rec.709 to the display's primaries;
 * out: A2B10G10R10_UNORM_PACK32 (alpha = 1). */
void orc_pq10_encode(const uint32_t *hdr, const uint32_t *ui, int w, int h, const float *primary16, float hdr_pre_exposure,
                     float ui_pre_exposure, float max_light_level, uint32_t *out, int y0, int y1);
/* hdr.cpp:580-593 compute_rec709_to_st2020 (math/transforms.cpp:352-370 compute_xyz_matrix): primaries8 =
 * display red.xy, green.xy, blue.xy, white.xy (VkHdrMetadataEXT); out9 = column-major mat3. */
void orc_rec709_to_display_primaries(const float *primaries8, float *out9);

/* ---- format helpers exported for tests ---- */
uint32_t orc_pack_r11g11b10(float r, float g, float b);
void orc_unpack_r11g11b10(uint32_t p, float *rgb);
uint16_t orc_f32_to_f16(float f);
float orc_f16_to_f32(uint16_t h);
uint32_t orc_linear_to_srgb8(float c);
float orc_srgb8_to_linear(uint32_t v);

#ifdef __cplusplus
}
#endif
/* SMAA (renderer/post/smaa.cpp:32-209, SMAA.hlsl): edge detection -> blending weights -> neighbourhood blending.
 * quality = SMAA_QUALITY 0..3 (presets Low / Medium / High / Ultra).  area: 160x560 R8G8, search: 64x16 R8 (the
 * reference's textures/smaa/{area,search}.gtx payloads). */
void orc_smaa_edge_detection(const uint32_t *color_unorm, int w, int h, int quality, uint8_t *edges_rg8, int y0, int y1);
void orc_smaa_blend_weights(const uint8_t *edges_rg8, int w, int h, const uint8_t *area_rg8, const uint8_t *search_r8, int quality,
                            uint32_t *weights_rgba8, int y0, int y1);
void orc_smaa_neighborhood_blend(const uint32_t *color_unorm, const uint32_t *weights_rgba8, int w, int h, uint32_t *out_srgb8, int y0, int y1);

/* ---- FSR 1 after the post chain: renderer/post/aa.cpp:34-174, assets/shaders/post/ffx-fsr/{upscale,sharpen}.frag,
 * ffx_fsr1.h (32-bit paths) ---- */
void orc_fsr_easu_constants(int w_in, int h_in, int w_out, int h_out, float *con16);  /* aa.cpp:33-61 */
void orc_fsr_rcas_constants(float sharpness, float *con4);                             /* aa.cpp:63-73 */
/* upscale.frag: src is the sRGB image read as UNORM; target_srgb = 1 stores decode_srgb(colour) into an sRGB target */
void orc_fsr_easu(const uint32_t *src_unorm, int w_in, int h_in, const float *con16, uint32_t *dst, int w_out, int h_out, int target_srgb, int y0, int y1);
/* sharpen.frag: srgb = 1 reads through an sRGB view (linear values) and stores into an sRGB target */
void orc_fsr_rcas(const uint32_t *src, int w, int h, const float *con4, uint32_t *dst, int srgb, int y0, int y1);

/* ---- volumetric fog, light-density pass: fog_light_density.comp, base variant (no fog regions, no temporal reprojection,
 * no floor lighting, no shadows); VolumetricFog::build_light_density (volumetric_fog.cpp:142-228) ---- */
typedef struct
{
	int width, height, depth;   /* VolumetricFog::set_resolution; the reference's default is 160 x 92 x 64 */
	int dither_offset;          /* layer of the 128 x 128 x N dither LUT */
	float slice_z_log2_scale;   /* 1 / log2(1 + z_range) (volumetric_fog.cpp:87-91) */
	float density_mod;          /* set_fog_density */
	float in_scatter_strength;  /* inscatter_mod */
} orc_fog_params_t;
void orc_fog_slice_extents(int depth, float slice_z_log2_scale, float *out);
/* out: depth x height x width RGBA16F = (in-scattered light, fog albedo); dither_lut_rgba8: N x 128 x 128 texels (R8G8B8A8_UNORM) */
void orc_fog_light_density(const orc_fog_params_t *f, const orc_camera_t *cam, const orc_cluster_params_t *p, const orc_light_t *lights,
                           const uint32_t *type_mask, const uint32_t *bitmask, const uint32_t *cluster_range, const float *dir_color3,
                           const float *dir_direction3, const float *slice_extents, const uint32_t *dither_lut_rgba8, uint16_t *out_rgba16f);

/* ---- volumetric fog, accumulation pass: fog_accumulate.comp + VolumetricFog::build_fog (volumetric_fog.cpp:236-254).
 * light / fog: R16G16B16A16_SFLOAT volumes of w x h x d texels, x fastest ---- */
void orc_fog_accumulate(const uint16_t *light_rgba16f, int w, int h, int d, uint16_t *fog_rgba16f);

#endif
