// grb_light_prep.cuh -- the per-light arithmetic of the host light prep (LightClusterer::refresh_bindless_prepare with
// PositionalLight / PointLight / SpotLight, AABB::transform, Frustum::intersects_fast, compute_uint_range) restated as
// __host__ __device__ functions over one light of a GrbLightList.  Every fp32 operation is written in the host code's
// association order; the device build uses -fmad=false and the host build -ffp-contract=off, so both round each
// operation on its own and give the host prep's bytes.  No transcendentals: + - * /, sqrtf, compares, floatToHalf.
#pragma once

#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/granite_b200.h"

namespace grb
{
namespace lp
{
struct V3
{
	float x, y, z;
};

__host__ __device__ inline uint32_t bits(float f)
{
	uint32_t u;
	memcpy(&u, &f, 4);
	return u;
}
__host__ __device__ inline V3 add(V3 a, V3 b) { return V3{ a.x + b.x, a.y + b.y, a.z + b.z }; }
__host__ __device__ inline V3 sub(V3 a, V3 b) { return V3{ a.x - b.x, a.y - b.y, a.z - b.z }; }
__host__ __device__ inline float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
// muglm's min / max: the first argument wins only on a strict compare
__host__ __device__ inline float mn(float a, float b) { return a < b ? a : b; }
__host__ __device__ inline float mx(float a, float b) { return a > b ? a : b; }

// muglm::floatToHalf (host/math.cpp): round half up on the magnitude
__host__ __device__ inline uint16_t float_to_half(float v)
{
	const uint32_t u = bits(v);
	const uint32_t sign = (u >> 16) & 0x8000u;
	const uint32_t mag = u & 0x7fffffffu;
	if (mag >= 0x7f800000u)
	{
		uint32_t payload = (mag & 0x7fffffu) >> 13;
		if ((mag & 0x7fffffu) != 0 && payload == 0)
			payload = 1;
		return (uint16_t)(sign | 0x7c00u | payload);
	}
	const int e = (int)(mag >> 23) - 112;
	if (e <= 0)
	{
		if (e < -10)
			return (uint16_t)sign;
		uint32_t m = ((mag & 0x7fffffu) | 0x800000u) >> (1 - e);
		return (uint16_t)(sign | ((m + 0x1000u) >> 13));
	}
	uint32_t h = (((uint32_t)e << 23) | (mag & 0x7fffffu)) + 0x1000u;
	h >>= 13;
	if (h >= 0x7c00u)
		h = 0x7c00u;
	return (uint16_t)(sign | h);
}

// One input light as the viewer's grbh_viewer_set_lights builds it: the node transform's three rows (a point light's
// rotation is the identity) and the PositionalLight state after set_maximum_range, set_color and, for a spot light,
// set_spot_parameters.
struct Light
{
	float row[3][4];
	V3 color;
	bool point;
	float inner, outer;  // clamped to [0.001, 1]
	float falloff;       // recompute_range: sqrt(max channel / 0.1)
	float reach;         // min(falloff, cutoff)
	float xy_range;      // spot: tan of the outer half-angle
	V3 lo, hi;           // the static AABB
};

__host__ __device__ inline Light load_light(const GrbLightList &l, int i)
{
	Light L;
	const float *p = l.position + 3 * i;
	L.color = V3{ l.color[3 * i], l.color[3 * i + 1], l.color[3 * i + 2] };
	L.point = l.is_point[i] != 0;
	if (L.point)
	{
		for (int c = 0; c < 3; c++)
		{
			for (int k = 0; k < 3; k++)
				L.row[c][k] = c == k ? 1.0f : 0.0f;
			L.row[c][3] = p[c];
		}
	}
	else
	{
		const float *r = l.rotation + 9 * i; // column-major 3x3
		for (int c = 0; c < 3; c++)
		{
			L.row[c][0] = r[c];
			L.row[c][1] = r[3 + c];
			L.row[c][2] = r[6 + c];
			L.row[c][3] = p[c];
		}
	}
	const float target_atten = 0.1f;
	const float max_color = mx(mx(L.color.x, L.color.y), L.color.z);
	L.falloff = sqrtf(max_color / target_atten);
	L.reach = mn(L.falloff, l.cutoff_range);
	L.inner = L.outer = 0.0f;
	L.xy_range = 0.0f;
	if (L.point)
	{
		L.lo = V3{ -L.reach, -L.reach, -L.reach };
		L.hi = V3{ L.reach, L.reach, L.reach };
	}
	else
	{
		L.inner = mn(mx(l.inner_cone[i], 0.001f), 1.0f);
		L.outer = mn(mx(l.outer_cone[i], 0.001f), 1.0f);
		L.xy_range = sqrtf(1.0f - L.outer * L.outer) / L.outer;
		const float side = L.xy_range * L.reach;
		L.lo = V3{ -side, -side, -L.reach };
		L.hi = V3{ side, side, 0.0f };
	}
	return L;
}

__host__ __device__ inline V3 translation(const Light &L) { return V3{ L.row[0][3], L.row[1][3], L.row[2][3] }; }

// AABB::transform then Frustum::intersects_fast (std::signbit of the plane distance)
__host__ __device__ inline bool visible(const Light &L, const float planes[24])
{
	float lo[3], hi[3];
	const float mn_[3] = { L.lo.x, L.lo.y, L.lo.z }, mx_[3] = { L.hi.x, L.hi.y, L.hi.z };
	for (int c = 0; c < 3; c++)
	{
		float h = L.row[c][3], l = L.row[c][3];
		for (int k = 0; k < 3; k++)
		{
			const float m = L.row[c][k];
			const bool positive = m > 0.0f;
			h = h + m * (positive ? mx_[k] : mn_[k]);
			l = l + m * (positive ? mn_[k] : mx_[k]);
		}
		hi[c] = h;
		lo[c] = l;
	}
	for (int q = 0; q < 6; q++)
	{
		const float *p = planes + 4 * q;
		const float dx = p[0] * (p[0] > 0.0f ? hi[0] : lo[0]);
		const float dy = p[1] * (p[1] > 0.0f ? hi[1] : lo[1]);
		const float dz = p[2] * (p[2] > 0.0f ? hi[2] : lo[2]);
		const float dw = p[3] * 1.0f;
		if (bits((dx + dy) + (dz + dw)) >> 31)
			return false;
	}
	return true;
}

// dot(translation, camera_front): the front-to-back sort key
__host__ __device__ inline float sort_key(const Light &L, const float front[3])
{
	return dot(translation(L), V3{ front[0], front[1], front[2] });
}

// The key as an unsigned integer that orders like the float's `<`: -0 and +0 compare equal, so both map to +0's code.
__host__ __device__ inline uint32_t radix_key(float key)
{
	if (key == 0.0f)
		key = 0.0f;
	const uint32_t u = bits(key);
	return (u >> 31) ? ~u : (u | 0x80000000u);
}

// The live length of a list of `capacity` entries whose count the caller wrote in device memory: a value written on the
// device cannot be refused, so one outside 0..capacity is clamped.
__host__ __device__ inline int live_count(int32_t count, int capacity) { return count < 0 ? 0 : (count > capacity ? capacity : count); }

// The cull kernel's 33-bit sort key of input light i when the first `live` entries are the light list: bit 32 set for a
// light the frustum culls, bits 0..31 the radix code of its sort key.  An entry at or past `live` is never loaded (it
// may hold anything) and gets the bare culled key, so it sorts behind every visible light and no slot packs it.
__host__ __device__ inline unsigned long long cull_key(const GrbLightList &lights, const GrbLightPrepView &view, int i, int live)
{
	if (i >= live)
		return 1ull << 32;
	const Light L = load_light(lights, i);
	const bool vis = !view.frustum_culling || visible(L, view.planes);
	return ((unsigned long long)(vis ? 0u : 1u) << 32) | radix_key(sort_key(L, view.camera_front));
}

// The light slot of a row-sharded frame's light channel (grb_light_slot_layout): the count word, then the six arrays of
// a GrbLightList of GRB_MAX_LIGHT_LIST entries in GrbLightList order, each from a multiple of 256 bytes.
constexpr int kLightArrays = 6;
// the element size of array a: color, position, is_point, rotation, inner_cone, outer_cone
__host__ __device__ inline int light_element_bytes(int a) { return a < 2 ? 12 : (a == 2 ? 1 : (a == 3 ? 36 : 4)); }
struct LightSlotLayout
{
	uint64_t count;
	uint64_t array[kLightArrays];
	uint64_t bytes;
};
// the offset of array a (a == kLightArrays: the slot's size)
__host__ __device__ inline uint64_t light_array_offset(int a)
{
	uint64_t at = 256;
	for (int k = 0; k < a; k++)
		at += ((uint64_t)GRB_MAX_LIGHT_LIST * (uint64_t)light_element_bytes(k) + 255) / 256 * 256;
	return at;
}
__host__ __device__ inline LightSlotLayout light_slot_layout()
{
	LightSlotLayout l;
	l.count = 0;
	for (int a = 0; a < kLightArrays; a++)
		l.array[a] = light_array_offset(a);
	l.bytes = light_array_offset(kLightArrays);
	return l;
}

// The shadowed light slot of grb_light_shadow_slot_layout: the light slot, then the shadow transforms and the map ids of
// GRB_MAX_LIGHT_LIST entries (arrays kLightArrays and kLightArrays + 1 of a shadowed push), each from a multiple of 256
// bytes.  The shadow part's element sizes and offsets are separate functions, so that the unshadowed push keeps its code.
constexpr int kShadowedLightArrays = kLightArrays + 2;
__host__ __device__ inline int shadow_element_bytes(int a) { return a == kLightArrays ? 64 : 4; }
// the offset of array a >= kLightArrays of a shadowed slot (a == kShadowedLightArrays: the shadowed slot's size)
__host__ __device__ inline uint64_t shadow_array_offset(int a)
{
	uint64_t at = light_array_offset(kLightArrays);
	for (int k = kLightArrays; k < a; k++)
		at += ((uint64_t)GRB_MAX_LIGHT_LIST * (uint64_t)shadow_element_bytes(k) + 255) / 256 * 256;
	return at;
}
// element size and slot offset of array a of a push of Arrays arrays (kLightArrays: the light slot's only)
template <int Arrays>
__host__ __device__ inline int push_element_bytes(int a)
{
	return Arrays == kLightArrays || a < kLightArrays ? light_element_bytes(a) : shadow_element_bytes(a);
}
template <int Arrays>
__host__ __device__ inline uint64_t push_array_offset(int a)
{
	return Arrays == kLightArrays || a < kLightArrays ? light_array_offset(a) : shadow_array_offset(a);
}

// What the push kernel of grb_light_list[_shadowed]_to_peers copies: the Arrays source arrays (the six of the light
// list, then for a shadowed list the transforms and the map ids), laid end to end in 16-byte chunks of which array a
// owns [start[a], start[a + 1]) (start[Arrays] = every chunk of the capacity), and whether array a moves in 16-byte
// words (vec16) or 4-byte words (vec4) -- both sides aligned -- or else byte by byte.
template <int Arrays>
struct LightPushArrays
{
	const uint8_t *src[Arrays];
	int start[Arrays + 1];
	unsigned vec16, vec4;
};
using LightPush = LightPushArrays<kLightArrays>;
using LightShadowPush = LightPushArrays<kShadowedLightArrays>;

// The push of `src` (capacity entries each): each array's source and chunk range, and the word size both sides allow
// (the slots are 16-byte aligned and every array of a slot starts on a multiple of 256 bytes).
template <int Arrays>
inline LightPushArrays<Arrays> light_push_arrays(const void *const *src, int capacity)
{
	LightPushArrays<Arrays> push = {};
	push.start[0] = 0;
	for (int a = 0; a < Arrays; a++)
	{
		push.src[a] = static_cast<const uint8_t *>(src[a]);
		const uintptr_t p = reinterpret_cast<uintptr_t>(src[a]);
		if ((p & 15) == 0)
			push.vec16 |= 1u << a;
		if (push_element_bytes<Arrays>(a) % 4 == 0 && (p & 3) == 0)
			push.vec4 |= 1u << a;
		push.start[a + 1] = push.start[a] + (capacity * push_element_bytes<Arrays>(a) + 15) / 16;
	}
	return push;
}
inline LightPush light_push(const GrbLightList &lights)
{
	const void *src[kLightArrays] = { lights.color, lights.position, lights.is_point, lights.rotation, lights.inner_cone, lights.outer_cone };
	return light_push_arrays<kLightArrays>(src, lights.count);
}
inline LightShadowPush light_shadow_push(const GrbLightList &lights, const GrbLightShadowIdList &ids)
{
	const void *src[kShadowedLightArrays] = { lights.color,      lights.position,   lights.is_point,  lights.rotation,
		                                      lights.inner_cone, lights.outer_cone, ids.transforms,   ids.map_ids };
	return light_push_arrays<kShadowedLightArrays>(src, lights.count);
}

// Thread t of the push: chunk t's bytes that lie below live x element size of its array, loaded once and stored at the
// same offset of that array in each of the `count` (<= GRB_MAX_PEERS) slots; nothing at or past it is read.  The loops
// over the arrays and the slots unroll, so that the kernel indexes its parameters with constants only.
template <int Arrays>
__host__ __device__ inline void push_light_chunk(const LightPushArrays<Arrays> &p, int live, int t, void *const *slots, int count)
{
	if (t >= p.start[Arrays])
		return;
	int a = 0;
	const uint8_t *src = p.src[0];
	int first = 0;
#pragma unroll
	for (int k = 1; k < Arrays; k++)
		if (t >= p.start[k])
		{
			a = k;
			src = p.src[k];
			first = p.start[k];
		}
	const uint64_t at = 16ull * (uint64_t)(t - first);
	const uint64_t end = (uint64_t)live * (uint64_t)push_element_bytes<Arrays>(a);
	if (at >= end)
		return;
	const int n = end - at < 16 ? (int)(end - at) : 16;
	const uint64_t dst = push_array_offset<Arrays>(a) + at;
	const uint8_t *s = src + at;
	if (n == 16 && ((p.vec16 >> a) & 1u))
	{
		const uint4 v = *reinterpret_cast<const uint4 *>(s);
#pragma unroll
		for (int r = 0; r < GRB_MAX_PEERS; r++)
			if (r < count)
				*reinterpret_cast<uint4 *>(static_cast<uint8_t *>(slots[r]) + dst) = v;
	}
	else if ((p.vec4 >> a) & 1u)
	{
		// n is a multiple of 4 here: the arrays that move in 4-byte words have elements of a multiple of 4 bytes
		for (int j = 0; j < n; j += 4)
		{
			const uint32_t v = *reinterpret_cast<const uint32_t *>(s + j);
#pragma unroll
			for (int r = 0; r < GRB_MAX_PEERS; r++)
				if (r < count)
					*reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(slots[r]) + dst + j) = v;
		}
	}
	else
		for (int j = 0; j < n; j++)
		{
			const uint8_t v = s[j];
#pragma unroll
			for (int r = 0; r < GRB_MAX_PEERS; r++)
				if (r < count)
					static_cast<uint8_t *>(slots[r])[dst + j] = v;
		}
}

// PointLight / SpotLight::get_shader_info, the model row (set_point_model_transform / SpotLight::build_model_matrix) and
// the Z-slice range (point_light_z_range / spot_light_z_range, then compute_uint_range)
__host__ __device__ inline void pack(const Light &L, const GrbLightPrepView &view, GrbPositionalLight &rec, float model[12], uint32_t zr[2])
{
	const float scale_factor = sqrtf(L.row[0][0] * L.row[0][0] + L.row[0][1] * L.row[0][1] + L.row[0][2] * L.row[0][2]);
	const float max_range = L.reach * scale_factor;
	const float s2 = scale_factor * scale_factor;
	rec.color[0] = L.color.x * s2;
	rec.color[1] = L.color.y * s2;
	rec.color[2] = L.color.z * s2;
	for (int c = 0; c < 3; c++)
		rec.position[c] = L.row[c][3];
	V3 forward{ -L.row[0][2], -L.row[1][2], -L.row[2][2] };
	if (L.point)
	{
		rec.spot_scale_bias[0] = rec.spot_scale_bias[1] = 0;
		rec.offset_radius[0] = float_to_half(0.0f);
		rec.offset_radius[1] = float_to_half(max_range);
	}
	else
	{
		const float spot_scale = 1.0f / mx(0.001f, L.inner - L.outer);
		const float spot_bias = -L.outer * spot_scale;
		const float tan2 = (1.0f - L.outer * L.outer) / (L.outer * L.outer);
		const float center_distance = ((tan2 + 1.0f) * max_range) * 0.5f;
		float spot_offset, spot_radius;
		if (center_distance < max_range)
		{
			spot_offset = center_distance;
			spot_radius = center_distance;
		}
		else
		{
			spot_offset = max_range;
			spot_radius = sqrtf(tan2) * max_range;
		}
		rec.spot_scale_bias[0] = float_to_half(spot_scale);
		rec.spot_scale_bias[1] = float_to_half(spot_bias);
		rec.offset_radius[0] = float_to_half(spot_offset);
		rec.offset_radius[1] = float_to_half(spot_radius);
		const float inv_len = 1.0f / sqrtf(dot(forward, forward));
		forward = V3{ forward.x * inv_len, forward.y * inv_len, forward.z * inv_len };
	}
	rec.direction[0] = forward.x;
	rec.direction[1] = forward.y;
	rec.direction[2] = forward.z;
	rec.inv_radius = 1.0f / max_range;

	const V3 cam{ view.camera_position[0], view.camera_position[1], view.camera_position[2] };
	const V3 front{ view.camera_front[0], view.camera_front[1], view.camera_front[2] };
	float lo, hi;
	if (L.point)
	{
		const float radius = 1.0f / rec.inv_radius;
		for (int k = 0; k < 12; k++)
			model[k] = 0.0f;
		model[0] = rec.position[0];
		model[1] = rec.position[1];
		model[2] = rec.position[2];
		model[3] = radius;
		const float z = dot(sub(translation(L), cam), front);
		lo = z - radius;
		hi = z + radius;
	}
	else
	{
		const float s[3] = { L.xy_range * L.reach, L.xy_range * L.reach, L.reach };
		for (int c = 0; c < 3; c++)
		{
			for (int k = 0; k < 3; k++)
				model[4 * c + k] = L.row[c][k] * s[k];
			model[4 * c + 3] = L.row[c][3];
		}
		const V3 base{ model[3], model[7], model[11] };
		const V3 x_off{ model[0], model[4], model[8] };
		const V3 y_off{ model[1], model[5], model[9] };
		const V3 z_base = add(base, V3{ -model[2], -model[6], -model[10] });
		const V3 hull[5] = { base, add(add(z_base, x_off), y_off), add(sub(z_base, x_off), y_off), sub(add(z_base, x_off), y_off),
			                 sub(sub(z_base, x_off), y_off) };
		lo = INFINITY;
		hi = -lo;
		for (int k = 0; k < 5; k++)
		{
			const float z = dot(sub(hull[k], cam), front);
			lo = mn(z, lo);
			hi = mx(z, hi);
		}
	}
	// compute_uint_range
	float x = lo / view.z_slice_extent, y = hi / view.z_slice_extent;
	if (y < 0.0f)
	{
		zr[0] = 0xffffffffu;
		zr[1] = 0u;
		return;
	}
	x = mx(x, 0.0f);
	// float -> uint32 as the x86-64 host converts it: through a signed 64-bit truncation
	zr[0] = (uint32_t)(int64_t)x;
	const uint32_t uy = (uint32_t)(int64_t)y;
	zr[1] = uy < (uint32_t)view.z_max_index ? uy : (uint32_t)view.z_max_index;
}

// Where the pack kernel's shadow part finds a light's map: by pointer (GrbLightShadowList, grb_light_prep_shadowed), or
// by id through this rank's table (ShadowIds, grb_light_prep_shadow_ids).  The unshadowed pack has no shadow part; its
// parameter keeps GrbLightShadowList's size, so that the kernel's parameter layout and code stay those of before.
struct NoShadows
{
	const void *unused[2];
};
struct ShadowIds
{
	GrbLightShadowIdList ids;
	const void *const *table;
	int table_size;
};
__host__ __device__ inline const float *shadow_transforms(const GrbLightShadowList &s) { return s.transforms; }
__host__ __device__ inline const float *shadow_transforms(const ShadowIds &s) { return s.ids.transforms; }
__host__ __device__ inline const void *shadow_map(const GrbLightShadowList &s, int src) { return s.maps[src]; }
// an id written on the device cannot be refused: one outside 0..table_size - 1 (negative ones included) means no shadow
__host__ __device__ inline const void *shadow_map(const ShadowIds &s, int src)
{
	const int32_t id = s.ids.map_ids[src];
	return (uint32_t)id < (uint32_t)s.table_size ? s.table[id] : nullptr;
}

// The shadow tables of slot s < slots: the transform and map of input light `src` (>= 0), or a zero matrix and a null
// map (src < 0).  The input transform is read one float at a time (it may be only 4-byte aligned); the output starts at
// packed_size(slots) of "cluster-transforms", 8-byte aligned for odd slot counts, so it is stored as float2.
template <class Shadows>
__host__ __device__ inline void pack_shadow(const Shadows &shadows, int src, int s, float *transforms_out, const void **maps_out)
{
	float2 *t = reinterpret_cast<float2 *>(transforms_out + 16 * (size_t)s);
	if (src >= 0)
	{
		const float *m = shadow_transforms(shadows) + 16 * (size_t)src;
		for (int k = 0; k < 8; k++)
			t[k] = make_float2(m[2 * k], m[2 * k + 1]);
		maps_out[s] = shadow_map(shadows, src);
	}
	else
	{
		for (int k = 0; k < 8; k++)
			t[k] = make_float2(0.0f, 0.0f);
		maps_out[s] = nullptr;
	}
}
} // namespace lp
} // namespace grb
