// grb_gbuffer.cu -- row copies of a G-buffer held in device memory: into the viewer's attachments on one device
// (grb_gbuffer_copy_rows), and from the rank that rasterised the whole frame into every rank's G-buffer slot through
// peer memory (grb_gbuffer_rows_to_peers; the protocol is grb_peer.cuh's).  Both are byte copies.
//
// One launch covers every listed row range of every present plane: blockIdx.z is the plane, blockIdx.y a row of the
// ranges laid end to end, and each thread moves 16 bytes of that row (one 16-byte load and store when the plane's
// pitches and bases allow it, whole texels otherwise and for the row's last bytes).  The ranges travel in the kernel
// parameters, a chunk of at most kMaxRanges per launch; a longer list takes more launches.
#include "grb_common.cuh"
#include "grb_peer.cuh"

#include <cstdio>
#include <type_traits>
#include <vector>

namespace grb
{
namespace
{
constexpr int kPlanes = GRB_GBUFFER_PLANES;
constexpr int kMaxRanges = 128;
constexpr int kMaxGridRows = 65535;
constexpr unsigned kSlotAlign = 256;

// the texel size plane p may have: emissive 4 (B10G11R11) or 8 (RGBA16F), pbr 2, every other plane 4
bool texel_fits_plane(int p, int texel) { return p == 0 ? (texel == 4 || texel == 8) : (p == 3 ? texel == 2 : texel == 4); }

int format_texel_bytes(int32_t format)
{
	switch (format)
	{
	case GRB_FORMAT_R8G8_UNORM: return 2;
	case GRB_FORMAT_R16G16B16A16_SFLOAT: return 8;
	case GRB_FORMAT_R8G8B8A8_UNORM:
	case GRB_FORMAT_R8G8B8A8_SRGB:
	case GRB_FORMAT_A2B10G10R10_UNORM_PACK32:
	case GRB_FORMAT_R16G16_SFLOAT:
	case GRB_FORMAT_B10G11R11_UFLOAT_PACK32:
	case GRB_FORMAT_D32_SFLOAT: return 4;
	default: return 0;
	}
}

struct PlaneArgs
{
	const uint8_t *src[kPlanes];
	uintptr_t dst[kPlanes]; // an address, or (peer copies) an offset into the slot of the range's rank
	int src_pitch[kPlanes];
	int dst_pitch[kPlanes];
	int row_bytes[kPlanes]; // 0: the plane is absent
	int texel[kPlanes];
	unsigned vec16; // bit p: plane p moves in 16-byte words
};

struct RangeChunk
{
	int count;
	int start[kMaxRanges + 1]; // first grid row of each range; start[count] = the grid rows in all
	int y0[kMaxRanges];
	uint8_t rank[kMaxRanges]; // peer copies: the rank whose slot takes the range
};

template <int Texel>
__device__ __forceinline__ void copy_texels(const uint8_t *s, uint8_t *d, int bytes)
{
	using T = typename std::conditional<Texel == 2, uint16_t, typename std::conditional<Texel == 4, uint32_t, uint2>::type>::type;
	for (int j = 0; j < 16 && j < bytes; j += Texel)
		*reinterpret_cast<T *>(d + j) = __ldg(reinterpret_cast<const T *>(s + j));
}

template <bool Peers>
__global__ void __launch_bounds__(256) gbuffer_rows_kernel(PlaneArgs planes, RangeChunk chunk, PeerTargets targets, int publish)
{
	__builtin_assume(threadIdx.y == 0); // 1-D blocks: peer_publish's leader test is threadIdx.x == 0
	const int p = (int)blockIdx.z;
	const int i = (int)blockIdx.y;
	const int x = 16 * (int)(blockIdx.x * blockDim.x + threadIdx.x);
	const int row_bytes = planes.row_bytes[p];
	if (x < row_bytes && i < chunk.start[chunk.count])
	{
		// the range of grid row i: the last k with start[k] <= i (ranges are never empty here)
		int lo = 0, hi = chunk.count - 1;
		while (lo < hi)
		{
			const int mid = (lo + hi + 1) >> 1;
			if (chunk.start[mid] <= i)
				lo = mid;
			else
				hi = mid - 1;
		}
		const int y = chunk.y0[lo] + (i - chunk.start[lo]);
		const uint8_t *s = planes.src[p] + (size_t)y * planes.src_pitch[p] + x;
		uintptr_t base = planes.dst[p];
		if (Peers)
			base += reinterpret_cast<uintptr_t>(targets.data[chunk.rank[lo]]);
		uint8_t *d = reinterpret_cast<uint8_t *>(base) + (size_t)y * planes.dst_pitch[p] + x;
		const int bytes = row_bytes - x;
		if (((planes.vec16 >> p) & 1u) && bytes >= 16)
			*reinterpret_cast<uint4 *>(d) = __ldg(reinterpret_cast<const uint4 *>(s));
		else if (planes.texel[p] == 2)
			copy_texels<2>(s, d, bytes);
		else if (planes.texel[p] == 4)
			copy_texels<4>(s, d, bytes);
		else
			copy_texels<8>(s, d, bytes);
	}
	if (Peers && publish)
		peer_publish(targets);
}

bool fail_arg(const char *fn, const char *what)
{
	char msg[256];
	std::snprintf(msg, sizeof(msg), "%s: %s", fn, what);
	set_last_error(msg);
	return false;
}

// Checks one set of planes: every present plane has the texel size its place allows, a pitch that is a multiple of
// its texel size and at least a row, a base aligned to its texel size, and the size of the first present plane.
// Fills the present mask, the common size and the texel sizes.
bool check_planes(const char *fn, const char *which, const GrbGBufferPlanes *g, unsigned &present, int &width, int &height, int texel[kPlanes])
{
	char msg[192];
	present = 0;
	for (int p = 0; p < kPlanes; p++)
	{
		const GrbImage &im = g->plane[p];
		texel[p] = 0;
		if (!im.data)
			continue;
		const int t = format_texel_bytes(im.format);
		if (!texel_fits_plane(p, t))
		{
			std::snprintf(msg, sizeof(msg), "%s plane %d has a format whose texel size does not fit that plane", which, p);
			return fail_arg(fn, msg);
		}
		if (im.width <= 0 || im.height <= 0 || im.row_pitch < im.width * t || im.row_pitch % t != 0 || reinterpret_cast<uintptr_t>(im.data) % (uintptr_t)t != 0)
		{
			std::snprintf(msg, sizeof(msg),
			              "%s plane %d needs a positive size, a row pitch that is a multiple of its texel size and at least a row, and a base aligned to its texel", which, p);
			return fail_arg(fn, msg);
		}
		if (!present)
		{
			width = im.width;
			height = im.height;
		}
		else if (im.width != width || im.height != height)
		{
			std::snprintf(msg, sizeof(msg), "%s plane %d differs in size from the planes before it", which, p);
			return fail_arg(fn, msg);
		}
		texel[p] = t;
		present |= 1u << p;
	}
	if (!present)
		return fail_arg(fn, "no plane is present");
	return true;
}

bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// The slot layout: the present planes one after another, each row width * texel bytes, each plane from a multiple of
// kSlotAlign bytes.  offsets[p] for the present planes; returns the slot's bytes.
uint64_t slot_offsets(const GrbGBufferPlanes *g, uint64_t offsets[kPlanes])
{
	uint64_t at = 0;
	for (int p = 0; p < kPlanes; p++)
	{
		offsets[p] = 0;
		const GrbImage &im = g->plane[p];
		if (!im.data)
			continue;
		offsets[p] = at;
		at += (uint64_t)im.width * (uint64_t)format_texel_bytes(im.format) * (uint64_t)im.height;
		at = (at + kSlotAlign - 1) / kSlotAlign * kSlotAlign;
	}
	return at;
}

struct Range
{
	GrbRows rows;
	int rank;
};

// Launches the kernel over `ranges` (none empty) in chunks of at most kMaxRanges ranges and kMaxGridRows grid rows; a
// peer copy publishes in its last launch only, and launches once with no rows to publish when there is nothing to copy.
template <bool Peers>
int32_t launch_chunks(const char *fn, const PlaneArgs &planes, const Range *ranges, int n, const PeerTargets &targets, void *stream)
{
	int max_row_bytes = 0;
	for (int p = 0; p < kPlanes; p++)
		max_row_bytes = planes.row_bytes[p] > max_row_bytes ? planes.row_bytes[p] : max_row_bytes;
	const unsigned grid_x = (unsigned)((max_row_bytes + 16 * 256 - 1) / (16 * 256));
	int k = 0;
	do
	{
		RangeChunk chunk;
		chunk.count = 0;
		int rows = 0;
		while (k < n && chunk.count < kMaxRanges && rows + (ranges[k].rows.y1 - ranges[k].rows.y0) <= kMaxGridRows)
		{
			chunk.start[chunk.count] = rows;
			chunk.y0[chunk.count] = ranges[k].rows.y0;
			chunk.rank[chunk.count] = (uint8_t)ranges[k].rank;
			rows += ranges[k].rows.y1 - ranges[k].rows.y0;
			chunk.count++;
			k++;
		}
		chunk.start[chunk.count] = rows;
		const bool last = k >= n;
		if (rows == 0 && !(Peers && last))
			break;
		const dim3 grid = rows > 0 ? dim3(grid_x, (unsigned)rows, (unsigned)kPlanes) : dim3(1, 1, 1);
		gbuffer_rows_kernel<Peers><<<grid, 256, 0, as_stream(stream)>>>(planes, chunk, targets, last ? 1 : 0);
		const int32_t rc = check_launch(fn);
		if (rc != GRB_OK)
			return rc;
	} while (k < n);
	return GRB_OK;
}

bool check_range(const char *fn, GrbRows r, int height)
{
	if (r.y0 < 0 || r.y1 < r.y0 || r.y1 > height)
		return fail_arg(fn, "a row range is not a range inside the image (empty allowed)");
	if (r.y1 - r.y0 > kMaxGridRows)
		return fail_arg(fn, "a row range holds more than 65535 rows");
	return true;
}
} // namespace
} // namespace grb

using namespace grb;

extern "C" int32_t grb_gbuffer_copy_rows(const GrbGBufferPlanes *src, const GrbGBufferPlanes *dst, const GrbRows *rows, int32_t range_count, void *stream)
{
	const char *fn = "grb_gbuffer_copy_rows";
	if (!src || !dst || range_count < 0 || (range_count > 0 && !rows))
	{
		fail_arg(fn, "null pointer or negative range count");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	unsigned src_present = 0, dst_present = 0;
	int w = 0, h = 0, dw = 0, dh = 0;
	int texel[kPlanes], dst_texel[kPlanes];
	if (!check_planes(fn, "src", src, src_present, w, h, texel) || !check_planes(fn, "dst", dst, dst_present, dw, dh, dst_texel))
		return GRB_ERR_INVALID_ARGUMENT;
	if (src_present != dst_present || w != dw || h != dh)
	{
		fail_arg(fn, "src and dst must have the same planes present, of one size");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	PlaneArgs planes = {};
	for (int p = 0; p < kPlanes; p++)
	{
		if (!(src_present & (1u << p)))
			continue;
		const GrbImage &s = src->plane[p], &d = dst->plane[p];
		if (s.format != d.format)
		{
			fail_arg(fn, "a plane has different formats in src and dst");
			return GRB_ERR_INVALID_ARGUMENT;
		}
		if (s.data == d.data)
		{
			fail_arg(fn, "a plane of dst is the same image as in src");
			return GRB_ERR_INVALID_ARGUMENT;
		}
		planes.src[p] = static_cast<const uint8_t *>(s.data);
		planes.dst[p] = reinterpret_cast<uintptr_t>(d.data);
		planes.src_pitch[p] = s.row_pitch;
		planes.dst_pitch[p] = d.row_pitch;
		planes.row_bytes[p] = w * texel[p];
		planes.texel[p] = texel[p];
		if (s.row_pitch % 16 == 0 && d.row_pitch % 16 == 0 && aligned16(s.data) && aligned16(d.data))
			planes.vec16 |= 1u << p;
	}
	std::vector<Range> ranges;
	for (int k = 0; k < range_count; k++)
	{
		if (!check_range(fn, rows[k], h))
			return GRB_ERR_INVALID_ARGUMENT;
		if (rows[k].y1 > rows[k].y0)
			ranges.push_back(Range{ rows[k], 0 });
	}
	return launch_chunks<false>(fn, planes, ranges.data(), (int)ranges.size(), PeerTargets{}, stream);
}

extern "C" int32_t grb_gbuffer_slot_layout(const GrbGBufferPlanes *layout, void *base, GrbGBufferPlanes *out, uint64_t *bytes)
{
	const char *fn = "grb_gbuffer_slot_layout";
	if (!layout || !bytes)
	{
		fail_arg(fn, "null pointer");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	unsigned present = 0;
	int w = 0, h = 0;
	int texel[kPlanes];
	if (!check_planes(fn, "layout", layout, present, w, h, texel))
		return GRB_ERR_INVALID_ARGUMENT;
	uint64_t offsets[kPlanes];
	*bytes = slot_offsets(layout, offsets);
	if (out)
		for (int p = 0; p < kPlanes; p++)
		{
			out->plane[p] = layout->plane[p];
			out->plane[p].data = (present & (1u << p)) && base ? static_cast<uint8_t *>(base) + offsets[p] : nullptr;
			out->plane[p].row_pitch = w * texel[p];
		}
	return GRB_OK;
}

extern "C" int32_t grb_gbuffer_rows_to_peers(const GrbGBufferPlanes *src, void *const *peer_slots, uint32_t *const *peer_flags, const GrbRows *rows,
                                             const int32_t *range_counts, int32_t peer_count, int32_t flag_index, uint32_t epoch,
                                             uint32_t *scratch_counter, void *stream)
{
	const char *fn = "grb_gbuffer_rows_to_peers";
	if (!src || !range_counts)
	{
		fail_arg(fn, "null pointer");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	PeerTargets targets;
	if (!peer_targets_from(fn, peer_slots, peer_flags, peer_count, flag_index, epoch, scratch_counter, targets))
		return GRB_ERR_INVALID_ARGUMENT;
	unsigned present = 0;
	int w = 0, h = 0;
	int texel[kPlanes];
	if (!check_planes(fn, "src", src, present, w, h, texel))
		return GRB_ERR_INVALID_ARGUMENT;
	int total = 0;
	for (int q = 0; q < peer_count; q++)
	{
		if (range_counts[q] < 0)
		{
			fail_arg(fn, "a negative range count");
			return GRB_ERR_INVALID_ARGUMENT;
		}
		total += range_counts[q];
	}
	if (total > 0 && !rows)
	{
		fail_arg(fn, "rows to copy need the row list");
		return GRB_ERR_INVALID_ARGUMENT;
	}
	uint64_t offsets[kPlanes];
	slot_offsets(src, offsets);
	PlaneArgs planes = {};
	bool slots16 = true;
	for (int q = 0; q < peer_count; q++)
		slots16 = slots16 && aligned16(peer_slots[q]);
	for (int p = 0; p < kPlanes; p++)
	{
		if (!(present & (1u << p)))
			continue;
		const GrbImage &s = src->plane[p];
		planes.src[p] = static_cast<const uint8_t *>(s.data);
		planes.dst[p] = (uintptr_t)offsets[p];
		planes.src_pitch[p] = s.row_pitch;
		planes.dst_pitch[p] = w * texel[p];
		planes.row_bytes[p] = w * texel[p];
		planes.texel[p] = texel[p];
		if (slots16 && s.row_pitch % 16 == 0 && planes.dst_pitch[p] % 16 == 0 && aligned16(s.data))
			planes.vec16 |= 1u << p;
	}
	std::vector<Range> ranges;
	for (int q = 0, at = 0; q < peer_count; q++)
		for (int k = 0; k < range_counts[q]; k++, at++)
		{
			if (!check_range(fn, rows[at], h))
				return GRB_ERR_INVALID_ARGUMENT;
			if (rows[at].y1 > rows[at].y0)
				ranges.push_back(Range{ rows[at], q });
		}
	return launch_chunks<true>(fn, planes, ranges.data(), (int)ranges.size(), targets, stream);
}
