// cuda_backend.hpp -- what stands where Granite's vulkan/ backend stood, for the passes of the
// hot path only: a Device that owns device memory, ImageView / Buffer handles for the physical
// resources of the render graph, and a CommandBuffer that is nothing but a CUDA stream on a
// device (SURVEY.md §8b: "Vulkan::CommandBuffer becomes a thin handle {cudaStream_t, device}").
//
// The class and method names follow the subset of the Vulkan:: API that the reference's pass
// builders call (get_image().get_create_info().width, get_format(), ...), so a builder written
// against Granite reads the same here.  `namespace Vulkan` is an alias of Granite::CUDA for that
// reason only -- there is no Vulkan anywhere in this build.
#pragma once

#include <cstddef>
#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/granite_b200.h"
#include "vk_compat.hpp"

struct CUstream_st;
struct CUevent_st;

namespace Granite
{
namespace CUDA
{
using Stream = CUstream_st *;
using Event = CUevent_st *;

struct ImageCreateInfo
{
	unsigned width = 0, height = 0;
	VkFormat format = VK_FORMAT_UNDEFINED;
};

class Device;

class Image
{
public:
	Image(Device &device, const ImageCreateInfo &info);
	// Wraps memory the caller owns (a swapchain image): rows of row_pitch bytes; never freed here.
	Image(Device &device, const ImageCreateInfo &info, void *external, unsigned row_pitch);
	~Image();
	Image(const Image &) = delete;
	void operator=(const Image &) = delete;
	const ImageCreateInfo &get_create_info() const { return info; }
	unsigned get_width() const { return info.width; }
	unsigned get_height() const { return info.height; }
	VkFormat get_format() const { return info.format; }
	void *get_device_pointer() const { return data; }
	size_t get_size() const { return size; }
	unsigned get_row_pitch() const { return row_pitch; }
	bool owns_memory() const { return owned; }

private:
	Device &device;
	ImageCreateInfo info;
	void *data = nullptr;
	size_t size = 0;
	unsigned row_pitch = 0;
	bool owned = true;
};

class ImageView
{
public:
	explicit ImageView(std::shared_ptr<Image> image_) : image(std::move(image_)) {}
	Image &get_image() { return *image; }
	const Image &get_image() const { return *image; }
	VkFormat get_format() const { return image->get_format(); }
	unsigned get_view_width() const { return image->get_width(); }
	unsigned get_view_height() const { return image->get_height(); }
	// The C-ABI descriptor of this view.
	GrbImage as_grb() const;
	// "set_unorm_texture": the same memory viewed with the non-sRGB twin of its format.
	GrbImage as_grb_unorm() const;
	const std::shared_ptr<Image> &get_image_handle() const { return image; }

private:
	std::shared_ptr<Image> image;
};

struct BufferCreateInfo
{
	size_t size = 0;
};

class Buffer
{
public:
	Buffer(Device &device, const BufferCreateInfo &info);
	~Buffer();
	Buffer(const Buffer &) = delete;
	void operator=(const Buffer &) = delete;
	const BufferCreateInfo &get_create_info() const { return info; }
	void *get_device_pointer() const { return data; }
	template <typename T>
	T *get() const { return static_cast<T *>(data); }

private:
	Device &device;
	BufferCreateInfo info;
	void *data = nullptr;
};
using BufferHandle = std::shared_ptr<Buffer>;
using ImageHandle = std::shared_ptr<Image>;

// One CUDA device + the stream the graph records on.  All allocations are zero-initialised,
// like the graph's buffers in the reference (renderer/render_graph.cpp:2587).
class Device
{
public:
	explicit Device(int cuda_device_index, Stream stream = nullptr);
	~Device();
	int get_device_index() const { return index; }
	Stream get_stream() const { return stream; }
	// Side streams for passes declared on the asynchronous queues (the reference's async-compute
	// queue): index 1 = RENDER_GRAPH_QUEUE_ASYNC_COMPUTE_BIT, 2 = RENDER_GRAPH_QUEUE_ASYNC_GRAPHICS_BIT,
	// 3 = RENDER_GRAPH_QUEUE_ASYNC_POST_COMPUTE_BIT.
	// Index 0 is the main stream.  Created on first use.
	Stream get_queue_stream(unsigned index);
	Stream get_async_stream() { return get_queue_stream(1); }
	void record_event_on(Event e, Stream s);
	void stream_wait_event(Stream s, Event e);
	// Makes the main stream wait for everything recorded so far on the side streams.
	void join_side_streams();
	ImageHandle create_image(const ImageCreateInfo &info);
	BufferHandle create_buffer(const BufferCreateInfo &info);
	void *allocate(size_t size);
	void free(void *ptr);
	void wait_idle();
	// GPU time intervals per tag (replaces Device::register_time_interval / timestamp_log).
	struct TimeInterval
	{
		std::string tag;
		Event begin, end;
	};
	void register_time_interval(const std::string &tag, Event begin, Event end);
	// Resolves and clears the registered intervals: (tag, milliseconds).
	std::vector<std::pair<std::string, float>> collect_time_intervals();
	// Same intervals as (tag, begin ms, end ms) relative to the first interval ever registered:
	// a GPU timeline (the counterpart of the reference's GRANITE_TIMELINE_TRACE for the GPU side).
	struct TimelineEntry
	{
		std::string tag;
		float begin_ms, end_ms;
	};
	std::vector<TimelineEntry> collect_timeline();
	Event request_event();
	void record_event(Event e);

private:
	int index;
	Stream stream;
	bool owns_stream = false;
	Stream side_streams[3] = { nullptr, nullptr, nullptr };
	Event join_events[3] = { nullptr, nullptr, nullptr };
	Event alloc_event = nullptr; // orders the zero fill of a fresh allocation before the side streams
	std::mutex lock;
	std::vector<TimeInterval> intervals;
	std::vector<Event> event_pool;
	Event epoch = nullptr;
};

// Thrown (host side only, never across the C ABI) when a kernel launch or CUDA call fails and
// the graph is configured to be strict; otherwise failures are logged and execution continues,
// as the reference does for runtime failures (render_graph.cpp:2220, 2678).
class CommandBuffer
{
public:
	CommandBuffer(Device &device_, Stream stream_) : device(device_), stream(stream_) {}
	Device &get_device() { return device; }
	Stream get_stream() const { return stream; }
	void *get_stream_handle() const { return stream; }
	// Checks a C-ABI return code; logs grb_last_error_string() on failure.
	bool check(int32_t grb_result, const char *what);
	unsigned get_error_count() const { return errors; }
	void begin_region(const char *name);
	void end_region();
	// Kept for source compatibility: stream order already provides the dependency.
	void barrier() {}

private:
	Device &device;
	Stream stream;
	unsigned errors = 0;
};

void log_error(const char *fmt, ...);
void log_info(const char *fmt, ...);
bool cuda_ok(int cuda_error, const char *what);

// Host-side section timer (GRB_HOST_PROFILE=1): accumulates wall time per named section of the
// frame recording and prints the averages when the report is requested.
struct HostProfile
{
	static bool enabled();
	static void add(const char *name, double microseconds);
	static void report(unsigned frames);
};

class ScopedHostTimer
{
public:
	explicit ScopedHostTimer(const char *name_);
	~ScopedHostTimer();

private:
	const char *name;
	double t0 = 0.0;
};
} // namespace CUDA
} // namespace Granite

namespace Vulkan = Granite::CUDA;
