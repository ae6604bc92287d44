#include "cuda_backend.hpp"

#include <nvtx3/nvToolsExt.h>

#include <cuda_runtime.h>

#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <stdexcept>

namespace Granite
{
namespace CUDA
{
void log_error(const char *fmt, ...)
{
	va_list va;
	va_start(va, fmt);
	std::fprintf(stderr, "[granite_b200 ERROR] ");
	std::vfprintf(stderr, fmt, va);
	va_end(va);
}

void log_info(const char *fmt, ...)
{
	va_list va;
	va_start(va, fmt);
	std::fprintf(stderr, "[granite_b200] ");
	std::vfprintf(stderr, fmt, va);
	va_end(va);
}

bool cuda_ok(int err, const char *what)
{
	if (err == cudaSuccess)
		return true;
	log_error("%s: %s\n", what, cudaGetErrorString((cudaError_t)err));
	return false;
}

namespace
{
std::map<std::string, std::pair<double, unsigned>> &profile_sections()
{
	static std::map<std::string, std::pair<double, unsigned>> sections;
	return sections;
}
double now_us()
{
	return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
} // namespace

bool HostProfile::enabled()
{
	static const bool on = std::getenv("GRB_HOST_PROFILE") != nullptr;
	return on;
}

void HostProfile::add(const char *name, double microseconds)
{
	auto &slot = profile_sections()[name];
	slot.first += microseconds;
	slot.second++;
}

void HostProfile::report(unsigned frames)
{
	if (!enabled() || !frames)
		return;
	std::fprintf(stderr, "[granite_b200] host profile over %u frames (us per frame, calls per frame):\n", frames);
	for (auto &kv : profile_sections())
		std::fprintf(stderr, "  %-36s %9.1f  %6.1f\n", kv.first.c_str(), kv.second.first / frames, double(kv.second.second) / frames);
	profile_sections().clear();
}

ScopedHostTimer::ScopedHostTimer(const char *name_) : name(name_)
{
	if (HostProfile::enabled())
		t0 = now_us();
}

ScopedHostTimer::~ScopedHostTimer()
{
	if (HostProfile::enabled())
		HostProfile::add(name, now_us() - t0);
}

Device::Device(int cuda_device_index, Stream stream_) : index(cuda_device_index), stream(stream_)
{
	if (!cuda_ok(cudaSetDevice(index), "cudaSetDevice"))
		throw std::runtime_error("granite_b200: cannot select the CUDA device");
	if (!stream)
	{
		cudaStream_t s;
		if (!cuda_ok(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking), "cudaStreamCreate"))
			throw std::runtime_error("granite_b200: cannot create a stream");
		stream = s;
		owns_stream = true;
	}
	if (grb_init() != GRB_OK)
		throw std::runtime_error(std::string("granite_b200: grb_init failed: ") + grb_last_error_string());
}

Device::~Device()
{
	cudaSetDevice(index);
	cudaStreamSynchronize(stream);
	for (auto &iv : intervals)
	{
		event_pool.push_back(iv.begin);
		event_pool.push_back(iv.end);
	}
	for (auto e : event_pool)
		cudaEventDestroy(e);
	for (auto &side : side_streams)
		if (side && side != stream)
		{
			cudaStreamSynchronize(side);
			cudaStreamDestroy(side);
		}
	for (auto e : join_events)
		if (e)
			cudaEventDestroy(e);
	if (owns_stream)
		cudaStreamDestroy(stream);
}

Stream Device::get_queue_stream(unsigned idx)
{
	if (idx == 0 || idx > 3)
		return stream;
	std::lock_guard<std::mutex> hold(lock);
	auto &side = side_streams[idx - 1];
	if (!side)
	{
		// Side streams get the highest priority: their kernels are short (cluster build) or HBM-bound
		// (post chain), and with priority the block scheduler hands them SM slots as the long,
		// ALU-bound lighting grid on the main stream retires CTAs -- without it a later kernel only
		// starts once the earlier grid has no CTAs left to issue, and nothing overlaps.
		int least = 0, greatest = 0;
		cudaDeviceGetStreamPriorityRange(&least, &greatest);
		cudaStream_t s;
		if (cuda_ok(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, greatest), "cudaStreamCreate(side)"))
			side = s;
		else
			side = stream;
	}
	return side;
}

void Device::join_side_streams()
{
	for (int i = 0; i < 3; i++)
	{
		if (!side_streams[i] || side_streams[i] == stream)
			continue;
		if (!join_events[i])
		{
			cudaEvent_t e;
			cuda_ok(cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "cudaEventCreate(join)");
			join_events[i] = e;
		}
		cuda_ok(cudaEventRecord(join_events[i], side_streams[i]), "cudaEventRecord(join)");
		cuda_ok(cudaStreamWaitEvent(stream, join_events[i], 0), "cudaStreamWaitEvent(join)");
	}
}

void Device::record_event_on(Event e, Stream s)
{
	cuda_ok(cudaEventRecord(e, s), "cudaEventRecord");
}

void Device::stream_wait_event(Stream s, Event e)
{
	cuda_ok(cudaStreamWaitEvent(s, e, 0), "cudaStreamWaitEvent");
}

void *Device::allocate(size_t size)
{
	void *p = nullptr;
	if (size == 0)
		size = 16;
	if (!cuda_ok(cudaMalloc(&p, size), "cudaMalloc"))
		throw std::runtime_error("granite_b200: out of device memory");
	// zero-initialised like the graph's buffers (render_graph.cpp:2587).  The fill runs on the graph
	// stream, but the first writer of a fresh resource may record on a side stream (cluster build,
	// pipelined G-buffer upload, bloom), and the graph's hazard tracking has no entry for a resource
	// that nobody has touched yet: make every side stream wait for the fill.
	cuda_ok(cudaMemsetAsync(p, 0, size, stream), "cudaMemsetAsync");
	bool has_side = false;
	for (auto side : side_streams)
		has_side = has_side || (side && side != stream);
	if (has_side)
	{
		if (!alloc_event)
		{
			cudaEvent_t e;
			cuda_ok(cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "cudaEventCreate(alloc)");
			alloc_event = e;
		}
		cuda_ok(cudaEventRecord(alloc_event, stream), "cudaEventRecord(alloc)");
		for (auto side : side_streams)
			if (side && side != stream)
				cuda_ok(cudaStreamWaitEvent(side, alloc_event, 0), "cudaStreamWaitEvent(alloc)");
	}
	return p;
}

void Device::free(void *ptr)
{
	if (ptr)
	{
		cudaStreamSynchronize(stream);
		cudaFree(ptr);
	}
}

void Device::wait_idle()
{
	for (auto side : side_streams)
		if (side && side != stream)
			cuda_ok(cudaStreamSynchronize(side), "cudaStreamSynchronize(side)");
	cuda_ok(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
}

ImageHandle Device::create_image(const ImageCreateInfo &info)
{
	return std::make_shared<Image>(*this, info);
}

BufferHandle Device::create_buffer(const BufferCreateInfo &info)
{
	return std::make_shared<Buffer>(*this, info);
}

Event Device::request_event()
{
	std::lock_guard<std::mutex> hold(lock);
	if (!event_pool.empty())
	{
		Event e = event_pool.back();
		event_pool.pop_back();
		return e;
	}
	cudaEvent_t e;
	cuda_ok(cudaEventCreate(&e), "cudaEventCreate");
	return e;
}

void Device::record_event(Event e)
{
	cuda_ok(cudaEventRecord(e, stream), "cudaEventRecord");
}

void Device::register_time_interval(const std::string &tag, Event begin, Event end)
{
	std::lock_guard<std::mutex> hold(lock);
	intervals.push_back({ tag, begin, end });
}

std::vector<std::pair<std::string, float>> Device::collect_time_intervals()
{
	std::vector<TimeInterval> local;
	{
		std::lock_guard<std::mutex> hold(lock);
		local.swap(intervals);
	}
	std::vector<std::pair<std::string, float>> out;
	for (auto &iv : local)
	{
		float ms = 0.0f;
		cudaEventSynchronize(iv.end);
		cudaEventElapsedTime(&ms, iv.begin, iv.end);
		out.emplace_back(iv.tag, ms);
		std::lock_guard<std::mutex> hold(lock);
		event_pool.push_back(iv.begin);
		event_pool.push_back(iv.end);
	}
	return out;
}

std::vector<Device::TimelineEntry> Device::collect_timeline()
{
	std::vector<TimeInterval> local;
	{
		std::lock_guard<std::mutex> hold(lock);
		local.swap(intervals);
	}
	std::vector<TimelineEntry> out;
	if (local.empty())
		return out;
	for (auto &iv : local)
		cudaEventSynchronize(iv.end);
	Event ref = local.front().begin;
	for (auto &iv : local)
	{
		TimelineEntry e;
		e.tag = iv.tag;
		cudaEventElapsedTime(&e.begin_ms, ref, iv.begin);
		cudaEventElapsedTime(&e.end_ms, ref, iv.end);
		out.push_back(e);
	}
	std::lock_guard<std::mutex> hold(lock);
	for (auto &iv : local)
	{
		event_pool.push_back(iv.begin);
		event_pool.push_back(iv.end);
	}
	return out;
}

Image::Image(Device &device_, const ImageCreateInfo &info_) : device(device_), info(info_)
{
	unsigned texel = format_texel_size(info.format);
	if (!texel || !info.width || !info.height)
		throw std::logic_error("granite_b200: unsupported image format or empty extent");
	row_pitch = info.width * texel;
	size = (size_t)row_pitch * info.height;
	data = device.allocate(size);
}

Image::Image(Device &device_, const ImageCreateInfo &info_, void *external, unsigned row_pitch_)
    : device(device_), info(info_), data(external), row_pitch(row_pitch_), owned(false)
{
	if (!format_texel_size(info.format) || !info.width || !info.height || !external || row_pitch < info.width * format_texel_size(info.format))
		throw std::logic_error("granite_b200: bad external image");
	size = (size_t)row_pitch * (info.height - 1) + (size_t)info.width * format_texel_size(info.format);
}

Image::~Image()
{
	if (owned)
		device.free(data);
}

Buffer::Buffer(Device &device_, const BufferCreateInfo &info_) : device(device_), info(info_)
{
	data = device.allocate(info.size);
}

Buffer::~Buffer()
{
	device.free(data);
}

GrbImage ImageView::as_grb() const
{
	GrbImage g;
	g.data = image->get_device_pointer();
	g.width = (int32_t)image->get_width();
	g.height = (int32_t)image->get_height();
	g.row_pitch = (int32_t)image->get_row_pitch();
	g.format = image->get_format();
	return g;
}

GrbImage ImageView::as_grb_unorm() const
{
	GrbImage g = as_grb();
	if (g.format == VK_FORMAT_R8G8B8A8_SRGB)
		g.format = VK_FORMAT_R8G8B8A8_UNORM;
	return g;
}

bool CommandBuffer::check(int32_t result, const char *what)
{
	if (result == GRB_OK)
		return true;
	errors++;
	log_error("%s failed (%d): %s\n", what, result, grb_last_error_string());
	return false;
}

// NVTX ranges around every pass callback (Vulkan::CommandBuffer::begin_region / end_region label
// the pass in RenderDoc; here it is what Nsight Systems / ncu --nvtx show).  Header-only NVTX3:
// without a profiler attached the calls are a pointer test.
void CommandBuffer::begin_region(const char *name) { nvtxRangePushA(name ? name : "pass"); }
void CommandBuffer::end_region() { nvtxRangePop(); }
} // namespace CUDA
} // namespace Granite
