// nccl_collectives.hpp -- RenderGraphCollectives over NCCL (NVLink 4 / NVSwitch), one rank per
// process/GPU.  libnccl is resolved at run time (dlopen of libnccl.so.2 -- the copy PyTorch
// already loaded when the host process is a torchrun rank), so the host library itself has no
// link-time NCCL dependency.  The unique id is created on rank 0 and distributed by the caller
// (bench.py / tests use torch.distributed for that plumbing).
#pragma once

#include <string>
#include <vector>

#include "render_graph.hpp"

namespace Granite
{
constexpr unsigned NcclUniqueIdBytes = 128;

class NcclCollectives : public RenderGraphCollectives
{
public:
	NcclCollectives() = default;
	~NcclCollectives() override;
	static bool get_unique_id(unsigned char out[NcclUniqueIdBytes], std::string &error);
	bool init(const unsigned char id[NcclUniqueIdBytes], unsigned rank, unsigned world_size, std::string &error);
	unsigned get_rank() const override { return rank; }
	unsigned get_world_size() const override { return world; }
	bool all_gather_rows(Vulkan::CommandBuffer &cmd, Vulkan::ImageView &image, const std::vector<GrbRows> &rows) override;
	bool all_reduce_sum(Vulkan::CommandBuffer &cmd, float *data, size_t count) override;
	// Peer-memory exchange: two image slots + a flag array per rank, cudaIpc-mapped into every
	// other rank (handles are exchanged with one ncclAllGather).  GRB_SHARD_EXCHANGE=nccl disables it.
	bool peer_exchange_begin_frame(size_t image_bytes, PeerSlot &slot) override;
	// Second channel, same set-up and teardown: the SMAA edge rows (host/post/smaa.cpp).
	bool smaa_edge_exchange_begin_frame(size_t image_bytes, PeerSlot &slot) override;
	// Third channel: the TAA history (host/post/temporal.cpp).
	bool taa_history_exchange_begin_frame(size_t image_bytes, PeerSlot &slot) override;
	// Fourth channel: the bands of the final image, pushed to the presenting rank (host/scene_viewer.cpp).
	bool present_exchange_begin_frame(size_t image_bytes, PeerSlot &slot) override;

private:
	bool collective_failed(const char *what);
	void *comm = nullptr;
	unsigned rank = 0, world = 1;

	struct PeerState
	{
		bool tried = false, ok = false;
		size_t image_bytes = 0;
		void *local_images[2] = {};
		uint32_t *local_flags = nullptr; // [world] flags followed by the scratch counter
		void *images[2][8] = {};
		uint32_t *flags[8] = {};
		std::vector<void *> opened;
		uint32_t epoch = 0;
	};
	PeerState bloom_d0;  // bloom d0 bands
	PeerState smaa_edge; // SMAA edge rows
	PeerState taa_history; // TAA history rows
	PeerState present;     // the final image on the presenting rank
	bool begin_frame(PeerState &channel, size_t image_bytes, PeerSlot &slot);
	bool setup_peer_exchange(PeerState &channel, size_t image_bytes);
	void release_peer_exchange(PeerState &channel);
};
} // namespace Granite
