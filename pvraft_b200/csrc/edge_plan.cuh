// The tiles of the SetConv edge kernel and their gather plan: edge_plan.cu builds the plan of a kNN graph once,
// setconv_edge.cu runs every launch on that graph from it.
//
// A tile is kEdgeTile consecutive positions of the processing order of one sample (a tile never straddles two samples; the
// last tile of a sample may be shorter).  It references kEdgeRefs rows of P: the 32 neighbours of each of its points, then
// the points themselves (the centres).  Its plan record, kEdgePlanBytes at byte offset ((b * tiles_per_sample) + tile) *
// kEdgePlanBytes, so that the records of a batch are sample-major and the first samples' records are a prefix:
//   int32  id[kEdgeRefs]      at 0               the distinct row ids in slot order (count of them are meaningful)
//   uint16 slot[kEdgeRefs]    at kEdgePlanSlots  the slot of each reference: neighbour e of point p at p * 32 + e, the centre
//                                                of point p at kEdgeTile * 32 + p (0 for the missing points of a short tile)
//   int32  count              at kEdgePlanCount  the number of distinct rows
// The plan depends on the graph (nbr, order) alone, not on the features nor on the channel count.
#pragma once
#include "common.cuh"

namespace pvraft {

constexpr int kEdgeTile = 32;                                  // points per tile
constexpr int kEdgeRefs = kEdgeTile * 33;                      // row references of a tile: 32 neighbours + the centre per point
constexpr int kEdgePlanSlots = kEdgeRefs * 4;                  // byte offsets in a tile's record (all multiples of 16: the
constexpr int kEdgePlanCount = kEdgePlanSlots + kEdgeRefs * 2; // edge kernel bulk-copies ids and slots)
constexpr int kEdgePlanBytes = kEdgePlanCount + 16;
static_assert(kEdgePlanSlots % 16 == 0 && kEdgePlanCount % 16 == 0, "bulk-copy alignment");

__host__ __device__ constexpr int edge_tiles_per_sample(int N) { return (N + kEdgeTile - 1) / kEdgeTile; }

}  // namespace pvraft
