// Slab plans: the H100-native replacement for the reference's MPI derived
// datatypes (MPI_Type_vector + create_resized, duplicated at reference
// csrc/extension.cpp:516-591, :651-726, :788-876).
//
// Every axis-aware collective (Gather, Allgather, Scatter, Alltoall,
// Reduce_scatter) is expressed as a list of strided box copies that THIS rank
// pulls out of peers' staged inputs.  A box is up to three outer loops around a
// contiguous run, all in 64-bit element units (no INT_MAX limits, cf.
// reference :530, :665, :810).  The same plan drives the CPU shared-memory
// backend (memcpy) and the sm_90a slab kernels (peer loads over NVLink).
#pragma once
#include <cstdint>
#include <vector>

namespace m4t {

struct SlabJob {
  int32_t peer = 0;        // rank whose staged buffer is read
  int64_t src_off = 0;     // element offset into the peer's staged input
  int64_t dst_off = 0;     // element offset into the local output
  int64_t n[3] = {1, 1, 1};   // outer loop extents (n[2] innermost)
  int64_t ss[3] = {0, 0, 0};  // source strides, elements
  int64_t ds[3] = {0, 0, 0};  // destination strides, elements
  int64_t run = 0;         // contiguous elements per row

  int64_t rows() const { return n[0] * n[1] * n[2]; }
  int64_t elems() const { return rows() * run; }
};

struct PullPlan {
  std::vector<SlabJob> jobs;  // boxes this rank pulls (may be empty, e.g. Gather off-root)
  int64_t stage_elems = 0;    // elements of this rank's input that peers will read (0 = none)
  int64_t out_elems = 0;      // elements of the local output
  int64_t max_stage_elems = 0;  // max over ranks of stage_elems (symmetric heap sizing)
  int64_t max_out_elems = 0;    // max over ranks of out_elems (rank-independent grid sizing)
  bool replicated_output = false;  // every rank receives the identical gathered tensor (Allgather)
  // Allgather only: the request the plan was built from (the hierarchical host backend re-plans it in two stages)
  int64_t before = 1, after = 1;
  std::vector<int64_t> axis_len;
};

// out = reduce over all peers p of staged_p[box]; all peers share one box shape.
struct ReducePlan {
  SlabJob box;               // peer field unused
  int64_t stage_elems = 0;   // identical on all ranks
  int64_t out_elems = 0;
  int64_t max_out_elems = 0;  // max over ranks (rank-independent grid sizing)
  // the request the plan was built from (transports that re-plan in stages - the hierarchical host backend - read it)
  int64_t before = 1, after = 1;
  std::vector<int64_t> numelem;
};

// Drops unit loops and folds loops that continue the contiguous run.
void normalize_job(SlabJob& j);

// [before, axis, after] decomposition of a shape around `axis`.
struct Axis3 {
  int64_t before = 1, axis = 1, after = 1;
};
Axis3 split_axis(const std::vector<int64_t>& shape, int64_t axis);

// axis_len[p] = length of the gather axis on rank p.
PullPlan plan_gather(int rank, int size, int root, int64_t before, int64_t after,
                     const std::vector<int64_t>& axis_len, bool all);
// numelem[p] = rows rank p receives; total = root's axis length.
PullPlan plan_scatter(int rank, int size, int root, int64_t before, int64_t after,
                      const std::vector<int64_t>& numelem);
// General all-to-all between two different axes.  `shape` is this rank's input
// shape; gather_len[p] = length of gatheraxis on rank p; numelem[p] = rows of
// scatteraxis rank p receives.
PullPlan plan_alltoall(int rank, int size, const std::vector<int64_t>& shape, int64_t gatheraxis,
                       int64_t scatteraxis, const std::vector<int64_t>& gather_len,
                       const std::vector<int64_t>& numelem);
// Same-axis all-to-all = re-partition of one global axis (reference :947-979).
PullPlan plan_repartition(int rank, int size, int64_t before, int64_t after,
                          const std::vector<int64_t>& cur_len, const std::vector<int64_t>& new_len);
// Reduce-scatter along an axis: every rank holds [before, sum(numelem), after].
ReducePlan plan_reduce_scatter(int rank, int size, int64_t before, int64_t after,
                               const std::vector<int64_t>& numelem);

}  // namespace m4t
