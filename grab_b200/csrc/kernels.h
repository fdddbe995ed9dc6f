// kernels.h -- host-callable launchers of the CUDA kernels (scan_kernels.cu, resolve_kernels.cu,
// corpus_gen.cu).  Internal to libgscan.so; the public surface is include/gscan.h.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "../../include/gscan.h"
#include "device_types.h"

namespace gscan {

size_t scan_smem_bytes(const ScanGeom &g, bool look_behind);
// kernel: the pattern's GSCAN_KERNEL_* value (include/gscan.h), picked once when the pattern is compiled
ScanGeom scan_geom(int kernel);
// the scan kernel instantiation for `kernel` and the pattern's filter: F (PAIR, TRIPLE, BALANCED; delta: its filter
// distance), H (HASH) or R (RUN); the other two are not read.  NONE is an error.
cudaError_t launch_scan(int kernel, const ScanArgs &A, const FixedParams &F, const HashParams &H, const RunParams &R, int delta,
                        int grid, cudaStream_t st);
// gscan_tma_probe: the null engine on geometry 0 (scan_geom(GSCAN_KERNEL_PAIR)) or 1 (scan_geom(GSCAN_KERNEL_RUN))
cudaError_t launch_scan_null(const ScanArgs &A, int geom, int grid, cudaStream_t st);

struct DevUnit {
	uint64_t ptr;        // device address of the unit's bytes
	uint64_t base_off;   // file offset of the unit (grab.cc:154 `off`)
	uint32_t len;
	uint32_t first_tile; // index of the unit's first tile
	uint32_t file_id;
	uint32_t pad;
};

// what goes back to the caller: byte-for-byte a gscan_match (include/gscan.h)
struct FinalRec {
	uint64_t start;      // base_off + pos == off + (start - content) + ovector[0]   (grab.cc:186)
	uint32_t file_id;
	uint32_t len;
};

// Which GSCAN_RESOLVE_* path (include/gscan.h) a batch takes is decided once, by plan_resolve (resolve_plan.h), and held in
// ResolveArgs::path.  WALK: one thread replays each unit's loop.  FLAT (ALL mode, RUN or a FIXED pattern whose matches can
// never overlap, no VM): every candidate of a unit is a match, except that the loop guard (grab.cc:175, Q1) can drop the
// unit's LAST one -- no replay needed, the write pass runs one thread per candidate (a 1 GiB window with 10^7 candidates
// resolves in microseconds).  The chain paths: see ResolveArgs.  The kernels and the launch sequence ask these questions:
__host__ __device__ inline bool path_chain(uint32_t p) { return p >= GSCAN_RESOLVE_CHAIN; }        // pointer doubling over a node list
__host__ __device__ inline bool path_vm_chain(uint32_t p) { return p >= GSCAN_RESOLVE_VM_ATTEMPTS; } // ... over the VM outcomes that matched
__host__ __device__ inline bool path_compacted(uint32_t p) { return p == GSCAN_RESOLVE_VM_DENSE || p == GSCAN_RESOLVE_VM_DENSE_TWO; } // k_vm_dense wrote that list
__host__ __device__ inline bool path_attempts(uint32_t p) { return path_vm_chain(p) && !path_compacted(p); } // k_vm_attempts writes it
__host__ __device__ inline bool path_two(uint32_t p) { return p == GSCAN_RESOLVE_VM_TWO || p == GSCAN_RESOLVE_VM_DENSE_TWO; } // outcomes A and B
__host__ __device__ inline bool path_run(uint32_t p) { return p == GSCAN_RESOLVE_VM_RUN_CHAIN; }

struct ResolveArgs {
	const TileDesc *tiles;
	const SegEntry *segs;
	uint32_t *occ;        // occupancy bits of segs (ScanArgs::occ); k_gather clears the words it reads
	uint32_t n_segs;
	uint32_t spt_shift;   // log2(slices per tile)
	uint32_t tag;         // generation of the scan that filled segs
	const Cand *cand;
	const DevUnit *units;
	uint32_t n_units;
	OutRec *ord;          // candidates in (unit, pos) order
	FinalRec *out;        // selected matches, same order (capacity known after the count pass)
	uint32_t *unit_start; // [n_units + 1] first candidate of each unit in ord
	uint32_t *unit_out;   // [n_units] matches per unit, then (exclusive scan) first output slot
	uint32_t *blk;        // block-sum scratch of the scans, reused from offset 0 by each
	uint32_t *totals;     // [0] candidates, [1] matches, [2] VM limit flag
	uint32_t path;        // GSCAN_RESOLVE_*, from plan_resolve
	uint32_t mode, minlen, engine, run_min;
	uint32_t bitmap[8];   // RUN class, for match-length extension
	uint32_t total_cand;  // known on the host after the scan kernel
	const uint32_t *vm_code; // general patterns: VM program (3 words per instruction) and byte classes (8 words each)
	const uint32_t *vm_sets;
	uint32_t vm_runstart; // candidates are run starts of `bitmap`: also try the search start itself when it lies inside a run
	uint32_t vm_dense;    // general pattern without a candidate filter: no candidate list, no segments; the WALK offers every position
	                      // whose byte is in `bitmap` (the first-byte set) to the VM
	// CHAIN (FIXED patterns whose matches can overlap, or LINE mode, with many candidates per unit) and the VM_* paths: the
	// selected matches of a unit are the chain c0 -> next(c0) -> ..., next(i) = first node at or after where the search
	// resumes behind i.  Pointer doubling marks every chain member in O(log n) passes over all nodes instead of one thread
	// walking a huge unit alone.  chain_buf: chain_levels x chain_cap jump tables, then the mark and rank arrays (VM_TWO,
	// VM_DENSE_TWO, VM_RUN_CHAIN: two more, see chain_bscan / chain_stop)
	uint32_t chain_levels, chain_cap;
	uint32_t *chain_buf;
	// VM_ATTEMPTS: patterns whose attempts do not depend on where the subject begins (Program::vm_start_free) with many
	// candidates per unit.  One anchored VM attempt per candidate, all at once (k_vm_attempts: outcome and match length into
	// ord[].pad / .len), the candidates that matched are compacted into vm_ord / vm_unit_start (exclusive scan of vm_flag), and
	// the chain kernels run over those: the selected matches of a unit are the chain from its first matching candidate,
	// next(i) = first matching candidate at or after where the loop resumes behind i.  A candidate whose match has a capturing
	// group set (Q2) or that ran into the VM's limits ends its unit's chain there and is not reported (grab.cc:179: rc <= 0 =>
	// break).
	OutRec *vm_ord;           // [total_cand] the candidates with pad != 0, (unit, pos) order
	uint32_t *vm_unit_start;  // [n_units + 1] into vm_ord
	uint32_t *vm_flag;        // [total_cand] pad != 0, then its exclusive scan
	unsigned long long *vm_budget; // [n_units] VM steps the unit's attempts may still take, all of them together
	// VM_DENSE: start-free programs without a candidate filter, units big enough that one thread per unit would walk for
	// seconds.  k_vm_dense runs the anchored attempts of 64 consecutive positions per thread over the whole batch, twice like
	// the serial walk (count, prefix sum, write): what comes out IS the compacted list of VM_ATTEMPTS (vm_ord / vm_unit_start,
	// totals[4]), and the chain kernels take it from there.
	uint32_t dense_blocks;    // 64-position blocks of the batch = n_tiles << (dense_tile_shift - 6)
	uint32_t dense_tile_shift;
	// VM_TWO / VM_DENSE_TWO: reach-1 programs (Program::vm_reach == 1: only the attempt whose subject begins at the candidate
	// itself differs from "any earlier start").  Every candidate p gets two outcomes, A(p): subject begins at p, and B(p):
	// subject begins before p (p >= 1).  The matching ones form one node list in (unit, pos, A before B) order; a search that
	// resumes at s continues at node (s, A) if A(s) matched, else at the first B node behind s.  Which nodes are B is kept
	// beside the chain tables (chain_bscan: exclusive count of B nodes, chain_blist: their indices, totals[5] of them), never
	// in OutRec.  vm_ord_b: [total_cand] the B outcomes of k_vm_attempts, before compaction.
	OutRec *vm_ord_b;
	// VM_RUN_CHAIN: class-repeat-led programs (vm_runstart, reach 0, greedy or possessive lead) on the chain: a search that
	// resumes inside a run tries one attempt there; if it matches it ends where the run start's own match ends (chain_stop:
	// where each node's search resumes, for chain_entry)
	uint32_t *vm_limit;   // VM_RUN_CHAIN: the VM limit flag (totals[2]; the chain kernels see totals + 4)
};

// count pass: segment scan and gather (not for vm_dense programs), then the path's count sequence; totals[1] = number of matches
cudaError_t launch_resolve_count(const ResolveArgs &R, cudaStream_t st, uint32_t *launches);
// write pass: the path's write kernel fills R.out
cudaError_t launch_resolve_write(const ResolveArgs &R, cudaStream_t st, uint32_t *launches);
// VM_DENSE*, before launch_resolve_count: count pass (matching positions per 64-position block into vm_flag, exclusive scan,
// total into totals[4]) and, once the host has sized vm_ord and the chain tables, the write pass (+ vm_unit_start)
cudaError_t launch_vm_dense_count(const ResolveArgs &R, cudaStream_t st, uint32_t *launches);
cudaError_t launch_vm_dense_write(const ResolveArgs &R, cudaStream_t st, uint32_t *launches);

cudaError_t launch_synth_corpus(uint8_t *dptr, uint64_t seed, uint64_t first_file_id, uint64_t n_files, uint64_t file_len,
                                uint64_t stride, const uint8_t *d_needle, uint32_t needle_len, uint32_t needle_every,
                                cudaStream_t st);
cudaError_t launch_fill_u32(uint32_t *p, size_t n, uint32_t v, cudaStream_t st);
cudaError_t launch_read_probe(const void *dptr, uint64_t bytes, unsigned long long *d_sum, int grid, cudaStream_t st);

} // namespace gscan
