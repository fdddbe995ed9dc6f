// resolve_plan.h -- which GSCAN_RESOLVE_* path resolves a batch, and the geometry of its chain tables.  Host only and
// header-inline: gscan_batch_scan and the CPU model checks (tests/model_check*.cc) plan with this same code.
#pragma once
#include <algorithm>
#include <cstdint>

#include "../../include/gscan.h"
#include "kernels.h"
#include "pattern.h"

namespace gscan {

enum ChainOverride { CHAIN_AUTO, CHAIN_ON, CHAIN_OFF }; // GSCAN_CHAIN unset / "1" (force the chain paths on small inputs) / other

constexpr uint64_t kChainTableBytes = 4ull << 30; // the chain tables of one call stay below this

struct ChainGeom {
	uint64_t nodes;   // list entries the tables cover
	uint32_t levels;  // jump tables (at least two: the second one doubles as the RUN entry positions)
	uint32_t arrays;  // levels + marks, ranks (+ the B scan and list / the resume points)
	bool fits;        // arrays x nodes words stay within kChainTableBytes
};

// n: candidates, or for VM_DENSE* the matching outcomes k_vm_dense counted.  VM_TWO: outcomes A and B of every candidate
inline ChainGeom chain_geom(uint32_t path, uint64_t n)
{
	ChainGeom g;
	g.nodes = path == GSCAN_RESOLVE_VM_TWO ? 2 * n : n;
	g.levels = 2;
	while ((1ull << g.levels) < g.nodes) g.levels++;
	g.arrays = g.levels + ((path_two(path) || path_run(path)) ? 4 : 2);
	g.fits = (uint64_t)g.arrays * g.nodes * 4 <= kChainTableBytes;
	return g;
}

// The path of one call.  n_cand: candidate slots the scan reserved (unused for dense programs, which have no scan);
// dense_blocks: 64-position blocks of the batch.  For VM_DENSE* the hit count is known only after k_vm_dense's count pass:
// the caller checks chain_geom(path, hits).fits then and falls back to the WALK when it does not fit.
inline uint32_t plan_resolve(const Program &p, uint32_t mode, uint64_t n_units, uint64_t bytes, uint64_t dense_blocks,
                             uint64_t n_cand, ChainOverride force)
{
	n_units = std::max<uint64_t>(n_units, 1);
	if (p.use_vm && p.vm_dense) {
		// no candidate filter: the attempts of all positions in parallel (k_vm_dense) when the units are big -- one thread per
		// unit would walk a 1 GiB window for minutes
		if (p.vm_reach > 1) return GSCAN_RESOLVE_WALK;
		const bool want = force == CHAIN_AUTO ? bytes / n_units >= (1u << 20) : force == CHAIN_ON;
		if (!want || bytes > kChainTableBytes || dense_blocks >= (1ull << 31)) return GSCAN_RESOLVE_WALK;
		return p.vm_reach == 1 ? GSCAN_RESOLVE_VM_DENSE_TWO : GSCAN_RESOLVE_VM_DENSE;
	}
	if (n_cand == 0) return GSCAN_RESOLVE_NONE;
	if (mode == GSCAN_MODE_ALL && !p.use_vm && (p.kind == ENGINE_RUN || p.disjoint)) return GSCAN_RESOLVE_FLAT;
	// the chain: FIXED patterns whose replay is sequential (overlapping matches, or LINE mode; RUN in LINE mode, where the search
	// resumes behind a line remainder, possibly inside a run), general patterns whose candidates come from a leading-sequence
	// filter and whose attempts depend on the search start at most through their first byte (reach <= 1), and the run starts
	// of a greedy / possessive leading class repeat -- with many candidates per unit
	uint32_t path = GSCAN_RESOLVE_WALK;
	if (!p.use_vm) {
		if ((p.kind == ENGINE_FIXED && (mode == GSCAN_MODE_ALL || mode == GSCAN_MODE_LINE)) || (p.kind == ENGINE_RUN && mode == GSCAN_MODE_LINE))
			path = GSCAN_RESOLVE_CHAIN;
	} else if (p.vm_runstart) {
		if (p.vm_reach == 0 && p.vm_lead != VM_Q_LAZY) path = GSCAN_RESOLVE_VM_RUN_CHAIN;
	} else if (p.vm_reach <= 1) {
		path = p.vm_reach == 1 ? GSCAN_RESOLVE_VM_TWO : GSCAN_RESOLVE_VM_ATTEMPTS;
	}
	if (path == GSCAN_RESOLVE_WALK) return path;
	const bool want = force == CHAIN_AUTO ? n_cand >= 65536 && n_cand / n_units >= 1024 : force == CHAIN_ON;
	return want && chain_geom(path, n_cand).fits ? path : GSCAN_RESOLVE_WALK;
}

} // namespace gscan
