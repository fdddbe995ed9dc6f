// model_host.h -- the resolve paths of resolve_kernels.cu on the CPU, for the model checks (model_check.cc,
// model_check_start.cc).  The test extracts the device source between the "device backtracking VM" and "4. generic u32 block
// sums" markers -- the VM, the resolve kernels and the launch sequence that runs them -- into vm_snippet.inc; it is compiled
// here with CUDA's qualifiers removed, the thread index a global that the host executor sets to each thread id in turn.
#pragma once
#include <algorithm>
#include <cstring>
#include <functional>
#include <vector>

#include "../include/gscan.h"
#include "../grab_b200/csrc/pattern.h"
#include "../grab_b200/csrc/kernels.h" // ResolveArgs, DevUnit, FinalRec, OutRec, TileDesc (host-includable: PODs + launcher prototypes)
#include "../grab_b200/csrc/resolve_plan.h"

#undef __host__
#undef __device__
#undef __global__
#undef __forceinline__
#undef __launch_bounds__
#define __host__
#define __device__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(...)
namespace gscan {
struct ModelIdx { uint32_t x; };
static ModelIdx model_blockIdx{0}, model_blockDim{1}, model_threadIdx{0};
#define blockIdx model_blockIdx
#define blockDim model_blockDim
#define threadIdx model_threadIdx
static inline uint32_t atomicOr(uint32_t *p, uint32_t v) { const uint32_t o = *p; *p |= v; return o; }
static inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { const unsigned long long o = *p; *p += v; return o; }
#include "vm_snippet.inc"
#undef blockIdx
#undef blockDim
#undef threadIdx
} // namespace gscan

using namespace gscan;

struct M { uint64_t pos; uint32_t len; };
typedef std::vector<uint8_t> Bytes;

static bool seq_at(const Sequence &q, const uint8_t *s, size_t len, size_t pos)
{
	if (pos + q.size() > len) return false;
	for (size_t i = 0; i < q.size(); i++) if (!q[i].has(s[pos + i])) return false;
	return true;
}

// What the scan kernels deliver for one unit, by contract (scan_kernels.cu): FIXED -- every position where an alternative
// (for general patterns: a leading-byte prefix) lies entirely inside the unit, with the length of the first one in preference
// order; RUN (and general patterns that begin with a class repeat) -- the first byte of every maximal class run of at least
// run_min bytes.  Position order.
static void candidates(const Program &p, const Bytes &b, uint32_t unit, std::vector<OutRec> &ord)
{
	const bool runs = p.kind == ENGINE_RUN || (p.use_vm && p.vm_runstart);
	for (size_t pos = 0; pos < b.size(); pos++) {
		if (runs) {
			if (!p.run_class.has(b[pos]) || (pos > 0 && p.run_class.has(b[pos - 1]))) continue;
			size_t k = 0;
			while (pos + k < b.size() && p.run_class.has(b[pos + k])) k++;
			if (k >= (size_t)p.run_min) ord.push_back(OutRec{unit, (uint32_t)pos, 0, 0});
		} else {
			for (auto &q : p.seqs)
				if (seq_at(q, b.data(), b.size(), pos)) { ord.push_back(OutRec{unit, (uint32_t)pos, (uint32_t)q.size(), 0}); break; }
		}
	}
}

static void exclusive(uint32_t *v, size_t n, uint32_t *total)
{
	uint32_t acc = 0;
	for (size_t i = 0; i < n; i++) { const uint32_t f = v[i]; v[i] = acc; acc += f; }
	if (total) *total = acc;
}

// the launch sequence's executor on the host: every kernel runs its thread ids 0 .. threads-1 one after another; the scans
// are plain prefix sums.  after_budget_init runs behind every k_vm_budget_init launch.
struct HostExec {
	std::function<void(const ResolveArgs &)> after_budget_init;
	template <class... P, class... A>
	void launch(void (*kernel)(P...), uint32_t threads, uint32_t, const ResolveArgs &R, A... more)
	{
		for (uint32_t t = 0; t < threads; t++) { model_threadIdx.x = t; kernel(R, more...); }
		model_threadIdx.x = 0;
		if (after_budget_init && (void *)kernel == (void *)&k_vm_budget_init) after_budget_init(R);
	}
	void exclusive_scan(uint32_t *v, uint32_t n, uint32_t *total_out) { exclusive(v, n, total_out); }
	void fill_zero(uint32_t *p, uint32_t n) { std::fill(p, p + n, 0u); }
	void copy(uint32_t *dst, const uint32_t *src, uint32_t n) { std::copy(src, src + n, dst); }
};

// One batch of subjects and the device memory of a resolve over it.  Unit u: base offset 1000 u, file id 7 + u; tiles of
// 256 bytes (the device's are 4 .. 64 KiB; the block -> tile -> unit arithmetic is the same), the last one of a unit partly
// filled.
struct ModelBatch {
	static constexpr uint32_t kTileShift = 8;
	std::vector<DevUnit> du;
	std::vector<TileDesc> tiles;
	std::vector<OutRec> cand;          // candidates by contract, (unit, pos) order (none for dense programs)
	std::vector<uint32_t> cand_start;  // [units + 1]
	uint64_t bytes = 0;
	// what a resolve leaves on the "device"
	std::vector<OutRec> ord, ord_b, vm_ord;
	std::vector<uint32_t> unit_start, unit_out, vm_unit_start, flag, chain;
	std::vector<unsigned long long> budget;
	uint32_t totals[10];

	ModelBatch(const Program &p, const std::vector<const Bytes *> &subj) : du(subj.size()), cand_start(1, 0u)
	{
		for (uint32_t u = 0; u < du.size(); u++) {
			const Bytes &b = *subj[u];
			memset(&du[u], 0, sizeof du[u]);
			du[u].ptr = (uint64_t)(uintptr_t)b.data();
			du[u].len = (uint32_t)b.size();
			du[u].base_off = 1000u * u;
			du[u].file_id = 7 + u;
			du[u].first_tile = (uint32_t)tiles.size();
			for (size_t off = 0; off < b.size(); off += (size_t)1 << kTileShift) {
				TileDesc t;
				memset(&t, 0, sizeof t);
				t.src = du[u].ptr + off; t.unit = u; t.off = (uint32_t)off;
				t.len = (uint32_t)std::min<size_t>((size_t)1 << kTileShift, b.size() - off); t.ulen = (uint32_t)b.size();
				tiles.push_back(t);
			}
			if (!(p.use_vm && p.vm_dense)) candidates(p, b, u, cand);
			cand_start.push_back((uint32_t)cand.size());
			bytes += b.size();
		}
	}
	uint64_t dense_blocks() const { return (uint64_t)tiles.size() << (kTileShift - 6); }
	uint32_t plan(const Program &p, uint32_t mode, ChainOverride force) const
	{
		return plan_resolve(p, mode, du.size(), bytes, dense_blocks(), cand.size(), force);
	}

	// gscan_batch_scan's set-up of a resolve: fresh device state, the candidates gathered (totals[0]), the buffers of `path`
	// except the node list and tables of VM_DENSE*, which wait for the count of k_vm_dense
	ResolveArgs args(const Program &p, uint32_t mode, uint32_t path)
	{
		const uint32_t nu = (uint32_t)du.size(), nc = (uint32_t)cand.size();
		ord = cand;
		unit_start = cand_start;
		unit_out.assign(nu + 1, 0u);
		vm_unit_start.assign(nu + 1, 0u);
		budget.assign(nu, 0ull);
		memset(totals, 0, sizeof totals);
		totals[0] = nc;
		ResolveArgs R;
		memset(&R, 0, sizeof R);
		R.tiles = tiles.data();
		R.units = du.data(); R.n_units = nu;
		R.ord = ord.data(); R.unit_start = unit_start.data(); R.unit_out = unit_out.data(); R.totals = totals;
		R.path = path;
		R.mode = mode; R.minlen = (uint32_t)p.minlen; R.engine = p.use_vm ? (uint32_t)GSCAN_ENGINE_VM : (uint32_t)p.kind;
		R.run_min = (uint32_t)p.run_min;
		for (int i = 0; i < 8; i++) R.bitmap[i] = (p.use_vm && p.vm_dense) ? p.first_set.w[i] : p.run_class.w[i];
		R.total_cand = nc;
		R.vm_code = p.vm_code.data(); R.vm_sets = p.vm_sets.data();
		R.vm_runstart = p.vm_runstart ? 1u : 0u;
		R.vm_dense = (p.use_vm && p.vm_dense) ? 1u : 0u;
		R.vm_limit = totals + 2;
		R.vm_budget = budget.data(); R.vm_unit_start = vm_unit_start.data();
		R.dense_tile_shift = kTileShift;
		if (path_compacted(path)) {
			flag.assign(dense_blocks() + 1, 0u);
			R.vm_flag = flag.data(); R.dense_blocks = (uint32_t)dense_blocks();
		} else if (path_chain(path)) {
			const ChainGeom g = chain_geom(path, nc);
			chain.assign((size_t)g.arrays * g.nodes, 0u);
			R.chain_levels = g.levels; R.chain_cap = (uint32_t)g.nodes; R.chain_buf = chain.data();
			vm_ord.assign(g.nodes, OutRec{0, 0, 0, 0}); flag.assign(g.nodes, 0u); ord_b.assign(nc, OutRec{0, 0, 0, 0});
			R.vm_ord = vm_ord.data(); R.vm_flag = flag.data(); R.vm_ord_b = ord_b.data();
		}
		return R;
	}

	// the resolve as gscan_batch_scan runs it, through the shipped launch sequence: out[u] = the matches of unit u.
	// 0 ok, -1 VM limit, -2 a record in another unit's slots
	int run(const Program &p, uint32_t mode, uint32_t path, HostExec &x, std::vector<std::vector<M>> &out)
	{
		out.assign(du.size(), std::vector<M>());
		if (path == GSCAN_RESOLVE_NONE) return 0;
		ResolveArgs R = args(p, mode, path);
		if (path_compacted(path)) {
			vm_dense_count_seq(x, R);
			if (totals[2]) return -1;
			const uint32_t hits = totals[4];
			if (hits == 0) return 0; // nothing to resolve: no count pass
			const ChainGeom g = chain_geom(path, hits);
			if (!g.fits) return -1;
			vm_ord.assign(hits, OutRec{0, 0, 0, 0});
			chain.assign((size_t)g.arrays * hits, 0u);
			R.vm_ord = vm_ord.data();
			R.chain_levels = g.levels; R.chain_cap = hits; R.chain_buf = chain.data();
			vm_dense_write_seq(x, R);
			R.total_cand = hits;
		}
		resolve_count_seq(x, R);
		if (totals[2]) return -1;
		const uint32_t n = totals[1];
		std::vector<FinalRec> fin(n + 1);
		R.out = fin.data();
		resolve_write_seq(x, R);
		if (totals[2]) return -1;
		for (uint32_t u = 0; u < du.size(); u++)
			for (uint32_t k = unit_out[u]; k < (u + 1 < du.size() ? unit_out[u + 1] : n); k++) {
				if (fin[k].file_id != du[u].file_id) return -2;
				out[u].push_back(M{fin[k].start - du[u].base_off, fin[k].len});
			}
		return 0;
	}
};
