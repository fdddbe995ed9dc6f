// resolve_kernels.cu -- turns the scan kernel's position-ordered segments into exactly the match
// sequence of the reference loop (/root/reference/src/grab.cc:175-213), entirely on the device:
//   1. exclusive prefix sum over the segment counts (three small kernels, no sort)
//   2. gather: candidates -> one array ordered by (unit, position)
//   3. select: per unit, replay the loop's control flow -- guard `start + minlen < end` (:175, quirk
//      Q1), leftmost candidate at or after `start` (:178), `start += ovector[1] + a` (:209), stop
//      after the first match in FIRST mode (:204-212), skip the rest of the line (<= 511 bytes) in
//      LINE mode (:194-196)
//   4. compact the kept records.
// Traffic: one occupancy bit per slice scanned, 8 bytes per non-empty slice for the segment table, plus O(candidates).
#include <cuda_runtime.h>
#include <cstdint>

#include "../../include/gscan.h"
#include "device_types.h"
#include "kernels.h"
#include "pattern.h"

namespace gscan {

constexpr int kScanBlock = 256;   // threads
constexpr int kPerThread = 8;     // items per thread
constexpr int kPerBlock = kScanBlock * kPerThread;

// block-wide exclusive scan of one value per thread; returns the block total via *total
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *total)
{
	__shared__ uint32_t warp_sums[kScanBlock / 32];
	__shared__ uint32_t block_total;
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t incl = v;
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
		if ((int)lane >= d) incl += t;
	}
	if (lane == 31) warp_sums[warp] = incl;
	__syncthreads();
	if (warp == 0) {
		uint32_t w = lane < kScanBlock / 32 ? warp_sums[lane] : 0u;
		uint32_t wi = w;
#pragma unroll
		for (int d = 1; d < 32; d <<= 1) {
			uint32_t t = __shfl_up_sync(0xffffffffu, wi, d);
			if ((int)lane >= d) wi += t;
		}
		if (lane < kScanBlock / 32) warp_sums[lane] = wi - w;
		if (lane == 31) block_total = wi;
	}
	__syncthreads();
	const uint32_t r = incl - v + warp_sums[warp];
	*total = block_total;
	__syncthreads();
	return r;
}

// a thread's kPerThread segments [base, base + 8) are 8 bits of one occupancy word: which of them the scan wrote.  Only
// those entries are read (a sparse pattern over 8 Mi segments reads 1 MiB of bits instead of 64 MiB of entries); a bit
// left over from an earlier scan is harmless, its entry's generation tag makes it count 0
static_assert(kPerThread == 8, "one byte of an occupancy word per thread");
__device__ __forceinline__ uint32_t occ_bits(const uint32_t *occ, uint32_t base, uint32_t n_segs)
{
	if (base >= n_segs) return 0u;
	uint32_t b = (occ[base >> 5] >> (base & 31u)) & 0xffu;
	if (n_segs - base < 8u) b &= (1u << (n_segs - base)) - 1u;
	return b;
}

// ---- 1. segment counts -> block sums ----
__global__ void k_seg_sums(const SegEntry *segs, const uint32_t *occ, uint32_t n_segs, uint32_t tag, uint32_t *blk)
{
	const uint32_t base = blockIdx.x * kPerBlock + threadIdx.x * kPerThread;
	const uint32_t bits = occ_bits(occ, base, n_segs);
	uint32_t s = 0;
#pragma unroll
	for (int i = 0; i < kPerThread; i++)
		if ((bits >> i) & 1u) s += seg_count(segs[base + i], tag);
	uint32_t total;
	block_exclusive_scan(s, &total);
	if (threadIdx.x == 0) blk[blockIdx.x] = total;
}

// single block: exclusive scan of blk[0..nb) in place, grand total to *total_out (and extra_out)
__global__ void k_scan_blk(uint32_t *blk, uint32_t nb, uint32_t *total_out, uint32_t *extra_out)
{
	__shared__ uint32_t carry;
	if (threadIdx.x == 0) carry = 0;
	__syncthreads();
	for (uint32_t base = 0; base < nb; base += kScanBlock) {
		const uint32_t i = base + threadIdx.x;
		const uint32_t v = i < nb ? blk[i] : 0u;
		uint32_t total;
		const uint32_t ex = block_exclusive_scan(v, &total);
		const uint32_t c = carry;
		if (i < nb) blk[i] = ex + c;
		__syncthreads();
		if (threadIdx.x == 0) carry = c + total;
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		*total_out = carry;
		if (extra_out) *extra_out = carry;
	}
}

// ---- 2. gather into (unit, pos) order ----
__global__ void k_gather(const ResolveArgs R)
{
	const uint32_t base = blockIdx.x * kPerBlock + threadIdx.x * kPerThread;
	const uint32_t bits = occ_bits(R.occ, base, R.n_segs);
	uint32_t cnt[kPerThread];
	uint32_t s = 0;
#pragma unroll
	for (int i = 0; i < kPerThread; i++) {
		cnt[i] = (bits >> i) & 1u ? seg_count(R.segs[base + i], R.tag) : 0u;
		s += cnt[i];
	}
	uint32_t total;
	uint32_t p = block_exclusive_scan(s, &total) + R.blk[blockIdx.x];
	// every thread of the block has read its occupancy byte (the scan above synchronises): clear the word for the next scan
	if ((base & 31u) == 0 && base < R.n_segs) R.occ[base >> 5] = 0u;
#pragma unroll
	for (int i = 0; i < kPerThread; i++) {
		const uint32_t seg = base + i;
		if (seg >= R.n_segs) break;
		const bool tile_start = (seg & ((1u << R.spt_shift) - 1u)) == 0;
		if (!tile_start && !cnt[i]) continue;
		const TileDesc td = R.tiles[seg >> R.spt_shift];
		if (tile_start && td.off == 0) R.unit_start[td.unit] = p; // first segment of a unit
		if (cnt[i]) {
			const Cand *src = R.cand + R.segs[seg].base;
			for (uint32_t k = 0; k < cnt[i]; k++) {
				OutRec o;
				o.unit = td.unit; o.pos = src[k].pos; o.len = src[k].len; o.pad = 0;
				R.ord[p + k] = o;
			}
			p += cnt[i];
		}
	}
}

// ---- device backtracking VM (general patterns) ----
// PCRE's matching strategy restated for one anchored attempt: alternatives in source order, greedy repeats take
// everything and give back one item at a time, lazy ones take one more on demand; explicit stack, no recursion.
// `subj` is the subject as the reference's pcre_exec call sees it: it begins at the moving search start
// (grab.cc:178), so ^, \A and \b at its first byte behave exactly as there.
constexpr int kVmStack = 2048; // entries of 12 bytes in thread-local memory (24 KiB per thread); the VM walk runs in its own low-occupancy kernel
// PCRE bounds the work of ONE pcre_exec call -- all start offsets of one search together (match limit, 10 million by
// default) -- and a unit additionally gets a total budget, so that a pathological pattern costs seconds, not hours, before
// the limit is reported (gscan_stats.vm_limit_hit; the unit stops there like the reference's loop on a pcre_exec error)
constexpr uint32_t kVmSearchSteps = 1u << 22;  // per search (from one search start to its match), plus 64 per byte of the unit
constexpr uint32_t kVmUnitSteps = 1u << 25;    // per unit and call, plus 128 per byte of the unit

__device__ __forceinline__ bool vm_in_set(const ResolveArgs &R, uint32_t set, uint32_t b) { return (R.vm_sets[set * 8 + (b >> 5)] >> (b & 31)) & 1u; }
__device__ __forceinline__ bool vm_is_word(uint32_t b) { return (b >= '0' && b <= '9') || (b >= 'A' && b <= 'Z') || (b >= 'a' && b <= 'z') || b == '_'; }

__device__ bool vm_assert(uint32_t kind, const uint8_t *s, uint32_t len, uint32_t sp)
{
	switch (kind) {
	case VM_A_BOL: case VM_A_SOS: return sp == 0;
	case VM_A_MBOL: return sp == 0 || s[sp - 1] == '\n';
	case VM_A_EOS: return sp == len;
	case VM_A_EOL: case VM_A_EOSNL: return sp == len || (sp + 1 == len && s[sp] == '\n');
	case VM_A_MEOL: return sp == len || s[sp] == '\n';
	default: {
		const bool before = sp > 0 && vm_is_word(s[sp - 1]);
		const bool after = sp < len && vm_is_word(s[sp]);
		return (before != after) == (kind == VM_A_WORDB);
	}
	}
}

// 1: match, *end set; 2: match in which a capturing group took part (VM_CAP on the successful path: pcre_exec with room
// for one offset pair returns 0 for it, quirk Q2); 0: no match at `at`; -1: stack / step limit
struct VmBudget {
	// both budgets grow with the unit (a linear scan of a big window must never trip them): + 64 steps per byte
	unsigned long long search, unit, per_search;
	// parallel attempts (k_vm_attempts): all attempts of a unit draw on ONE unit budget in device memory, a slice at a time,
	// and hand back what they did not use -- the work a pathological pattern can cause stays bounded per unit exactly as on
	// the serial walk, however many attempts run at once (signed arithmetic: an overdrawn counter stays negative)
	unsigned long long *shared;
	unsigned long long slice = 32;
	__device__ explicit VmBudget(unsigned long long ulen) : search(kVmSearchSteps + 64ull * ulen), unit(kVmUnitSteps + 128ull * ulen), per_search(kVmSearchSteps + 64ull * ulen), shared(nullptr) {}
	__device__ VmBudget(unsigned long long ulen, unsigned long long *unit_budget) : search(kVmSearchSteps + 64ull * ulen), unit(0), per_search(kVmSearchSteps + 64ull * ulen), shared(unit_budget) {}
	__device__ static unsigned long long unit_total(unsigned long long ulen) { return kVmUnitSteps + 128ull * ulen; }
	__device__ void new_search() { search = per_search; }
	__device__ bool refill()
	{
		if (!shared) return false;
		// slices grow with the attempt (32, 64, ... 512 steps): the attempts in flight -- tens of thousands of short ones on a
		// big unit -- must not hold the whole budget between them while each uses a few dozen steps of its slice (with 4096-step
		// slices 37 000 resident threads parked 155 M steps: every unit below 1 MiB "ran out" at once)
		const unsigned long long want = slice;
		if (slice < 512) slice <<= 1;
		const long long before = (long long)atomicAdd(shared, (unsigned long long)(-(long long)want));
		if (before <= 0) { atomicAdd(shared, want); return false; } // nothing left: undo, so that what others hand back counts
		unit = before < (long long)want ? (unsigned long long)before : want;
		if (before < (long long)want) atomicAdd(shared, want - unit); // took the rest only
		return true;
	}
	__device__ void give_back()
	{
		if (shared && unit) atomicAdd(shared, unit);
		unit = 0;
	}
};

__device__ int vm_exec(const ResolveArgs &R, const uint8_t *s, uint32_t len, uint32_t at, uint32_t *end, VmBudget &budget)
{
	// st_pc: pc | kind << 16 (0 plain, 1 give-back, 2 take-more) | capture flag at push time << 24
	uint32_t st_pc[kVmStack], st_sp[kVmStack], st_lo[kVmStack];
	int top = 0;
	uint32_t pc = 0, sp = at, cap = 0;
	for (;;) {
		if (budget.search == 0 || (budget.unit == 0 && !budget.refill())) return -1;
		budget.search--;
		budget.unit--;
		const uint32_t w0 = R.vm_code[3 * pc], a = R.vm_code[3 * pc + 1], b = R.vm_code[3 * pc + 2];
		const uint32_t op = w0 & 0xffu, kind = (w0 >> 8) & 0xffu, set = w0 >> 16;
		bool fail = false;
		switch (op) {
		case VM_MATCH: *end = sp; return cap ? 2 : 1;
		case VM_CAP: cap = 1u << 24; pc++; break;
		case VM_SET:
			if (sp < len && vm_in_set(R, set, s[sp])) { sp++; pc++; } else fail = true;
			break;
		case VM_ASSERT:
			if (vm_assert(kind, s, len, sp)) pc++; else fail = true;
			break;
		case VM_JMP: pc = a; break;
		case VM_LOOK: { // kind: VM_LK_*, a: pc behind the construct, b: bytes to step back (lookbehind)
			const bool behind = kind == VM_LK_BEHIND || kind == VM_LK_BEHIND_NEG;
			if (behind && sp < b) {
				// fewer bytes before sp than the branch needs (the subject begins at the moving search start): it cannot match
				if (kind == VM_LK_BEHIND) fail = true; else pc = a;
				break;
			}
			if (top == kVmStack) return -1;
			st_pc[top] = a | (3u << 16) | cap; st_sp[top] = sp; st_lo[top] = kind; top++;
			if (behind) sp -= b;
			pc++;
			break;
		}
		case VM_LOOKEND: {
			// the body matched: the choice points it left are dropped (an assertion / atomic group is never re-entered)
			int L = top;
			while (L > 0 && ((st_pc[L - 1] >> 16) & 0xffu) != 3u) L--;
			if (L == 0) return -1; // cannot happen: every LOOKEND has its frame
			const uint32_t fk = st_lo[L - 1], fsp = st_sp[L - 1], fcap = st_pc[L - 1] & (1u << 24);
			top = L - 1;
			if (fk == VM_LK_AHEAD_NEG || fk == VM_LK_BEHIND_NEG) { cap = fcap; fail = true; break; } // the negative assertion is false
			if (fk != VM_LK_ATOMIC) sp = fsp; // assertions consume nothing
			pc++;
			break;
		}
		case VM_SPLIT:
			if (top == kVmStack) return -1;
			st_pc[top] = b | cap; st_sp[top] = sp; st_lo[top] = 0; top++;
			pc = a;
			break;
		default: { // VM_REP: one byte class, a = min, b = max
			const uint32_t avail = len - sp, mx = b == 0xffffffffu ? avail : (b < avail ? b : avail);
			uint32_t k = 0;
			if (kind == VM_Q_LAZY) {
				while (k < a && k < avail && vm_in_set(R, set, s[sp + k])) k++;
				if (k < a) { fail = true; break; }
				if (b > a) { // may take more later: remember how many
					if (top == kVmStack) return -1;
					st_pc[top] = pc | (2u << 16) | cap; st_sp[top] = sp + k; st_lo[top] = b == 0xffffffffu ? 0xffffffffu : b - a; top++;
				}
				sp += k; pc++;
			} else {
				while (k < mx && vm_in_set(R, set, s[sp + k])) k++;
				if (k < a) { fail = true; break; }
				if (kind == VM_Q_GREEDY && k > a) {
					if (top == kVmStack) return -1;
					st_pc[top] = (pc + 1) | (1u << 16) | cap; st_sp[top] = sp + k; st_lo[top] = sp + a; top++;
				}
				sp += k; pc++;
			}
			break;
		}
		}
		if (!fail) continue;
		for (;;) { // backtrack
			if (top == 0) return 0;
			const uint32_t e = st_pc[top - 1], ek = (e >> 16) & 0xffu;
			cap = e & (1u << 24); // whatever closed after this choice point is undone
			if (ek == 0) { pc = e & 0xffffu; sp = st_sp[top - 1]; top--; break; }
			if (ek == 3) { // the body of an assertion / atomic group failed for good
				const uint32_t fk = st_lo[top - 1];
				const uint32_t back_to = st_sp[top - 1];
				top--;
				if (fk != VM_LK_AHEAD_NEG && fk != VM_LK_BEHIND_NEG) continue; // positive assertion / atomic group: the failure goes on
				pc = e & 0xffffu; sp = back_to;                                 // the negative assertion holds: go on behind it
				break;
			}
			if (ek == 1) { // greedy repeat gives one item back
				if (st_sp[top - 1] > st_lo[top - 1]) {
					sp = --st_sp[top - 1];
					pc = e & 0xffffu;
					if (st_sp[top - 1] == st_lo[top - 1]) top--;
					break;
				}
				top--;
				continue;
			}
			{ // lazy repeat takes one more item
				const uint32_t rpc = e & 0xffffu, rset = R.vm_code[3 * rpc] >> 16;
				if (st_lo[top - 1] > 0 && st_sp[top - 1] < len && vm_in_set(R, rset, s[st_sp[top - 1]])) {
					sp = ++st_sp[top - 1];
					if (st_lo[top - 1] != 0xffffffffu) st_lo[top - 1]--;
					pc = rpc + 1;
					if (st_lo[top - 1] == 0) top--;
					break;
				}
				top--;
			}
		}
	}
}

// ---- 3. per-unit replay of the reference loop ----
// Pass 1 (WRITE=false) counts the matches of every unit, pass 2 writes them at the unit's slot of
// the output (exclusive scan of the counts in between): the output can hold matches that are not
// candidates -- in LINE mode the RUN engine restarts up to 511 bytes after a match, possibly in
// the middle of a run, and PCRE then reports a match at that very byte.
__device__ __forceinline__ bool in_class(const ResolveArgs &R, uint32_t b) { return (R.bitmap[b >> 5] >> (b & 31)) & 1u; }

template <bool WRITE>
__global__ void k_walk(const ResolveArgs R)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= R.n_units) return;
	uint32_t i = R.unit_start[u];
	const uint32_t end = R.unit_start[u + 1];
	uint32_t n = 0;
	FinalRec *o = WRITE ? R.out + R.unit_out[u] : nullptr;
	if (i != end) {
		const DevUnit du = R.units[u];
		const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
		const uint64_t ulen = du.len;
		const bool run = R.engine == GSCAN_ENGINE_RUN;
		uint64_t start = 0;
		if (!WRITE && R.path == GSCAN_RESOLVE_FLAT) {
			// ALL mode, no two matches can overlap: every candidate is a match as long as the loop guard start + minlen < ulen
			// (grab.cc:175, Q1) holds.  Runs never touch each other (a non-class byte separates them), so for RUN it can only
			// bite before the first search; for FIXED it can also drop the LAST candidate (the one that exactly fills what the
			// previous match left).  Counted here in O(1); the write pass is k_write_flat, one thread per candidate.
			n = (R.minlen < ulen) ? end - i : 0u;
			if (!run && n >= 2u) {
				const OutRec prev = R.ord[end - 2];
				if (!((uint64_t)prev.pos + prev.len + R.minlen < ulen)) n--;
			}
		} else
		for (;;) {
			if (!(start + R.minlen < ulen)) break;                 // grab.cc:175 (strict '<': Q1)
			uint64_t pos = 0, e = 0;
			bool found = false;
			if (run && R.mode == GSCAN_MODE_LINE && start > 0 && in_class(R, data[start - 1]) && in_class(R, data[start])) {
				// `start` lies inside a run: the leftmost match, if the rest of the run is long enough, is AT start
				e = start;
				while (e < ulen && in_class(R, data[e])) e++;
				if (e - start >= R.run_min) { pos = start; found = true; }
			}
			if (!found) {
				while (i < end && R.ord[i].pos < start) i++;       // candidates swallowed by the previous match / skip
				if (i == end) break;
				pos = R.ord[i].pos;
				e = pos + R.ord[i].len;
				if (run) {                                         // greedy: extend to the end of the run
					e = pos + R.run_min;
					while (e < ulen && in_class(R, data[e])) e++;
				}
				i++;
			}
			if (WRITE) { FinalRec r; r.start = du.base_off + pos; r.file_id = du.file_id; r.len = (uint32_t)(e - pos); o[n] = r; }
			n++;
			if (R.mode == GSCAN_MODE_FIRST) break;                 // grab.cc:206 / :211
			if (R.mode == GSCAN_MODE_LINE) {                       // grab.cc:194-196: a = bytes to '\n', <= 511
				uint32_t a = 0;
				while (e + a < ulen && a < 511 && data[e + a] != '\n') a++;
				e += a;
			}
			start = e;                                             // grab.cc:209
		}
	}
	if (!WRITE) R.unit_out[u] = n;
}

// write pass of GSCAN_RESOLVE_FLAT: one thread per candidate
__global__ void k_write_flat(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.total_cand) return;
	const OutRec c = R.ord[i];
	const DevUnit du = R.units[c.unit];
	const uint64_t ulen = du.len;
	const uint32_t first = R.unit_start[c.unit], idx = i - first;
	if (!(R.minlen < ulen)) return;                                 // grab.cc:175 before the first search
	uint32_t len = c.len;
	if (R.engine == GSCAN_ENGINE_RUN) {                             // greedy: extend to the end of the run
		const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
		uint64_t e = (uint64_t)c.pos + R.run_min;
		while (e < ulen && in_class(R, data[e])) e++;
		len = (uint32_t)(e - c.pos);
	} else if (idx >= 1u && i + 1u == R.unit_start[c.unit + 1]) {    // the unit's last candidate: the guard after its predecessor (Q1)
		const OutRec prev = R.ord[i - 1];
		if (!((uint64_t)prev.pos + prev.len + R.minlen < ulen)) return;
	}
	FinalRec r;
	r.start = du.base_off + c.pos;
	r.file_id = du.file_id;
	r.len = len;
	R.out[R.unit_out[c.unit] + idx] = r;
}

// ---- chain paths: the per-unit replay as pointer doubling over all candidates (GSCAN_RESOLVE_CHAIN and the VM_* paths) ----
constexpr uint32_t kChainEnd = 0xffffffffu;
__host__ __device__ __forceinline__ uint32_t *chain_level(const ResolveArgs &R, uint32_t k) { return R.chain_buf + (size_t)k * R.chain_cap; }
__host__ __device__ __forceinline__ uint32_t *chain_mark(const ResolveArgs &R) { return R.chain_buf + (size_t)R.chain_levels * R.chain_cap; }
__host__ __device__ __forceinline__ uint32_t *chain_rank(const ResolveArgs &R) { return R.chain_buf + (size_t)(R.chain_levels + 1) * R.chain_cap; }
// VM_TWO / VM_DENSE_TWO: is-B flag of every node, then (in place) its exclusive scan; the B nodes' indices in order.
// VM_RUN_CHAIN: where each node's search resumes, and the outcome of the attempt there (k_vm_resume)
__host__ __device__ __forceinline__ uint32_t *chain_bscan(const ResolveArgs &R) { return R.chain_buf + (size_t)(R.chain_levels + 2) * R.chain_cap; }
__device__ __forceinline__ uint32_t *chain_blist(const ResolveArgs &R) { return R.chain_buf + (size_t)(R.chain_levels + 3) * R.chain_cap; }
__device__ __forceinline__ uint32_t *chain_stop(const ResolveArgs &R) { return chain_bscan(R); }
__device__ __forceinline__ uint32_t *chain_resume(const ResolveArgs &R) { return chain_blist(R); }

// two outcomes, chain view (totals[0]: nodes, totals[1]: B nodes): node j is a B node when the exclusive count steps behind it
__device__ __forceinline__ bool two_is_b(const ResolveArgs &R, uint32_t j)
{
	const uint32_t *bs = chain_bscan(R);
	return (j + 1 < R.totals[0] ? bs[j + 1] : R.totals[1]) != bs[j];
}
// two outcomes: where a search that resumes at `s` goes on -- lo: the unit's first node at or after s, uend: the unit's end.  Node
// (s, A) if A(s) matched; else the first B node behind s (B(s) itself is never taken: the subject began AT s)
__device__ __forceinline__ uint32_t two_next(const ResolveArgs &R, uint32_t lo, uint32_t uend, uint64_t s)
{
	if (lo < uend && R.ord[lo].pos == s && !two_is_b(R, lo)) return lo;
	while (lo < uend && R.ord[lo].pos == s) lo++; // at most the two nodes of s
	if (lo >= uend) return kChainEnd;
	const uint32_t j = chain_bscan(R)[lo];
	if (j >= R.totals[1]) return kChainEnd;
	const uint32_t b = chain_blist(R)[j];
	return b < uend ? b : kChainEnd;
}

// next(i): where the loop resumes behind match i (grab.cc:209; LINE mode: behind the line remainder, <= 511 bytes,
// grab.cc:194-196), the guard of the next iteration (grab.cc:175), then the first candidate of the unit at or after it
__global__ void k_chain_next(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	const OutRec c = R.ord[i];
	if (path_vm_chain(R.path) && c.pad >= 2u) { chain_level(R, 0)[i] = kChainEnd; return; } // this match ends its unit's loop (Q2 / VM limit)
	const DevUnit du = R.units[c.unit];
	const uint64_t ulen = du.len;
	const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
	const bool run = R.engine == GSCAN_ENGINE_RUN;
	uint64_t stop = (uint64_t)c.pos + c.len;
	if (run) { // greedy: the match reaches the end of the run, wherever inside the run it began (kept for the later passes)
		stop = (uint64_t)c.pos + R.run_min;
		while (stop < ulen && in_class(R, data[stop])) stop++;
		R.ord[i].len = (uint32_t)(stop - c.pos);
	}
	if (R.mode == GSCAN_MODE_LINE) {
		uint32_t a = 0;
		while (stop + a < ulen && a < 511 && data[stop + a] != '\n') a++;
		stop += a;
	}
	if (run) R.ord[i].pad = (uint32_t)stop; // where the search resumes behind this match (k_chain_entry)
	uint32_t nx = kChainEnd;
	if (path_run(R.path) && chain_resume(R)[i] == 2u) stop = ulen; // the attempt where the search resumes ran into the VM limit
	if (stop + R.minlen < ulen) {
		// RUN: the search may resume INSIDE a run (behind a line remainder); if what is left of that run is long enough the
		// leftmost match is at `stop` itself -- it ends where the run's own candidate ends, so the chain goes on from that
		// candidate and only the reported start differs (chain_entry).  VM_RUN_CHAIN: k_vm_resume ran the attempt there
		bool inside = false;
		if (run && stop > 0 && in_class(R, data[stop - 1]) && in_class(R, data[stop])) {
			uint64_t e = stop;
			while (e < ulen && in_class(R, data[e])) e++;
			inside = e - stop >= R.run_min;
		}
		if (path_run(R.path)) inside = chain_resume(R)[i] == 1u;
		const uint32_t uend = R.unit_start[c.unit + 1];
		uint32_t lo = i + 1, hi = uend; // candidates are ordered by position inside the unit
		while (lo < hi) {
			const uint32_t mid = lo + ((hi - lo) >> 1);
			if (R.ord[mid].pos < stop) lo = mid + 1; else hi = mid;
		}
		if (path_two(R.path)) nx = two_next(R, lo, uend, stop);
		else if (inside) nx = lo > i + 1 ? lo - 1 : kChainEnd; // the run that holds `stop`: the last one that starts before it (behind i's own run)
		else if (lo < uend) nx = lo;
	}
	chain_level(R, 0)[i] = nx;
}

// level k: jump 2^k matches ahead
__global__ void k_chain_double(const ResolveArgs R, uint32_t k)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	const uint32_t *prev = chain_level(R, k - 1);
	const uint32_t j = prev[i];
	chain_level(R, k)[i] = j == kChainEnd ? kChainEnd : prev[j];
}

// the first candidate of every unit starts its chain (the guard before the first search: grab.cc:175)
__global__ void k_chain_heads(const ResolveArgs R)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= R.n_units) return;
	const uint32_t first = R.unit_start[u], end = R.unit_start[u + 1];
	if (first == end || !(R.minlen < (uint64_t)R.units[u].len)) return;
	const uint32_t h = path_two(R.path) ? two_next(R, first, end, 0u) : first; // two outcomes: the first search begins at 0
	if (h != kChainEnd) chain_mark(R)[h] = 1u;
}

// descending levels: after level k every chain member whose distance from the head has no bit below k is marked.
// Marks set by other threads of the same pass are harmless (whatever a marked candidate jumps to is on the chain too).
__global__ void k_chain_spread(const ResolveArgs R, uint32_t k)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	if (!chain_mark(R)[i]) return;
	const uint32_t j = chain_level(R, k)[i];
	if (j != kChainEnd) chain_mark(R)[j] = 1u;
}

// RUN: where every chain member's match is reported -- at its run's first byte, or, when its predecessor's search resumed
// inside the run, there (level 1 of the jump tables is free once the marks are spread: it holds the entry positions)
__device__ __forceinline__ uint32_t *chain_entry(const ResolveArgs &R) { return chain_level(R, 1); }
__global__ void k_chain_entry_init(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	chain_entry(R)[i] = R.ord[i].pos;
}
__global__ void k_chain_entry(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	if (!chain_mark(R)[i]) return;
	const uint32_t nx = chain_level(R, 0)[i];
	if (nx == kChainEnd) return;
	const uint32_t stop = path_run(R.path) ? chain_stop(R)[i] : R.ord[i].pad;
	if (stop > R.ord[nx].pos) chain_entry(R)[nx] = stop; // one marked predecessor per chain member: no two writers
}

// VM_* paths: a candidate that ends its unit's loop (pad 2: a capturing group was set, pcre_exec returns 0; pad 3: VM limit,
// pcre_exec returns an error) is on the chain -- nothing behind it is -- but is not a reported match
__global__ void k_chain_unmark(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	if (R.ord[i].pad >= 2u) chain_mark(R)[i] = 0u;
}

// matches per unit from the exclusive scan of the marks (rank)
__global__ void k_chain_count(const ResolveArgs R)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= R.n_units) return;
	const uint32_t first = R.unit_start[u], end = R.unit_start[u + 1];
	uint32_t n = 0;
	if (first != end) n = chain_rank(R)[end - 1] + chain_mark(R)[end - 1] - chain_rank(R)[first];
	R.unit_out[u] = n;
}

__global__ void k_chain_write(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.total_cand) return;
	if (!chain_mark(R)[i]) return;
	const OutRec c = R.ord[i];
	const DevUnit du = R.units[c.unit];
	const uint32_t k = chain_rank(R)[i] - chain_rank(R)[R.unit_start[c.unit]];
	const uint32_t from = (R.engine == GSCAN_ENGINE_RUN || path_run(R.path)) ? chain_entry(R)[i] : c.pos;
	FinalRec r;
	r.start = du.base_off + from;
	r.file_id = du.file_id;
	r.len = c.pos + c.len - from;
	R.out[R.unit_out[c.unit] + k] = r;
}

// ---- general patterns on the chain paths (GSCAN_RESOLVE_VM_*) ----
// One anchored attempt per candidate, every candidate of the batch at once.  The subject of the attempt begins at the
// candidate itself: for a start-free program (no ^, \A, \b, \B, (?m)^, look-behind) the result is the one pcre_exec
// reaches from any search start at or before the candidate (grab.cc:178).
__global__ void __launch_bounds__(64, 4) k_vm_attempts(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	const OutRec c = R.ord[i];
	const DevUnit du = R.units[c.unit];
	const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
	VmBudget budget(du.len, R.vm_budget + c.unit);
	uint32_t e = 0;
	int rc = vm_exec(R, data + c.pos, du.len - c.pos, 0u, &e, budget);
	budget.give_back();
	if (rc < 0) { atomicOr(R.totals + 2, 1u); rc = 3; }
	R.ord[i].len = e;             // the subject began at the candidate: the end offset is the match length
	R.ord[i].pad = (uint32_t)rc;  // 0: no match here, 1: match, 2: match with a capturing group set (Q2), 3: VM limit
	if (!path_two(R.path)) { R.vm_flag[i] = rc != 0 ? 1u : 0u; return; }
	// VM_TWO: B(p), the subject begins one byte before the candidate -- what every earlier search start sees (reach 1)
	OutRec b;
	b.unit = c.unit; b.pos = c.pos; b.len = 0; b.pad = 0;
	if (c.pos >= 1u) {
		budget.new_search();
		uint32_t eb = 0;
		int rb = vm_exec(R, data + c.pos - 1u, du.len - c.pos + 1u, 1u, &eb, budget);
		budget.give_back();
		if (rb < 0) { atomicOr(R.totals + 2, 1u); rb = 3; }
		if (rb == 1 || rb == 2) b.len = eb - 1u;
		b.pad = (uint32_t)rb;
	}
	R.vm_ord_b[i] = b;
	R.vm_flag[2 * i] = rc != 0 ? 1u : 0u;
	R.vm_flag[2 * i + 1] = b.pad != 0 ? 1u : 0u;
}

// two outcomes / VM_RUN_CHAIN: the budget covers two attempts per position (A and B; a run start and a search resuming inside its
// run), twice what the serial walk gets -- it makes one attempt per position and search
__global__ void k_vm_budget_init(const ResolveArgs R)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= R.n_units) return;
	R.vm_budget[u] = VmBudget::unit_total(R.units[u].len) << ((path_two(R.path) || path_run(R.path)) ? 1 : 0);
}

// vm_flag holds its own exclusive scan by now: the candidates that matched, in order (VM_TWO: A then B of every candidate,
// and the node's kind into chain_bscan)
__global__ void k_vm_compact(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	const OutRec c = R.ord[i];
	if (!path_two(R.path)) {
		if (c.pad) R.vm_ord[R.vm_flag[i]] = c;
		return;
	}
	const OutRec b = R.vm_ord_b[i];
	if (c.pad) { R.vm_ord[R.vm_flag[2 * i]] = c; chain_bscan(R)[R.vm_flag[2 * i]] = 0u; }
	if (b.pad) { R.vm_ord[R.vm_flag[2 * i + 1]] = b; chain_bscan(R)[R.vm_flag[2 * i + 1]] = 1u; }
}

// first matching candidate of every unit (R.totals[4]: how many matched in all)
__global__ void k_vm_unit_starts(const ResolveArgs R)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u > R.n_units) return;
	const uint32_t s = R.unit_start[u];
	R.vm_unit_start[u] = s < R.totals[0] ? R.vm_flag[path_two(R.path) ? 2 * s : s] : R.totals[4];
}

// two outcomes, chain view, chain_bscan scanned: the index of every B node at its rank among them
__global__ void k_two_blist(const ResolveArgs R)
{
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= R.totals[0]) return;
	if (two_is_b(R, j)) chain_blist(R)[chain_bscan(R)[j]] = j;
}

// VM_RUN_CHAIN, chain view: where the search resumes behind node i, and -- when that lies inside a run of the leading class
// (the test of k_walk_vm) -- the attempt there: 1 match (it ends where the run start's own match ends: a greedy or possessive
// C{n,} from inside the run tries a subset of the run start's split points, in the same order), 0 none, 2 VM limit.  Own
// kernel: the VM's thread-local stack stays out of the chain kernels
__global__ void __launch_bounds__(64, 4) k_vm_resume(const ResolveArgs R)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R.totals[0]) return;
	const OutRec c = R.ord[i];
	const DevUnit du = R.units[c.unit];
	const uint64_t ulen = du.len;
	const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
	uint64_t stop = (uint64_t)c.pos + c.len;
	if (R.mode == GSCAN_MODE_LINE) {
		uint32_t a = 0;
		while (stop + a < ulen && a < 511 && data[stop + a] != '\n') a++;
		stop += a;
	}
	chain_stop(R)[i] = (uint32_t)stop;
	uint32_t res = 0;
	if (c.pad < 2u && stop + R.minlen < ulen && stop > 0 && in_class(R, data[stop - 1]) && in_class(R, data[stop])) {
		VmBudget budget(ulen, R.vm_budget + c.unit);
		uint32_t e = 0;
		const int rc = vm_exec(R, data + stop, (uint32_t)(ulen - stop), 0u, &e, budget);
		budget.give_back();
		if (rc < 0) { atomicOr(R.vm_limit, 1u); res = 2; }
		else res = rc != 0 ? 1u : 0u;
	}
	chain_resume(R)[i] = res;
}

// ---- dense general patterns on the chain path (GSCAN_RESOLVE_VM_DENSE*) ----
// No candidate list: every position whose byte can start a match gets its anchored attempt (what pcre_exec's own search
// loop does, grab.cc:178), 64 consecutive positions per thread, all blocks of the batch at once.  The count pass leaves the
// number of matching positions per block in vm_flag; after the exclusive scan the write pass replays the attempts and
// writes the matching positions in order -- the compacted list the chain kernels expect.  Both passes start from the same
// per-unit step budget; should the budget run out (nondeterministically, the attempts of a unit share it) the write pass
// never writes more than was counted and pads what is missing with chain-ending entries.
constexpr uint32_t kDenseShift = 6;
template <bool WRITE>
__global__ void __launch_bounds__(64, 4) k_vm_dense(const ResolveArgs R)
{
	const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= R.dense_blocks) return;
	const uint32_t bpt = R.dense_tile_shift - kDenseShift; // log2(blocks per tile)
	const TileDesc td = R.tiles[b >> bpt];
	const uint32_t lo = td.off + ((b & ((1u << bpt) - 1u)) << kDenseShift), tile_end = td.off + td.len;
	uint32_t n = 0;
	const uint32_t cnt = WRITE ? ((b + 1 < R.dense_blocks ? R.vm_flag[b + 1] : R.totals[4]) - R.vm_flag[b]) : 0u;
	OutRec *o = WRITE ? R.vm_ord + R.vm_flag[b] : nullptr;
	if (lo < tile_end && (!WRITE || cnt)) {
		const DevUnit du = R.units[td.unit];
		const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
		const uint32_t ulen = du.len;
		const uint32_t hi = lo + (1u << kDenseShift) < tile_end ? lo + (1u << kDenseShift) : tile_end;
		VmBudget budget(ulen, R.vm_budget + td.unit);
		// VM_DENSE_TWO: both outcomes of every position, A (subject begins at pos) before B (subject begins at pos - 1); the write
		// pass records each node's kind in chain_bscan
		const uint32_t kinds = path_two(R.path) ? 2u : 1u;
		for (uint32_t pos = lo; pos < hi && !(WRITE && n == cnt); pos++) {
			if ((uint64_t)pos + R.minlen > ulen) break;                                 // an attempt with fewer bytes left cannot succeed
			if (!in_class(R, data[pos])) continue;
			for (uint32_t k = 0; k < kinds; k++) {
				if (k == 1u && pos == 0u) break;
				uint32_t e = 0;
				int rc = vm_exec(R, data + pos - k, ulen - pos + k, k, &e, budget);
				budget.new_search();
				if (rc < 0) { atomicOr(R.totals + 2, 1u); rc = 3; }
				if (rc == 0) continue;
				if (WRITE) {
					if (n == cnt) break;
					OutRec r;
					r.unit = td.unit; r.pos = pos; r.len = rc == 3 ? 0u : e - k; r.pad = (uint32_t)rc;
					o[n] = r;
					if (path_two(R.path)) chain_bscan(R)[R.vm_flag[b] + n] = k;
				}
				n++;
			}
		}
		budget.give_back();
		if (WRITE) for (; n < cnt; n++) {
			OutRec r; r.unit = td.unit; r.pos = hi - 1u; r.len = 0; r.pad = 3u; o[n] = r;
			if (path_two(R.path)) chain_bscan(R)[R.vm_flag[b] + n] = 1u; // keeps the (pos, A before B) order
		}
	}
	if (!WRITE) R.vm_flag[b] = n;
}

// first matching position of every unit in vm_ord: the offset of the unit's first block
__global__ void k_vm_dense_unit_starts(const ResolveArgs R)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u > R.n_units) return;
	if (u == R.n_units) { R.vm_unit_start[u] = R.totals[4]; return; }
	const uint32_t blk0 = R.units[u].first_tile << (R.dense_tile_shift - kDenseShift);
	R.vm_unit_start[u] = blk0 < R.dense_blocks ? R.vm_flag[blk0] : R.totals[4];
}

// general patterns: every match starts at a candidate (a leading-byte prefix hit).  The count pass runs the VM
// and records the outcome in the candidate array, the write pass only copies.  Own kernel: the VM's backtrack
// stack is thread-local memory, so occupancy is capped to keep the reservation small.
template <bool WRITE>
__global__ void __launch_bounds__(64, 4) k_walk_vm(const ResolveArgs R)
{
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= R.n_units) return;
	uint32_t i = R.vm_dense ? 0u : R.unit_start[u];
	const uint32_t end = R.vm_dense ? 0u : R.unit_start[u + 1];
	uint32_t n = 0;
	FinalRec *o = WRITE ? R.out + R.unit_out[u] : nullptr;
	VmBudget budget(R.units[u].len); // the count and the write pass replay the same searches with the same budgets: same outcome
	if (R.vm_dense) {
		// no candidate list: PCRE's own search loop -- one anchored attempt per position whose byte can start a match, from
		// the moving search start; both passes replay it
		const DevUnit du = R.units[u];
		const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
		const uint64_t ulen = du.len;
		uint64_t start = 0;
		for (;;) {
			if (!(start + R.minlen < ulen)) break;                                      // grab.cc:175
			uint64_t pos = start;
			uint32_t e = 0;
			int rc = 0;
			for (; pos + R.minlen <= ulen; pos++) {                                     // (an attempt with fewer bytes left cannot succeed)
				if (!in_class(R, data[pos])) continue;
				rc = vm_exec(R, data + start, (uint32_t)(ulen - start), (uint32_t)(pos - start), &e, budget); // grab.cc:178
				if (rc != 0) break;
			}
			if (rc < 0) { atomicOr(R.totals + 2, 1u); break; }
			if (rc != 1) break;                                                         // no match, or Q2 (rc 2)
			uint64_t me = start + e;
			if (WRITE) { FinalRec r; r.start = du.base_off + pos; r.file_id = du.file_id; r.len = (uint32_t)(me - pos); o[n] = r; }
			n++;
			if (R.mode == GSCAN_MODE_FIRST) break;
			if (R.mode == GSCAN_MODE_LINE) {
				uint32_t a = 0;
				while (me + a < ulen && a < 511 && data[me + a] != '\n') a++;
				me += a;
			}
			start = me;                                                                 // grab.cc:209
			budget.new_search();
		}
	} else if (i != end && R.vm_runstart) {
		// candidates are run starts; a match may also begin at the search start when that lies inside a run, so the
		// outcome cannot be recorded in the candidate array: both passes replay the loop (the VM runs twice)
		const DevUnit du = R.units[u];
		const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
		const uint64_t ulen = du.len;
		uint64_t start = 0;
		for (;;) {
			if (!(start + R.minlen < ulen)) break;                                      // grab.cc:175
			uint64_t pos = 0;
			uint32_t e = 0;
			bool found = false;
			if (start > 0 && in_class(R, data[start - 1]) && in_class(R, data[start])) {
				const int rc = vm_exec(R, data + start, (uint32_t)(ulen - start), 0u, &e, budget);
				if (rc < 0) { atomicOr(R.totals + 2, 1u); break; }
				if (rc == 2) break;                                                     // Q2: pcre_exec returns 0, the loop leaves the window
				if (rc == 1) { pos = start; found = true; }
			}
			while (!found) {
				while (i < end && R.ord[i].pos < start) i++;
				if (i == end) break;
				pos = R.ord[i++].pos;
				const int rc = vm_exec(R, data + start, (uint32_t)(ulen - start), (uint32_t)(pos - start), &e, budget); // grab.cc:178
				if (rc < 0) { atomicOr(R.totals + 2, 1u); i = end; break; }
				if (rc == 2) { i = end; break; }                                        // Q2
				found = rc == 1;
			}
			if (!found) break;
			uint64_t me = start + e;
			if (WRITE) { FinalRec r; r.start = du.base_off + pos; r.file_id = du.file_id; r.len = (uint32_t)(me - pos); o[n] = r; }
			n++;
			if (R.mode == GSCAN_MODE_FIRST) break;
			if (R.mode == GSCAN_MODE_LINE) {
				uint32_t a = 0;
				while (me + a < ulen && a < 511 && data[me + a] != '\n') a++;
				me += a;
			}
			start = me;                                                                 // grab.cc:209
			budget.new_search();
		}
	} else 	if (i != end) {
		const DevUnit du = R.units[u];
		if (!WRITE) {
			const uint8_t *data = reinterpret_cast<const uint8_t *>(du.ptr);
			const uint64_t ulen = du.len;
			uint64_t start = 0;
			for (; i < end; i++) {
				if (!(start + R.minlen < ulen)) break;                                  // grab.cc:175
				const uint32_t pos = R.ord[i].pos;
				if (pos < start) continue;
				uint32_t e = 0;
				const int rc = vm_exec(R, data + start, (uint32_t)(ulen - start), (uint32_t)(pos - start), &e, budget); // grab.cc:178
				if (rc < 0) { atomicOr(R.totals + 2, 1u); break; }                      // limit: this unit stops here (pcre_exec error => break, grab.cc:179 / Q5)
				if (rc == 0) continue;                                                  // next start offset, like PCRE
				if (rc == 2) break;                                                     // Q2: a group was set => rc 0 => grab.cc:179 breaks
				uint64_t me = start + e;
				R.ord[i].len = (uint32_t)(me - pos);
				R.ord[i].pad = 1;
				n++;
				if (R.mode == GSCAN_MODE_FIRST) break;
				if (R.mode == GSCAN_MODE_LINE) {
					uint32_t a = 0;
					while (me + a < ulen && a < 511 && data[me + a] != '\n') a++;
					me += a;
				}
				start = me;                                                             // grab.cc:209
				budget.new_search();
			}
		} else {
			for (; i < end; i++)
				if (R.ord[i].pad) { FinalRec r; r.start = du.base_off + R.ord[i].pos; r.file_id = du.file_id; r.len = R.ord[i].len; o[n++] = r; }
		}
	}
	if (!WRITE) R.unit_out[u] = n;
}

// ---- the resolve launch sequence, written once over an executor X ----
// The device runs it through DeviceExec (launch_* below); the CPU model checks (tests/model_host.h) run the same
// sequence with every thread id in turn.  X provides
//   launch(kernel, threads, block, args...)  one thread per index in [0, threads), blocks of `block`
//   exclusive_scan(v, n, total_out)          in place; the sum of all n values into *total_out
//   fill_zero(p, n), copy(dst, src, n)       u32 words
// what the chain kernels see: the candidate list itself, or (VM_* paths) the compacted list of the outcomes that matched with
// its own count (totals[4]) and rank-total scratch (totals[7])
inline ResolveArgs chain_view(const ResolveArgs &R)
{
	ResolveArgs C = R;
	if (path_vm_chain(R.path)) { C.ord = R.vm_ord; C.unit_start = R.vm_unit_start; C.totals = R.totals + 4; }
	return C;
}

// count pass, behind the gather (VM_DENSE*: behind vm_dense_write): per-unit match counts into unit_out, their exclusive
// scan (the output slots), totals[1] = number of matches
template <class X>
void resolve_count_seq(X &x, const ResolveArgs &R)
{
	if (path_chain(R.path)) {
		// grids cover the reserved node slots; the kernels stop at the exact count (totals[0], on the device by now)
		const uint32_t cap = R.chain_cap;
		if (path_attempts(R.path)) {
			x.fill_zero(R.vm_flag, cap); // VM_TWO: cap is two slots per candidate
			if (path_two(R.path)) x.fill_zero(chain_bscan(R), cap);
			x.launch(k_vm_budget_init, R.n_units, 256, R);
			x.launch(k_vm_attempts, cap, 64, R);
			x.exclusive_scan(R.vm_flag, cap, R.totals + 4);
			x.launch(k_vm_compact, cap, 256, R);
			x.launch(k_vm_unit_starts, R.n_units + 1, 256, R);
		}
		const ResolveArgs C = chain_view(R);
		if (path_two(R.path)) { // which nodes are B: exclusive count (total: totals[5]) and the list of their indices
			x.exclusive_scan(chain_bscan(C), cap, R.totals + 5);
			x.launch(k_two_blist, cap, 256, C);
		}
		const bool follow = R.mode != GSCAN_MODE_FIRST; // FIRST: the head of every unit's chain is all there is
		x.fill_zero(chain_mark(C), cap);                // (the ranks are a copy of the marks, below)
		if (follow) {
			if (path_run(R.path)) x.launch(k_vm_resume, cap, 64, C);
			x.launch(k_chain_next, cap, 256, C);
			for (uint32_t k = 1; k < C.chain_levels; k++) x.launch(k_chain_double, cap, 256, C, k);
		}
		x.launch(k_chain_heads, R.n_units, 256, C);
		if (follow) for (uint32_t k = C.chain_levels; k-- > 0;) x.launch(k_chain_spread, cap, 256, C, k);
		if (path_vm_chain(R.path)) x.launch(k_chain_unmark, cap, 256, C);
		if (R.engine == GSCAN_ENGINE_RUN || path_run(R.path)) {
			x.launch(k_chain_entry_init, cap, 256, C);
			if (follow) x.launch(k_chain_entry, cap, 256, C);
		}
		x.copy(chain_rank(C), chain_mark(C), cap);
		x.exclusive_scan(chain_rank(C), cap, C.totals + 3);
		x.launch(k_chain_count, R.n_units, 256, C);
	} else if (R.engine == GSCAN_ENGINE_VM) {
		x.launch(k_walk_vm<false>, R.n_units, 64, R);
	} else {
		x.launch(k_walk<false>, R.n_units, 128, R);
	}
	x.exclusive_scan(R.unit_out, R.n_units, R.totals + 1);
}

// VM_DENSE*: the matching positions per 64-position block into vm_flag, exclusive scan, total into totals[4]
template <class X>
void vm_dense_count_seq(X &x, const ResolveArgs &R)
{
	x.launch(k_vm_budget_init, R.n_units, 256, R);
	x.launch(k_vm_dense<false>, R.dense_blocks, 64, R);
	x.exclusive_scan(R.vm_flag, R.dense_blocks, R.totals + 4);
}

// VM_DENSE*, once vm_ord and the chain tables are sized: the node list and vm_unit_start
template <class X>
void vm_dense_write_seq(X &x, const ResolveArgs &R)
{
	x.launch(k_vm_budget_init, R.n_units, 256, R);
	x.launch(k_vm_dense<true>, R.dense_blocks, 64, R);
	x.launch(k_vm_dense_unit_starts, R.n_units + 1, 256, R);
}

// write pass: the records into R.out, at the slots of the count pass
template <class X>
void resolve_write_seq(X &x, const ResolveArgs &R)
{
	if (path_chain(R.path)) {
		ResolveArgs C = chain_view(R);
		if (path_two(R.path)) C.total_cand = R.chain_cap; // two node slots per candidate; the slots behind the nodes are unmarked
		x.launch(k_chain_write, C.total_cand, 256, C);
	} else if (R.path == GSCAN_RESOLVE_FLAT) {
		x.launch(k_write_flat, R.total_cand, 256, R);
	} else if (R.engine == GSCAN_ENGINE_VM) {
		x.launch(k_walk_vm<true>, R.n_units, 64, R);
	} else {
		x.launch(k_walk<true>, R.n_units, 128, R);
	}
}

// ---- 4. generic u32 block sums / exclusive scan (per-unit match counts -> output slots) ----
__global__ void k_u32_sums(const uint32_t *v, uint32_t n, uint32_t *blk)
{
	const uint32_t base = blockIdx.x * kPerBlock + threadIdx.x * kPerThread;
	uint32_t s = 0;
#pragma unroll
	for (int i = 0; i < kPerThread; i++)
		if (base + i < n) s += v[base + i];
	uint32_t total;
	block_exclusive_scan(s, &total);
	if (threadIdx.x == 0) blk[blockIdx.x] = total;
}

__global__ void k_u32_exclusive(uint32_t *v, uint32_t n, const uint32_t *blk)
{
	const uint32_t base = blockIdx.x * kPerBlock + threadIdx.x * kPerThread;
	uint32_t x[kPerThread];
	uint32_t s = 0;
#pragma unroll
	for (int i = 0; i < kPerThread; i++) { x[i] = base + i < n ? v[base + i] : 0u; s += x[i]; }
	uint32_t total;
	uint32_t p = block_exclusive_scan(s, &total) + blk[blockIdx.x];
#pragma unroll
	for (int i = 0; i < kPerThread; i++)
		if (base + i < n) { v[base + i] = p; p += x[i]; }
}

__global__ void k_fill_zero(uint32_t *p, uint32_t n)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) p[i] = 0u;
	if (i + gridDim.x * blockDim.x < n) p[i + gridDim.x * blockDim.x] = 0u;
}
// the executor of the launch sequence on the device: the grids cover `threads` in blocks of `block`; every scan is
// k_u32_sums -> k_scan_blk -> k_u32_exclusive with its block sums in R.blk from offset 0 (the stream orders the scans)
struct DeviceExec {
	cudaStream_t st;
	uint32_t *blk;
	uint32_t launches = 0;
	cudaError_t err = cudaSuccess;
	template <class... P, class... A>
	void launch(void (*kernel)(P...), uint32_t threads, uint32_t block, A... args)
	{
		kernel<<<(threads + block - 1) / block, block, 0, st>>>(args...);
		launches++;
	}
	void exclusive_scan(uint32_t *v, uint32_t n, uint32_t *total_out)
	{
		const uint32_t nb = (n + kPerBlock - 1) / kPerBlock;
		k_u32_sums<<<nb, kScanBlock, 0, st>>>(v, n, blk);
		k_scan_blk<<<1, kScanBlock, 0, st>>>(blk, nb, total_out, nullptr);
		k_u32_exclusive<<<nb, kScanBlock, 0, st>>>(v, n, blk);
		launches += 3;
	}
	void fill_zero(uint32_t *p, uint32_t n)
	{
		k_fill_zero<<<(n + 255) / 256, 256, 0, st>>>(p, n);
		launches++;
	}
	void copy(uint32_t *dst, const uint32_t *src, uint32_t n)
	{
		const cudaError_t e = cudaMemcpyAsync(dst, src, (size_t)n * 4, cudaMemcpyDeviceToDevice, st);
		if (err == cudaSuccess) err = e;
	}
	cudaError_t finish(uint32_t *n_launches)
	{
		if (n_launches) *n_launches = launches;
		const cudaError_t e = cudaGetLastError();
		return err != cudaSuccess ? err : e;
	}
};

cudaError_t launch_resolve_count(const ResolveArgs &R, cudaStream_t st, uint32_t *launches)
{
	DeviceExec x{st, R.blk};
	if (!R.vm_dense) { // segment prefix sum and gather; k_gather reads the segment scan's block sums
		const uint32_t nb_seg = (R.n_segs + kPerBlock - 1) / kPerBlock;
		k_seg_sums<<<nb_seg, kScanBlock, 0, st>>>(R.segs, R.occ, R.n_segs, R.tag, R.blk);
		k_scan_blk<<<1, kScanBlock, 0, st>>>(R.blk, nb_seg, R.totals, R.unit_start + R.n_units);
		k_gather<<<nb_seg, kScanBlock, 0, st>>>(R);
		x.launches += 3;
	}
	resolve_count_seq(x, R);
	return x.finish(launches);
}

cudaError_t launch_vm_dense_count(const ResolveArgs &R, cudaStream_t st, uint32_t *launches)
{
	DeviceExec x{st, R.blk};
	vm_dense_count_seq(x, R);
	return x.finish(launches);
}

cudaError_t launch_vm_dense_write(const ResolveArgs &R, cudaStream_t st, uint32_t *launches)
{
	DeviceExec x{st, R.blk};
	vm_dense_write_seq(x, R);
	return x.finish(launches);
}

cudaError_t launch_resolve_write(const ResolveArgs &R, cudaStream_t st, uint32_t *launches)
{
	DeviceExec x{st, R.blk};
	resolve_write_seq(x, R);
	return x.finish(launches);
}

} // namespace gscan
