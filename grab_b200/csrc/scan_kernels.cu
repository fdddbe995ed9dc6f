// scan_kernels.cu -- the hot path: hand-written sm_90a kernels that replace the match loop of
// /root/reference/src/grab.cc:175-213 (one pcre_exec per match) with one persistent streaming
// pass over every byte of a batch of scan units.
//
// Structure (one CTA per SM, persistent, every warp an independent scanner):
//   each warp owns a ring of Geom::kRing shared-memory slots.  Lane 0 issues one 1-D TMA bulk copy
//   (cp.async.bulk, SASS UBLKCP) per slice (Geom::kSlice bytes, 512-byte aligned on both sides) plus,
//   where the engine needs them, two 16-byte copies of the bytes right before / after the slice, all
//   completing on the slot's mbarrier (complete_tx::bytes); the warp waits on the barrier, reads the
//   slice with conflict-free 16-byte LDS (lane l <- bytes [16l,16l+16) of a 512-byte row), runs the
//   engine's SWAR filter (4 bytes per 32-bit op) and, on the rare flagged row, verifies; then lane 0
//   re-arms the slot for the slice kRing steps ahead.  No producer warp, no __syncthreads in the loop.
//   Engines: FixedEngine (byte-pair filter), Fixed3Engine (byte-triple filter), HashEngine (perfect-hash
//   membership of the leading bytes, large alternations), RunEngine (byte-class runs), NullEngine (probe).
// Output order: each warp appends its candidates in position order to a private scratch list and,
// at the end of its slice, reserves a contiguous range of the global candidate buffer with one
// atomicAdd and records (base, n | generation tag) in the segment table.  Segment ids are position
// ordered, so the resolve pass needs no sort.
// Code size: every instantiation stays under 32 KB of SASS (out-of-line single-copy slow paths), so the
// rarely executed verification code is still in the SM's instruction cache when a match finally shows up.
//
// HBM traffic: every byte once; 8 bytes of segment table and one occupancy bit per NON-EMPTY slice; candidates
// only where they exist.
#include <cuda_runtime.h>
#include <atomic>
#include <cstdint>
#include <cstdlib>

#include "device_types.h"
#include "swar.h"
#include "kernels.h"

namespace gscan {

// ------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier + TMA bulk copy
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
	asm volatile(
	    "{\n"
	    ".reg .pred p;\n"
	    "WAIT_%=:\n"
	    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
	    "@p bra DONE_%=;\n"
	    "bra WAIT_%=;\n"
	    "DONE_%=:\n"
	    "}\n" ::"r"(smem_u32(bar)),
	    "r"(parity)
	    : "memory");
}
// one LOP3 with the given truth table (a = 0xF0, b = 0xCC, c = 0xAA)
template <int LUT>
__device__ __forceinline__ uint32_t lop3(uint32_t a, uint32_t b, uint32_t c)
{
	uint32_t d;
	asm("lop3.b32 %0, %1, %2, %3, %4;" : "=r"(d) : "r"(a), "r"(b), "r"(c), "n"(LUT));
	return d;
}
// L2 eviction policy for the corpus stream: every byte is read exactly once, so its lines are the first to go.
// Without it the stream (the whole 50 MB L2 turns over every ~15 us) evicts the rarely executed slow-path code and
// the pattern tables from L2, and a warp that finally hits a match fetches its instructions from DRAM one line at a
// time.  On an H100 (80GB HBM3, 400 W limit) evict_first also lifts the literal scan kernel from 2.87 to 2.95 TB/s and
// the null-consumer ring from 2.95 to 2.98 TB/s against evict_normal (tools/step_budget.py, DESIGN.md section 6).
__device__ __forceinline__ uint64_t l2_stream_policy()
{
	uint64_t p;
	asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
	return p;
}
// global -> shared bulk copy executed by the TMA unit; bytes and both addresses multiples of 16
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar, uint64_t policy)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
	                 smem_u32(smem_dst)),
	             "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
	             : "memory");
}

// ------------------------------------------------------------------------------------------
// shared-memory layout: every warp owns kRing slots of 16 + kSlice + 16 bytes, one mbarrier and one slice
// descriptor per slot.  The slice itself arrives as ONE bulk copy that is 512-byte aligned on both sides;
// the 16 bytes after it (shifted filter stream, run look-ahead) and, for the RUN engine, the 16 bytes
// before it (is the previous byte in the class?) arrive as separate 16-byte bulk copies on the same
// mbarrier.  Whatever else a verification touches is read from global memory (L2).  Nothing is shared
// between warps.
constexpr uint32_t kHalo = 16;
// ------------------------------------------------------------------------------------------
struct __align__(16) SlotCtl {
	uint64_t full;
	uint64_t src; // global address of tile byte 0
	uint32_t off, ulen, tile_len, begin, niter;
	uint32_t slice; // the slice in the slot; kNoSlice: none, the warp is done once it reaches this slot
};
constexpr uint32_t kNoSlice = 0xffffffffu;

// a slot: [16 bytes before the slice, engines with a look-behind only] slice [16 bytes after it]
size_t scan_smem_bytes(const ScanGeom &g, bool look_behind)
{
	return (size_t)g.warps * g.ring * ((size_t)g.slice + (look_behind ? 2 : 1) * kHalo + sizeof(SlotCtl)) + 64;
}

// what a warp knows about the slice it is scanning
struct Slice {
	const uint8_t *tile;  // shared-memory address of the tile's byte 0 (only the slice itself is resident)
	const uint8_t *gtile; // global address of the tile's byte 0 (neighbouring bytes, verification)
	const uint8_t *extra; // engine-private shared memory (hash table)
	uint32_t off;        // offset of the tile in its unit
	uint32_t ulen;       // unit length
	uint32_t tile_len;
	uint32_t begin, niter; // slice = [begin, begin + niter*512) in tile coordinates
};

struct Emitter {
	Cand *scratch; // this warp's private list (global memory, L2 resident)
	uint32_t n;    // warp-uniform

	// mm: per-lane 16-bit mask of matched bytes of the lane's chunk; lens via callback.
	// Appends in (lane, bit) order == position order at dst; returns how many the warp wrote.
	template <class LenFn>
	static __device__ __forceinline__ uint32_t emit_at(Cand *dst, uint32_t mm, uint32_t pos0, LenFn len_of, uint32_t lane)
	{
		uint32_t cnt = __popc(mm), incl = cnt;
#pragma unroll
		for (int d = 1; d < 32; d <<= 1) {
			uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
			if ((int)lane >= d) incl += v;
		}
		uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
		uint32_t idx = incl - cnt;
		while (mm) {
			uint32_t b = __ffs(mm) - 1;
			mm &= mm - 1;
			Cand c;
			c.pos = pos0 + b;
			c.len = len_of(b);
			dst[idx++] = c;
		}
		return total;
	}

	// Space in the global candidate buffer is reserved a CHUNK at a time (one atomicAdd per A.chunk candidates, not one
	// per slice): with one reservation per slice the warp sat on the atomic's round trip in four slices out of five of a
	// dense pattern -- 35 % of all stall samples of the RUN kernel (profiles/r02_run16_v1_ncu.txt).  What a warp leaves
	// unused of its last chunk is wasted (the host sizes for it); candidates of one slice stay contiguous.
	uint32_t chunk_base = 0, chunk_left = 0;
	uint32_t aux0 = 0, aux1 = 0; // engine-private state that lives across a warp's slices (hashed engine: dense-path back-off)

	__device__ __forceinline__ void flush(const ScanArgs &A, uint32_t seg, uint32_t lane)
	{
		if (n) {
			if (n > chunk_left) { // warp-uniform
				const uint32_t want = n > A.chunk ? n : A.chunk;
				unsigned long long b64 = 0;
				if (lane == 0) b64 = atomicAdd(A.cursor, (unsigned long long)want);
				b64 = __shfl_sync(0xffffffffu, b64, 0);
				// past the end of the buffer: nothing is written, the host sees cursor > cand_cap, grows the buffer and re-runs
				chunk_left = b64 + want <= (unsigned long long)A.cand_cap ? want : 0u;
				chunk_base = (uint32_t)b64;
			}
			__syncwarp();
			if (n <= chunk_left) {
				const uint32_t base = chunk_base;
				for (uint32_t i = lane; i < n; i += 32) A.cand[base + i] = scratch[i];
				// only non-empty segments are written; the entry carries this scan's generation tag, so stale entries of
				// earlier scans read as empty and the table never has to be cleared between scans
				// the occupancy bit lets the resolve skip the empty segments without reading them; the atomicOr's result
				// is unused, so it issues as a fire-and-forget reduction and the warp does not wait for it
				if (lane == 0) {
					A.segs[seg] = SegEntry{base, n | (A.tag << 16)};
					atomicOr(&A.occ[seg >> 5], 1u << (seg & 31u));
				}
				chunk_base += n;
				chunk_left -= n;
			}
		}
		n = 0;
	}
};

// ------------------------------------------------------------------------------------------
// FIXED engine: alternation of fixed-length byte-class sequences
// ------------------------------------------------------------------------------------------
// what a slow path needs to read bytes around a candidate: the slot (shared memory, fast) when the bytes
// lie inside the resident window, global memory (L2) otherwise
struct ByteSrc {
	const uint8_t *stile; // shared-memory address of tile byte 0
	const uint8_t *gtile; // global address of tile byte 0
	int lo, hi;           // tile coordinates resident in shared memory: [lo, hi)
};

// first sequence (in preference order) matching with its anchor byte at tile position p; 0: none
static __device__ __noinline__ uint32_t fixed_verify(const FixedParams &P, const ByteSrc &B, uint32_t off, uint32_t ulen, int p)
{
	const int q = p - (int)P.anchor;              // match start in tile coordinates (may be < 0: previous tile)
	const long long qu = (long long)off + q;      // ... in unit coordinates
	if (qu < 0) return 0;
	const uint8_t *src = (q >= B.lo && q + (int)P.maxlen <= B.hi) ? B.stile : B.gtile;
	for (uint32_t s = 0; s < P.nseq; s++) {
		const uint32_t len = P.seq_len[s];
		if ((unsigned long long)qu + len > ulen) continue;
		const uint32_t *pp = P.seq_pos + P.seq_off[s];
		uint32_t i = 0;
		for (; i < len; i++) {
			const uint32_t e = pp[i];
			const uint32_t b = src[q + (int)i];
			const uint32_t cls = e >> 16;
			bool ok;
			if (cls == 0xffffu) ok = (b & (e & 0xffu)) == ((e >> 8) & 0xffu);
			else ok = (P.cls_bm[cls * 8 + (b >> 5)] >> (b & 31)) & 1u;
			if (!ok) break;
		}
		if (i == len) return len;
	}
	return 0;
}

// rare path shared by the pair and the triple filter: verify the flagged bytes of one row, append in order
static __device__ __noinline__ uint32_t fixed_slow_row(const FixedParams &P, const uint8_t *stile, const uint8_t *gtile, int lo, int hi,
                                                       uint32_t off, uint32_t ulen, uint32_t tile_len, Cand *dst, uint32_t lane,
                                                       uint32_t c0, uint32_t f0, uint32_t f1, uint32_t f2, uint32_t f3)
{
	const ByteSrc B{stile, gtile, lo, hi};
	const uint32_t f[4] = {f0 & kHigh, f1 & kHigh, f2 & kHigh, f3 & kHigh};
	uint32_t mm = 0;
#pragma unroll
	for (int j = 0; j < 4; j++) {
		uint32_t t = f[j];
		while (t) {
			const int byte = (__ffs(t) - 1) >> 3;
			t &= t - 1;
			const int p = (int)c0 + j * 4 + byte;
			if (p < (int)tile_len && fixed_verify(P, B, off, ulen, p)) mm |= 1u << (j * 4 + byte);
		}
	}
	const uint32_t pos0 = off + c0 - P.anchor; // unit offset of a match anchored at chunk byte 0
	return Emitter::emit_at(dst, mm, pos0, [&](uint32_t b) -> uint32_t {
		return P.uniform_len ? P.uniform_len : fixed_verify(P, B, off, ulen, (int)(c0 + b));
	}, lane);
}

template <int D, int K, bool EX>
struct FixedEngine {
	typedef FixedParams Params;
	static constexpr bool kLookBehind = false, kLookAhead = D != 0, kMergeCopies = false;
	static __device__ __forceinline__ void prologue(const FixedParams &, uint8_t *) {}

	// first sequence (in preference order) matching with its anchor byte at tile position p; 0: none
	// Stage-1 SWAR filter of one word pair: bit 7 of a byte of the result set (superset) where some test
	// passes at that byte.  EX: every mask is 0xff, two LOP3 per test instead of three.  The decrement of
	// the zero-byte trick is written t * one + 0xfefefeff (one == 1, opaque to the compiler) so that it
	// issues as IMAD on the FMA pipe instead of crowding the ALU pipe the LOP3/SHF already fill.
	static __device__ __forceinline__ uint32_t word_flags(const FixedParams &P, uint32_t w, uint32_t s)
	{
		uint32_t f = 0;
#pragma unroll
		for (int k = 0; k < K; k++) {
			const uint32_t t = EX ? ((w ^ P.v0[k]) | (s ^ P.v1[k])) : (((w & P.m0[k]) ^ P.v0[k]) | ((s & P.m1[k]) ^ P.v1[k]));
			f |= (t * P.one + 0xfefefeffu) & ~t;
		}
		return f;
	}

	// the bytes D positions further on: D == 4 is the next word itself (no funnel shift at all)
	static __device__ __forceinline__ uint32_t second(uint32_t lo, uint32_t hi)
	{
		return D == 0 ? lo : (D == 4 ? hi : __funnelshift_r(lo, hi, 8 * (D & 3)));
	}

	static __device__ __forceinline__ uint32_t row_any(const FixedParams &P, const uint32_t (&w)[5])
	{
		uint32_t acc = 0;
#pragma unroll
		for (int j = 0; j < 4; j++) acc |= word_flags(P, w[j], second(w[j], w[j + 1]));
		return acc;
	}

	// Rare path for one flagged 512-byte row (warp-converged).  Stage 2 first narrows the flags with a
	// third pattern byte (SWAR again), only then are the survivors verified byte by byte.
	static __device__ __noinline__ uint32_t slow_row(const FixedParams &P, const uint8_t *stile, const uint8_t *gtile, int lo, int hi,
	                                                 uint32_t off, uint32_t ulen, uint32_t tile_len, Cand *dst, uint32_t lane, uint32_t c0,
	                                                 uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t w4)
	{
		const uint32_t w[5] = {w0, w1, w2, w3, w4};
		uint32_t f[4];
#pragma unroll
		for (int j = 0; j < 4; j++) f[j] = word_flags(P, w[j], second(w[j], w[j + 1])) & kHigh;
		for (uint32_t k = 0; P.n2 && k < 1; k++) { // stage 2 (one pass; the loop only scopes the constants)
			uint32_t g[4] = {0, 0, 0, 0};
			for (uint32_t t3 = 0; t3 < P.n2; t3++) {
				const uint32_t m0 = P.t2_m0[t3], v0 = P.t2_v0[t3], m1 = P.t2_m1[t3], v1 = P.t2_v1[t3], m2 = P.t2_m2[t3], v2 = P.t2_v2[t3];
#pragma unroll
				for (int j = 0; j < 4; j++) {
					const uint32_t s1 = second(w[j], w[j + 1]);
					const uint32_t s2 = __funnelshift_r(w[j], w[j + 1], 8 * P.d2);
					const uint32_t t = ((w[j] & m0) ^ v0) | ((s1 & m1) ^ v1) | ((s2 & m2) ^ v2);
					g[j] |= (t - kOnes) & ~t;
				}
			}
#pragma unroll
			for (int j = 0; j < 4; j++) f[j] &= g[j];
		}
		if (!__any_sync(0xffffffffu, (f[0] | f[1] | f[2] | f[3]) != 0)) return 0;
		return fixed_slow_row(P, stile, gtile, lo, hi, off, ulen, tile_len, dst, lane, c0, f[0], f[1], f[2], f[3]);
	}

	// lane's 16 bytes + the 4 bytes after them (next lane's / next row's first word; after the last chunk of the
	// slice: the 16-byte look-ahead copy that sits right behind the slice in the slot)
	static __device__ __forceinline__ void load_row(const Slice &S, uint32_t c0, uint32_t (&w)[5])
	{
		const uint4 a = *reinterpret_cast<const uint4 *>(S.tile + c0);
		w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
		w[4] = D ? *reinterpret_cast<const uint32_t *>(S.tile + c0 + 16) : 0u;
	}

	template <class G>
	static __device__ __forceinline__ void run(const FixedParams &P, const Slice &S, Emitter &E, uint32_t lane)
	{
		constexpr int kRows = G::kSlice / 512;
		if (S.niter == 0) return;
		const uint32_t base = S.begin + lane * 16;
		if (S.niter == (uint32_t)kRows) {
			// full slice: groups of 4 rows -- all 8 loads of a group first, one vote per group
			constexpr int kGroup = 4;
#pragma unroll 1
			for (int g0 = 0; g0 < kRows; g0 += kGroup) {
				uint32_t w[kGroup][5];
#pragma unroll
				for (int r = 0; r < kGroup; r++) load_row(S, base + (g0 + r) * 512, w[r]);
				uint32_t acc = 0, ra[kGroup];
#pragma unroll
				for (int r = 0; r < kGroup; r++) { ra[r] = row_any(P, w[r]); acc |= ra[r]; }
				if (__any_sync(0xffffffffu, (acc & kHigh) != 0)) {
#pragma unroll
					for (int r = 0; r < kGroup; r++) {
						if (__any_sync(0xffffffffu, (ra[r] & kHigh) != 0))
							E.n += slow_row(P, S.tile, S.gtile, (int)S.begin, (int)(S.begin + S.niter * 512 + (D ? kHalo : 0u)), S.off, S.ulen, S.tile_len,
							                E.scratch + E.n, lane, base + (g0 + r) * 512, w[r][0], w[r][1], w[r][2], w[r][3], w[r][4]);
					}
				}
			}
			return;
		}
		for (uint32_t it = 0; it < S.niter; it++) {
			uint32_t w[5];
			load_row(S, base + it * 512, w);
			if (__any_sync(0xffffffffu, (row_any(P, w) & kHigh) != 0))
				E.n += slow_row(P, S.tile, S.gtile, (int)S.begin, (int)(S.begin + S.niter * 512 + (D ? kHalo : 0u)), S.off, S.ulen, S.tile_len,
				                E.scratch + E.n, lane, base + it * 512, w[0], w[1], w[2], w[3], w[4]);
		}
	}
};

// ------------------------------------------------------------------------------------------
// FIXED engine, triple filter: when the best byte pair would flag too many rows (short or
// case-insensitive patterns, several alternatives) stage 1 tests three pattern bytes (anchor, anchor + d1,
// anchor + d2, all within one word of each other) -- 2 funnel shifts and 4 ops per test and word, and the
// slow path is entered ~100x less often.
// ------------------------------------------------------------------------------------------
template <int K, bool EX>
struct Fixed3Engine {
	typedef FixedParams Params;
	static constexpr bool kLookBehind = false, kLookAhead = true, kMergeCopies = true;
	static __device__ __forceinline__ void prologue(const FixedParams &, uint8_t *) {}

	static __device__ __forceinline__ uint32_t word_flags(const FixedParams &P, uint32_t w, uint32_t s1, uint32_t s2)
	{
		uint32_t f = 0;
#pragma unroll
		for (int k = 0; k < K; k++) {
			const uint32_t t = EX ? ((w ^ P.t2_v0[k]) | (s1 ^ P.t2_v1[k]) | (s2 ^ P.t2_v2[k]))
			                      : (((w & P.t2_m0[k]) ^ P.t2_v0[k]) | ((s1 & P.t2_m1[k]) ^ P.t2_v1[k]) | ((s2 & P.t2_m2[k]) ^ P.t2_v2[k]));
			f |= (t * P.one + 0xfefefeffu) & ~t;
		}
		return f;
	}
	static __device__ __forceinline__ uint32_t row_any(const FixedParams &P, const uint32_t (&w)[5], uint32_t (&f)[4])
	{
		uint32_t acc = 0;
#pragma unroll
		for (int j = 0; j < 4; j++) {
			f[j] = word_flags(P, w[j], __funnelshift_r(w[j], w[j + 1], P.sh1), __funnelshift_r(w[j], w[j + 1], P.sh2));
			acc |= f[j];
		}
		return acc;
	}

	template <class G>
	static __device__ __forceinline__ void run(const FixedParams &P, const Slice &S, Emitter &E, uint32_t lane)
	{
		const uint32_t base = S.begin + lane * 16;
#pragma unroll 2
		for (uint32_t it = 0; it < S.niter; it++) {
			const uint32_t c0 = base + it * 512;
			uint32_t w[5], f[4];
			const uint4 a = *reinterpret_cast<const uint4 *>(S.tile + c0);
			w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
			w[4] = *reinterpret_cast<const uint32_t *>(S.tile + c0 + 16);
			if (__any_sync(0xffffffffu, (row_any(P, w, f) & kHigh) != 0))
				E.n += fixed_slow_row(P, S.tile, S.gtile, (int)S.begin, (int)(S.begin + S.niter * 512 + kHalo), S.off, S.ulen, S.tile_len,
				                      E.scratch + E.n, lane, c0, f[0], f[1], f[2], f[3]);
		}
	}
};

// ------------------------------------------------------------------------------------------
// FIXED engine, balanced pair filter (exact byte pairs, 2..8 alternatives: `foo|bar|baz|quux`, BASELINE
// configs[2]).  The pair and triple filters above are ALU-pipe bound (LOP3/SHF issue at half rate): the triple
// filter spends 17 ALU-pipe instructions per word on three alternatives.  Here
//   * equality is a subtraction on the FMA pipe.  w80 = w | 0x80808080 (bit 7 forced), a = w80 - V0, b = s80 - V1
//     with V = the pattern byte & 0x7f replicated: no byte borrows (0x80+x - v >= 1) and a byte of a is 0x80 iff
//     the text byte equals the pattern byte (mod bit 7: a superset, the verification is exact).  One LOP3 then
//     forms t = (a | b) ^ 0x80808080 -- zero byte iff both match -- and the usual zero-byte test (IMAD + LOP3)
//     ORs it into the row's flag word: 2 ALU-pipe + 3 FMA-pipe instructions per test and word instead of 3 + 1;
//   * the cheap pair test flags one row in six on random text, so the third byte is NOT tested up front but in an
//     inline stage 2 on the flagged rows only, reusing the kept t words (t | third-byte mismatch), and only rows
//     that survive both stages visit the out-of-line verification.
// ------------------------------------------------------------------------------------------
template <int D, int K, bool ALIGNED>
struct FixedBEngine {
	typedef FixedParams Params;
	static constexpr bool kLookBehind = false, kLookAhead = true, kMergeCopies = true;
	static __device__ __forceinline__ void prologue(const FixedParams &, uint8_t *) {}

	// t words of one text word: zero byte <=> pair test k passes at that byte (bit 7 of the text ignored).  Bit 7 of every
	// byte of t is clear by construction (a | b is never 0x00, so masking bit 7 leaves a zero byte exactly where
	// a == b == 0x80), which halves the zero-byte test: t - 0x01 sets bit 7 where t is zero (or above a zero byte: a
	// superset), no "& ~t" needed.
	static __device__ __forceinline__ void word_t(const FixedParams &P, uint32_t w80, uint32_t s80, uint32_t (&t)[K])
	{
#pragma unroll
		for (int k = 0; k < K; k++) {
			const uint32_t a = w80 * P.one + P.b_c0[k], b = s80 * P.one + P.b_c1[k];
			t[k] = (a | b) & kLow7;
		}
	}
	static __device__ __forceinline__ uint32_t dec(const FixedParams &P, uint32_t t) { return t * P.one + 0xfefefeffu; }
	// general zero-byte test (stage 2: the third-byte term can have bit 7 set)
	static __device__ __forceinline__ uint32_t zero_flags(const FixedParams &P, uint32_t t, uint32_t f)
	{
		return ((t * P.one + 0xfefefeffu) & ~t) | f;
	}

	template <class G>
	static __device__ __forceinline__ void run(const FixedParams &P, const Slice &S, Emitter &E, uint32_t lane)
	{
		const uint32_t base = S.begin + lane * 16;
#pragma unroll 2
		for (uint32_t it = 0; it < S.niter; it++) {
			const uint32_t c0 = base + it * 512;
			uint32_t w[5], w80[5], t[4][K];
			const uint4 a = *reinterpret_cast<const uint4 *>(S.tile + c0);
			w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
			w[4] = *reinterpret_cast<const uint32_t *>(S.tile + c0 + 16);
#pragma unroll
			for (int j = 0; j < 5; j++) w80[j] = w[j] | kHigh;
			uint32_t f = 0;
#pragma unroll
			for (int j = 0; j < 4; j++) {
				const uint32_t s80 = D == 4 ? w80[j + 1] : __funnelshift_r(w80[j], w80[j + 1], 8 * D);
				word_t(P, w80[j], s80, t[j]);
#pragma unroll
				for (int k = 0; k < K; k++) f |= dec(P, t[j][k]);
			}
			if (!__any_sync(0xffffffffu, (f & kHigh) != 0)) continue;
			// ---- stage 2 (flagged rows): per-word flags, narrowed by the third byte of every alternative ----
			uint32_t g[4];
#pragma unroll
			for (int j = 0; j < 4; j++) {
				g[j] = 0;
				if (ALIGNED) {
					const uint32_t s2 = __funnelshift_r(w[j], w[j + 1], P.b_sh2);
#pragma unroll
					for (int k = 0; k < K; k++) g[j] = zero_flags(P, t[j][k] | ((s2 & P.b_m2[k]) ^ P.b_v2[k]), g[j]);
				} else {
#pragma unroll
					for (int k = 0; k < K; k++) g[j] |= dec(P, t[j][k]);
				}
			}
			if (!__any_sync(0xffffffffu, ((g[0] | g[1] | g[2] | g[3]) & kHigh) != 0)) continue;
			E.n += fixed_slow_row(P, S.tile, S.gtile, (int)S.begin, (int)(S.begin + S.niter * 512 + kHalo), S.off, S.ulen, S.tile_len,
			                      E.scratch + E.n, lane, c0, g[0], g[1], g[2], g[3]);
		}
	}
};

// ------------------------------------------------------------------------------------------
// HASH engine: FIXED with many alternatives (literal sets).  The first L = 2 or 3 bytes at every position
// are looked up in a perfect-hash table in shared memory -- exact membership, one multiply (FMA pipe),
// one LDS and four ALU ops per position, independent of how many alternatives there are.  Only true
// key hits are verified, against the alternatives that share the key, in preference order.
// Two paths per 1 KiB block: DENSE (every position probed: 6.25 issue slots each) and, when all key bytes lie in one
// narrow byte range, SPARSE (a SWAR class test first, the table probed only where three class bytes in a row leave a
// key possible -- ~2 % of printable text); the kernel picks per block, see "sparse path" below.
//
// Small tables are replicated across the shared-memory banks: 32 copies (stride 128 B, lane l reads bank l: one
// wavefront per lookup) up to 256 slots, 16 copies (two lanes per bank: two wavefronts) up to 512.  With a single
// copy the 32 random slots of a warp cost ~3.4 wavefronts and the shared-memory data pipe is the bottleneck (95 %
// busy, profiles/r01_scan_v5_lits8_single_table_ncu.txt).
// ------------------------------------------------------------------------------------------
struct HashEngine {
	typedef HashParams Params;
	static constexpr bool kLookBehind = false, kLookAhead = true, kMergeCopies = true;

	static __device__ __forceinline__ void prologue(const HashParams &P, uint8_t *extra)
	{
		uint32_t *t = reinterpret_cast<uint32_t *>(extra);
		const uint32_t copies = P.stride >> 2; // 32, 16 or 1 (power of two): slot s, copy c at word s * copies + c
		for (uint32_t i = threadIdx.x; i < P.nslots * copies; i += blockDim.x) t[i] = P.table[i / copies];
		__syncthreads();
	}

	// first alternative (preference order) with this key that matches at tile position p; 0: none
	static __device__ __noinline__ uint32_t verify(const HashParams &P, const uint8_t *tile, uint32_t off, uint32_t ulen, int p, uint32_t slot)
	{
		const unsigned long long qu = (unsigned long long)off + (unsigned)p;
		// the pattern tables are read-only for the whole launch: the non-coherent path keeps them in L1 (a verification is a
		// chain of dependent loads: from L2 every link costs ~250 cycles)
		const uint32_t first = __ldg(P.slot_first + slot), cnt = __ldg(P.slot_count + slot);
		for (uint32_t k = 0; k < cnt; k++) {
			const uint32_t s = __ldg(P.slot_seqs + first + k);
			const uint32_t len = __ldg(P.seq_len + s);
			if (qu + len > ulen) continue;
			const uint32_t *pp = P.seq_pos + __ldg(P.seq_off + s);
			uint32_t i = 0;
			for (; i < len; i++) {
				const uint32_t e = __ldg(pp + i);
				const uint32_t b = tile[p + (int)i];
				const uint32_t cls = e >> 16;
				bool ok;
				if (cls == 0xffffu) ok = (b & (e & 0xffu)) == ((e >> 8) & 0xffu);
				else ok = (P.cls_bm[cls * 8 + (b >> 5)] >> (b & 31)) & 1u;
				if (!ok) break;
			}
			if (i == len) return len;
		}
		return 0;
	}

	// the 32-bit window at byte k of the word pair; the bytes beyond the key fall off the top of window * mulsh
	static __device__ __forceinline__ uint32_t window(uint32_t lo, uint32_t hi, int k) { return k ? __funnelshift_r(lo, hi, 8 * k) : lo; }
	static __device__ __forceinline__ uint32_t slot_of(const HashParams &P, uint32_t h) { return __umulhi(h, P.nslots); }
	// tbl: the table in shared memory, for a replicated table already advanced to this lane's bank (+ lane * 4).
	// Hash, slot and address are three IMADs (FMA pipe); zero <=> the position holds a key of the set.  SUB: the
	// comparison as entry - h on the FMA pipe instead of entry ^ h on the ALU pipe (two of every 4 positions).
	template <bool SUB>
	static __device__ __forceinline__ uint32_t probe(const HashParams &P, const uint8_t *tbl, uint32_t y)
	{
		const uint32_t h = y * P.mulsh;
		const uint32_t e = *reinterpret_cast<const uint32_t *>(tbl + slot_of(P, h) * P.stride);
		return SUB ? h * P.neg1 + e : e ^ h;
	}

	// min over the 16 positions of (table[slot(h)] ^ h), two positions per 3-input minimum; d[] keeps the 16 words for the
	// rare row that has a hit (its positions then cost a compare each instead of a second round of lookups)
	static __device__ __forceinline__ uint32_t row_min(const HashParams &P, const uint8_t *tbl, const uint32_t (&w)[5], uint32_t (&d)[16])
	{
		uint32_t mn = 0xffffffffu;
#pragma unroll
		for (int j = 0; j < 4; j++) {
			d[4 * j + 0] = probe<true>(P, tbl, window(w[j], w[j + 1], 0));
			d[4 * j + 1] = probe<true>(P, tbl, window(w[j], w[j + 1], 1));
			d[4 * j + 2] = probe<false>(P, tbl, window(w[j], w[j + 1], 2));
			d[4 * j + 3] = probe<false>(P, tbl, window(w[j], w[j + 1], 3));
			mn = __vimin3_u32(mn, d[4 * j + 0], d[4 * j + 1]);
			mn = __vimin3_u32(mn, d[4 * j + 2], d[4 * j + 3]);
		}
		return mn;
	}

	static __device__ __noinline__ uint32_t slow_row(const HashParams &P, const uint8_t *tbl, const uint8_t *gtile, uint32_t off,
	                                                 uint32_t ulen, uint32_t tile_len, Cand *dst, uint32_t lane, uint32_t c0,
	                                                 uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t w4, uint32_t hits)
	{
		// hits: positions whose leading bytes are a key of the set (from the comparison words the fast path kept)
		const uint32_t w[5] = {w0, w1, w2, w3, w4};
		uint32_t mm = 0;
		// the slot at position b for a run-time b (rolled loops below: the slow path stays small)
		auto slot_rt = [&](int b) -> uint32_t { return slot_of(P, __funnelshift_r(w[b >> 2], w[(b >> 2) + 1], 8 * (b & 3)) * P.mulsh); };
		uint32_t len_a = 0, len_b = 0, bit_a = 32, bit_b = 32; // lengths of the lane's first two matches (a third one verifies again)
		while (hits) { // verify() is out of line: one copy, the kernel stays instruction-cache resident
			const int b = __ffs(hits) - 1;
			hits &= hits - 1;
			const int p = (int)c0 + b;
			const uint32_t len = p < (int)tile_len ? verify(P, gtile, off, ulen, p, slot_rt(b)) : 0u;
			if (len) {
				mm |= 1u << b;
				if (bit_a == 32) { bit_a = (uint32_t)b; len_a = len; }
				else if (bit_b == 32) { bit_b = (uint32_t)b; len_b = len; }
			}
		}
		return Emitter::emit_at(dst, mm, off + c0, [&](uint32_t b) -> uint32_t {
			if (b == bit_a) return len_a;
			if (b == bit_b) return len_b;
			return verify(P, gtile, off, ulen, (int)(c0 + b), slot_rt((int)b));
		}, lane);
	}

	// ---- sparse path ----------------------------------------------------------------------------------------------
	// Probing every position costs ~6 issue slots each (~155 instructions per 512-byte row: issue-bound well below the
	// HBM roofline).  When all key bytes lie in one narrow range (a set of lowercase words) most positions cannot hold
	// a key at all: a SWAR class test -- 3 instructions per word, carry-tolerant, a superset -- leaves ~2 % of the positions of
	// printable text, and only those are hashed and looked up, two per lane and round.  Text that passes the class test
	// nearly everywhere (prose against lowercase keys) is noticed per block: the warp then runs the dense path for a
	// while (8 .. 64 blocks, doubling) before it tries the class test again.
	// A block is 1 KiB: every lane owns 32 CONTIGUOUS bytes (8 words + the word behind them).

	// bit 7 of a byte set where lo <= byte <= hi + 1 may hold; never clear for a byte in [lo, hi] whatever its neighbours
	// are (a carry out of a byte >= 0x80 below adds one to both sums: the upper bound is one too wide for that reason)
	static __device__ __forceinline__ uint32_t pre_flags(const HashParams &P, uint32_t x)
	{
		return lop3<0x20>(x * P.one + P.pre_ge, x * P.one + P.pre_gt, kHigh); // a & ~b & 0x80808080
	}
	static __device__ __forceinline__ uint32_t bfind(uint32_t x) // index of the highest set bit, 0xffffffff for 0 (one FLO)
	{
		uint32_t r;
		asm("bfind.u32 %0, %1;" : "=r"(r) : "r"(x));
		return r;
	}
	static __device__ __forceinline__ uint32_t shl_clamp(uint32_t x, uint32_t n) // x << n, 0 for n >= 32
	{
		uint32_t r;
		asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(x), "r"(n));
		return r;
	}
	// Positions of a lane's 32 bytes whose hash_len bytes all pass the class test, INTERLEAVED: position 4k + j (word k,
	// byte j) at bit 8j + k.  The flag words of the 8 text words only have to be shifted by 7 - k and added (IMAD.HI, FMA
	// pipe), and "the flag of the next position at this position's bit" is one funnel shift for all 32 positions.
	static __device__ __forceinline__ uint32_t pre_block(const HashParams &P, const uint32_t (&w)[9])
	{
		uint32_t c = pre_flags(P, w[7]);
#pragma unroll
		for (int k = 0; k < 7; k++) c = __umulhi(pre_flags(P, w[k]), P.pre_mul[k]) + c; // flags >> (7 - k): disjoint bits
		const uint32_t r8 = pre_flags(P, w[8]); // bit 7: position 32, bit 15: position 33
		// next(): bits 8j + k, j < 3 take bit 8(j + 1) + k; bit 24 + k takes bit k + 1, bit 31 the first position behind the lane
		const uint32_t n1 = __funnelshift_r(c, lop3<0xCA>(0x7fu, c >> 1, r8), 8);
		uint32_t f = c & n1;
		if (P.hash_len == 3) f &= __funnelshift_r(n1, lop3<0xCA>(0x7fu, n1 >> 1, r8 >> 8), 8);
		return f;
	}
	static constexpr uint32_t kPreMax = 12; // more flagged positions than this in one lane (of 32): the dense path is cheaper

	// Rare (a key of the set really is in the block, one 1 KiB block in eight on printable noise): decide the lanes' key
	// hits and append the matches in position order.  A key hit is first held against the slot's TAIL entry -- what the 8
	// bytes at the position must look like for any alternative of that key to match: one 16-byte table load and the text
	// from shared memory, against a chain of dependent global loads in verify() (the out-of-line verification used to be
	// 40 % of the kernel's time).  For a slot with a single all-literal alternative of up to 7 bytes the tail entry IS the
	// verification and carries the length; only other slots' survivors visit verify().
	// hc: key hits in the interleaved layout of pre_block
	static __device__ __noinline__ uint32_t slow_block(const HashParams &P, const uint8_t *tile, const uint8_t *gtile, uint32_t off,
	                                                   uint32_t ulen, uint32_t tile_len, Cand *dst, uint32_t lane, uint32_t c0, uint32_t hc)
	{
		const uint8_t *lb = tile + c0; // the lane's 32 bytes in shared memory
		// length of the match at linear position b of the lane's bytes (a key position), 0: none
		auto len_at = [&](uint32_t b) -> uint32_t {
			const uint8_t *wp = lb + (b & ~3u);
			const uint32_t x0 = *reinterpret_cast<const uint32_t *>(wp), x1 = *reinterpret_cast<const uint32_t *>(wp + 4),
			               x2 = *reinterpret_cast<const uint32_t *>(wp + 8);
			const uint32_t sh = 8u * (b & 3u);
			const uint32_t y0 = __funnelshift_r(x0, x1, sh), y1 = __funnelshift_r(x1, x2, sh);
			const uint32_t slot = slot_of(P, y0 * P.mulsh);
			const uint4 te = __ldg(P.tail + slot);
			if (((y0 ^ te.y) & te.x) | ((y1 ^ te.w) & te.z)) return 0u; // no alternative of this key matches here
			const int p = (int)(c0 + b);
			if (p >= (int)tile_len) return 0u;
			const uint32_t simple = te.w >> 24; // the slot's only alternative, all literal: its length (the bytes just compared)
			if (simple) return (unsigned long long)off + (unsigned)p + simple <= ulen ? simple : 0u;
			return verify(P, gtile, off, ulen, p, slot);
		};
		uint32_t mm = 0, len_a = 0, bit_a = 32; // length of the lane's first match (a second one is decided again when emitted)
		while (hc) {
			const uint32_t t = bfind(hc);
			hc ^= 1u << t;
			const uint32_t b = (t & 7u) * 4u + (t >> 3);
			const uint32_t len = len_at(b);
			if (len) {
				mm |= 1u << b;
				if (b < bit_a) { bit_a = b; len_a = len; }
			}
		}
		if (!__any_sync(0xffffffffu, mm != 0)) return 0;
		return Emitter::emit_at(dst, mm, off + c0, [&](uint32_t b) -> uint32_t { return b == bit_a ? len_a : len_at(b); }, lane);
	}

	static __device__ __forceinline__ void load_row(const Slice &S, uint32_t c0, uint32_t (&w)[5])
	{
		const uint4 a = *reinterpret_cast<const uint4 *>(S.tile + c0);
		w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
		w[4] = *reinterpret_cast<const uint32_t *>(S.tile + c0 + 16);
	}

	// every position probed (the path for sets without a usable byte range and for text the class test cannot thin out)
	static __device__ __forceinline__ void dense_row(const HashParams &P, const uint8_t *tbl, const Slice &S, Emitter &E, uint32_t lane,
	                                                 uint32_t c0)
	{
		uint32_t w[5], d[16];
		load_row(S, c0, w);
		const uint32_t mn = row_min(P, tbl, w, d);
		if (__any_sync(0xffffffffu, mn == 0)) {
			uint32_t hits = 0;
#pragma unroll
			for (int b = 0; b < 16; b++) hits |= (d[b] == 0u ? 1u : 0u) << b;
			E.n += slow_row(P, tbl, S.gtile, S.off, S.ulen, S.tile_len, E.scratch + E.n, lane, c0, w[0], w[1], w[2], w[3], w[4], hits);
		}
	}

	// two 32-bit shared-memory loads at a and a + 4, executed only where on != 0 (the lanes that have no flagged position left
	// in a probe round would otherwise all read word 7 of their 32 bytes: lanes l, l + 4, l + 8, ... on one bank, 8-way
	// conflicts -- the shared-memory pipe was 85 % busy and the top stall reason, profiles/r02_lits100_sparse_v1_ncu.txt)
	static __device__ __forceinline__ void lds2_if(uint32_t a, uint32_t on, uint32_t &x0, uint32_t &x1)
	{
		asm volatile(
		    "{\n"
		    ".reg .pred q;\n"
		    "setp.ne.u32 q, %3, 0;\n"
		    "@q ld.shared.u32 %0, [%2];\n"
		    "@q ld.shared.u32 %1, [%2+4];\n"
		    "}\n"
		    : "=r"(x0), "=r"(x1) // left as they were where on == 0: the caller ignores what such a lane computes
		    : "r"(a), "r"(on));
	}

	template <class G>
	static __device__ __forceinline__ void run(const HashParams &P, const Slice &S, Emitter &E, uint32_t lane)
	{
		const uint8_t *tbl = S.extra + ((lane * 4u) & (P.stride - 1u)); // this lane's copy of the table
		uint32_t it = 0;
		// E.aux0: blocks still to run dense before the class test is tried again, E.aux1: how many the last give-up asked for
		// (doubling, 8 .. 64: prose against lowercase keys pays one wasted class test per 64 blocks, text that changes its
		// character is re-probed within 8)
		if (P.pre_enable) {
			// the probe loop's constants in vector registers (as kernel parameters the compiler reloads them from the constant
			// bank every round: issue slots).  z is zero in every lane, but the compiler cannot know (P.one is opaque)
			const uint32_t z = (P.one - 1u) * lane;
			const uint32_t mulsh = P.mulsh + z, nslots = P.nslots + z, stride = P.stride + z, k1 = P.one + z, k4 = k1 << 2;
			while (it + 2 <= S.niter) {
				if (E.aux0) { // warp-uniform
					E.aux0--;
					dense_row(P, tbl, S, E, lane, S.begin + it * 512 + lane * 16);
					dense_row(P, tbl, S, E, lane, S.begin + (it + 1) * 512 + lane * 16);
					it += 2;
					continue;
				}
				const uint32_t c0 = S.begin + it * 512 + lane * 32;
				const uint8_t *lb = S.tile + c0;
				uint32_t w[9];
				{
					const uint4 a = *reinterpret_cast<const uint4 *>(lb), b = *reinterpret_cast<const uint4 *>(lb + 16);
					w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
					w[8] = *reinterpret_cast<const uint32_t *>(lb + 32);
				}
				uint32_t c = pre_block(P, w);
				if (__any_sync(0xffffffffu, __popc(c) > (int)kPreMax)) {
					E.aux1 = E.aux1 ? (E.aux1 < 64u ? E.aux1 * 2u : 64u) : 8u;
					E.aux0 = E.aux1;
					continue; // this block and the next aux1 - 1 run dense
				}
				E.aux1 = 0;
				it += 2;
				uint32_t hc = 0;
				const uint32_t lbr = smem_u32(lb) + z; // the block's shared-memory address in one register
#pragma unroll 1
				for (uint32_t round = 0; round < (kPreMax + 1) / 2; round++) {
					// two flagged positions per lane and round: two independent chains of FLO -> LDS -> hash -> LDS in flight, one
					// vote for both (a lane that has none left keeps what its registers held and hashes that: m is 0 for it)
					const uint32_t on0 = c, t0 = bfind(c), m0 = shl_clamp(k1, t0);
					c ^= m0;
					const uint32_t on1 = c, t1 = bfind(c), m1 = shl_clamp(k1, t1);
					c ^= m1;
					uint32_t x0, x1, y0, y1;
					lds2_if((t0 & 7u) * k4 + lbr, on0, x0, x1); // LOP3 + IMAD
					lds2_if((t1 & 7u) * k4 + lbr, on1, y0, y1);
					const uint32_t h0 = __funnelshift_r(x0, x1, t0 & 0x18u) * mulsh, h1 = __funnelshift_r(y0, y1, t1 & 0x18u) * mulsh;
					const uint32_t e0 = *reinterpret_cast<const uint32_t *>(tbl + __umulhi(h0, nslots) * stride); // own bank: conflict free
					const uint32_t e1 = *reinterpret_cast<const uint32_t *>(tbl + __umulhi(h1, nslots) * stride);
					hc |= (e0 == h0 ? m0 : 0u) | (e1 == h1 ? m1 : 0u);
					if (!__any_sync(0xffffffffu, c != 0)) break; // no lane has more than kPreMax: the loop bound is never the exit
				}
				if (__any_sync(0xffffffffu, hc != 0))
					E.n += slow_block(P, S.tile, S.gtile, S.off, S.ulen, S.tile_len, E.scratch + E.n, lane, c0, hc);
			}
		}
		for (; it < S.niter; it++) dense_row(P, tbl, S, E, lane, S.begin + it * 512 + lane * 16);
	}
};

// ------------------------------------------------------------------------------------------
// RUN engine: one byte class repeated {n,}: one candidate per maximal run of >= n class bytes
// ------------------------------------------------------------------------------------------
template <int NLO, int NHI, int NFO>
struct RunEngine {
	typedef RunParams Params;
	static constexpr bool kLookBehind = true, kLookAhead = true, kMergeCopies = true;
	static __device__ __forceinline__ void prologue(const RunParams &, uint8_t *) {}

	static __device__ __forceinline__ uint32_t class_flags(const RunParams &P, uint32_t x)
	{
		const uint32_t x7 = x & kLow7;
		uint32_t lo = 0, hi = 0;
#pragma unroll
		for (int r = 0; r < NLO; r++) {
			// adds as IMAD (x7 * one + c, one == 1 opaque): FMA pipe, the ALU pipe is the bottleneck; keep the
			// first add on the ALU pipe for balance
			const uint32_t ge = r == 0 ? x7 + P.add_ge_lo[r] : x7 * P.one + P.add_ge_lo[r];
			const uint32_t gt = x7 * P.one + P.add_gt_lo[r];
			lo |= ge & ~gt;
		}
		if (NFO) {
			// one range test serves two ranges that differ only in bit 5 ([A-Z] and [a-z]): test x | 0x20 against the upper one
			const uint32_t y = x7 | 0x20202020u;
			lo |= (y * P.one + P.add_ge_fold) & ~(y * P.one + P.add_gt_fold);
		}
#pragma unroll
		for (int r = 0; r < NHI; r++) hi |= (x7 * P.one + P.add_ge_hi[r]) & ~(x7 * P.one + P.add_gt_hi[r]);
		if (NHI) return ((lo & ~x) | (hi & x)) & kHigh;
		return lo & ~x & kHigh;
	}
	// The same for words whose bytes are all below 0x80 (plain ASCII text, checked per slice by the caller) and a class
	// without high ranges: membership is the PARITY of the thresholds lo, hi + 1 at or below the byte, each one bit 7 of
	// x + (0x80 - threshold) (an IMAD, no carry leaves a byte since x <= 0x7f), so all ranges reduce with 3-input XORs:
	// 5 ALU-pipe instructions per word instead of 8 ([A-Za-z0-9_]: one OR for the case fold, three XOR3, the nibble insert).
	static __device__ __forceinline__ uint32_t class_flags_ascii(const RunParams &P, uint32_t x)
	{
		constexpr int kTerms = 2 * NLO + 2 * NFO; // >= 2
		uint32_t t[kTerms];
#pragma unroll
		for (int r = 0; r < NLO; r++) { t[2 * r] = x * P.one + P.add_ge_lo[r]; t[2 * r + 1] = x * P.one + P.add_gt_lo[r]; }
		if (NFO) {
			const uint32_t y = x | 0x20202020u;
			t[2 * NLO] = y * P.one + P.add_ge_fold;
			t[2 * NLO + 1] = y * P.one + P.add_gt_fold;
		}
		// XOR3 chain, the last step fused with the bit-7 mask: (kTerms + 1) / 2 LOP3 in all (inline PTX: the compiler
		// would otherwise pair the terms first and spend one more)
		uint32_t acc = t[0];
		int i = 1;
#pragma unroll
		for (; i + 2 < kTerms; i += 2) acc = lop3<0x96>(acc, t[i], t[i + 1]);
		if (i + 1 < kTerms) { acc = lop3<0x96>(acc, t[i], t[i + 1]); return acc & kHigh; }
		return lop3<0x28>(acc, t[i], kHigh); // (acc ^ t) & 0x80808080
	}
	static __device__ __forceinline__ bool in_class(const RunParams &P, uint32_t b)
	{
		return (P.bitmap[b >> 5] >> (b & 31)) & 1u;
	}
	// class mask of 16 ASCII bytes inside the unit; `seen` collects the words so the caller can tell whether the slice was ASCII
	static __device__ __forceinline__ uint32_t mask16_ascii(const RunParams &P, const uint8_t *p, uint32_t &seen)
	{
		const uint4 a = *reinterpret_cast<const uint4 *>(p);
		seen |= a.x | a.y;
		seen |= a.z | a.w;
		uint32_t r = pack_top_nibble(class_flags_ascii(P, a.w)) >> 28;
		r = __funnelshift_l(pack_top_nibble(class_flags_ascii(P, a.z)), r, 4);
		r = __funnelshift_l(pack_top_nibble(class_flags_ascii(P, a.y)), r, 4);
		return __funnelshift_l(pack_top_nibble(class_flags_ascii(P, a.x)), r, 4);
	}
	// 16-bit class mask of the 16 bytes at tile position c, bytes at or past the unit end read as 0
	static __device__ __forceinline__ uint32_t mask16(const RunParams &P, const Slice &S, uint32_t c)
	{
		const uint4 a = *reinterpret_cast<const uint4 *>(S.tile + c);
		uint32_t r = pack_top_nibble(class_flags(P, a.w)) >> 28;
		r = __funnelshift_l(pack_top_nibble(class_flags(P, a.z)), r, 4);
		r = __funnelshift_l(pack_top_nibble(class_flags(P, a.y)), r, 4);
		r = __funnelshift_l(pack_top_nibble(class_flags(P, a.x)), r, 4);
		const long long rem = (long long)S.ulen - (long long)S.off - (long long)c;
		const uint32_t valid = rem >= 16 ? 0xffffu : (rem <= 0 ? 0u : ((1u << (int)rem) - 1u));
		return r & valid; // the tail of the last 16-byte granule of a unit is whatever follows it in memory
	}

	// class mask of 16 bytes that are known to lie inside the unit
	static __device__ __forceinline__ uint32_t mask16_inner(const RunParams &P, const uint8_t *p)
	{
		const uint4 a = *reinterpret_cast<const uint4 *>(p);
		uint32_t r = pack_top_nibble(class_flags(P, a.w)) >> 28;
		r = __funnelshift_l(pack_top_nibble(class_flags(P, a.z)), r, 4);
		r = __funnelshift_l(pack_top_nibble(class_flags(P, a.y)), r, 4);
		return __funnelshift_l(pack_top_nibble(class_flags(P, a.x)), r, 4);
	}

	// positions whose bit and the following run_min-1 bits are set (window: own 16 bits + next 16): five
	// AND-with-shift steps whose shift amounts the host derived from run_min (doubling, then the remainder)
	static __device__ __forceinline__ uint32_t runs(const RunParams &P, uint32_t w)
	{
#pragma unroll
		for (int i = 0; i < 5; i++) w &= w >> P.sh[i];
		return w;
	}

	// candidates of one row -> private list, in position order.  Common case (every lane has at most one):
	// rank by ballot; otherwise the general prefix sum.
	// candidates of one row -> private list, in position order; returns how many
	static __device__ __forceinline__ uint32_t emit_row(const RunParams &P, const uint8_t *gtile, uint32_t off, uint32_t ulen, Cand *dst,
	                                                 uint32_t lane, uint32_t cand, uint32_t c0)
	{
		if (P.run_min > 17u) {
			// long minimum: confirm bytes 17..n-1 (global memory: they may lie in another warp's slice)
			uint32_t keep = 0, t = cand;
			while (t) {
				const uint32_t b = __ffs(t) - 1;
				t &= t - 1;
				const uint32_t p = c0 + b;
				bool ok = (unsigned long long)off + p + P.run_min <= ulen;
				for (uint32_t i = 17; ok && i < P.run_min; i++) ok = in_class(P, gtile[p + i]);
				if (ok) keep |= 1u << b;
			}
			cand = keep;
		}
		if (!__any_sync(0xffffffffu, (cand & (cand - 1)) != 0)) {
			const uint32_t has = __ballot_sync(0xffffffffu, cand != 0);
			if (cand) {
				Cand c;
				c.pos = off + c0 + (__ffs(cand) - 1);
				c.len = 0;
				dst[__popc(has & ((1u << lane) - 1u))] = c;
			}
			return __popc(has);
		}
		return Emitter::emit_at(dst, cand, off + c0, [](uint32_t) -> uint32_t { return 0u; }, lane);
	}

	// rare: several candidates in one lane's 64 bytes -- general prefix sum, lane-major, low word first == position order
	static __device__ __noinline__ uint32_t emit_block_multi(Cand *dst, uint32_t lane, uint32_t clo, uint32_t chi, uint32_t pos0)
	{
		const uint32_t cnt = __popc(clo) + __popc(chi);
		uint32_t incl = cnt;
#pragma unroll
		for (int d = 1; d < 32; d <<= 1) {
			const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
			if ((int)lane >= d) incl += v;
		}
		const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
		uint32_t idx = incl - cnt;
		for (uint32_t t = clo; t; t &= t - 1) { Cand c; c.pos = pos0 + (__ffs(t) - 1); c.len = 0; dst[idx++] = c; }
		for (uint32_t t = chi; t; t &= t - 1) { Cand c; c.pos = pos0 + 32 + (__ffs(t) - 1); c.len = 0; dst[idx++] = c; }
		return total;
	}
	// long minimum: confirm bytes 17..n-1 of every candidate (global memory: they may lie in another warp's slice)
	static __device__ __noinline__ uint32_t confirm_long(const RunParams &P, const uint8_t *gtile, uint32_t off, uint32_t ulen, uint32_t cand, uint32_t c0)
	{
		uint32_t keep = 0;
		for (uint32_t t = cand; t; t &= t - 1) {
			const uint32_t b = __ffs(t) - 1, p = c0 + b;
			bool ok = (unsigned long long)off + p + P.run_min <= ulen;
			for (uint32_t i = 17; ok && i < P.run_min; i++) ok = in_class(P, gtile[p + i]);
			if (ok) keep |= 1u << b;
		}
		return keep;
	}
	// candidates of one 2 KiB block (64 bytes per lane: clo = bytes 0..31, chi = bytes 32..63) -> private list, in
	// position order; returns how many.  Common case (no lane has two): rank by ballot.
	static __device__ __forceinline__ uint32_t emit_block(const RunParams &P, const uint8_t *gtile, uint32_t off, uint32_t ulen, Cand *dst,
	                                                   uint32_t lane, uint32_t clo, uint32_t chi, uint32_t c0)
	{
		if (P.run_min > 17u) {
			clo = confirm_long(P, gtile, off, ulen, clo, c0);
			chi = confirm_long(P, gtile, off, ulen, chi, c0 + 32);
		}
		const uint32_t any = clo | chi;
		const bool one = (clo & (clo - 1)) == 0 && (chi & (chi - 1)) == 0 && (clo == 0 || chi == 0);
		if (__all_sync(0xffffffffu, one)) {
			const uint32_t has = __ballot_sync(0xffffffffu, any != 0);
			if (any) {
				Cand c;
				c.pos = off + c0 + (clo ? __ffs(clo) - 1 : 32 + __ffs(chi) - 1);
				c.len = 0;
				dst[__popc(has & ((1u << lane) - 1u))] = c;
			}
			return __popc(has);
		}
		return emit_block_multi(dst, lane, clo, chi, off + c0);
	}

	// One slice.  Full slices inside their unit run 2 KiB per warp step: every lane classifies 64 CONTIGUOUS bytes (four
	// 16-byte loads, the order rotated per lane pair so that a quarter warp still covers all 32 banks) into a 64-bit class
	// mask -- the cross-lane stitching (two shuffles), the "n ones start here" shifts and the vote are then paid once per
	// 64 bytes instead of once per 16.
	template <class G>
	static __device__ __forceinline__ void run(const RunParams &P, const Slice &S, Emitter &E, uint32_t lane)
	{
		constexpr int kRows = G::kSlice / 512, kBlocks = G::kSlice / 2048;
		static_assert(kBlocks >= 1 && kBlocks * 2048 == G::kSlice, "RUN scans blocks of 2 KiB");
		if (S.niter == 0) return;
		// is the byte just before the slice in the class?  (the unit's first byte has no predecessor)
		uint32_t prevbit = 0;
		if (S.off + S.begin > 0) prevbit = in_class(P, S.tile[(int)S.begin - 1]); // 16-byte look-behind copy
		const uint32_t send = S.begin + S.niter * 512;
		if (S.niter == (uint32_t)kRows && (unsigned long long)S.off + send <= S.ulen) {
			// ---- full slice inside the unit (also its last one: a 16 KiB file is four of these): no validity masks but on
			// the look-ahead bytes, everything in registers ----
			const unsigned long long after = (unsigned long long)S.ulen - S.off - send; // bytes of the unit behind the slice
			const uint32_t la_valid = after >= 16 ? 0xffffu : ((1u << (uint32_t)after) - 1u);
			const uint32_t rot = (lane >> 1) & 3u; // this lane loads its pieces in the order rot, rot + 1, ... (mod 4)
			const uint32_t sel_lo = (uint32_t)(0x5432765410763210ull >> (16 * rot)) & 0xffffu; // undo the rotation: byte selectors
			const uint32_t sel_hi = (uint32_t)(0x1076321054327654ull >> (16 * rot)) & 0xffffu; // for the low / high mask word
			uint32_t mlo[kBlocks], mhi[kBlocks], seen = 0;
#pragma unroll
			for (int b = 0; b < kBlocks; b++) {
				const uint8_t *base = S.tile + S.begin + b * 2048 + lane * 64;
				uint32_t m[4];
#pragma unroll
				for (int k = 0; k < 4; k++) {
					const uint8_t *pp = base + 16u * ((rot + (uint32_t)k) & 3u);
					m[k] = NHI == 0 ? mask16_ascii(P, pp, seen) : mask16_inner(P, pp);
				}
				const uint32_t a = __byte_perm(m[0], m[1], 0x5410), c = __byte_perm(m[2], m[3], 0x5410);
				mlo[b] = __byte_perm(a, c, sel_lo);
				mhi[b] = __byte_perm(a, c, sel_hi);
			}
			uint32_t la; // class mask of the 16 bytes after the slice: correct in lanes 0..3, consumed from lane 0 (by lane 31)
			{
				const uint32_t x = la_valid ? *reinterpret_cast<const uint32_t *>(S.tile + send + (lane & 3) * 4) : 0u; // no copy behind the unit's end
				seen |= x;
				uint32_t nib = (pack_top_nibble(NHI == 0 ? class_flags_ascii(P, x) : class_flags(P, x)) >> 28) << ((lane & 3) * 4);
				nib |= __shfl_xor_sync(0xffffffffu, nib, 1);
				nib |= __shfl_xor_sync(0xffffffffu, nib, 2);
				la = nib & la_valid;
			}
			if (NHI == 0 && __any_sync(0xffffffffu, (seen & kHigh) != 0)) {
				// a byte >= 0x80: the ASCII classification is void (carries between bytes) -- general out-of-line path
				E.n += run_tail(P, S.tile, S.gtile, S.off, S.ulen, S.begin, S.niter, prevbit, E.scratch + E.n, lane);
				return;
			}
			const uint32_t nxt_lane = (lane + 1) & 31, prv_lane = (lane + 31) & 31;
#pragma unroll
			for (int b = 0; b < kBlocks; b++) {
				// one shuffle brings the next lane's first 16 class bits and (for lane 31) lane 0's of the next block / the look-ahead
				const uint32_t follow = b + 1 < kBlocks ? (mlo[b + 1 < kBlocks ? b + 1 : b] & 0xffffu) : la;
				const uint32_t v = __shfl_sync(0xffffffffu, (mlo[b] & 0xffffu) | (follow << 16), nxt_lane);
				uint32_t ext = lane == 31 ? v >> 16 : v & 0xffffu;
				// one shuffle brings the previous lane's last bit and (for lane 0) lane 31's last bit of the previous block
				const uint32_t below = b ? mhi[b ? b - 1 : 0] >> 31 : prevbit;
				const uint32_t u = __shfl_sync(0xffffffffu, (mhi[b] >> 31) | (below << 1), prv_lane);
				const uint32_t pv = lane == 0 ? u >> 1 : u & 1u;
				// bits where at least min(run_min, 17) ones start, on the 80-bit window (own 64 + 16 of the follower)
				uint32_t rlo = mlo[b], rhi = mhi[b];
#pragma unroll
				for (int i = 0; i < 5; i++) {
					const uint32_t sh = P.sh[i];
					if (sh == 0) break; // the schedule is front-packed: nothing after the first zero
					rlo &= __funnelshift_r(rlo, rhi, sh);
					rhi &= __funnelshift_r(rhi, ext, sh);
					ext &= ext >> sh;
				}
				// run starts: class bit with the previous bit clear
				const uint32_t clo = rlo & mlo[b] & ~((mlo[b] << 1) | pv);
				const uint32_t chi = rhi & mhi[b] & ~__funnelshift_l(mlo[b], mhi[b], 1);
				if (__any_sync(0xffffffffu, (clo | chi) != 0))
					E.n += emit_block(P, S.gtile, S.off, S.ulen, E.scratch + E.n, lane, clo, chi, S.begin + b * 2048 + lane * 64);
			}
			return;
		}
		// ---- slices at the end of a unit / short tiles: same logic with per-byte validity, out of line ----
		E.n += run_tail(P, S.tile, S.gtile, S.off, S.ulen, S.begin, S.niter, prevbit, E.scratch + E.n, lane);
	}

	static __device__ __noinline__ uint32_t run_tail(const RunParams &P, const uint8_t *tile, const uint8_t *gtile, uint32_t off, uint32_t ulen,
	                                                 uint32_t begin, uint32_t niter, uint32_t prevbit, Cand *dst, uint32_t lane)
	{
		Slice S;
		S.tile = tile; S.gtile = gtile; S.extra = nullptr; S.off = off; S.ulen = ulen; S.tile_len = 0; S.begin = begin; S.niter = niter;
		const uint32_t send = begin + niter * 512;
		uint32_t n = 0;
		uint32_t cm_next = mask16(P, S, S.begin + lane * 16);
		for (uint32_t it = 0; it < S.niter; it++) {
			const uint32_t c0 = S.begin + it * 512 + lane * 16;
			const uint32_t cm = cm_next;
			if (it + 1 < S.niter) {
				cm_next = mask16(P, S, c0 + 512);
			} else {
				const uint32_t cb = send + (lane & 3) * 4;
				const long long rem = (long long)S.ulen - (long long)S.off - (long long)send;
				const uint32_t x = *reinterpret_cast<const uint32_t *>(S.tile + cb); // look-ahead copy (masked by `valid`)
				uint32_t nib = (pack_top_nibble(class_flags(P, x)) >> 28) << ((lane & 3) * 4);
				nib |= __shfl_xor_sync(0xffffffffu, nib, 1);
				nib |= __shfl_xor_sync(0xffffffffu, nib, 2);
				const uint32_t valid = rem >= 16 ? 0xffffu : (rem <= 0 ? 0u : ((1u << (int)rem) - 1u));
				cm_next = nib & valid;
			}
			const uint32_t la = __shfl_sync(0xffffffffu, cm_next, 0);
			uint32_t nx = __shfl_down_sync(0xffffffffu, cm, 1);
			if (lane == 31) nx = la;
			uint32_t pv = __shfl_up_sync(0xffffffffu, cm, 1) >> 15;
			if (lane == 0) pv = prevbit;
			prevbit = __shfl_sync(0xffffffffu, cm, 31) >> 15;
			const uint32_t starts = cm & ~((cm << 1) | pv);
			const uint32_t cand = starts & runs(P, cm | (nx << 16)) & 0xffffu;
			if (__any_sync(0xffffffffu, cand != 0)) n += emit_row(P, gtile, off, ulen, dst + n, lane, cand, c0);
		}
		return n;
	}
};

// ------------------------------------------------------------------------------------------
// NULL engine: moves every slice through the ring and looks at nothing.  Measures what the TMA
// streaming structure itself can pull from HBM (gscan_tma_probe) -- the ceiling of the scan kernels.
// ------------------------------------------------------------------------------------------
struct NullParams { uint32_t unused; };
struct NullEngine {
	typedef NullParams Params;
	static constexpr bool kLookBehind = false, kLookAhead = false, kMergeCopies = false;
	static __device__ __forceinline__ void prologue(const NullParams &, uint8_t *) {}
	template <class G>
	static __device__ __forceinline__ void run(const NullParams &, const Slice &S, Emitter &E, uint32_t lane)
	{
		// touch one word per row so the copy cannot be elided and the slot is really consumed
		uint32_t x = 0;
		for (uint32_t it = 0; it < S.niter; it++) x ^= *reinterpret_cast<const uint32_t *>(S.tile + S.begin + it * 512 + lane * 16);
		if (x == 0x9e3779b9u && S.ulen == 0xffffffffu) E.n += 1; // never true; keeps x alive
	}
};

// ------------------------------------------------------------------------------------------
// the persistent kernel: warp-private TMA rings
// ------------------------------------------------------------------------------------------
// Slice s = (tile << spt_shift) + j is the j-th kSlice-byte part of a tile.  Warp g (of all G warps of the grid) starts with
// slices g, g + G, ..., g + (kRing - 1) G and then takes runs of slices from a shared counter.  Each warp keeps kRing slices
// in flight: after finishing a slice its lane 0 re-arms the slot's mbarrier and issues the bulk copy for the warp's next
// slice.  No producer warp, no "empty" barriers, no __syncthreads.
template <class G>
__device__ __forceinline__ void slice_geometry(const TileDesc &d, uint32_t j, uint32_t &begin, uint32_t &niter)
{
	// slice j of a tile is its bytes [j * kSlice, (j + 1) * kSlice): full slices wherever the unit has the bytes
	// (a 16 KiB file in a 16 KiB tile is 4 slices of 8 rows), an empty one (niter 0) past the end of a short tile
	begin = j * (uint32_t)G::kSlice;
	niter = 0;
	if (begin < d.len) {
		const uint32_t end = begin + (uint32_t)G::kSlice < d.len ? begin + (uint32_t)G::kSlice : d.len;
		niter = (end - begin + 511u) >> 9;
	}
}

template <class Eng, class G>
__global__ void __launch_bounds__(G::kThreads, 1)
scan_kernel(const __grid_constant__ ScanArgs A, const __grid_constant__ typename Eng::Params P)
{
	extern __shared__ __align__(128) uint8_t smem[];
	const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	constexpr uint32_t kPre = Eng::kLookBehind ? kHalo : 0u;
	constexpr uint32_t slot_bytes = G::kSlice + kPre + kHalo;
	uint8_t *my = smem + (size_t)warp * G::kRing * slot_bytes;
	SlotCtl *ctl = reinterpret_cast<SlotCtl *>(smem + (size_t)G::kWarps * G::kRing * slot_bytes) + warp * G::kRing;
	uint8_t *extra = smem + (size_t)G::kWarps * G::kRing * (slot_bytes + sizeof(SlotCtl)) + 64;
	Eng::prologue(P, extra);

	const uint32_t total = A.n_tiles << A.spt_shift, spt_mask = (1u << A.spt_shift) - 1u;
	const uint32_t stride = gridDim.x * G::kWarps;
	const uint32_t first = blockIdx.x * G::kWarps + warp;

	if (lane == 0) {
		for (int s = 0; s < G::kRing; s++) mbar_init(&ctl[s].full, 1);
		mbar_fence_init();
	}
	__syncwarp();

	const uint64_t policy = l2_stream_policy();
	// lane 0: describe slice `s` in slot `slot` and start its copy
	auto issue = [&](uint32_t slot, uint32_t s, const TileDesc &d) {
		uint32_t begin, niter;
		slice_geometry<G>(d, s & spt_mask, begin, niter);
		SlotCtl *c = &ctl[slot];
		c->slice = s;
		c->src = d.src; c->off = d.off; c->ulen = d.ulen; c->tile_len = d.len; c->begin = begin; c->niter = niter;
		if (niter == 0) { mbar_arrive(&c->full); return; }
		const uint32_t rest = (d.ulen - d.off - begin + 15u) & ~15u; // rest of the unit from the slice start, padded to 16
		const uint32_t bytes = rest > niter * 512u ? niter * 512u : rest;
		const bool behind = Eng::kLookBehind && (d.off + begin) != 0;
		const bool ahead = Eng::kLookAhead && rest >= niter * 512u + kHalo;
		uint8_t *dst = my + (size_t)slot * slot_bytes + kPre;
		mbar_arrive_expect_tx(&c->full, bytes + (behind ? kHalo : 0u) + (ahead ? kHalo : 0u));
		if constexpr (Eng::kMergeCopies) {
			// the bytes before / after the slice are contiguous with it on both sides: ONE bulk copy.  (The issue-bound engines
			// save ~20 instructions per extra copy; the HBM-bound pair filter keeps its 512-byte aligned slice copy -- an
			// unaligned one re-reads the boundary sectors.)
			const uint32_t pre = behind ? kHalo : 0u;
			tma_load_1d(dst - pre, reinterpret_cast<const void *>(d.src + begin - pre), bytes + pre + (ahead ? kHalo : 0u), &c->full, policy);
		} else {
			tma_load_1d(dst, reinterpret_cast<const void *>(d.src + begin), bytes, &c->full, policy);
			if (behind) tma_load_1d(dst - kHalo, reinterpret_cast<const void *>(d.src + begin - kHalo), kHalo, &c->full, policy);
			if (ahead) tma_load_1d(dst + niter * 512u, reinterpret_cast<const void *>(d.src + begin + niter * 512u), kHalo, &c->full, policy);
		}
	};

	if (lane == 0) {
		for (uint32_t k = 0; k < (uint32_t)G::kRing; k++) {
			const uint32_t s = first + k * stride;
			if (s < total) issue(k, s, A.tiles[s >> A.spt_shift]);
			else ctl[k].slice = kNoSlice;
		}
	}
	__syncwarp();
	// the first kRing slices of every warp are static (above); every later one comes from a shared counter, kDynRun
	// consecutive slices per atomicAdd (one counter serves ~500 M atomics/s: one per 4 KiB slice would cap the kernel near
	// 2 TB/s), so the warps stay together in the stream and an SM that runs ahead takes more slices instead of idling at
	// the end.  A warp takes its slices in increasing order, so once a slot has no slice, no later slot has one.
	constexpr uint32_t kDynRun = 4; // a power of two
	const uint32_t dyn0 = G::kRing * stride;
	uint32_t run_next = dyn0; // lane 0: the warp's next slice; a new run is taken whenever it reaches a run boundary

	Emitter E;
	E.scratch = A.scratch + ((size_t)blockIdx.x * G::kWarps + warp) * G::kSlice;
	E.n = 0;
	uint32_t slot = 0, phase = 0;
	for (;;) {
		const uint32_t s = ctl[slot].slice;
		if (s == kNoSlice) break;
		// the slice that will reuse this slot and its descriptor: taken now, needed after the scan
		uint32_t nxt = kNoSlice;
		TileDesc dn;
		if (lane == 0) {
			if (((run_next - dyn0) & (kDynRun - 1u)) == 0) run_next = dyn0 + atomicAdd(A.next_slice, kDynRun);
			nxt = run_next < total ? run_next : kNoSlice;
			run_next++;
			if (nxt < total) dn = A.tiles[nxt >> A.spt_shift];
		}

		mbar_wait(&ctl[slot].full, phase);
		Slice S;
		S.off = ctl[slot].off;
		S.ulen = ctl[slot].ulen;
		S.tile_len = ctl[slot].tile_len;
		S.begin = ctl[slot].begin;
		S.niter = ctl[slot].niter;
		S.tile = my + (size_t)slot * slot_bytes + kPre - S.begin; // address of tile byte 0 (only the slice window is resident)
		S.gtile = reinterpret_cast<const uint8_t *>(ctl[slot].src);
		S.extra = extra;
		Eng::template run<G>(P, S, E, lane);
		E.flush(A, s, lane);
		__syncwarp(); // every lane is done reading the slot before it is overwritten
		if (lane == 0) {
			if (nxt < total) issue(slot, nxt, dn);
			else ctl[slot].slice = kNoSlice;
		}
		__syncwarp(); // the slot's slice number is visible to every lane when the warp comes back to it
		if (++slot == (uint32_t)G::kRing) { slot = 0; phase ^= 1u; }
	}
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
constexpr int kMaxDevices = 64;

template <class G>
static ScanGeom geom_of() { return ScanGeom{G::kWarps, G::kRing, G::kSlice}; }

template <class Eng, class G>
static cudaError_t launch_g(const ScanArgs &A, const typename Eng::Params &P, int grid, cudaStream_t st)
{
	const int smem = (int)(scan_smem_bytes(geom_of<G>(), Eng::kLookBehind) + A.extra_smem);
	// the shared-memory limit is a property of the kernel on a device: raised once per instantiation and device, not per
	// launch (the largest size asked for so far; the hashed engine's table size varies with the pattern)
	static std::atomic<int> smem_set[kMaxDevices];
	int dev = 0;
	cudaError_t e = cudaGetDevice(&dev);
	if (e != cudaSuccess) return e;
	if (dev >= kMaxDevices || smem > smem_set[dev].load(std::memory_order_acquire)) {
		e = cudaFuncSetAttribute(scan_kernel<Eng, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
		if (e != cudaSuccess) return e;
		if (dev < kMaxDevices) smem_set[dev].store(smem, std::memory_order_release);
	}
	scan_kernel<Eng, G><<<grid, G::kThreads, smem, st>>>(A, P);
	return cudaGetLastError();
}

// which geometry a kernel (GSCAN_KERNEL_*) runs with: the Geom its case of launch_scan below instantiates
ScanGeom scan_geom(int kernel)
{
	switch (kernel) {
	case GSCAN_KERNEL_BALANCED: return geom_of<GeomPair>();
	case GSCAN_KERNEL_HASH: return geom_of<GeomHash>();
	case GSCAN_KERNEL_RUN: return geom_of<GeomBalanced>();
	default: return geom_of<GeomStream>(); // PAIR, TRIPLE; NONE runs no scan kernel
	}
}

cudaError_t launch_scan_null(const ScanArgs &A, int geom, int grid, cudaStream_t st)
{
	NullParams P{0};
	if (geom == 0) return launch_g<NullEngine, GeomStream>(A, P, grid, st);
	return launch_g<NullEngine, GeomBalanced>(A, P, grid, st);
}

// the per-family K tables of launch_scan: an engine instantiated for K tests runs any count up to K (unused tests never pass)
template <int D, bool EX>
static cudaError_t launch_pair(const ScanArgs &A, const FixedParams &P, int grid, cudaStream_t st)
{
	switch (P.ntests) {
	case 1: return launch_g<FixedEngine<D, 1, EX>, GeomStream>(A, P, grid, st);
	case 2: return launch_g<FixedEngine<D, 2, EX>, GeomStream>(A, P, grid, st);
	case 3: return launch_g<FixedEngine<D, 3, EX>, GeomStream>(A, P, grid, st);
	case 4: return launch_g<FixedEngine<D, 4, EX>, GeomStream>(A, P, grid, st);
	case 5: case 6: return launch_g<FixedEngine<D, 6, EX>, GeomStream>(A, P, grid, st);
	default: return launch_g<FixedEngine<D, 8, EX>, GeomStream>(A, P, grid, st);
	}
}

template <bool EX>
static cudaError_t launch_triple(const ScanArgs &A, const FixedParams &P, int grid, cudaStream_t st)
{
	switch (P.n2) {
	case 1: return launch_g<Fixed3Engine<1, EX>, GeomStream>(A, P, grid, st);
	case 2: return launch_g<Fixed3Engine<2, EX>, GeomStream>(A, P, grid, st);
	case 3: return launch_g<Fixed3Engine<3, EX>, GeomStream>(A, P, grid, st);
	case 4: return launch_g<Fixed3Engine<4, EX>, GeomStream>(A, P, grid, st);
	case 5: case 6: return launch_g<Fixed3Engine<6, EX>, GeomStream>(A, P, grid, st);
	default: return launch_g<Fixed3Engine<8, EX>, GeomStream>(A, P, grid, st);
	}
}

template <int D, bool AL>
static cudaError_t launch_balanced(const ScanArgs &A, const FixedParams &P, int grid, cudaStream_t st)
{
	switch (P.ntests) {
	case 2: return launch_g<FixedBEngine<D, 2, AL>, GeomPair>(A, P, grid, st);
	case 3: return launch_g<FixedBEngine<D, 3, AL>, GeomPair>(A, P, grid, st);
	case 4: return launch_g<FixedBEngine<D, 4, AL>, GeomPair>(A, P, grid, st);
	case 5: case 6: return launch_g<FixedBEngine<D, 6, AL>, GeomPair>(A, P, grid, st);
	default: return launch_g<FixedBEngine<D, 8, AL>, GeomPair>(A, P, grid, st);
	}
}

template <int NHI, int NFO>
static cudaError_t launch_run(const ScanArgs &A, const RunParams &P, int grid, cudaStream_t st)
{
	switch (P.nlo) {
	case 0: case 1: return launch_g<RunEngine<1, NHI, NFO>, GeomBalanced>(A, P, grid, st);
	case 2: return launch_g<RunEngine<2, NHI, NFO>, GeomBalanced>(A, P, grid, st);
	case 3: return launch_g<RunEngine<3, NHI, NFO>, GeomBalanced>(A, P, grid, st);
	case 4: return launch_g<RunEngine<4, NHI, NFO>, GeomBalanced>(A, P, grid, st);
	case 5: case 6: return launch_g<RunEngine<6, NHI, NFO>, GeomBalanced>(A, P, grid, st);
	default: return launch_g<RunEngine<8, NHI, NFO>, GeomBalanced>(A, P, grid, st);
	}
}

cudaError_t launch_scan(int kernel, const ScanArgs &A, const FixedParams &F, const HashParams &H, const RunParams &R, int delta,
                        int grid, cudaStream_t st)
{
	switch (kernel) {
	case GSCAN_KERNEL_PAIR:
		switch (delta) {
		case 0: return launch_pair<0, false>(A, F, grid, st); // a single-byte filter is never exact (gscan_compile)
		case 1: return F.exact ? launch_pair<1, true>(A, F, grid, st) : launch_pair<1, false>(A, F, grid, st);
		case 2: return F.exact ? launch_pair<2, true>(A, F, grid, st) : launch_pair<2, false>(A, F, grid, st);
		case 3: return F.exact ? launch_pair<3, true>(A, F, grid, st) : launch_pair<3, false>(A, F, grid, st);
		default: return F.exact ? launch_pair<4, true>(A, F, grid, st) : launch_pair<4, false>(A, F, grid, st);
		}
	case GSCAN_KERNEL_TRIPLE: return F.exact3 ? launch_triple<true>(A, F, grid, st) : launch_triple<false>(A, F, grid, st);
	case GSCAN_KERNEL_BALANCED:
		switch (delta) {
		case 1: return F.b_aligned ? launch_balanced<1, true>(A, F, grid, st) : launch_balanced<1, false>(A, F, grid, st);
		case 2: return F.b_aligned ? launch_balanced<2, true>(A, F, grid, st) : launch_balanced<2, false>(A, F, grid, st);
		case 3: return F.b_aligned ? launch_balanced<3, true>(A, F, grid, st) : launch_balanced<3, false>(A, F, grid, st);
		default: return F.b_aligned ? launch_balanced<4, true>(A, F, grid, st) : launch_balanced<4, false>(A, F, grid, st);
		}
	case GSCAN_KERNEL_HASH: return launch_g<HashEngine, GeomHash>(A, H, grid, st);
	case GSCAN_KERNEL_RUN:
		switch (R.nhi) {
		case 0: return R.nfold ? launch_run<0, 1>(A, R, grid, st) : launch_run<0, 0>(A, R, grid, st);
		case 1: return R.nfold ? launch_run<1, 1>(A, R, grid, st) : launch_run<1, 0>(A, R, grid, st);
		default: return R.nfold ? launch_run<2, 1>(A, R, grid, st) : launch_run<2, 0>(A, R, grid, st);
		}
	}
	return cudaErrorInvalidValue; // GSCAN_KERNEL_NONE: the pattern has no scan kernel
}

} // namespace gscan
