// device_types.h -- PODs shared by host code and kernels (layout in HBM; see DESIGN.md).
#pragma once
#include <cstdint>

namespace gscan {

// Geometry.  A tile (the planning unit, one 32-byte descriptor) is up to 2^tile_shift bytes of one unit --
// 64 KiB for batches of big units, down to 4 KiB for batches of many small files (the batch planner picks
// the power of two next to the average unit length, so a 16 KiB file is four full 4 KiB slices and not a
// sixteenth of a 64 KiB tile each); the scan kernel cuts a tile into slices of Geom::kSlice bytes, the
// amount one warp scans per step.  Geometry is a template parameter of the kernel, chosen per engine
// (memory-bound filters want a deep ring, instruction-bound ones want as many warps as fit).
constexpr int kTileBytes = 65536;     // largest tile
constexpr int kMinTileShift = 12, kMaxTileShift = 16;
constexpr int kSmemBudget = 227 * 1024;

template <int W, int R, int S>
struct Geom {
	static constexpr int kWarps = W;          // warps per CTA, every one an independent scanner
	static constexpr int kRing = R;           // slices in flight per warp
	static constexpr int kSlice = S;          // bytes one warp scans per step (rows of 512)
	static_assert(S >= 512 && S <= (1 << kMinTileShift) && (S & (S - 1)) == 0, "a slice is a power of two that divides the smallest tile");
	static constexpr int kThreads = W * 32;
};
typedef Geom<16, 3, 4096> GeomStream;  // memory-bound: the FIXED filters
// RUN (class runs): ALU/issue-bound, 24 warps; 4 KiB slices with a 2-deep ring do half the ring work per byte of
// <24, 4, 2048>
typedef Geom<24, 2, 4096> GeomBalanced;
// hashed engine: issue-bound, wants warps (20 = 5 per scheduler) and
// long slices (fewer ring refills per byte): 2 x 4 KiB per warp, which leaves 32 KiB for the table
typedef Geom<20, 2, 4096> GeomHash;
// balanced pair filter (FixedBEngine): issue-bound like the hashed engine
typedef Geom<20, 2, 4096> GeomPair;

struct ScanGeom { int warps, ring, slice; }; // host-side mirror of the chosen Geom

// One tile of one unit.  Built on the host when a batch is planned, 32 bytes.
struct TileDesc {
	uint64_t src;   // global address of the tile's first byte (16-byte aligned)
	uint32_t unit;  // index into the batch's unit table
	uint32_t off;   // offset of the tile inside the unit
	uint32_t len;   // bytes of the unit inside this tile (<= kTileBytes)
	uint32_t ulen;  // length of the unit
	uint32_t pad[2];
};
static_assert(sizeof(TileDesc) == 32, "TileDesc layout");

// One segment == one slice; candidates of a segment are contiguous and ordered in the candidate
// buffer.  seg id = (tile << spt_shift) + slice.
struct SegEntry { uint32_t base, n; }; // n: low 16 bits count (<= slice bytes), high 16 bits generation tag of the scan that wrote it
__host__ __device__ inline uint32_t seg_count(const SegEntry &e, uint32_t tag) { return (e.n >> 16) == tag ? (e.n & 0xffffu) : 0u; }

// A candidate / match inside a unit.
struct Cand { uint32_t pos, len; };

// An ordered, resolved match: what goes back to the host.
struct OutRec { uint32_t unit, pos, len, pad; };

struct FixedParams {
	uint32_t one;         // == 1, opaque to the compiler: x * one + c issues as IMAD (FMA pipe) instead of IADD (ALU pipe)
	uint32_t exact;       // every filter mask is 0xff
	uint32_t ntests;
	uint32_t m0[8], v0[8], m1[8], v1[8]; // byte replicated x4
	uint32_t anchor;      // pattern byte the filter stream is anchored on
	uint32_t nseq;
	uint32_t uniform_len; // != 0: every sequence has this length
	uint32_t maxlen;
	const uint16_t *seq_len;  // [nseq]
	const uint32_t *seq_off;  // [nseq] index into seq_pos
	const uint32_t *seq_pos;  // per position: mask | val << 8 | cls << 16 (cls 0xffff: none)
	const uint32_t *cls_bm;   // [ncls][8] bitmaps for positions that are not a masked equality
	// triples (anchor, anchor + delta, anchor + d2): stage 2 of the pair filter (flagged rows only), or the stage-1
	// filter itself (Fixed3Engine; sh1/sh2 = 8*delta, 8*d2 funnel-shift amounts, 8-byte aligned: the triple filter reads
	// them with one 64-bit load)
	uint32_t n2, d2, sh1, sh2, exact3;
	// balanced pair filter (FixedBEngine): test k is (w | 0x80..) + b_c0[k]; the third byte of alternative k (stage 2,
	// aligned with test k) is ((s2 & b_m2[k]) ^ b_v2[k]) == 0, s2 = the bytes b_sh2 / 8 further on
	uint32_t b_aligned, b_sh2;
	uint32_t b_c0[8], b_c1[8], b_m2[8], b_v2[8];
	uint32_t t2_m0[16], t2_v0[16], t2_m1[16], t2_v1[16], t2_m2[16], t2_v2[16];
};

// FIXED, hashed: exact membership of the 2 or 3 bytes at every position in a perfect-hash table held in
// shared memory; hits are verified against the alternatives sharing the key
struct HashParams {
	uint32_t mulsh;      // h = window * mulsh (mulsh = mul << 8 * (4 - L): the bytes beyond the key fall off the top, no mask);
	uint32_t nslots;     //   slot = umulhi(h, nslots): IMADs only, nothing on the ALU pipe
	uint32_t stride;     // bytes between slots in shared memory: 128 when the table is replicated per bank, else 4
	uint32_t neg1;       // == 0xffffffff, opaque to the compiler: h * neg1 + entry is an IMAD (FMA pipe) where a XOR would be ALU
	// class prefilter (sparse path): every key byte lies in [pre_lo, pre_hi] (one range inside 0x01-0x7d); a position can
	// only hold a key when its hash_len bytes all pass x in [pre_lo, pre_hi + 1] -- tested SWAR, the table is then probed
	// at the surviving positions only.  pre_enable == 0: no usable range, every position is probed (dense path).
	uint32_t one;        // == 1, opaque: x * one + c issues as IMAD
	uint32_t hash_len;   // key bytes (2 or 3)
	uint32_t pre_enable;
	uint32_t pre_ge, pre_gt;  // (0x80 - lo) x4, (0x7e - hi) x4: bit 7 of x + pre_ge set and of x + pre_gt clear <=> lo <= x <= hi + 1
	uint32_t pre_mul[7];      // 1 << (25 + k): umulhi(flags, pre_mul[k]) == flags >> (7 - k) on the FMA pipe
	const uint4 *tail;        // [nslots] {mask_lo, val_lo, mask_hi, val_hi}: bytes 0..7 behind a key position must satisfy
	                          // ((y_lo ^ val_lo) & mask_lo) | ((y_hi ^ val_hi) & mask_hi) == 0 for ANY alternative of the key to
	                          // match (all-zero masks: no cheap statement) -- drops most key hits before the verification
	const uint32_t *table;      // [nslots] h of the slot's key, or 0xffffffff (copied to shared memory at kernel start)
	const uint32_t *slot_first; // [nslots] first index into slot_seqs
	const uint32_t *slot_count; // [nslots]
	const uint32_t *slot_seqs;  // alternatives of a key, preference order
	const uint16_t *seq_len;
	const uint32_t *seq_off;
	const uint32_t *seq_pos;
	const uint32_t *cls_bm;
};
constexpr int kHashMaxSlots = 8192;
// copies of the table in shared memory (slot s, copy c at word s * copies + c; lane l reads copy l): 32 copies put every
// lane of a warp on its own bank -- one wavefront per lookup instead of ~3.4 for random slots (and 2 with 16 copies: at
// 16 lookups per 512-byte row that alone caps the kernel's throughput).  512 slots x 128 bytes = 64 KiB, beside a 20-warp ring
// of 2 x 4 KiB slots
constexpr uint32_t kHashReplicatedSlots = 512;
static inline uint32_t hash_table_copies(uint32_t nslots) { return nslots <= kHashReplicatedSlots ? 32u : 1u; }

struct RunParams {
	uint32_t one;         // == 1, opaque (see FixedParams)
	uint32_t nlo, nhi;
	uint32_t add_ge_lo[8], add_gt_lo[8]; // (0x80-lo)*0x01010101, (0x7f-hi)*0x01010101 for ranges in 0x00-0x7f
	uint32_t add_ge_hi[2], add_gt_hi[2]; // same for ranges in 0x80-0xff (after clearing bit 7)
	uint32_t nfold, add_ge_fold, add_gt_fold; // one pair of ranges that differ only in bit 5, tested once on x | 0x20
	uint32_t run_min;
	uint32_t sh[5];      // w &= w >> sh[i], i = 0..4: leaves the bits where min(run_min, 17) ones start (0 = no-op)
	uint32_t bitmap[8];
};

struct ScanArgs {
	const TileDesc *tiles;
	uint32_t n_tiles;
	Cand *cand;
	uint32_t cand_cap;
	unsigned long long *cursor; // [0]: candidate slots reserved so far (in chunks: an upper bound of the candidates written)
	uint32_t chunk;             // slots a warp reserves per atomicAdd
	uint32_t *next_slice;       // zero at launch: slices taken from the shared counter so far (the kernel's dynamic schedule)
	SegEntry *segs;
	uint32_t *occ;  // one bit per segment, set with every entry written: the resolve reads only the entries whose bit is set
	Cand *scratch;  // [gridDim.x * warps][slice bytes]: one private list per warp
	uint32_t spt_shift;  // log2(slices per tile) = batch tile_shift - log2(Geom::kSlice)
	uint32_t extra_smem; // bytes of engine-private shared memory behind the rings (hash table)
	uint32_t tag;        // generation of this scan (1..65535), stored in the segment entries it writes
};

} // namespace gscan
