// pattern.h -- host-side pattern compiler: PCRE subset -> device automaton tables.
//
// Replaces what FileGrep::prepare gets from libpcre (/root/reference/src/grab.cc:101-123):
// pcre_compile(regex, options = 0, ...), pcre_study and PCRE_INFO_MINLENGTH.  Semantics are
// PCRE's with options 0: bytes (no UTF), case-sensitive unless (?i), '.' excludes '\n',
// "C"-locale classes (pcre_maketables() without setlocale, grab.cc:106), leftmost-first
// alternation.  Instead of byte code for a backtracking interpreter the output is one of two
// data-parallel programs:
//   FIXED : ordered list of fixed-length byte-class sequences (literals, alternations, classes,
//           bounded repeats expanded in backtracking order) + a SWAR byte-pair filter
//   RUN   : one byte class repeated {n,} greedily, as SWAR range tests
// Anything else is rejected loudly: there is no CPU fallback for the scan.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

namespace gscan {

struct ByteSet {
	uint32_t w[8];
	ByteSet() { for (auto &x : w) x = 0; }
	void add(unsigned c) { w[(c & 255) >> 5] |= 1u << (c & 31); }
	bool has(unsigned c) const { return (w[(c & 255) >> 5] >> (c & 31)) & 1u; }
	void add_range(unsigned lo, unsigned hi) { for (unsigned c = lo; c <= hi; c++) add(c); }
	void invert() { for (auto &x : w) x = ~x; }
	void unite(const ByteSet &o) { for (int i = 0; i < 8; i++) w[i] |= o.w[i]; }
	bool intersects(const ByteSet &o) const { for (int i = 0; i < 8; i++) if (w[i] & o.w[i]) return true; return false; }
	bool subset_of(const ByteSet &o) const { for (int i = 0; i < 8; i++) if (w[i] & ~o.w[i]) return false; return true; }
	bool operator==(const ByteSet &o) const { for (int i = 0; i < 8; i++) if (w[i] != o.w[i]) return false; return true; }
	int count() const { int n = 0; for (auto x : w) n += __builtin_popcount(x); return n; }
	bool empty() const { return count() == 0; }
};

// {x : (x & mask) == val}; exact == true when that set equals the class itself
struct MaskedEq {
	uint8_t mask, val;
	bool exact;
	int size; // number of bytes passing the test
};
MaskedEq masked_superset(const ByteSet &s);

struct ByteRange { uint8_t lo, hi; };
std::vector<ByteRange> to_ranges(const ByteSet &s);

typedef std::vector<ByteSet> Sequence;

struct FilterTest {
	uint8_t m0, v0, m1, v1; // (byte[p] & m0) == v0 && (byte[p+d] & m1) == v1
	bool operator==(const FilterTest &o) const { return m0 == o.m0 && v0 == o.v0 && m1 == o.m1 && v1 == o.v1; }
};

enum EngineKind { ENGINE_FIXED = 1, ENGINE_RUN = 2, ENGINE_NONE = 3 };

// device VM (resolve_kernels.cu) instruction set
enum { VM_SET = 0, VM_SPLIT = 1, VM_JMP = 2, VM_REP = 3, VM_ASSERT = 4, VM_MATCH = 5, VM_CAP = 6 /* a capturing group closed (Q2) */,
       VM_LOOK = 7 /* kind: VM_LK_*, a: pc behind the construct, b: bytes to step back (lookbehind) */, VM_LOOKEND = 8 };
enum { VM_LK_AHEAD = 0, VM_LK_AHEAD_NEG = 1, VM_LK_BEHIND = 2, VM_LK_BEHIND_NEG = 3, VM_LK_ATOMIC = 4 };
enum { VM_Q_GREEDY = 0, VM_Q_LAZY = 1, VM_Q_POSSESSIVE = 2 };
enum { VM_A_BOL = 0, VM_A_EOL = 1, VM_A_SOS = 2, VM_A_EOS = 3, VM_A_EOSNL = 4, VM_A_WORDB = 5, VM_A_NWORDB = 6, VM_A_MBOL = 7, VM_A_MEOL = 8 };

constexpr int kMaxFilterTests = 8;
constexpr int kMaxPatternLen = 1024;   // longest sequence the smem halo can verify
constexpr int kMaxSequences = 4096;
constexpr int kMaxRunRangesLow = 8, kMaxRunRangesHigh = 2;

struct Program {
	EngineKind kind = ENGINE_FIXED;
	int minlen = 0, maxlen = 0; // maxlen -1: unbounded
	int captures = 0;
	bool strict_q2 = false;
	bool cap_stops = false;   // Q2, mixed: only some matches set a capturing group -- the VM reports which, the first such match ends its unit

	// FIXED
	std::vector<Sequence> seqs;       // in PCRE preference order
	std::vector<FilterTest> tests;    // deduplicated
	int anchor = 0, delta = 0;        // filter bytes are pattern[anchor], pattern[anchor+delta]
	struct Triple { uint8_t m0, v0, m1, v1, m2, v2; };
	std::vector<Triple> triples;      // stage-2 refinement with a third byte at anchor+delta2 (empty: none)
	int delta2 = 0;
	double pair_flag_prior = 0;       // estimated probability that the pair filter flags a byte (static text prior)
	bool disjoint = false;            // no two matches can ever overlap => resolve is a pure copy

	// FIXED, hashed variant (many alternatives): the first hash_len bytes of every alternative are keys of
	// a perfect-hash table; membership of the text's bytes at p is EXACT, then only the alternatives that
	// share the key are verified
	bool use_hash = false;
	int hash_len = 0;                       // 2 or 3 key bytes
	uint32_t hash_mul = 0, hash_slots = 0;  // slot = umulhi(key * (mul << 8 * (4 - hash_len)) mod 2^32, slots)
	std::vector<uint32_t> hash_table;       // [slots] key, 0xffffffff = empty
	std::vector<uint32_t> slot_first, slot_count, slot_seqs; // alternatives per slot, preference order

	// RUN
	ByteSet run_class;
	int run_min = 0;
	std::vector<ByteRange> ranges_low, ranges_high; // within 0x00-0x7F / 0x80-0xFF

	// general patterns: seqs are the leading-byte prefixes (candidate filter), matches are decided by the VM
	bool use_vm = false;
	bool vm_runstart = false;      // candidates are the starts of runs of run_class (pattern begins with C{n,})
	bool vm_dense = false;         // no useful candidate filter (the match can begin with (almost) any byte): the VM walk tries every
	                               // position whose byte is in first_set itself, no scan kernel runs -- PCRE does the same on the CPU
	ByteSet first_set;             // vm_dense: bytes a match can start with
	int vm_reach = 0;              // sound upper bound L: an attempt at p has the same outcome for every subject beginning s <= p - L
	                               // (only ^ \A \b \B (?m)^ and look-behinds near the attempt's first byte look at s; 1: the
	                               // attempt at s itself differs from "any earlier start", resolve: GSCAN_RESOLVE_VM_TWO)
	bool vm_start_free = false;    // vm_reach == 0: an anchored attempt at a position gives the same result wherever the subject
	                               // begins, so the attempts of a unit's candidates can run in parallel (resolve: GSCAN_RESOLVE_VM_ATTEMPTS)
	int vm_lead = 0;               // vm_runstart: VM_Q_* of the leading repeat (after (?U))
	std::vector<uint32_t> vm_code; // 3 words per instruction
	std::vector<uint32_t> vm_sets; // 8 words per byte class

	uint64_t id = 0; // unique per compiled pattern (device-table cache key)
};

// Returns true and fills `out`; false and `err` otherwise.
bool compile_pattern(const char *pat, size_t len, uint32_t flags, Program &out, std::string &err);

} // namespace gscan
