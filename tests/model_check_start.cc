// model_check_start.cc -- CPU check of the resolve paths for general patterns whose attempts look at or before their first
// byte (Program::vm_reach) and of class-repeat-led patterns (Program::vm_runstart), with the device's own source (the VM and
// the chain kernels of resolve_kernels.cu, extracted by tests/test_model_start.py) compiled for the host:
//   1. reach soundness: an attempt at p gives the same outcome from every subject beginning s <= p - vm_reach; and the check
//      catches a reach reported one too small (it must find a disagreement for patterns whose reach is exact)
//   2. reach-1 programs, two outcomes per candidate (vm_two): filtered (k_vm_attempts) and dense (k_vm_dense), then the chain
//   3. greedy / possessive class-repeat-led programs on the chain (vm_chain_run, k_vm_resume)
// against the oracle's loop in all three modes (ALL / FIRST / LINE), for single units and two-unit batches, with and without
// the capturing-group quirk (Q2, STRICT_REF).
// Usage: model_check_start PATTERN_FILE   (one pattern per line)
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "../include/gscan.h"
#include "../grab_b200/csrc/pattern.h"
#include "../grab_b200/csrc/kernels.h"
extern "C" {
#include "../oracle/grab_oracle.h"
}

#undef __device__
#undef __global__
#undef __forceinline__
#undef __launch_bounds__
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

static uint64_t rng_state = 0x9e3779b97f4a7c15ull;
static uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (uint32_t)(rng_state >> 9); }

struct M { uint64_t pos; uint32_t len; };
typedef std::vector<uint8_t> Bytes;

// steps an attempt, or all attempts of a unit together, may take here: pathological patterns of the random grammar end in the
// VM limit (those checks are skipped) in milliseconds instead of seconds
constexpr unsigned long long kModelSteps = 200000;

// ---- 1. reach soundness ----
// outcome of the attempt at p when the subject begins at s: rc and absolute end
static std::pair<int, uint64_t> attempt(const Program &p, const Bytes &b, size_t s, size_t pos)
{
	ResolveArgs R;
	memset(&R, 0, sizeof R);
	R.vm_code = p.vm_code.data();
	R.vm_sets = p.vm_sets.data();
	VmBudget budget(b.size());
	budget.search = budget.unit = kModelSteps; // the same path takes the same steps: a sound reach agrees on the limit too
	uint32_t e = 0;
	const int rc = vm_exec(R, b.data() + s, (uint32_t)(b.size() - s), (uint32_t)(pos - s), &e, budget);
	return {rc, rc > 0 ? s + e : 0};
}

static long g_reach_checks = 0;
// number of (p, s) where an attempt from s <= p - reach differs from the one from p - reach.  Every s on short subjects, the
// ones next to 0 and to p - reach on longer ones (an attempt tells the starts behind p - reach apart only through sp == 0)
static long reach_violations(const Program &p, const std::vector<Bytes> &subjects, int reach)
{
	long bad = 0;
	for (auto &b : subjects) {
		const size_t n = b.size();
		for (size_t pos = (size_t)reach; pos < n; pos++) {
			const size_t s0 = pos - (size_t)reach;
			const auto want = attempt(p, b, s0, pos);
			for (size_t s = 0; s < s0; s++) {
				if (n > 16 && s > 2 && s + 3 < s0) continue;
				g_reach_checks++;
				if (attempt(p, b, s, pos) != want) bad++;
			}
		}
	}
	return bad;
}

// ---- 2./3. the chain paths ----
static bool seq_at(const Sequence &q, const uint8_t *s, size_t len, size_t pos)
{
	if (pos + q.size() > len) return false;
	for (size_t i = 0; i < q.size(); i++) if (!q[i].has(s[pos + i])) return false;
	return true;
}

// what the scan kernels deliver by contract: leading-sequence hits, or the first byte of every class run >= run_min
static void candidates(const Program &p, const Bytes &b, uint32_t unit, std::vector<OutRec> &ord)
{
	for (size_t pos = 0; pos < b.size(); pos++) {
		if (p.vm_runstart) {
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

enum Path { P_TWO, P_DENSE_TWO, P_RUN };
static const char *path_name[3] = {"two-outcome", "dense two-outcome", "class-repeat chain"};

// launch_resolve_count + launch_resolve_write of resolve_kernels.cu for one batch, on the host (the device's block scans are
// plain prefix sums here).  0 ok, -1 VM limit
static int run_path(const Program &p, const std::vector<const Bytes *> &subj, uint32_t mode, Path path, std::vector<std::vector<M>> &out)
{
	const uint32_t nu = (uint32_t)subj.size();
	std::vector<DevUnit> du(nu);
	for (uint32_t u = 0; u < nu; u++) {
		memset(&du[u], 0, sizeof du[u]);
		du[u].ptr = (uint64_t)(uintptr_t)subj[u]->data();
		du[u].len = (uint32_t)subj[u]->size();
		du[u].base_off = 1000u * u;
		du[u].file_id = 7 + u;
	}
	ResolveArgs R;
	memset(&R, 0, sizeof R);
	uint32_t tot[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
	std::vector<unsigned long long> vbud(nu);
	std::vector<uint32_t> us(nu + 1, 0u), vus(nu + 1, 0u), uo(nu + 1, 0u), flag, buf;
	std::vector<OutRec> ord, ordb, vord;
	std::vector<TileDesc> tds;
	R.units = du.data(); R.n_units = nu; R.totals = tot; R.vm_limit = tot + 2; R.vm_budget = vbud.data();
	R.unit_out = uo.data(); R.mode = mode; R.minlen = (uint32_t)p.minlen; R.engine = GSCAN_ENGINE_VM; R.run_min = (uint32_t)p.run_min;
	for (int i = 0; i < 8; i++) R.bitmap[i] = path == P_DENSE_TWO ? p.first_set.w[i] : p.run_class.w[i];
	R.vm_code = p.vm_code.data(); R.vm_sets = p.vm_sets.data();
	R.vm_par = 1; R.vm_two = path != P_RUN; R.vm_chain_run = path == P_RUN;
	auto each = [&](uint32_t n, auto fn) { for (uint32_t i = 0; i < n; i++) { model_threadIdx.x = i; fn(); } model_threadIdx.x = 0; };
	out.assign(nu, std::vector<M>());
	uint32_t cap = 0, levels = 2;
	if (path != P_DENSE_TWO) {
		for (uint32_t u = 0; u < nu; u++) { candidates(p, *subj[u], u, ord); us[u + 1] = (uint32_t)ord.size(); }
		const uint32_t nc = (uint32_t)ord.size();
		if (nc == 0) return 0;
		cap = R.vm_two ? 2 * nc : nc;
		while ((1u << levels) < cap) levels++;
		buf.assign((size_t)(levels + 4) * cap, 0u); flag.assign(cap, 0u); vord.assign(cap, OutRec{0, 0, 0, 0}); ordb.assign(nc, OutRec{0, 0, 0, 0});
		R.ord = ord.data(); R.unit_start = us.data(); R.total_cand = nc;
		R.chain = 1; R.chain_levels = levels; R.chain_cap = cap; R.chain_buf = buf.data();
		R.vm_ord = vord.data(); R.vm_flag = flag.data(); R.vm_unit_start = vus.data(); R.vm_ord_b = ordb.data();
		tot[0] = nc;
		each(nu, [&] { k_vm_budget_init(R); });
		for (auto &v : vbud) v = std::min(v, kModelSteps);
		each(nc, [&] { k_vm_attempts(R); });
		exclusive(flag.data(), cap, &tot[4]);
		each(nc, [&] { k_vm_compact(R); });
		each(nu + 1, [&] { k_vm_unit_starts(R); });
	} else {
		// tiles of 256 bytes (the device's are 4 .. 64 KiB; the block -> tile -> unit arithmetic is the same)
		const uint32_t tshift = 8;
		for (uint32_t u = 0; u < nu; u++) {
			du[u].first_tile = (uint32_t)tds.size();
			const size_t len = subj[u]->size();
			for (size_t off = 0; off < len; off += (size_t)1 << tshift) {
				TileDesc t;
				memset(&t, 0, sizeof t);
				t.src = du[u].ptr + off; t.unit = u; t.off = (uint32_t)off;
				t.len = (uint32_t)std::min<size_t>((size_t)1 << tshift, len - off); t.ulen = (uint32_t)len;
				tds.push_back(t);
			}
		}
		const uint32_t blocks = (uint32_t)tds.size() << (tshift - 6);
		flag.assign(blocks + 1, 0u);
		R.tiles = tds.data(); R.dense_tile_shift = tshift; R.dense_blocks = blocks; R.vm_flag = flag.data(); R.vm_unit_start = vus.data();
		each(nu, [&] { k_vm_budget_init(R); });
		for (auto &v : vbud) v = std::min(v, kModelSteps);
		each(blocks, [&] { k_vm_dense<false>(R); });
		if (tot[2]) return -1;
		exclusive(flag.data(), blocks, &tot[4]);
		cap = tot[4];
		if (cap == 0) return 0;
		while ((1u << levels) < cap) levels++;
		buf.assign((size_t)(levels + 4) * cap, 0u); vord.assign(cap, OutRec{0, 0, 0, 0});
		R.vm_ord = vord.data();
		R.chain = 1; R.chain_levels = levels; R.chain_cap = cap; R.chain_buf = buf.data();
		each(nu, [&] { k_vm_budget_init(R); });
		for (auto &v : vbud) v = std::min(v, kModelSteps);
		each(blocks, [&] { k_vm_dense<true>(R); });
		each(nu + 1, [&] { k_vm_dense_unit_starts(R); });
		R.vm_ready = 1; R.total_cand = cap;
	}
	if (tot[2]) return -1;
	ResolveArgs C = R;
	C.ord = R.vm_ord; C.unit_start = R.vm_unit_start; C.totals = R.totals + 4; // chain_view()
	const uint32_t nodes = tot[4];
	uint32_t *mark = buf.data() + (size_t)levels * cap, *rank = mark + cap;
	if (R.vm_two) {
		exclusive(buf.data() + (size_t)(levels + 2) * cap, cap, &tot[5]);
		each(nodes, [&] { k_two_blist(C); });
	}
	const bool follow = mode != GSCAN_MODE_FIRST;
	if (follow) {
		if (R.vm_chain_run) each(nodes, [&] { k_vm_resume(C); });
		each(nodes, [&] { k_chain_next(C); });
		for (uint32_t k = 1; k < levels; k++) each(nodes, [&] { k_chain_double(C, k); });
	}
	each(nu, [&] { k_chain_heads(C); });
	if (follow) for (uint32_t k = levels; k-- > 0;) each(nodes, [&] { k_chain_spread(C, k); });
	each(nodes, [&] { k_chain_unmark(C); });
	if (R.vm_chain_run) {
		each(nodes, [&] { k_chain_entry_init(C); });
		if (follow) each(nodes, [&] { k_chain_entry(C); });
	}
	if (tot[2]) return -1;
	std::copy(mark, mark + cap, rank);
	exclusive(rank, cap, nullptr);
	each(nu, [&] { k_chain_count(C); });
	std::vector<uint32_t> cnt(uo.begin(), uo.begin() + nu);
	uint32_t total = 0;
	exclusive(uo.data(), nu, &total);
	std::vector<FinalRec> fin(total + 1);
	C.out = fin.data();
	C.total_cand = cap;
	each(cap, [&] { k_chain_write(C); });
	for (uint32_t u = 0; u < nu; u++)
		for (uint32_t k = 0; k < cnt[u]; k++) {
			const FinalRec &r = fin[uo[u] + k];
			if (r.file_id != du[u].file_id) return -2;
			out[u].push_back(M{r.start - du[u].base_off, r.len});
		}
	return 0;
}

static bool same(const std::vector<M> &g, const go_matches &w)
{
	if (g.size() != w.n) return false;
	for (size_t i = 0; i < g.size(); i++) if (g[i].pos != w.v[i].start || g[i].len != w.v[i].len) return false;
	return true;
}

static void show(const Bytes &b)
{
	printf("\"");
	for (size_t i = 0; i < b.size() && i < 200; i++) printf(b[i] == '\n' ? "\\n" : b[i] == '\t' ? "\\t" : "%c", b[i]);
	printf(b.size() > 200 ? "...\"" : "\"");
}

int main(int argc, char **argv)
{
	if (argc < 2) return 2;
	std::ifstream f(argv[1]);
	std::vector<Bytes> subjects;
	const char *alphas[] = {"abc", "abcx \n", "ab", "abc abc\n\n", "aabbcc_x1 \t\n", "ab\n", "a@b.c1 \n", "ab=:\\\" \n"};
	const int lens[] = {1, 2, 3, 4, 5, 7, 9, 16, 17, 33, 64, 130, 257};
	for (int k = 0; k < 78; k++) {
		const char *al = alphas[k % 8];
		const size_t na = strlen(al), ln = (size_t)lens[k % 13];
		Bytes b(ln);
		for (auto &c : b) c = (uint8_t)al[rnd() % na];
		subjects.push_back(b);
	}
	// lines longer than the 511 bytes the reference prints behind a match: in LINE mode the search resumes in the middle of a
	// line -- inside a run, or right behind a '\n'
	std::vector<Bytes> long_lines;
	for (int k = 0; k < 6; k++) {
		const char *al = k % 3 == 0 ? "ab" : (k % 3 == 1 ? "abc " : "aab_1 @.");
		const size_t na = strlen(al), ln = k < 3 ? 700 : 1500;
		Bytes b(ln);
		for (auto &c : b) c = (uint8_t)al[rnd() % na];
		if (k >= 3) { b[ln / 2] = '\n'; b[ln / 2 + 520] = '\n'; }
		long_lines.push_back(b);
	}
	std::vector<Bytes> all = subjects;
	all.insert(all.end(), long_lines.begin(), long_lines.end());

	const int modes[3] = {GO_MODE_ALL, GO_MODE_FIRST, GO_MODE_LINE};
	const uint32_t dmodes[3] = {GSCAN_MODE_ALL, GSCAN_MODE_FIRST, GSCAN_MODE_LINE};
	long n_path[3] = {0, 0, 0}, n_two_unit = 0, n_limit = 0, n_reach_pat = 0, n_reach1 = 0, n_caught = 0, n_strict = 0;
	int bad = 0, n_pat = 0;
	std::string pat;
	while (std::getline(f, pat)) {
		if (pat.empty()) continue;
		n_pat++;
		char oerr[200];
		go_regex *re = go_compile(pat.data(), pat.size(), 0, oerr, sizeof oerr);
		if (!re) continue;
		for (int strict = 0; strict < 2; strict++) {
			Program p;
			std::string err;
			if (!compile_pattern(pat.data(), pat.size(), strict ? GSCAN_STRICT_REF : 0u, p, err) || !p.use_vm) continue;
			if (strict && !p.cap_stops) continue; // the same program as without STRICT_REF
			n_strict += strict;
			if (!strict) {
				n_reach_pat++;
				const long v = reach_violations(p, subjects, p.vm_reach);
				if (v) { printf("REACH UNSOUND %s: reach %d, %ld disagreements\n", pat.c_str(), p.vm_reach, v); bad++; }
				// a reach reported one too small must be caught (it is exact for the programs of reach 1 tried here when the
				// subjects show the difference -- counted, the caller checks that it happens)
				if (p.vm_reach >= 1) {
					n_reach1 += p.vm_reach == 1;
					if (reach_violations(p, subjects, p.vm_reach - 1) > 0) n_caught++;
				}
			}
			Path path;
			if (p.vm_runstart) {
				if (p.vm_reach != 0 || p.vm_lead == VM_Q_LAZY) continue;
				path = P_RUN;
			} else if (p.vm_reach == 1) path = p.vm_dense ? P_DENSE_TWO : P_TWO;
			else continue;
			for (int m = 0; m < 3; m++) {
				for (size_t k = 0; k < all.size(); k++) {
					go_matches w = {0, 0, 0};
					if (go_scan_window(re, all[k].data(), all[k].size(), 0, 0, modes[m], strict, &w) != 0) { go_matches_free(&w); n_limit++; continue; }
					std::vector<std::vector<M>> got;
					const int rc = run_path(p, {&all[k]}, dmodes[m], path, got);
					if (rc == -1) { n_limit++; go_matches_free(&w); continue; }
					if (rc != 0 || !same(got[0], w)) {
						bad++;
						printf("%s MISMATCH %s strict %d mode %d on ", path_name[path], pat.c_str(), strict, m);
						show(all[k]);
						printf(": got %zu want %zu\n", rc == 0 ? got[0].size() : (size_t)0, w.n);
						if (bad > 20) return 1;
					}
					n_path[path]++;
					go_matches_free(&w);
				}
				// two units in one batch: unit borders in the searches, the heads, the B list, the output slots
				for (size_t k = 0; k + 1 < all.size(); k += 3) {
					go_matches w[2] = {{0, 0, 0}, {0, 0, 0}};
					const bool ok0 = go_scan_window(re, all[k].data(), all[k].size(), 0, 0, modes[m], strict, &w[0]) == 0;
					const bool ok1 = go_scan_window(re, all[k + 1].data(), all[k + 1].size(), 0, 0, modes[m], strict, &w[1]) == 0;
					std::vector<std::vector<M>> got;
					const int rc = ok0 && ok1 ? run_path(p, {&all[k], &all[k + 1]}, dmodes[m], path, got) : -1;
					if (rc == -1) n_limit++;
					else if (rc != 0 || !same(got[0], w[0]) || !same(got[1], w[1])) {
						bad++;
						printf("TWO-UNIT %s MISMATCH %s strict %d mode %d subjects %zu,%zu\n", path_name[path], pat.c_str(), strict, m, k, k + 1);
						if (bad > 20) return 1;
					} else n_two_unit++;
					go_matches_free(&w[0]);
					go_matches_free(&w[1]);
				}
			}
		}
		go_free(re);
	}
	printf("reach checks %ld over %ld patterns; reach-1 patterns %ld; under-reported reach caught %ld; ", g_reach_checks, n_reach_pat, n_reach1, n_caught);
	printf("two-outcome checks %ld; dense two-outcome checks %ld; class-repeat chain checks %ld; two-unit checks %ld; strict programs %ld; ",
	       n_path[P_TWO], n_path[P_DENSE_TWO], n_path[P_RUN], n_two_unit, n_strict);
	printf("patterns %d, limit skips %ld, mismatches %d\n", n_pat, n_limit, bad);
	if (bad == 0) printf("model ok\n");
	return bad ? 1 : 0;
}
