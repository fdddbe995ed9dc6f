// model_check_start.cc -- CPU check of the resolve paths for general patterns whose attempts look at or before their first
// byte (Program::vm_reach) and of class-repeat-led patterns (Program::vm_runstart), with the device's own source (the VM, the
// resolve kernels and their launch sequence in resolve_kernels.cu, extracted by tests/test_model_start.py, model_host.h)
// compiled for the host:
//   1. reach soundness: an attempt at p gives the same outcome from every subject beginning s <= p - vm_reach; and the check
//      catches a reach reported one too small (it must find a disagreement for patterns whose reach is exact)
//   2. reach-1 programs, two outcomes per candidate: filtered (VM_TWO, k_vm_attempts) and dense (VM_DENSE_TWO, k_vm_dense),
//      then the chain
//   3. greedy / possessive class-repeat-led programs on the chain (VM_RUN_CHAIN, k_vm_resume)
// against the oracle's loop in all three modes (ALL / FIRST / LINE), for single units and two-unit batches, with and without
// the capturing-group quirk (Q2, STRICT_REF).
// Usage: model_check_start PATTERN_FILE   (one pattern per line)
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>

#include "model_host.h"
extern "C" {
#include "../oracle/grab_oracle.h"
}

static uint64_t rng_state = 0x9e3779b97f4a7c15ull;
static uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (uint32_t)(rng_state >> 9); }

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
enum { P_TWO, P_DENSE_TWO, P_RUN };
static const char *path_name[3] = {"two-outcome", "dense two-outcome", "class-repeat chain"};

// the batch through the shipped launch sequence on the path the planner picks with the chain paths forced on (what
// GSCAN_CHAIN=1 selects), the unit budgets clamped to kModelSteps.  0 ok, -1 VM limit
static int run_path(const Program &p, const std::vector<const Bytes *> &subj, uint32_t mode, std::vector<std::vector<M>> &out)
{
	ModelBatch b(p, subj);
	HostExec x;
	x.after_budget_init = [](const ResolveArgs &R) { for (uint32_t u = 0; u < R.n_units; u++) R.vm_budget[u] = std::min(R.vm_budget[u], kModelSteps); };
	return b.run(p, mode, b.plan(p, mode, CHAIN_ON), x, out);
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
			// the paths of this check (reach 0 without a leading class repeat: model_check.cc); a batch with no candidates plans NONE
			const uint32_t planned = plan_resolve(p, GSCAN_MODE_ALL, 1, 1, 1, 1, CHAIN_ON);
			const int path = planned == GSCAN_RESOLVE_VM_TWO ? P_TWO : planned == GSCAN_RESOLVE_VM_DENSE_TWO ? P_DENSE_TWO
			               : planned == GSCAN_RESOLVE_VM_RUN_CHAIN ? P_RUN : -1;
			if (path < 0) continue;
			for (int m = 0; m < 3; m++) {
				for (size_t k = 0; k < all.size(); k++) {
					go_matches w = {0, 0, 0};
					if (go_scan_window(re, all[k].data(), all[k].size(), 0, 0, modes[m], strict, &w) != 0) { go_matches_free(&w); n_limit++; continue; }
					std::vector<std::vector<M>> got;
					const int rc = run_path(p, {&all[k]}, dmodes[m], got);
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
					const int rc = ok0 && ok1 ? run_path(p, {&all[k], &all[k + 1]}, dmodes[m], got) : -1;
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
