// model_check.cc -- CPU check of what the pattern compiler (grab_b200/csrc/pattern.cc) hands to the device, against
// the oracle: the compiled Program is interpreted on the host exactly as the resolve kernels interpret it -- FIXED:
// first sequence in preference order at the leftmost position; RUN: greedy class run of at least run_min; general
// patterns: the device VM, whose source is extracted verbatim from resolve_kernels.cu by tests/test_model.py
// (vm_snippet.inc, model_host.h) and compiled here for the host -- inside the reference's loop (moving search start, strict
// '<' guard, grab.cc:175-213).  Then the device's own launch sequence (same extraction) fed with the candidates the scan
// kernels deliver by contract, in all three modes (ALL / FIRST / LINE): the per-unit walk against the oracle, and the path
// the engine's planner picks with the chain paths forced on against the walk, for single units and two-unit batches.  Also
// checks that the candidate filter of general patterns (leading-byte sequences / run starts) never rejects a position where
// the VM matches.
// Usage: model_check PATTERN_FILE   (one pattern per line)
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>

#include "model_host.h"
extern "C" {
#include "../oracle/grab_oracle.h"
}

static uint64_t rng_state = 0x1234567ull;
static uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (uint32_t)(rng_state >> 9); }

// 0 ok, -1 VM limit, -2 filter soundness violated
static int emulate(const Program &p, const uint8_t *s, size_t len, std::vector<M> &out, std::string &why)
{
	ResolveArgs R;
	memset(&R, 0, sizeof R);
	R.vm_code = p.vm_code.data();
	R.vm_sets = p.vm_sets.data();
	size_t start = 0;
	while (start + (size_t)p.minlen < len) { // grab.cc:175
		bool found = false;
		size_t pos = start, mend = 0;
		VmBudget budget(len);
		for (; pos < len; pos++) {
			if (p.use_vm) {
				uint32_t e = 0;
				const int rc = vm_exec(R, s + start, (uint32_t)(len - start), (uint32_t)(pos - start), &e, budget);
				if (rc < 0) return -1;
				if (rc == 1) { found = true; mend = start + e; }
			} else if (p.kind == ENGINE_RUN) {
				size_t k = 0;
				while (pos + k < len && p.run_class.has(s[pos + k])) k++;
				if (k >= (size_t)p.run_min) { found = true; mend = pos + k; }
			} else {
				for (auto &q : p.seqs)
					if (seq_at(q, s, len, pos)) { found = true; mend = pos + q.size(); break; }
			}
			if (found) break;
		}
		if (!found) break;
		if (p.use_vm) { // the scan kernel (dense: the first-byte test of the walk) must have offered this position to the VM walk
			bool offered = false;
			if (p.vm_dense) offered = p.first_set.has(s[pos]);
			else if (p.vm_runstart) offered = p.run_class.has(s[pos]) && (pos == start || !p.run_class.has(s[pos - 1]));
			else for (auto &q : p.seqs) offered = offered || seq_at(q, s, len, pos);
			if (!offered) { why = "candidate filter rejects a matching position"; return -2; }
		}
		if (mend <= pos) { why = "empty match"; return -2; }
		out.push_back(M{pos, (uint32_t)(mend - pos)});
		start = mend;
	}
	return 0;
}

static int g_flat_checks = 0, g_chain_checks = 0, g_vmpar_checks = 0, g_densepar_checks = 0, g_two_unit_checks = 0;

static bool same(const std::vector<std::vector<M>> &g, const std::vector<std::vector<M>> &w)
{
	bool ok = g.size() == w.size();
	for (size_t u = 0; ok && u < g.size(); u++) {
		ok = g[u].size() == w[u].size();
		for (size_t i = 0; ok && i < g[u].size(); i++) ok = g[u][i].pos == w[u][i].pos && g[u][i].len == w[u][i].len;
	}
	return ok;
}

// the dense write pass with LESS budget than the count pass had (the attempts of a unit share it: on the device the two passes
// can run out at different places): never more records than counted, what is missing padded with chain-ending entries,
// nothing written past the list.  One unit.
static bool dense_write_starved(ModelBatch &b, const Program &p, uint32_t mode, uint32_t path)
{
	HostExec x;
	const ResolveArgs R = b.args(p, mode, path);
	vm_dense_count_seq(x, R);
	const uint32_t cap = b.totals[4];
	if (b.totals[2] || cap == 0) return true;
	std::vector<OutRec> guarded(cap + 4, OutRec{0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu});
	const ChainGeom g = chain_geom(path, cap);
	std::vector<uint32_t> tables((size_t)g.arrays * cap, 0u); // VM_DENSE_TWO: the nodes' kinds
	uint32_t wtot[10];
	memcpy(wtot, b.totals, sizeof wtot);
	ResolveArgs W = R;
	W.totals = wtot; W.vm_ord = guarded.data();
	W.chain_levels = g.levels; W.chain_cap = cap; W.chain_buf = tables.data();
	b.budget[0] = 40; // steps for the whole unit
	for (uint32_t k = 0; k < W.dense_blocks; k++) { model_threadIdx.x = k; k_vm_dense<true>(W); }
	model_threadIdx.x = 0;
	bool ok = true; // (40 steps can be enough for a tiny subject: then nothing is flagged and the list is complete)
	for (uint32_t i = 0; ok && i < cap; i++) ok = guarded[i].unit == 0 && guarded[i].pos < b.du[0].len && guarded[i].pad >= 1 && guarded[i].pad <= 3;
	for (uint32_t i = cap; ok && i < cap + 4; i++) ok = guarded[i].unit == 0xdeadbeefu;
	return ok;
}

// The per-unit walk (GSCAN_RESOLVE_WALK) through the shipped launch sequence into `out`, then the path the engine's planner
// picks with the chain paths forced on (what GSCAN_CHAIN=1 selects) into *path: the same records.  0 ok, -1 VM limit on the
// walk, -2 VM limit on the planned path (`out` is complete), -3 the planned path differs
static int walk(const Program &p, const std::vector<const Bytes *> &subj, uint32_t mode, std::vector<std::vector<M>> &out, uint32_t *path)
{
	ModelBatch b(p, subj);
	HostExec x;
	*path = GSCAN_RESOLVE_WALK;
	if (b.run(p, mode, GSCAN_RESOLVE_WALK, x, out) != 0) return -1;
	*path = b.plan(p, mode, CHAIN_ON);
	if (*path == GSCAN_RESOLVE_WALK) return 0;
	std::vector<unsigned long long> budget0;
	x.after_budget_init = [&](const ResolveArgs &R) { budget0.assign(R.vm_budget, R.vm_budget + R.n_units); };
	std::vector<std::vector<M>> got;
	const int rc = b.run(p, mode, *path, x, got);
	if (rc == -1) return -2;
	if (rc != 0 || !same(got, out)) return -3;
	if (*path == GSCAN_RESOLVE_VM_ATTEMPTS || *path == GSCAN_RESOLVE_VM_TWO) {
		// every attempt hands back what it did not use: never more than there was (nothing behind k_vm_attempts runs the VM)
		for (size_t u = 0; u < subj.size(); u++)
			if (b.budget[u] > budget0[u] || b.budget[u] == 0) return -3;
	}
	if (path_compacted(*path) && subj.size() == 1 && !dense_write_starved(b, p, mode, *path)) return -3;
	if (*path == GSCAN_RESOLVE_NONE) return 0;
	if (subj.size() > 1) g_two_unit_checks++;
	else if (*path == GSCAN_RESOLVE_FLAT) g_flat_checks++;
	else if (*path == GSCAN_RESOLVE_CHAIN) g_chain_checks++;
	else if (path_compacted(*path)) g_densepar_checks++;
	else g_vmpar_checks++;
	return 0;
}

static void show(const std::vector<uint8_t> &b)
{
	printf("\"");
	for (uint8_t c : b) printf(c == '\n' ? "\\n" : c == '\t' ? "\\t" : "%c", c);
	printf("\"");
}

static bool same_as_oracle(const std::vector<M> &g, const go_matches &w)
{
	bool ok = g.size() == w.n;
	for (size_t i = 0; ok && i < g.size(); i++) ok = g[i].pos == w.v[i].start && g[i].len == w.v[i].len;
	return ok;
}

int main(int argc, char **argv)
{
	if (argc < 2) return 2;
	std::ifstream f(argv[1]);
	std::string pat;
	std::vector<Bytes> subjects;
	const char *alphas[] = {"abc", "abcx \n", "ab", "abc abc\n\n", "aabbcc_x1 \t\n", "ab\n"};
	const int lens[] = {1, 2, 3, 4, 5, 7, 9, 16, 17, 33, 64, 130, 257};
	for (int k = 0; k < 78; k++) {
		const char *al = alphas[k % 6];
		const size_t na = strlen(al), ln = (size_t)lens[k % 13];
		std::vector<uint8_t> b(ln);
		for (auto &c : b) c = (uint8_t)al[rnd() % na];
		subjects.push_back(b);
	}
	// lines longer than the 511 bytes the reference prints behind a match (grab.cc:194-196): in LINE mode the search resumes
	// in the middle of the line, for class runs possibly in the middle of a run
	for (int k = 0; k < 6; k++) {
		const char *al = k % 3 == 0 ? "ab" : (k % 3 == 1 ? "abc " : "aab_1 ");
		const size_t na = strlen(al), ln = k < 3 ? 700 : 1500;
		std::vector<uint8_t> b(ln);
		for (auto &c : b) c = (uint8_t)al[rnd() % na];
		if (k >= 3) b[ln / 2] = '\n';
		subjects.push_back(b);
	}
	int n_dense = 0, n_pat = 0, n_served = 0, n_vm = 0, n_cmp = 0, n_walk = 0, n_limit = 0, bad = 0, n_strict = 0;
	while (std::getline(f, pat)) {
		if (pat.empty()) continue;
		n_pat++;
		Program p;
		std::string err;
		if (!compile_pattern(pat.data(), pat.size(), 0, p, err)) continue; // rejected loudly: nothing to check
		char oerr[200];
		go_regex *re = go_compile(pat.data(), pat.size(), 0, oerr, sizeof oerr);
		if (!re) continue;
		if (go_nullable(re)) { printf("MISMATCH %s: compiled but the oracle says it can match the empty string\n", pat.c_str()); bad++; go_free(re); continue; }
		if (go_minlen(re) != p.minlen) { printf("MISMATCH %s: minlen %d, oracle %d\n", pat.c_str(), p.minlen, go_minlen(re)); bad++; }
		n_served++;
		// the device's launch sequence on `subj` in mode m against the oracle (walk: the per-unit walk, then the planned path);
		// false: too many mismatches
		auto check_walk = [&](const Program &prog, const std::vector<const Bytes *> &subj, int m, int strict) {
			const int modes[3] = {GO_MODE_ALL, GO_MODE_FIRST, GO_MODE_LINE};
			const uint32_t dmodes[3] = {GSCAN_MODE_ALL, GSCAN_MODE_FIRST, GSCAN_MODE_LINE};
			std::vector<go_matches> w(subj.size(), go_matches{0, 0, 0});
			bool limit = false;
			for (size_t u = 0; u < subj.size(); u++)
				limit = go_scan_window(re, subj[u]->data(), subj[u]->size(), 0, 0, modes[m], strict, &w[u]) != 0 || limit;
			std::vector<std::vector<M>> g;
			uint32_t path = 0;
			const int rc = limit ? -1 : walk(prog, subj, dmodes[m], g, &path);
			bool ok = rc != -3;
			if (rc == -1 || rc == -2) n_limit++;
			if (rc != -1) {
				for (size_t u = 0; ok && u < subj.size(); u++) ok = same_as_oracle(g[u], w[u]);
				n_walk++;
			}
			if (!ok) {
				bad++;
				printf("%s MISMATCH %s mode %d path %u (engine %d vm %d runstart %d) on", rc == -3 ? "PATH" : "WALK", pat.c_str(), m, path,
				       (int)prog.kind, (int)prog.use_vm, (int)prog.vm_runstart);
				for (auto *b : subj) { printf(" "); show(*b); }
				printf(strict ? " (STRICT_REF)\n" : "\n");
			}
			for (auto &x : w) go_matches_free(&x);
			return bad <= 20;
		};
		n_vm += p.use_vm;
		n_dense += p.use_vm && p.vm_dense;
		for (auto &sb : subjects) {
			go_matches want = {0, 0, 0};
			if (go_scan_window(re, sb.data(), sb.size(), 0, 0, GO_MODE_ALL, 0, &want) != 0) { go_matches_free(&want); n_limit++; continue; }
			std::vector<M> got;
			std::string why;
			const int rc = emulate(p, sb.data(), sb.size(), got, why);
			if (rc == -1) { n_limit++; go_matches_free(&want); continue; }
			bool same = rc == 0 && got.size() == want.n;
			for (size_t i = 0; same && i < got.size(); i++) same = got[i].pos == want.v[i].start && got[i].len == want.v[i].len;
			n_cmp++;
			if (!same) {
				bad++;
				printf("MISMATCH %s (engine %d vm %d runstart %d) on ", pat.c_str(), (int)p.kind, (int)p.use_vm, (int)p.vm_runstart);
				show(sb);
				printf(": %s got %zu want %zu\n", why.c_str(), got.size(), want.n);
				if (bad > 20) { go_matches_free(&want); go_free(re); return 1; }
			}
			go_matches_free(&want);
			for (int m = 0; m < 3; m++) if (!check_walk(p, {&sb}, m, 0)) { go_free(re); return 1; }
		}
		// two units in one batch: consecutive subjects pairwise, all modes
		for (size_t k = 0; k + 1 < subjects.size(); k += 5)
			for (int m = 0; m < 3; m++) if (!check_walk(p, {&subjects[k], &subjects[k + 1]}, m, 0)) { go_free(re); return 1; }
		// Q2 in full (STRICT_REF): patterns with capturing groups -- the first match in which a group took part ends the
		// window; the device's launch sequence against the oracle with strict_q2 on
		if (p.captures > 0) {
			Program ps;
			std::string e2;
			if (compile_pattern(pat.data(), pat.size(), GSCAN_STRICT_REF, ps, e2)) {
				n_strict++;
				if (ps.kind != ENGINE_NONE)
					for (auto &sb : subjects)
						for (int m = 0; m < 3; m++) if (!check_walk(ps, {&sb}, m, 1)) { go_free(re); return 1; }
			}
		}
		go_free(re);
	}
	printf("two-unit chain checks %d; dense vm chain checks %d; vm chain checks %d; chain checks %d; dense VM patterns %d; ", g_two_unit_checks, g_densepar_checks, g_vmpar_checks, g_chain_checks, n_dense);
	printf("flat write checks %d; strict (Q2) patterns %d; ", g_flat_checks, n_strict);
	printf("patterns %d, served %d (%d through the VM), comparisons %d + %d through the walk kernels, limit skips %d, mismatches %d\n", n_pat, n_served, n_vm, n_cmp, n_walk, n_limit, bad);
	if (bad == 0) printf("model ok\n");
	return bad ? 1 : 0;
}
