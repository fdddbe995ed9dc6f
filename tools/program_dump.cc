#include PATTERN_H
#include <cstdio>
#include <fstream>
#include <string>
using namespace gscan;
static uint64_t h = 1469598103934665603ull;
static void mix(const void *p, size_t n) { const unsigned char *b = (const unsigned char *)p; for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 1099511628211ull; } }
int main(int argc, char **argv) {
	std::ifstream f(argv[1]); std::string pat;
	while (std::getline(f, pat)) {
		Program p; std::string err;
		h = 1469598103934665603ull;
		if (!compile_pattern(pat.data(), pat.size(), 0, p, err)) { printf("REJ %s | %s\n", pat.c_str(), err.c_str()); continue; }
		int k = p.kind; mix(&k, 4); mix(&p.minlen, 4); mix(&p.maxlen, 4); mix(&p.captures, 4);
		for (auto &s : p.seqs) { size_t n = s.size(); mix(&n, 8); for (auto &b : s) mix(b.w, 32); }
		for (auto &t : p.tests) mix(&t, sizeof t);
		mix(&p.anchor, 4); mix(&p.delta, 4); mix(&p.delta2, 4);
		for (auto &t : p.triples) mix(&t, sizeof t);
		bool b2 = p.disjoint, b3 = p.use_hash, b4 = p.use_vm, b5 = p.vm_runstart; mix(&p.pair_flag_prior, 8); mix(&b2,1); mix(&b3,1); mix(&b4,1); mix(&b5,1);
		mix(&p.hash_len, 4); mix(&p.hash_mul, 4); mix(&p.hash_slots, 4);
		if (!p.hash_table.empty()) mix(p.hash_table.data(), p.hash_table.size() * 4);
		if (!p.slot_seqs.empty()) mix(p.slot_seqs.data(), p.slot_seqs.size() * 4);
		mix(p.run_class.w, 32); mix(&p.run_min, 4);
		if (!p.vm_code.empty()) mix(p.vm_code.data(), p.vm_code.size() * 4);
		if (!p.vm_sets.empty()) mix(p.vm_sets.data(), p.vm_sets.size() * 4);
		printf("%016llx %s\n", (unsigned long long)h, pat.c_str());
	}
}
