// pattern.cc -- see pattern.h.  Host C++ only (no CUDA).
#include "pattern.h"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <memory>

#include "../../include/gscan.h"

namespace gscan {

// ------------------------------------------------------------------------------------------
// byte-class helpers
// ------------------------------------------------------------------------------------------

MaskedEq masked_superset(const ByteSet &s)
{
	MaskedEq r{0, 0, false, 256};
	int first = -1;
	unsigned varying = 0;
	for (int c = 0; c < 256; c++) {
		if (!s.has(c)) continue;
		if (first < 0) first = c;
		varying |= (unsigned)(c ^ first);
	}
	if (first < 0) { r.mask = 0xff; r.val = 0; r.size = 0; r.exact = false; return r; }
	r.mask = (uint8_t)(~varying & 0xff);
	r.val = (uint8_t)(first & r.mask);
	r.size = 1 << __builtin_popcount(varying & 0xff);
	r.exact = (r.size == s.count());
	return r;
}

std::vector<ByteRange> to_ranges(const ByteSet &s)
{
	std::vector<ByteRange> out;
	int c = 0;
	while (c < 256) {
		if (!s.has(c)) { c++; continue; }
		int lo = c;
		while (c < 256 && s.has(c)) c++;
		out.push_back(ByteRange{(uint8_t)lo, (uint8_t)(c - 1)});
	}
	return out;
}

namespace {

bool is_upper(unsigned c) { return c >= 'A' && c <= 'Z'; }
bool is_lower(unsigned c) { return c >= 'a' && c <= 'z'; }
bool is_alpha(unsigned c) { return is_upper(c) || is_lower(c); }
bool is_digit(unsigned c) { return c >= '0' && c <= '9'; }
bool is_alnum(unsigned c) { return is_alpha(c) || is_digit(c); }
bool is_word(unsigned c) { return is_alnum(c) || c == '_'; }
bool is_space(unsigned c) { return c == ' ' || (c >= 9 && c <= 13); }
bool is_xdigit(unsigned c) { return is_digit(c) || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'); }
bool is_punct(unsigned c) { return c > 32 && c < 127 && !is_alnum(c); }
bool is_print(unsigned c) { return c >= 32 && c < 127; }
bool is_graph(unsigned c) { return c > 32 && c < 127; }
bool is_cntrl(unsigned c) { return c < 32 || c == 127; }
bool is_blank(unsigned c) { return c == ' ' || c == '\t'; }

ByteSet from_pred(bool (*p)(unsigned), bool negate = false)
{
	ByteSet s;
	for (unsigned c = 0; c < 256; c++)
		if (p(c) != negate) s.add(c);
	return s;
}

void fold_case(ByteSet &s)
{
	for (unsigned c = 'a'; c <= 'z'; c++) {
		if (s.has(c)) s.add(c - 32);
		if (s.has(c - 32)) s.add(c);
	}
}

// ------------------------------------------------------------------------------------------
// syntax tree
// ------------------------------------------------------------------------------------------

struct Node;
typedef std::unique_ptr<Node> NodeP;

struct Node {
	enum Kind { SET, CAT, ALT, REP, GROUP, ASSERT, EMPTY, LOOK /* (?=) (?!) (?<=) (?<!) */, ATOMIC /* (?>...), possessive groups */ } kind;
	ByteSet set;
	std::vector<NodeP> kids;
	uint32_t rmin = 0, rmax = 0; // rmax == UINT32_MAX: unbounded
	bool lazy = false, possessive = false;
	bool capturing = false;
	bool ahead = false, neg = false; // LOOK
	int akind = 0; // ASSERT: one of VM_A_*
	explicit Node(Kind k) : kind(k) {}
};

constexpr uint32_t kInf = UINT32_MAX;
const Node *peel_noncapturing(const Node *n);

struct Flags { bool icase = false, dotall = false, multiline = false, ungreedy = false, extended = false; };

class Parser {
public:
	Parser(const uint8_t *p, size_t n) : p_(p), end_(p + n) {}
	NodeP parse(std::string &err)
	{
		NodeP r = alternation(Flags());
		if (ok_ && p_ < end_) fail("unmatched )");
		if (!ok_) { err = err_; return nullptr; }
		return r;
	}
	int captures() const { return captures_; }

private:
	const uint8_t *p_, *end_;
	bool ok_ = true;
	std::string err_;
	int captures_ = 0, depth_ = 0;

	void fail(const char *m) { if (ok_) { ok_ = false; err_ = m; } }
	bool more() const { return p_ < end_; }

	static int hex(int c)
	{
		if (c >= '0' && c <= '9') return c - '0';
		if (c >= 'a' && c <= 'f') return c - 'a' + 10;
		if (c >= 'A' && c <= 'F') return c - 'A' + 10;
		return -1;
	}

	// after '\': 1 = single byte in ch, 2 = class in set, 3 = assertion (unsupported by the device engines)
	int escape(bool in_class, unsigned &ch, ByteSet &set)
	{
		if (!more()) { fail("\\ at end of pattern"); return 0; }
		unsigned c = *p_++;
		switch (c) {
		case 'd': set = from_pred(is_digit); return 2;
		case 'D': set = from_pred(is_digit, true); return 2;
		case 'w': set = from_pred(is_word); return 2;
		case 'W': set = from_pred(is_word, true); return 2;
		case 's': set = from_pred(is_space); return 2;
		case 'S': set = from_pred(is_space, true); return 2;
		case 'h': set = ByteSet(); set.add(' '); set.add('\t'); set.add(0xa0); return 2;
		case 'H': set = ByteSet(); set.add(' '); set.add('\t'); set.add(0xa0); set.invert(); return 2;
		case 'v': set = ByteSet(); set.add_range(10, 13); set.add(0x85); return 2;
		case 'V': set = ByteSet(); set.add_range(10, 13); set.add(0x85); set.invert(); return 2;
		case 'N':
			if (in_class) { fail("\\N is not allowed in a class"); return 0; }
			set = ByteSet(); set.invert(); set.w[0] &= ~(1u << 10); return 2;
		case 'n': ch = '\n'; return 1;
		case 't': ch = '\t'; return 1;
		case 'r': ch = '\r'; return 1;
		case 'f': ch = '\f'; return 1;
		case 'a': ch = 7; return 1;
		case 'e': ch = 27; return 1;
		case 'c': {
			if (!more()) { fail("\\c at end of pattern"); return 0; }
			unsigned x = *p_++;
			if (is_lower(x)) x -= 32;
			ch = x ^ 0x40;
			return 1;
		}
		case 'x': {
			unsigned v = 0;
			if (more() && *p_ == '{') {
				const uint8_t *q = p_ + 1;
				int nd = 0;
				while (q < end_ && hex(*q) >= 0) { v = v * 16 + (unsigned)hex(*q); q++; nd++; if (v > 255) break; }
				if (q >= end_ || *q != '}' || nd == 0 || v > 255) { fail("bad \\x{..} (bytes only)"); return 0; }
				p_ = q + 1;
			} else {
				for (int nd = 0; nd < 2 && more() && hex(*p_) >= 0; nd++) v = v * 16 + (unsigned)hex(*p_++);
			}
			ch = v;
			return 1;
		}
		case '0': {
			unsigned v = 0;
			for (int nd = 0; nd < 2 && more() && *p_ >= '0' && *p_ <= '7'; nd++) v = v * 8 + (unsigned)(*p_++ - '0');
			ch = v & 255;
			return 1;
		}
		case 'b':
			if (in_class) { ch = 8; return 1; }
			ch = VM_A_WORDB;
			return 3;
		case 'B': case 'A': case 'z': case 'Z':
			if (in_class) { fail("assertion escape inside a class"); return 0; }
			ch = c == 'B' ? VM_A_NWORDB : c == 'A' ? VM_A_SOS : c == 'z' ? VM_A_EOS : VM_A_EOSNL;
			return 3;
		case 'G':
			fail("\\G is not supported");
			return 0;
		default:
			if (c >= '1' && c <= '9') { fail("back references are not supported"); return 0; }
			if (is_alnum(c)) { fail("unsupported escape sequence"); return 0; }
			ch = c;
			return 1;
		}
	}

	NodeP make_char(unsigned c, const Flags &f)
	{
		NodeP n(new Node(Node::SET));
		n->set.add(c);
		if (f.icase) fold_case(n->set);
		return n;
	}

	NodeP char_class(const Flags &f)
	{
		static const struct { const char *name; bool (*pred)(unsigned); } posix[] = {
			{"alpha", is_alpha}, {"digit", is_digit}, {"alnum", is_alnum}, {"upper", is_upper}, {"lower", is_lower},
			{"space", is_space}, {"xdigit", is_xdigit}, {"punct", is_punct}, {"print", is_print},
			{"graph", is_graph}, {"cntrl", is_cntrl}, {"blank", is_blank}, {"word", is_word}};
		NodeP n(new Node(Node::SET));
		bool negate = false, first = true;
		if (more() && *p_ == '^') { negate = true; p_++; }
		for (;;) {
			if (!more()) { fail("missing terminating ] for character class"); return n; }
			unsigned c = *p_;
			if (c == ']' && !first) { p_++; break; }
			first = false;
			unsigned lo = 0;
			if (c == '[' && p_ + 1 < end_ && p_[1] == ':') {
				const uint8_t *q = p_ + 2;
				bool neg = false;
				if (q < end_ && *q == '^') { neg = true; q++; }
				const uint8_t *name = q;
				while (q < end_ && is_lower(*q)) q++;
				if (q + 1 < end_ && q[0] == ':' && q[1] == ']') {
					bool found = false;
					for (auto &pc : posix)
						if (strlen(pc.name) == (size_t)(q - name) && !memcmp(pc.name, name, (size_t)(q - name))) {
							n->set.unite(from_pred(pc.pred, neg));
							found = true;
						}
					if (!found) { fail("unknown POSIX class name"); return n; }
					p_ = q + 2;
					continue;
				}
			}
			if (c == '\\') {
				p_++;
				ByteSet t;
				unsigned ch = 0;
				int k = escape(true, ch, t);
				if (k == 0) return n;
				if (k == 2) { n->set.unite(t); continue; }
				lo = ch;
			} else {
				lo = c;
				p_++;
			}
			if (p_ + 1 < end_ && p_[0] == '-' && p_[1] != ']') {
				const uint8_t *save = p_;
				p_++;
				unsigned hi = 0;
				if (*p_ == '\\') {
					p_++;
					ByteSet t;
					int k = escape(true, hi, t);
					if (k == 0) return n;
					if (k == 2) { n->set.add(lo); n->set.add('-'); n->set.unite(t); continue; }
				} else if (*p_ == '[' && p_ + 1 < end_ && p_[1] == ':') {
					p_ = save;
					n->set.add(lo);
					continue;
				} else {
					hi = *p_++;
				}
				if (hi < lo) { fail("range out of order in character class"); return n; }
				n->set.add_range(lo, hi);
			} else {
				n->set.add(lo);
			}
		}
		if (f.icase) fold_case(n->set);
		if (negate) n->set.invert();
		return n;
	}

	// 1: quantifier consumed, 0: '{' is a literal, -1: error
	int braces(uint32_t &mn, uint32_t &mx)
	{
		const uint8_t *q = p_ + 1;
		if (q >= end_ || !is_digit(*q)) return 0;
		unsigned long a = 0, b = 0;
		while (q < end_ && is_digit(*q)) { a = a * 10 + (unsigned long)(*q++ - '0'); if (a > 65535) return -1; }
		if (q < end_ && *q == '}') { mn = mx = (uint32_t)a; p_ = q + 1; return 1; }
		if (q >= end_ || *q != ',') return 0;
		q++;
		if (q < end_ && *q == '}') { mn = (uint32_t)a; mx = kInf; p_ = q + 1; return 1; }
		if (q >= end_ || !is_digit(*q)) return 0;
		while (q < end_ && is_digit(*q)) { b = b * 10 + (unsigned long)(*q++ - '0'); if (b > 65535) return -1; }
		if (q >= end_ || *q != '}') return 0;
		if (b < a) return -1;
		mn = (uint32_t)a; mx = (uint32_t)b; p_ = q + 1;
		return 1;
	}

	// returns nullptr with flag_only set when the atom was an inline option like (?i)
	NodeP atom(Flags &f, bool &flag_only)
	{
		flag_only = false;
		unsigned c = *p_++;
		switch (c) {
		case '(': {
			bool capturing = true;
			Flags inner = f;
			if (more() && *p_ == '?') {
				p_++;
				if (!more()) { fail("unterminated (?"); return nullptr; }
				if (*p_ == ':') { capturing = false; p_++; }
				else if (*p_ == 'P' && p_ + 1 < end_ && p_[1] == '<') {
					p_ += 2;
					while (more() && *p_ != '>') p_++;
					if (!more()) { fail("unterminated group name"); return nullptr; }
					p_++;
				} else if ((*p_ == '<' || *p_ == '\'') && p_ + 1 < end_ && p_[1] != '=' && p_[1] != '!') {
					unsigned close = *p_ == '<' ? '>' : '\'';
					p_++;
					while (more() && *p_ != close) p_++;
					if (!more()) { fail("unterminated group name"); return nullptr; }
					p_++;
				} else if (*p_ == '#') { // (?#comment): up to the next ')'
					while (more() && *p_ != ')') p_++;
					if (!more()) { fail("missing ) after comment"); return nullptr; }
					p_++;
					flag_only = true;
					return nullptr;
				} else if (*p_ == '=' || *p_ == '!' || *p_ == '>' || (*p_ == '<' && p_ + 1 < end_ && (p_[1] == '=' || p_[1] == '!'))) {
					// lookahead (?= (?!, lookbehind (?<= (?<!, atomic group (?> -- none of them captures
					int kind = 0; // 0 ahead, 1 behind, 2 atomic
					bool neg = false;
					if (*p_ == '>') { kind = 2; p_++; }
					else if (*p_ == '<') { kind = 1; neg = p_[1] == '!'; p_ += 2; }
					else { neg = *p_ == '!'; p_++; }
					if (++depth_ > 200) { fail("parentheses nested too deeply"); return nullptr; }
					NodeP body = alternation(inner);
					depth_--;
					if (!ok_) return nullptr;
					if (!more() || *p_ != ')') { fail("missing )"); return nullptr; }
					p_++;
					NodeP g(new Node(kind == 2 ? Node::ATOMIC : Node::LOOK));
					g->ahead = kind == 0;
					g->neg = neg;
					g->kids.push_back(std::move(body));
					return g;
				} else if (strchr("<|R(&C+0123456789", (int)*p_)) {
					fail("recursive / conditional groups are not supported by the device engines");
					return nullptr;
				} else {
					bool on = true;
					Flags nf = f;
					for (;;) {
						if (!more()) { fail("unterminated inline option"); return nullptr; }
						unsigned o = *p_++;
						if (o == '-') { on = false; continue; }
						if (o == 'i') { nf.icase = on; continue; }
						if (o == 's') { nf.dotall = on; continue; }
						if (o == 'm') { nf.multiline = on; continue; }
						if (o == 'U') { nf.ungreedy = on; continue; } // PCRE_UNGREEDY: greedy <-> lazy
						if (o == 'x') { nf.extended = on; continue; } // PCRE_EXTENDED: white space and #-comments ignored
						if (o == ')') { f = nf; flag_only = true; return nullptr; }
						if (o == ':') { inner = nf; capturing = false; break; }
						fail("unsupported inline option");
						return nullptr;
					}
				}
			}
			if (capturing) captures_++;
			if (++depth_ > 200) { fail("parentheses nested too deeply"); return nullptr; }
			NodeP body = alternation(inner);
			depth_--;
			if (!ok_) return nullptr;
			if (!more() || *p_ != ')') { fail("missing )"); return nullptr; }
			p_++;
			NodeP g(new Node(Node::GROUP));
			g->capturing = capturing;
			g->kids.push_back(std::move(body));
			return g;
		}
		case '[': return char_class(f);
		case '.': {
			NodeP n(new Node(Node::SET));
			n->set.invert();
			if (!f.dotall) n->set.w[0] &= ~(1u << 10);
			return n;
		}
		case '^': case '$': {
			NodeP n(new Node(Node::ASSERT));
			n->akind = c == '^' ? (f.multiline ? VM_A_MBOL : VM_A_BOL) : (f.multiline ? VM_A_MEOL : VM_A_EOL);
			return n;
		}
		case '\\': {
			if (more() && *p_ == 'Q') {
				p_++;
				NodeP cat(new Node(Node::CAT));
				while (more()) {
					if (p_ + 1 < end_ && p_[0] == '\\' && p_[1] == 'E') { p_ += 2; break; }
					cat->kids.push_back(make_char(*p_++, f));
				}
				return cat;
			}
			if (more() && *p_ == 'E') { p_++; return NodeP(new Node(Node::EMPTY)); }
			ByteSet t;
			unsigned ch = 0;
			int k = escape(false, ch, t);
			if (k == 0) return nullptr;
			if (k == 1) return make_char(ch, f);
			if (k == 2) { NodeP n(new Node(Node::SET)); n->set = t; return n; }
			NodeP n(new Node(Node::ASSERT));
			n->akind = (int)ch;
			return n;
		}
		case '*': case '+': case '?':
			fail("quantifier does not follow a repeatable item");
			return nullptr;
		default: return make_char(c, f);
		}
	}

	// (?x): outside character classes white space is ignored and # starts a comment that ends at the next newline
	// (?#...) comments vanish wherever they stand, also between an item and its quantifier ("a(?#x)+" is "a+")
	void skip_extended(const Flags &f)
	{
		while (more()) {
			const unsigned c = *p_;
			if (c == '(' && p_ + 2 < end_ && p_[1] == '?' && p_[2] == '#') {
				const uint8_t *q = p_ + 3;
				while (q < end_ && *q != ')') q++;
				if (q >= end_) return; // unterminated: atom() reports it
				p_ = q + 1;
				continue;
			}
			if (!f.extended) break;
			if (c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\f' || c == '\v') { p_++; continue; }
			if (c == '#') { while (more() && *p_ != '\n') p_++; continue; }
			break;
		}
	}

	NodeP concatenation(Flags &f)
	{
		NodeP cat(new Node(Node::CAT));
		for (;;) {
			skip_extended(f);
			if (!(ok_ && more() && *p_ != '|' && *p_ != ')')) break;
			bool flag_only = false;
			NodeP a = atom(f, flag_only);
			if (!ok_) break;
			if (flag_only) continue;
			if (!a) break;
			skip_extended(f);
			if (more()) {
				uint32_t mn = 0, mx = 0;
				bool q = false;
				if (*p_ == '*') { mn = 0; mx = kInf; p_++; q = true; }
				else if (*p_ == '+') { mn = 1; mx = kInf; p_++; q = true; }
				else if (*p_ == '?') { mn = 0; mx = 1; p_++; q = true; }
				else if (*p_ == '{') {
					int r = braces(mn, mx);
					if (r < 0) { fail("bad {n,m} quantifier"); break; }
					q = r == 1;
				}
				if (q) {
					NodeP r(new Node(Node::REP));
					r->rmin = mn;
					r->rmax = mx;
					r->lazy = f.ungreedy;
					if (more() && *p_ == '?') { r->lazy = !f.ungreedy; p_++; }
					else if (more() && *p_ == '+') { r->possessive = true; r->lazy = false; p_++; }
					if (a->kind == Node::ASSERT || a->kind == Node::LOOK) { fail("quantified assertion"); break; }
					r->kids.push_back(std::move(a));
					a = std::move(r);
					if (a->possessive && peel_noncapturing(a->kids[0].get())->kind != Node::SET) {
						// X*+ on anything but a single byte class is the atomic group (?>X*)
						a->possessive = false;
						NodeP at(new Node(Node::ATOMIC));
						at->kids.push_back(std::move(a));
						a = std::move(at);
					}
				}
			}
			cat->kids.push_back(std::move(a));
		}
		return cat;
	}

	NodeP alternation(Flags f)
	{
		NodeP alt(new Node(Node::ALT));
		Flags cur = f;
		for (;;) {
			alt->kids.push_back(concatenation(cur));
			if (!ok_) break;
			if (more() && *p_ == '|') { p_++; continue; }
			break;
		}
		if (alt->kids.size() == 1) return std::move(alt->kids[0]);
		return alt;
	}
};

// ------------------------------------------------------------------------------------------
// analysis
// ------------------------------------------------------------------------------------------

uint64_t min_length(const Node *n)
{
	uint64_t m = 0;
	switch (n->kind) {
	case Node::EMPTY: case Node::ASSERT: return 0;
	case Node::SET: return 1;
	case Node::CAT: for (auto &k : n->kids) m += min_length(k.get()); return m;
	case Node::ALT:
		m = UINT64_MAX;
		for (auto &k : n->kids) m = std::min(m, min_length(k.get()));
		return m;
	case Node::REP: return (uint64_t)n->rmin * min_length(n->kids[0].get());
	case Node::GROUP: case Node::ATOMIC: return min_length(n->kids[0].get());
	case Node::LOOK: return 0;
	}
	return 0;
}

// every match of n has the same length (what a lookbehind branch must have)
bool fixed_length(const Node *n, uint64_t &len)
{
	uint64_t a = 0, b = 0;
	switch (n->kind) {
	case Node::EMPTY: case Node::ASSERT: case Node::LOOK: len = 0; return true;
	case Node::SET: len = 1; return true;
	case Node::CAT:
		for (auto &k : n->kids) { if (!fixed_length(k.get(), b)) return false; a += b; }
		len = a;
		return true;
	case Node::ALT:
		if (n->kids.empty() || !fixed_length(n->kids[0].get(), a)) return false;
		for (size_t i = 1; i < n->kids.size(); i++) if (!fixed_length(n->kids[i].get(), b) || b != a) return false;
		len = a;
		return true;
	case Node::REP:
		if (n->rmin != n->rmax || !fixed_length(n->kids[0].get(), a)) return false;
		len = a * n->rmin;
		return true;
	case Node::GROUP: case Node::ATOMIC: return fixed_length(n->kids[0].get(), len);
	}
	return false;
}

// assertions, look-arounds and atomic groups: only the VM serves them
bool has_assert(const Node *n)
{
	if (n->kind == Node::ASSERT || n->kind == Node::LOOK || n->kind == Node::ATOMIC) return true;
	for (auto &k : n->kids) if (has_assert(k.get())) return true;
	return false;
}

// strips groups and single-child CAT/ALT wrappers
const Node *peel(const Node *n)
{
	for (;;) {
		if (n->kind == Node::GROUP) { n = n->kids[0].get(); continue; }
		if ((n->kind == Node::CAT || n->kind == Node::ALT) && n->kids.size() == 1) { n = n->kids[0].get(); continue; }
		return n;
	}
}

// like peel(), but a capturing group stays (the VM must see it close when capture participation matters, Q2)
const Node *peel_noncapturing(const Node *n)
{
	for (;;) {
		if (n->kind == Node::GROUP && !n->capturing) { n = n->kids[0].get(); continue; }
		if ((n->kind == Node::CAT || n->kind == Node::ALT) && n->kids.size() == 1) { n = n->kids[0].get(); continue; }
		return n;
	}
}

// does EVERY match of n close at least one capturing group?  (pcre_exec with room for one offset pair returns 0 for
// exactly the matches in which a group was set: quirk Q2)
bool always_captures(const Node *n)
{
	switch (n->kind) {
	case Node::SET: case Node::EMPTY: case Node::ASSERT: case Node::LOOK: return false;
	case Node::ATOMIC: return always_captures(n->kids[0].get());
	case Node::GROUP: return n->capturing || always_captures(n->kids[0].get());
	case Node::CAT: for (auto &k : n->kids) if (always_captures(k.get())) return true; return false;
	case Node::ALT: for (auto &k : n->kids) if (!always_captures(k.get())) return false; return !n->kids.empty();
	case Node::REP: return n->rmin >= 1 && always_captures(n->kids[0].get());
	}
	return false;
}

struct Expander {
	size_t budget_seqs = kMaxSequences;
	size_t budget_bytes = 1u << 20;
	bool overflow = false;
	bool general = false; // the pattern is fine, it just is not a list of fixed-length sequences: use the VM
	std::string why;

	typedef std::vector<Sequence> List;

	bool charge(const List &l)
	{
		if (l.size() > budget_seqs) { overflow = true; why = "pattern expands to too many alternatives"; return false; }
		size_t b = 0;
		for (auto &s : l) {
			b += s.size();
			if (s.size() > (size_t)kMaxPatternLen) { overflow = true; why = "alternative longer than 1024 bytes"; return false; }
		}
		if (b > budget_bytes) { overflow = true; why = "pattern expands to too many bytes"; return false; }
		return true;
	}

	// ordered product a x b (a-major: PCRE backtracks the right-hand side first)
	List product(const List &a, const List &b)
	{
		List out;
		if (overflow) return out;
		if (a.size() * b.size() > budget_seqs) { overflow = true; why = "pattern expands to too many alternatives"; return out; }
		out.reserve(a.size() * b.size());
		for (auto &x : a)
			for (auto &y : b) {
				Sequence s = x;
				s.insert(s.end(), y.begin(), y.end());
				out.push_back(std::move(s));
			}
		charge(out);
		return out;
	}

	// alternatives of `count` more iterations of `body` having done `done`, in backtracking order
	List rest(const List &body, uint32_t done, uint32_t mn, uint32_t mx, bool lazy)
	{
		List out;
		if (overflow) return out;
		List more;
		if (done < mx) more = product(body, rest(body, done + 1, mn, mx, lazy));
		List stop;
		if (done >= mn) stop.push_back(Sequence());
		if (lazy) { out = stop; out.insert(out.end(), more.begin(), more.end()); }
		else { out = more; out.insert(out.end(), stop.begin(), stop.end()); }
		charge(out);
		return out;
	}

	List expand(const Node *n)
	{
		List out;
		if (overflow) return out;
		switch (n->kind) {
		case Node::EMPTY: out.push_back(Sequence()); return out;
		case Node::ASSERT: case Node::LOOK: case Node::ATOMIC: overflow = true; general = true; return out;
		case Node::SET:
			if (n->set.empty()) return out; // can never match: contributes no alternative
			out.push_back(Sequence(1, n->set));
			return out;
		case Node::GROUP: return expand(n->kids[0].get());
		case Node::CAT: {
			out.push_back(Sequence());
			for (auto &k : n->kids) {
				out = product(out, expand(k.get()));
				if (overflow) break;
			}
			return out;
		}
		case Node::ALT:
			for (auto &k : n->kids) {
				List l = expand(k.get());
				out.insert(out.end(), l.begin(), l.end());
				if (!charge(out)) break;
			}
			return out;
		case Node::REP: {
			if (n->rmax == kInf) { overflow = true; general = true; return out; }
			List body = expand(n->kids[0].get());
			if (overflow) return out;
			// a possessive bounded repeat of single-byte bodies behaves like greedy without give-back;
			// expanding it as greedy could add matches PCRE would not find, so refuse
			if (n->possessive) { overflow = true; general = true; return out; }
			return rest(body, 0, n->rmin, n->rmax, n->lazy);
		}
		}
		return out;
	}
};

// crude byte-frequency prior (text / source code) used only to pick the rarest filter bytes
double byte_prior(unsigned c)
{
	static const char *common = " etaoinsrhldcumfpgwybvkxjqz";
	if (c == ' ') return 0.15;
	if (c == '\n') return 0.02;
	if (is_lower(c)) {
		const char *p = strchr(common, (int)c);
		int rank = p ? (int)(p - common) : 26;
		return 0.09 * (1.0 - rank / 30.0) + 0.002;
	}
	if (is_upper(c)) return 0.004;
	if (is_digit(c)) return 0.006;
	if (c > 32 && c < 127) return 0.004;
	if (c == '\t') return 0.005;
	if (c == 0) return 0.002;
	return 0.0005;
}

double test_prior(const MaskedEq &m)
{
	double p = 0;
	for (unsigned c = 0; c < 256; c++)
		if ((c & m.mask) == m.val) p += byte_prior(c);
	return p;
}

// can sequence b match `shift` bytes after sequence a started, with both matches overlapping?
bool can_overlap(const Sequence &a, const Sequence &b, size_t shift)
{
	for (size_t i = 0; shift + i < a.size() && i < b.size(); i++)
		if (!a[shift + i].intersects(b[i])) return false;
	return true;
}

// ------------------------------------------------------------------------------------------
// general patterns: backtracking VM program + leading-byte prefixes
// ------------------------------------------------------------------------------------------
// Anything the FIXED / RUN programs cannot express (unbounded repeats inside a sequence, assertions, lazy
// quantifiers, repeated groups) runs as: (1) a scan for the fixed-length leading byte sequences every match
// must start with (same kernels as FIXED), (2) the backtracking VM below, executed on the device at each
// candidate in position order by the resolve walk -- PCRE's own strategy (first-code-unit scan, then the
// interpreter), with PCRE's preference order: alternatives in source order, greedy takes all and gives back.

struct VmGen {
	std::vector<uint32_t> code; // 3 words per instruction: op | kind << 8 | set << 16, a, b
	std::vector<ByteSet> sets;
	bool track_caps = false;    // emit VM_CAP where a capturing group closes
	bool failed = false;
	std::string why;

	uint32_t emit(uint32_t op, uint32_t kind, uint32_t set, uint32_t a, uint32_t b)
	{
		if (code.size() / 3 >= 4096) { failed = true; why = "pattern too large for the device VM (more than 4096 instructions)"; return 0; }
		code.push_back(op | (kind << 8) | (set << 16));
		code.push_back(a);
		code.push_back(b);
		return (uint32_t)(code.size() / 3 - 1);
	}
	uint32_t set_id(const ByteSet &s)
	{
		for (size_t i = 0; i < sets.size(); i++) if (sets[i] == s) return (uint32_t)i;
		sets.push_back(s);
		return (uint32_t)sets.size() - 1;
	}
	void gen(const Node *n)
	{
		if (failed) return;
		switch (n->kind) {
		case Node::EMPTY: return;
		case Node::SET: emit(VM_SET, 0, set_id(n->set), 0, 0); return;
		case Node::ASSERT: emit(VM_ASSERT, (uint32_t)n->akind, 0, 0, 0); return;
		case Node::GROUP:
			gen(n->kids[0].get());
			if (track_caps && n->capturing) emit(VM_CAP, 0, 0, 0, 0);
			return;
		case Node::ATOMIC: {
			const uint32_t l = emit(VM_LOOK, VM_LK_ATOMIC, 0, 0, 0);
			gen(n->kids[0].get());
			emit(VM_LOOKEND, 0, 0, 0, 0);
			if (!failed) code[3 * l + 1] = (uint32_t)(code.size() / 3);
			return;
		}
		case Node::LOOK: {
			if (n->ahead) {
				const uint32_t l = emit(VM_LOOK, n->neg ? VM_LK_AHEAD_NEG : VM_LK_AHEAD, 0, 0, 0);
				gen(n->kids[0].get());
				emit(VM_LOOKEND, 0, 0, 0, 0);
				if (!failed) code[3 * l + 1] = (uint32_t)(code.size() / 3);
				return;
			}
			// lookbehind: every top-level branch has its own fixed length (PCRE's rule): (?<=a|bc) is (?:(?<=a)|(?<=bc)),
			// (?<!a|bc) is (?<!a)(?<!bc)
			const Node *body = peel_noncapturing(n->kids[0].get());
			std::vector<const Node *> branches;
			if (body->kind == Node::ALT) for (auto &k : body->kids) branches.push_back(k.get());
			else branches.push_back(body);
			std::vector<uint32_t> jmps;
			for (size_t i = 0; i < branches.size() && !failed; i++) {
				uint64_t len = 0;
				if (!fixed_length(branches[i], len) || len > 65535) { failed = true; why = "lookbehind assertion is not fixed length"; return; }
				uint32_t split = 0;
				const bool more_branches = !n->neg && i + 1 < branches.size();
				if (more_branches) split = emit(VM_SPLIT, 0, 0, 0, 0);
				const uint32_t l = emit(VM_LOOK, n->neg ? VM_LK_BEHIND_NEG : VM_LK_BEHIND, 0, 0, (uint32_t)len);
				gen(branches[i]);
				emit(VM_LOOKEND, 0, 0, 0, 0);
				if (failed) return;
				code[3 * l + 1] = (uint32_t)(code.size() / 3);
				if (more_branches) {
					jmps.push_back(emit(VM_JMP, 0, 0, 0, 0));
					code[3 * split + 1] = split + 1;
					code[3 * split + 2] = (uint32_t)(code.size() / 3);
				}
			}
			for (uint32_t j : jmps) code[3 * j + 1] = (uint32_t)(code.size() / 3);
			return;
		}
		case Node::CAT: for (auto &k : n->kids) gen(k.get()); return;
		case Node::ALT: {
			std::vector<uint32_t> jmps;
			for (size_t i = 0; i < n->kids.size() && !failed; i++) {
				if (i + 1 < n->kids.size()) {
					const uint32_t s = emit(VM_SPLIT, 0, 0, 0, 0);
					gen(n->kids[i].get());
					jmps.push_back(emit(VM_JMP, 0, 0, 0, 0));
					if (failed) return;
					code[3 * s + 1] = s + 1;
					code[3 * s + 2] = (uint32_t)(code.size() / 3);
				} else {
					gen(n->kids[i].get());
				}
			}
			for (uint32_t j : jmps) code[3 * j + 1] = (uint32_t)(code.size() / 3);
			return;
		}
		case Node::REP: {
			const Node *body = track_caps ? peel_noncapturing(n->kids[0].get()) : peel(n->kids[0].get());
			const uint32_t kind = n->lazy ? VM_Q_LAZY : n->possessive ? VM_Q_POSSESSIVE : VM_Q_GREEDY;
			if (body->kind == Node::SET) { emit(VM_REP, kind, set_id(body->set), n->rmin, n->rmax); return; }
			if (n->possessive) { failed = true; why = "possessive quantifier on a group is not supported"; return; }
			if (n->rmax == kInf && min_length(n->kids[0].get()) == 0) { failed = true; why = "unbounded repeat of an empty-matchable group is not supported"; return; }
			if (n->rmin > 256 || (n->rmax != kInf && n->rmax > 256)) { failed = true; why = "group repeat count above 256 is not supported"; return; }
			for (uint32_t i = 0; i < n->rmin && !failed; i++) gen(n->kids[0].get());
			if (n->rmax == kInf) {
				const uint32_t L = emit(VM_SPLIT, 0, 0, 0, 0);
				gen(n->kids[0].get());
				emit(VM_JMP, 0, 0, L, 0);
				if (failed) return;
				const uint32_t out = (uint32_t)(code.size() / 3);
				code[3 * L + 1] = n->lazy ? out : L + 1;
				code[3 * L + 2] = n->lazy ? L + 1 : out;
			} else {
				std::vector<uint32_t> splits;
				for (uint32_t i = n->rmin; i < n->rmax && !failed; i++) {
					splits.push_back(emit(VM_SPLIT, 0, 0, 0, 0));
					gen(n->kids[0].get());
				}
				const uint32_t out = (uint32_t)(code.size() / 3);
				for (uint32_t sp : splits) {
					code[3 * sp + 1] = n->lazy ? out : sp + 1;
					code[3 * sp + 2] = n->lazy ? sp + 1 : out;
				}
			}
			return;
		}
		}
	}
};

// Reach of a VM program (Program::vm_reach): an attempt at p reads the subject's beginning s only where a back-looking
// construct runs close to it -- an assertion that tests sp == 0 or the byte before sp (^ \A (?m)^ \b \B), or a look-behind
// of b bytes, which fails / holds at once when fewer than b bytes precede sp.  Run at offset o >= m from p, such a construct
// sees the same as from any earlier start once s <= p + m - 1 (assertions) or s <= p + m - b (look-behinds).  `m` is the
// least offset at which the node can begin (negative inside a look-behind body); returns the least offset behind it.
int64_t reach_walk(const Node *n, int64_t m, int64_t &reach)
{
	switch (n->kind) {
	case Node::EMPTY: return m;
	case Node::SET: return m + 1;
	case Node::ASSERT:
		if (n->akind == VM_A_BOL || n->akind == VM_A_SOS || n->akind == VM_A_MBOL || n->akind == VM_A_WORDB || n->akind == VM_A_NWORDB)
			reach = std::max<int64_t>(reach, 1 - m);
		return m;
	case Node::GROUP: case Node::ATOMIC: return reach_walk(n->kids[0].get(), m, reach);
	case Node::LOOK: {
		if (n->ahead) { reach_walk(n->kids[0].get(), m, reach); return m; }
		const Node *body = peel_noncapturing(n->kids[0].get()); // one fixed length per top-level branch, as VmGen emits it
		std::vector<const Node *> branches;
		if (body->kind == Node::ALT) for (auto &k : body->kids) branches.push_back(k.get());
		else branches.push_back(body);
		for (const Node *br : branches) {
			uint64_t len = 0;
			fixed_length(br, len);
			reach = std::max<int64_t>(reach, (int64_t)len - m);
			reach_walk(br, m - (int64_t)len, reach);
		}
		return m;
	}
	case Node::CAT:
		for (auto &k : n->kids) m = reach_walk(k.get(), m, reach);
		return m;
	case Node::ALT: {
		int64_t lo = INT64_MAX;
		for (auto &k : n->kids) lo = std::min(lo, reach_walk(k.get(), m, reach));
		return lo;
	}
	case Node::REP: // later iterations begin at or behind the first one: the first bounds them all
		reach_walk(n->kids[0].get(), m, reach);
		return m + (int64_t)n->rmin * (int64_t)min_length(n->kids[0].get());
	}
	return m;
}

int vm_reach(const Node *root)
{
	int64_t reach = 0;
	reach_walk(root, 0, reach);
	return (int)std::min<int64_t>(reach, 1 << 20);
}

// byte-class sequences (length <= L) every match of `n` starts with; `done`: the node is consumed exactly by
// the sequence, so what follows the node may extend it
struct Pref { Sequence seq; bool done; };

bool prefixes(const Node *n, size_t L, std::vector<Pref> &out)
{
	out.clear();
	switch (n->kind) {
	case Node::EMPTY: case Node::ASSERT: case Node::LOOK: out.push_back(Pref{Sequence(), true}); return true;
	case Node::ATOMIC: return prefixes(n->kids[0].get(), L, out);
	case Node::SET:
		if (n->set.empty()) return true; // can never match: no prefix at all
		out.push_back(Pref{Sequence(1, n->set), true});
		return true;
	case Node::GROUP: return prefixes(n->kids[0].get(), L, out);
	case Node::ALT:
		for (auto &k : n->kids) {
			std::vector<Pref> t;
			if (!prefixes(k.get(), L, t)) return false;
			out.insert(out.end(), t.begin(), t.end());
			if (out.size() > 256) return false;
		}
		return true;
	case Node::CAT: {
		out.push_back(Pref{Sequence(), true});
		for (auto &k : n->kids) {
			bool any_open = false;
			for (auto &p : out) any_open = any_open || (p.done && p.seq.size() < L);
			if (!any_open) break;
			std::vector<Pref> t, next;
			if (!prefixes(k.get(), L, t)) return false;
			for (auto &p : out) {
				if (!p.done || p.seq.size() >= L) { next.push_back(Pref{p.seq, false}); continue; }
				for (auto &q : t) {
					Pref r{p.seq, q.done};
					for (auto &cls : q.seq) {
						if (r.seq.size() >= L) { r.done = false; break; }
						r.seq.push_back(cls);
					}
					next.push_back(r);
				}
			}
			if (next.size() > 256) return false;
			out.swap(next);
		}
		return true;
	}
	case Node::REP: {
		const Node *body = peel(n->kids[0].get());
		if (n->rmax == 0) { out.push_back(Pref{Sequence(), true}); return true; }
		if (body->kind == Node::SET && !body->set.empty()) {
			// a class repeated: min copies are certain
			const size_t take = std::min<size_t>(n->rmin, L);
			if (n->rmin == 0) {
				out.push_back(Pref{Sequence(), true});              // skipped: what follows starts the match
				out.push_back(Pref{Sequence(1, body->set), false}); // or at least one
			} else {
				out.push_back(Pref{Sequence(take, body->set), n->rmin == n->rmax && n->rmin <= L});
			}
			return true;
		}
		std::vector<Pref> t;
		if (!prefixes(n->kids[0].get(), L, t)) return false;
		if (n->rmin == 0) out.push_back(Pref{Sequence(), true});
		for (auto &p : t) out.push_back(Pref{p.seq, p.done && n->rmin == 1 && n->rmax == 1});
		return true;
	}
	}
	return false;
}

std::atomic<uint64_t> g_next_id{1};

uint32_t umulhi32(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }

// Perfect hash over the distinct values of the first L bytes (little endian, like a 32-bit load) of all
// alternatives.  Classes in the leading positions are enumerated (e.g. (?i) doubles per letter).
bool build_hash(Program &out, int L)
{
	std::vector<std::pair<uint32_t, uint32_t>> kv; // (key, sequence index)
	size_t total = 0;
	for (size_t si = 0; si < out.seqs.size(); si++) {
		const Sequence &s = out.seqs[si];
		size_t combos = 1;
		for (int i = 0; i < L; i++) combos *= (size_t)s[i].count();
		total += combos;
		if (combos == 0 || total > 4096) return false;
		std::vector<uint32_t> keys(1, 0);
		for (int i = 0; i < L; i++) {
			std::vector<uint32_t> next;
			for (uint32_t k : keys)
				for (unsigned b = 0; b < 256; b++)
					if (s[i].has(b)) next.push_back(k | (b << (8 * i)));
			keys.swap(next);
		}
		for (uint32_t k : keys) kv.push_back(std::make_pair(k, (uint32_t)si));
	}
	std::vector<uint32_t> distinct;
	for (auto &e : kv) distinct.push_back(e.first);
	std::sort(distinct.begin(), distinct.end());
	distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
	uint64_t rng = 0x9E3779B97F4A7C15ull ^ (distinct.size() * 0xD1B54A32D192ED03ull);
	const uint32_t kEmpty = 0xffffffffu; // never a key: keys are at most 3 bytes
	// slot = umulhi(h, slots), h = key * (mul << 8 * (4 - L)) mod 2^32: multiplicative hashing on the LOW product word
	// (every key bit reaches its top bits; text keys differ mostly in their low bits) and a multiply-high range
	// reduction, so the kernel computes the slot with two IMADs and no ALU-pipe instruction, and `slots` need not be a
	// power of two.  The multiplier carries the shift that pushes the bytes beyond the key out of the word: the kernel
	// hashes the raw 32-bit window at every position without masking it, and the device table holds h, not the key.
	std::vector<uint32_t> table;
	auto search = [&](uint32_t ns, int attempts) -> bool {
		for (int attempt = 0; attempt < attempts; attempt++) {
			rng = rng * 6364136223846793005ull + 1442695040888963407ull;
			const uint32_t mul = (uint32_t)(rng >> 32) | 1u;
			table.assign(ns, kEmpty);
			bool ok = true;
			for (uint32_t k : distinct) {
				const uint32_t sl = umulhi32(k * (mul << (8 * (4 - L))), ns);
				if (table[sl] != kEmpty) { ok = false; break; }
				table[sl] = k;
			}
			if (!ok) continue;
			out.use_hash = true;
			out.hash_len = L;
			out.hash_mul = mul;
			out.hash_slots = ns;
			out.hash_table = table;
			out.slot_first.assign(ns, 0);
			out.slot_count.assign(ns, 0);
			out.slot_seqs.clear();
			for (uint32_t sl = 0; sl < ns; sl++) {
				if (table[sl] == kEmpty) continue;
				out.slot_first[sl] = (uint32_t)out.slot_seqs.size();
				for (auto &e : kv) // kv is in preference order of the alternatives
					if (e.first == table[sl]) { out.slot_seqs.push_back(e.second); out.slot_count[sl]++; }
			}
			return true;
		}
		return false;
	};
	// tables of up to kHashReplicatedSlots (512) slots are replicated once per shared-memory bank by the kernel
	// (conflict-free lookups; with random slots the shared-memory data pipe is the bottleneck: ~3.4 wavefronts per
	// lookup), so a small table is worth a long search: P(no collision) ~ exp(-n^2 / 2 slots) per try
	const size_t n = distinct.size();
	if (n + n / 8 <= 256 && search(256, 20000)) return true;
	if (n + n / 8 <= 384 && search(384, 100000)) return true;
	if (n + n / 8 <= 512 && search(512, 1000000)) return true;
	for (uint32_t ns = 1024; ns <= 8192; ns <<= 1)
		if (search(ns, 4000)) return true;
	return false;
}

} // namespace

bool compile_pattern(const char *pat, size_t len, uint32_t flags, Program &out, std::string &err)
{
	out = Program();
	out.id = g_next_id.fetch_add(1);
	out.strict_q2 = (flags & GSCAN_STRICT_REF) != 0;
	if (memchr(pat, 0, len)) { err = "pattern contains a NUL byte (the reference passes a C string, grab.cc:106)"; return false; }

	NodeP root;
	int captures = 0;
	if (flags & GSCAN_LITERAL) {
		root.reset(new Node(Node::CAT));
		for (size_t i = 0; i < len; i++) {
			NodeP n(new Node(Node::SET));
			n->set.add((uint8_t)pat[i]);
			root->kids.push_back(std::move(n));
		}
	} else {
		Parser ps((const uint8_t *)pat, len);
		root = ps.parse(err);
		if (!root) return false;
		captures = ps.captures();
	}
	out.captures = captures;

	uint64_t ml = min_length(root.get());
	if (ml == 0) {
		err = "pattern can match the empty string: the reference never terminates on it (grab.cc:209); rejected";
		return false;
	}
	out.minlen = ml > 65535 ? 65535 : (int)ml; // PCRE2's study caps MINLENGTH at 65535

	if (out.strict_q2 && captures > 0 && always_captures(root.get())) {
		// Q2: every match sets a capturing group, pcre_exec (ovecsize 3) returns 0 for every match => the loop breaks
		// before printing anything (grab.cc:179)
		out.kind = ENGINE_NONE;
		out.maxlen = -1;
		return true;
	}
	// Q2, mixed: `foo|(bar)`, `(x)?foo` -- pcre_exec returns 0 only for the matches in which a group took part: the loop
	// prints until the first such match and then leaves the window.  Which match that is depends on the path taken, so
	// these patterns run on the VM, which reports the flag with every match.
	const bool cap_stops = out.strict_q2 && captures > 0;
	out.cap_stops = cap_stops;

	// RUN: the whole pattern is one byte class repeated {n,}
	const Node *core = peel(root.get());
	if (!cap_stops && core->kind == Node::REP && core->rmax == kInf && !core->lazy) {
		const Node *body = peel(core->kids[0].get());
		if (body->kind == Node::SET && core->rmin >= 1) {
			if (core->rmin > (uint32_t)kMaxPatternLen) { err = "run minimum above 1024"; return false; }
			out.kind = ENGINE_RUN;
			out.run_class = body->set;
			out.run_min = (int)core->rmin;
			out.maxlen = -1;
			out.disjoint = true;
			for (auto r : to_ranges(body->set)) {
				if (r.lo < 0x80) out.ranges_low.push_back(ByteRange{r.lo, (uint8_t)std::min<int>(r.hi, 0x7f)});
				if (r.hi >= 0x80) out.ranges_high.push_back(ByteRange{(uint8_t)std::max<int>(r.lo, 0x80), r.hi});
			}
			if ((int)out.ranges_low.size() > kMaxRunRangesLow || (int)out.ranges_high.size() > kMaxRunRangesHigh) {
				err = "byte class of the run needs too many ranges for the SWAR class test";
				return false;
			}
			if (body->set.empty()) { err = "empty byte class"; return false; }
			return true;
		}
	}

	// FIXED: expand into fixed-length sequences in backtracking (preference) order
	Expander ex;
	std::vector<Sequence> seqs;
	if (!has_assert(root.get()) && !cap_stops) seqs = ex.expand(root.get());
	else { ex.overflow = true; ex.general = true; }
	if (ex.overflow && !ex.general) { err = ex.why; return false; }
	if (ex.overflow) {
		// general pattern: VM program + leading-byte prefixes as the candidate filter
		VmGen g;
		g.track_caps = cap_stops;
		g.gen(root.get());
		g.emit(VM_MATCH, 0, 0, 0, 0);
		if (g.failed) { err = g.why; return false; }
		out.vm_reach = vm_reach(root.get());
		out.vm_start_free = out.vm_reach == 0;
		// a pattern that begins with a greedy/lazy/possessive byte-class repeat C{n,}: if an attempt succeeds anywhere
		// inside a run of C it also succeeds at the run's first byte (C{n,} simply takes the bytes in between), so
		// PCRE's leftmost match starts at a run start -- or at the search start itself when that lies inside a run.
		// Candidates are then the run starts (RUN scan kernel), far fewer than "every byte of the class".
		{
			const Node *top = peel(root.get());
			if (!cap_stops && top->kind == Node::CAT && top->kids.size() >= 2) {
				const Node *lead = top->kids[0].get();
				while (lead->kind == Node::GROUP) lead = lead->kids[0].get();
				const Node *body = lead->kind == Node::REP ? peel(lead->kids[0].get()) : nullptr;
				if (body && body->kind == Node::SET && !body->set.empty() && lead->rmin >= 1 && lead->rmax == kInf && lead->rmin <= (uint32_t)kMaxPatternLen) {
					std::vector<ByteRange> lo, hi;
					for (auto r : to_ranges(body->set)) {
						if (r.lo < 0x80) lo.push_back(ByteRange{r.lo, (uint8_t)std::min<int>(r.hi, 0x7f)});
						if (r.hi >= 0x80) hi.push_back(ByteRange{(uint8_t)std::max<int>(r.lo, 0x80), r.hi});
					}
					if ((int)lo.size() <= kMaxRunRangesLow && (int)hi.size() <= kMaxRunRangesHigh) {
						out.kind = ENGINE_RUN;
						out.run_class = body->set;
						out.run_min = (int)lead->rmin;
						out.ranges_low = lo;
						out.ranges_high = hi;
						out.maxlen = -1;
						out.use_vm = true;
						out.vm_runstart = true;
						out.vm_lead = lead->lazy ? VM_Q_LAZY : lead->possessive ? VM_Q_POSSESSIVE : VM_Q_GREEDY;
						out.vm_code = g.code;
						for (auto &s : g.sets) for (int i = 0; i < 8; i++) out.vm_sets.push_back(s.w[i]);
						return true;
					}
				}
			}
		}
		std::vector<Pref> pf;
		out.use_vm = true;
		out.vm_code = g.code;
		for (auto &s : g.sets) for (int i = 0; i < 8; i++) out.vm_sets.push_back(s.w[i]);
		bool dense = !prefixes(root.get(), 4, pf) || pf.empty();
		seqs.clear();
		out.first_set = ByteSet();
		for (auto &p : pf) {
			if (p.seq.empty()) dense = true; // a match can begin with any byte (leading optional item or bare assertion)
			else { seqs.push_back(p.seq); out.first_set.unite(p.seq[0]); }
		}
		if (dense) {
			// no candidate filter at all: the walk offers every position to the VM (what pcre_exec does without a
			// first-code-unit optimisation)
			out.first_set = ByteSet();
			out.first_set.invert();
			out.vm_dense = true;
			out.kind = ENGINE_FIXED;
			out.seqs.clear();
			out.maxlen = -1;
			return true;
		}
	}
	// drop exact duplicates (a later identical alternative can never win) and never-matching ones
	std::vector<Sequence> uniq;
	for (auto &s : seqs) {
		if (s.empty()) { err = "internal: empty alternative"; return false; }
		bool dup = false;
		for (auto &u : uniq)
			if (u.size() <= s.size()) {
				// u shadows s if u is a prefix-wise superset: whenever s matches at q, u (earlier) does too
				bool shadow = true;
				for (size_t i = 0; i < u.size() && shadow; i++) shadow = s[i].subset_of(u[i]);
				if (shadow) { dup = true; break; }
			}
		if (!dup) uniq.push_back(s);
	}
	// alternatives of equal length that differ in exactly one position are one alternative with the union class
	// there: same start, same length, so which of them PCRE would have preferred does not show ("a|b|c" == "[abc]")
	// (an optimisation only, quadratic per merge: skipped for sets far beyond what the engines serve anyway)
	for (bool merged = uniq.size() <= 512; merged;) {
		merged = false;
		for (size_t i = 0; i < uniq.size() && !merged; i++)
			for (size_t j = i + 1; j < uniq.size() && !merged; j++) {
				if (uniq[i].size() != uniq[j].size()) continue;
				int diff = -1, ndiff = 0;
				for (size_t k = 0; k < uniq[i].size(); k++)
					if (!(uniq[i][k] == uniq[j][k])) { diff = (int)k; ndiff++; }
				if (ndiff != 1) continue;
				// only safe if nothing between them in preference order could win at a position where j matches:
				// merging moves j's matches up to i's rank, which changes the result only if an alternative k in (i, j)
				// of a DIFFERENT length also matches there -- so require all alternatives in between to have this length
				bool ok = true;
				for (size_t k = i + 1; k < j && ok; k++) ok = uniq[k].size() == uniq[i].size();
				if (!ok) continue;
				uniq[i][diff].unite(uniq[j][diff]);
				uniq.erase(uniq.begin() + (long)j);
				merged = true;
			}
	}
	if (uniq.empty()) { err = "pattern can never match"; return false; }
	out.kind = ENGINE_FIXED;
	out.seqs = uniq;
	size_t mn = SIZE_MAX, mx = 0;
	for (auto &s : out.seqs) { mn = std::min(mn, s.size()); mx = std::max(mx, s.size()); }
	out.maxlen = out.use_vm ? -1 : (int)mx;
	// (minlen from the tree equals mn unless shadowing removed the shortest: keep PCRE's figure)

	// ---- choose the SWAR filter: anchor byte + second byte `delta` further on ----
	double best_score = 1e300, best_p = 1.0;
	int best_a = 0, best_d = 0;
	std::vector<FilterTest> best_tests;
	for (int d = (mn >= 2 ? 1 : 0); d <= 4; d++) {
		for (int a = 0; a + d < (int)mn && a <= 224; a++) {
			std::vector<FilterTest> tests;
			double p = 0, cost = 0;
			for (auto &s : out.seqs) {
				MaskedEq e0 = masked_superset(s[a]);
				MaskedEq e1 = d ? masked_superset(s[a + d]) : MaskedEq{0, 0, false, 256};
				FilterTest t{e0.mask, e0.val, e1.mask, e1.val};
				if (std::find(tests.begin(), tests.end(), t) == tests.end()) {
					tests.push_back(t);
					p += test_prior(e0) * (d ? test_prior(e1) : 1.0);
					// a test of two plain bytes is cheaper than one with a mask (and an all-exact multi-test filter runs on the
					// balanced pair engine, half the ALU-pipe work): prefer `ba` over `b.[rz]` when the priors are close
					cost += (e0.mask == 0xff && (!d || e1.mask == 0xff)) ? 1.0 : 2.0;
				}
			}
			if ((int)tests.size() > kMaxFilterTests) continue;
			// each test costs ~4 ALU ops per 4 bytes (a distance of exactly one word needs no funnel shift:
			// ~20 % cheaper); each flagged position costs a slow-path visit
			double score = (p * 4000.0 + cost) * (d == 4 ? 0.8 : 1.0);
			if (score < best_score) { best_score = score; best_a = a; best_d = d; best_tests = tests; best_p = p; }
		}
		if (mn < 2) break;
	}
	// many distinct byte pairs: the pair filter gets slow (4 ops per test and word) -- switch to the hashed engine
	if ((best_tests.empty() || best_tests.size() > 4) && mn >= 2 && build_hash(out, (int)std::min<size_t>(mn, 3))) {
		out.anchor = 0;
		out.delta = 0;
		out.tests.clear();
	} else if (best_tests.empty() && out.use_vm) {
		out.vm_dense = true; // too many distinct leading sequences for either filter: the VM walk tries the positions itself
		out.seqs.clear();
		return true;
	} else if (best_tests.empty()) {
		err = "alternation needs more than 8 distinct byte-pair filter tests and its leading bytes cannot be hashed "
		      "(an alternative shorter than 2 bytes, or more than 4096 distinct leading byte combinations)";
		return false;
	}
	if (out.use_hash) {
		bool dj = out.seqs.size() <= 256;
		for (size_t i = 0; i < out.seqs.size() && dj; i++)
			for (size_t j = 0; j < out.seqs.size() && dj; j++)
				for (size_t sh = 1; sh < out.seqs[i].size() && dj; sh++)
					if (can_overlap(out.seqs[i], out.seqs[j], sh)) dj = false;
		out.disjoint = dj;
		return true;
	}
	out.anchor = best_a;
	out.delta = best_d;
	out.tests = best_tests;

	// ---- stage 2: a third byte (anchor + d2, d2 in 0..3 other than 0 and delta) narrows flagged rows ----
	{
		double best_p = 1e300;
		for (int d2 = 1; d2 <= 3; d2++) {
			if (d2 == out.delta || out.anchor + d2 >= (int)mn) continue;
			std::vector<Program::Triple> tr;
			double p = 0;
			for (auto &s : out.seqs) {
				MaskedEq e0 = masked_superset(s[out.anchor]);
				MaskedEq e1 = out.delta ? masked_superset(s[out.anchor + out.delta]) : MaskedEq{0, 0, false, 256};
				MaskedEq e2 = masked_superset(s[out.anchor + d2]);
				Program::Triple t{e0.mask, e0.val, e1.mask, e1.val, e2.mask, e2.val};
				bool dup = false;
				for (auto &x : tr) dup = dup || !memcmp(&x, &t, sizeof(t));
				if (!dup) { tr.push_back(t); p += test_prior(e0) * (out.delta ? test_prior(e1) : 1.0) * test_prior(e2); }
			}
			if (tr.size() <= 16 && p < best_p) { best_p = p; out.triples = tr; out.delta2 = d2; }
		}
	}

	if (out.use_vm && best_p > 0.30) {
		// the leading bytes are so common that the candidate list would hold every other position: skip the scan kernel and
		// let the VM walk try the positions itself (first-byte test in registers), as pcre_exec does
		out.vm_dense = true;
		out.seqs.clear();
		out.tests.clear();
		out.triples.clear();
		return true;
	}
	out.pair_flag_prior = best_p;

	// ---- can two matches overlap?  If not, the greedy resolve keeps every candidate ----
	bool disjoint = true;
	for (auto &a : out.seqs) {
		for (auto &b : out.seqs) {
			for (size_t sh = 1; sh < a.size() && disjoint; sh++)
				if (can_overlap(a, b, sh)) disjoint = false;
			if (!disjoint) break;
		}
		if (!disjoint) break;
	}
	out.disjoint = disjoint;
	return true;
}

} // namespace gscan
